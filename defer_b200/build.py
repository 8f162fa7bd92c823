"""Build libdefer_b200.so in-tree with nvcc for sm_90a (ahead of time: nothing is compiled when the library loads)."""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIB = HERE / "lib" / "libdefer_b200.so"
SOURCES = ["stage.cu", "kernels_simt.cu", "conv_umma.cu", "api_kernels.cu", "jpeg.cu", "png.cu", "image.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC,-fvisibility=hidden", "-DDEFER_BUILD"]


def _stale(obj: Path, src: Path) -> bool:
    if not obj.exists():
        return True
    t = obj.stat().st_mtime
    deps = [src] + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + [HERE.parent / "include" / "defer_b200.h"]
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objdir = HERE / "lib" / "obj"
    objdir.mkdir(parents=True, exist_ok=True)
    objs, procs = [], []
    for name in SOURCES:
        src, obj = CSRC / name, objdir / (name + ".o")
        objs.append(obj)
        if force or _stale(obj, src):
            cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
                print(" ".join(cmd), flush=True)
            procs.append((name, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for name, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc {name} failed ---\n{out}\n")
        elif verbose and out:
            print(out)
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or not LIB.exists():
        cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), "-Xlinker", "--exclude-libs,ALL", "-lcudart_static",
               "-lpthread", "-ldl", "-lrt"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
