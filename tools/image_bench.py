"""Mixed JPEG and PNG decode on the GPU: `defer_k_image_decode` against the single-format decodes, per microbatch of 32
photo-like files (CUDA events, median of --reps after a warm-up), at bounds of 480x640 and 1080x1920:
  - 32 JPEGs through `defer_k_jpeg_decode` and through the image op: the cost of the sample filter and of the PNG
    kernels' CTAs that exit at once;
  - 32 PNGs through `defer_k_png_decode` and through the image op, for the same reason;
  - 16 JPEG + 16 PNG and 31 JPEG + 1 PNG through the image op, against the sum of the single-format decodes of the same
    files (16 + 16, 31 + 1).
The JPEGs are the committed photo fixtures of each size (tests/golden/jpeg), the PNGs `png_photo` of tests/test_gpu_png.py
(Sub-filtered rows, zlib level 6).  Every image op result is checked against `image.decode_image` before timing.  Card
name and power limit are read in the same run.  One JSON line.

    python tools/image_bench.py [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import image  # noqa: E402
from test_gpu_image import Decode  # noqa: E402
from test_gpu_png import png_photo  # noqa: E402

JPEG_PHOTO = {(480, 640): "photo_480x640_420_q75.jpg", (1080, 1920): "photo_1080x1920_420_q50.jpg"}


def _time(dec: Decode, files, reps: int) -> float:
    dec.run(files)                                                       # warm-up
    return float(np.median([dec.run(files, timed=True) for _ in range(reps)]))


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    out = {"card": card, "files_per_call": 32, "ms": {}}
    for H, W in ((480, 640), (1080, 1920)):
        j = (ROOT / "tests" / "golden" / "jpeg" / JPEG_PHOTO[(H, W)]).read_bytes()
        p = png_photo(H, W, 1)
        want = {"jpeg": image.decode_image(j), "png": image.decode_image(p)}
        single = {}

        def one(kind, n):
            if (kind, n) not in single:
                single[kind, n] = Decode(kind, n, H, W)
            return _time(single[kind, n], [j if kind == "jpeg" else p] * n, a.reps)
        dec = Decode("image", 32, H, W)
        res = {}
        for name, nj in (("jpeg32", 32), ("png32", 0), ("mix16+16", 16), ("mix31+1", 31)):
            files = [j] * nj + [p] * (32 - nj)
            dec.run(files)
            for i in (0, 31):
                kind = "jpeg" if i < nj else "png"
                assert np.array_equal(dec.rgb(i, H, W), want[kind]), (name, i)
            t = _time(dec, files, a.reps)
            ref = (one("jpeg", nj) if nj else 0.0) + (one("png", 32 - nj) if nj < 32 else 0.0)
            res[name] = {"image_op": round(t, 3), "single_format": round(ref, 3)}
        out["ms"][f"{H}x{W}"] = res
        del dec, single
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
