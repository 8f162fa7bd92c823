"""Time of the GPU JPEG decode on its worst case for self-synchronisation, next to encoder-made files.

The worst case (tests/jpeg_craft.py ``long_code_stream``): a valid 1080x1920 grayscale file with one-symbol 16-bit
Huffman codes and all-zero entropy bits, 1476-bit blocks and entropy data filling 96 % of the compressed slot.  Every bit
position decodes, so a decoder started in the wrong phase never resynchronises: the sync takes one round per
subsequence of 8192 bits, thousands of rounds, and the entropy kernel is close to a sequential decode.  For comparison,
32 files of 480x640 q90 4:2:0 from Pillow (tools/jpeg_bench.py's files) take 2 rounds each.

``defer_k_jpeg_decode`` (all three kernels) is timed with CUDA events, one warm-up launch and ``--reps`` timed ones,
at the 1080x1920 bound; it prints one JSON line with the median and spread per case, the rounds and subsequences from
the kernel's counters, and the card and its power limit.

    python tools/jpeg_worst_case.py --reps 3
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests"), str(ROOT / "tools")]

from defer_b200 import _cabi as A  # noqa: E402
from defer_b200 import jpeg  # noqa: E402
from ingress_bench import card  # noqa: E402
import jpeg_craft  # noqa: E402

BOUND = (1080, 1920)


def time_decode(files, reps):
    """(ms per launch of every rep, stats [n, 5]) of defer_k_jpeg_decode over ``files`` at the bound."""
    import torch
    lib = A.load()
    H, W = BOUND
    n, slot = len(files), H * W * 3
    slots = np.zeros((n, slot), np.uint8)
    blocks = np.zeros((n, jpeg.BLOCK_INTS), np.int32)
    for i, d in enumerate(files):
        slots[i, :len(d)] = np.frombuffer(d, np.uint8)
        blocks[i] = jpeg.pack_block(jpeg.parse(d))
    total, stride = C.c_uint64(), C.c_uint64()
    A.check(lib.defer_k_jpeg_workspace(H, W, n, C.byref(total), C.byref(stride), None, None))
    ws = torch.zeros(total.value, dtype=torch.uint8, device="cuda")
    x = torch.from_numpy(slots.reshape(-1)).cuda()
    b = torch.from_numpy(blocks.reshape(-1)).cuda()
    y = torch.zeros(n * slot, dtype=torch.uint8, device="cuda")
    s = torch.cuda.default_stream()
    ts = []
    for r in range(reps + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record(s)
        A.check(lib.defer_k_jpeg_decode(x.data_ptr(), b.data_ptr(), n, H, W, ws.data_ptr(), y.data_ptr(), None))
        ev[1].record(s)
        torch.cuda.synchronize()
        if r:
            ts.append(ev[0].elapsed_time(ev[1]))
    stats = ws.view(n, stride.value)[:, :20].cpu().numpy().view(np.int32)
    return ts, stats


def summary(ts, stats, files):
    return {"files": len(files), "mean_file_bytes": int(np.mean([len(d) for d in files])),
            "ms_median": round(statistics.median(ts), 2), "ms_min": round(min(ts), 2), "ms_max": round(max(ts), 2),
            "rounds_max": int(stats[:, 3].max()), "subsequences_max": int(stats[:, 2].max())}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from jpeg_bench import files as bench_files
    worst = jpeg_craft.long_code_stream(*BOUND)
    q90 = bench_files((480, 640), 90)
    out = {"card": card(), "bound": f"{BOUND[0]}x{BOUND[1]}"}
    for key, fs in (("worst_1080x1920_x1", [worst]), ("worst_1080x1920_x32", [worst] * 32),
                    ("pillow_480x640_q90_420_x32", q90)):
        out[key] = summary(*time_decode(fs, args.reps), fs)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
