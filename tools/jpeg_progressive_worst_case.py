"""Time of the GPU decode of a progressive file whose AC refinement data fills most of the compressed slot.

AC refinement scans decode sequentially (one thread per restart interval), so their worst case is one large refinement
scan without restart intervals.  The file here is a valid 1080x1920 grayscale progressive file: a DC first scan, an AC
first scan of zigzag 1..63 at Al = 1 that sends nothing (one EOB run over every block), then one AC refinement scan of
1..63 under a one-symbol table with a 16-bit code for (run 0, size 1): every coefficient of every block is a 17-bit new
-1.  That is 1071 bits per block, 4.3 MB of entropy data in the 6.2 MB slot.  For comparison, 32 Pillow-written
progressive 480x640 q90 4:2:0 files.

``--sync`` times the worst case of the first-scan self-synchronisation instead (tests/jpeg_craft_progressive.py
``worst_first``): a valid 1080x1920 grayscale file whose AC first scan of zigzag 1..63 is 1071-bit blocks of 17-bit
symbols over all-zero bits, so every bit offset starts a valid symbol and the sync takes one round per subsequence.

``defer_k_jpeg_decode`` (all three kernels) is timed with CUDA events as tools/jpeg_worst_case.py times it; one JSON line
with the card and its power limit.

    python tools/jpeg_progressive_worst_case.py --reps 3
    python tools/jpeg_progressive_worst_case.py --sync --reps 3
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests"), str(ROOT / "tools")]

from defer_b200 import jpeg  # noqa: E402
from ingress_bench import card  # noqa: E402
from jpeg_craft import _seg, one_symbol, pack, stuff  # noqa: E402
from jpeg_worst_case import BOUND, summary, time_decode  # noqa: E402


def _dht(cls: int, t) -> bytes:
    counts, syms = t
    return _seg(0xC4, bytes([cls << 4]) + bytes(counts) + bytes(syms))


def _sos(ss: int, se: int, ah: int, al: int) -> bytes:
    return _seg(0xDA, bytes([1, 1, 0x00, ss, se, (ah << 4) | al]))


def refinement_stream(h: int, w: int) -> bytes:
    blocks = -(-h // 8) * -(-w // 8)
    assert blocks <= 32767
    out = b"\xff\xd8" + _seg(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")
    out += _seg(0xDB, bytes([0]) + bytes([1] * 64))
    out += _seg(0xC2, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([1, 1, 0x11, 0]))
    out += _dht(0, one_symbol(0)) + _sos(0, 0, 0, 0) + stuff(pack("0" * blocks))               # DC differences 0
    out += _dht(1, one_symbol(0xE0)) + _sos(1, 63, 0, 1) + stuff(pack("0" + "1" * 14))         # EOB run of 32767
    out += _dht(1, one_symbol(0x01, 16)) + _sos(1, 63, 1, 0)                                   # 63 new -1 per block
    out += stuff(pack(np.zeros(blocks * 63 * 17, np.uint8)))
    return out + b"\xff\xd9"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sync", action="store_true", help="time the AC first self-synchronisation worst case")
    args = ap.parse_args()
    if args.sync:
        from jpeg_craft_progressive import worst_first
        worst = worst_first(*BOUND, "gray", "ac")[0]
        out = {"card": card(), "bound": f"{BOUND[0]}x{BOUND[1]}", "ac_first_bytes": jpeg.parse(worst).scans[1].length,
               "slot_bytes": BOUND[0] * BOUND[1] * 3,
               "ac_first_sync_1080x1920_x1": summary(*time_decode([worst], args.reps), [worst])}
        print(json.dumps(out))
        return
    from jpeg_bench import files as bench_files
    worst = refinement_stream(*BOUND)
    info = jpeg.parse(worst)
    q90 = bench_files((480, 640), 90, progressive=True)
    out = {"card": card(), "bound": f"{BOUND[0]}x{BOUND[1]}",
           "refinement_bytes": info.scans[-1].length, "slot_bytes": BOUND[0] * BOUND[1] * 3}
    for key, fs in (("refine_1080x1920_x1", [worst]), ("pillow_progressive_480x640_q90_420_x32", q90)):
        out[key] = summary(*time_decode(fs, args.reps), fs)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
