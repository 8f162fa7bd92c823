"""Progressive test files the tests share: the committed fixtures and a seeded corpus of corrupt ones.

``corrupt_corpus`` takes Pillow-written progressive fixtures apart at their scans and damages them: bit flips inside a
scan's entropy data, a scan cut short, a DHT segment dropped between scans, RST markers dropped or renumbered.  Every
file it returns still passes ``jpeg.parse``, so its decode is the defined result for corrupt data of ``jpeg.py``."""
from __future__ import annotations

from pathlib import Path
from typing import List, Tuple

import numpy as np

from defer_b200 import jpeg

GOLDEN = Path(__file__).resolve().parent / "golden" / "jpeg_progressive"


def fixture_names() -> List[str]:
    return sorted(p.name for p in GOLDEN.glob("*.jpg"))


def fixture(name: str) -> bytes:
    return (GOLDEN / name).read_bytes()


def _flip(data: bytes, sc: jpeg.Scan, rng) -> bytes:
    a = bytearray(data)
    for _ in range(int(rng.integers(1, 4))):
        i = sc.offset + int(rng.integers(0, max(sc.length, 1)))
        if i >= sc.offset + sc.length:
            continue
        v = a[i] ^ (1 << int(rng.integers(0, 8)))
        if a[i] != 0xFF and v != 0xFF and not (i > 0 and a[i - 1] == 0xFF):     # keep every marker and stuffing
            a[i] = v
    return bytes(a)


def corrupt_corpus(seed: int = 0) -> List[Tuple[str, bytes]]:
    rng = np.random.default_rng(seed)
    out = []
    srcs = ["photo_61x75_420_q75.jpg", "photo_61x75_444_q75_rb1.jpg", "photo_61x75_gray_q50_rr1.jpg",
            "photo_61x75_422_q90_opt.jpg", "photo_223x225_420_q100.jpg"]
    for name in srcs:
        d = fixture(name)
        info = jpeg.parse(d)
        for s, sc in enumerate(info.scans):
            if sc.length > 4:
                out.append((f"{name}: bits flipped in scan {s}", _flip(d, sc, rng)))
        sc = info.scans[int(rng.integers(len(info.scans)))]
        cut = sc.offset + sc.length // 2
        if d[cut - 1] == 0xFF:
            cut -= 1
        out.append((f"{name}: a scan cut in half", d[:cut] + d[sc.offset + sc.length:]))
        for i in (1, 2):                                   # DHT segments between scans
            hits = [k for k in range(len(d) - 1) if d[k] == 0xFF and d[k + 1] == 0xC4 and k > info.scans[0].offset]
            if len(hits) >= i:
                k = hits[-i]
                ln = int.from_bytes(d[k + 2:k + 4], "big")
                out.append((f"{name}: DHT dropped between scans", d[:k] + d[k + 2 + ln:]))
        rst = [k for k in range(info.offset, len(d) - 1) if d[k] == 0xFF and 0xD0 <= d[k + 1] <= 0xD7]
        if rst:
            k = rst[int(rng.integers(len(rst)))]
            out.append((f"{name}: an RST marker dropped", d[:k] + d[k + 2:]))
            out.append((f"{name}: an RST marker renumbered", d[:k + 1] + bytes([0xD0 + (d[k + 1] + 3) % 8]) + d[k + 2:]))
    kept = []
    for nm, f in out:
        try:
            jpeg.parse(f)
        except ValueError:
            continue
        kept.append((nm, f))
    return kept
