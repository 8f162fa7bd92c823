"""A seeded corpus of corrupt PNG streams: real zlib and crafted streams, truncated, bit-flipped, overwritten and spliced.

``bases()`` are small valid files (a few KB of scanlines) whose streams cover stored, fixed and dynamic blocks: zlib at
levels 0, 1, 6 and 9 and with the Z_RLE, Z_HUFFMAN_ONLY and Z_FIXED strategies, a stream of one stored, one fixed and
one dynamic block written by ``png_craft.BitWriter``, and the crafted valid files of ``png_craft.valid_cases`` of at
most ``MAX_RAW`` scanline bytes.  ``mutants()`` corrupts each base stream and wraps it in a PNG of the base's geometry:
  - truncated at every byte of a stream of at most ``TRUNCATE_ALL`` bytes, and at seeded positions of longer ones;
  - one bit flipped at every bit of its first dynamic block header (block type bits to the last code length);
  - one bit flipped at seeded positions;
  - one to four bytes overwritten with seeded values at seeded positions;
  - spliced: a seeded prefix of the stream followed by a seeded suffix of another base's stream.
The two zlib header bytes are never changed (the parser refuses a bad one before anything is inflated), so every
mutant is a file ``png.parse`` accepts.  The corpus is the same on every run: a fixed seed, and zlib's output for a
fixed input, level and strategy.
"""
from __future__ import annotations

import zlib
from typing import Dict, List, Optional, Tuple

import numpy as np

from defer_b200 import png
import png_craft as PC

MAX_RAW = 4096
TRUNCATE_ALL = 400
SEED = 2026

# (name, w, h, depth, colour type): filter units 3 and 8, at most 2 KB of scanlines
GEOMETRIES = [("rgb8", 24, 20, 8, 2), ("rgba16", 11, 14, 16, 6)]
# (name, level, strategy)
ZLIB = [("z0", 0, zlib.Z_DEFAULT_STRATEGY), ("z1", 1, zlib.Z_DEFAULT_STRATEGY), ("z6", 6, zlib.Z_DEFAULT_STRATEGY),
        ("z9", 9, zlib.Z_DEFAULT_STRATEGY), ("rle", 6, zlib.Z_RLE), ("huff", 6, zlib.Z_HUFFMAN_ONLY),
        ("fixed", 6, zlib.Z_FIXED)]


def _scanlines(w: int, h: int, depth: int, ctype: int, seed: int) -> bytes:
    """Smooth rows with some noise, each with a seeded filter type 0..4: runs and repeats for zlib to match."""
    rng = np.random.default_rng(seed)
    bpr = PC.bytes_per_row(w, depth, ctype)
    x = np.arange(bpr)
    rows = []
    for y in range(h):
        v = (40 * np.sin(x / 7 + y / 5) + 100 + rng.integers(0, 4, bpr)).astype(np.uint8)
        v[rng.random(bpr) < 0.1] = 0
        rows.append(bytes([int(rng.integers(0, 5))]) + v.tobytes())
    return b"".join(rows)


def _compress(raw: bytes, level: int, strategy: int) -> bytes:
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    return c.compress(raw) + c.flush()


def bases() -> Dict[str, Tuple[bytes, Tuple[int, int, int, int]]]:
    """name -> (valid zlib stream, (w, h, depth, colour type)) of every base."""
    out = {}
    for gi, (gname, w, h, depth, ctype) in enumerate(GEOMETRIES):
        raw = _scanlines(w, h, depth, ctype, gi)
        for zname, level, strategy in ZLIB:
            out[f"{gname}_{zname}"] = (_compress(raw, level, strategy), (w, h, depth, ctype))
    w, h, depth, ctype = GEOMETRIES[0][1:]
    raw = _scanlines(w, h, depth, ctype, 7)
    bw = PC.BitWriter()                                               # one block of each type
    bw.stored(raw[:400])
    bw.huffman(list(raw[400:900]))
    bw.huffman(list(raw[900:]), final=True, lit_lens=PC.lit_lengths_for(raw[900:]), dist_lens=[1])
    out["mixed_blocks"] = (bw.zlib(raw), (w, h, depth, ctype))
    seen = {s for s, _ in out.values()}
    for name, d in sorted(PC.valid_cases().items()):
        info = png.parse(d)
        s = png.gather(d, info)
        if info.raw_bytes <= MAX_RAW and s not in seen:              # the same stream in other IDAT chunks: once
            seen.add(s)
            out[f"crafted_{name}"] = (s, (info.w, info.h, info.depth, info.ctype))
    return out


def first_dynamic_header(stream: bytes) -> Optional[Tuple[int, int]]:
    """Bit range [start, end) of the stream's first block, from its type bits to its last code length, when that block
    is dynamic."""
    r = png._Bits(stream)
    start = r.pos
    r.take(1)
    if r.take(2) != 2:
        return None
    png._dynamic(r)
    return start, r.pos


def _flip(s: bytes, bit: int) -> bytes:
    b = bytearray(s)
    b[bit >> 3] ^= 1 << (bit & 7)
    return bytes(b)


def mutants() -> List[Tuple[str, bytes]]:
    """(name, PNG file) of every mutant, in a fixed order."""
    rng = np.random.default_rng(SEED)
    bs = bases()
    names = sorted(bs)
    out = []
    for name in names:
        s, (w, h, depth, ctype) = bs[name]
        n = len(s)
        ms: List[Tuple[str, bytes]] = []
        cuts = range(2, n) if n <= TRUNCATE_ALL else sorted(set(rng.integers(2, n, 48).tolist()))
        ms += [(f"cut{k}", s[:k]) for k in cuts]
        hdr = first_dynamic_header(s)
        if hdr is not None:
            ms += [(f"hdrflip{b}", _flip(s, b)) for b in range(*hdr)]
        ms += [(f"flip{b}", _flip(s, b)) for b in sorted(set(rng.integers(16, 8 * n, 48).tolist()))]
        for _ in range(24):
            k = int(rng.integers(1, 5))
            p = int(rng.integers(2, max(3, n - k)))
            b = bytearray(s)
            b[p:p + k] = rng.integers(0, 256, k, dtype=np.uint8).tobytes()
            ms.append((f"over{p}x{k}", bytes(b[:n])))
        for _ in range(12):
            other, _g = bs[names[int(rng.integers(0, len(names)))]]
            p, q = int(rng.integers(2, n + 1)), int(rng.integers(2, len(other) + 1))
            ms.append((f"splice{p}+{q}", s[:p] + other[q:]))
        out += [(f"{name}/{k}", PC.png_file(w, h, depth, ctype, m)) for k, m in ms]
    return out
