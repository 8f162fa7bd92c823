"""Write the PNG fixtures of tests/golden/png/ with zlib (and Pillow for one file), deterministically (seeded content,
fixed encoder options).

    python tools/make_png_fixtures.py            # (re)writes tests/golden/png/*.png

The GPU tests read these files, so they need no Pillow.  Each name says what the file covers:
<content>_<h>x<w>_c<colour type>_d<bit depth>[_f<filter>][_z<level><strategy>][_p<palette entries>].png.  The scanlines
are filtered here (each row's filter type drawn at random unless ``_f`` names one) and compressed by zlib at the level
and strategy named (default level 6); ``pillow_`` files are written by Pillow itself.  Other zlib builds may produce
other bytes; the tests compare the GPU decode with the host restatement of these bytes and Pillow with that, so the files
need not be reproduced exactly.
"""
from __future__ import annotations

import io
import struct
import sys
import zlib
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
OUT = ROOT / "tests" / "golden" / "png"
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
STRATEGIES = {"": zlib.Z_DEFAULT_STRATEGY, "fixed": zlib.Z_FIXED, "huff": zlib.Z_HUFFMAN_ONLY, "rle": zlib.Z_RLE}


def photo(h: int, w: int, seed: int, noise: float = 12.0) -> np.ndarray:
    """float64 [h, w, 3] in 0..1: gradients, waves and some noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([128 + 100 * np.sin(x / (7 + c * 5) + y / (11 + c * 3) + c) for c in range(3)], axis=2)
    img += 60 * (x / max(w - 1, 1) - 0.5)[..., None] + rng.normal(0, noise, (h, w, 3))
    return np.clip(img / 255.0, 0, 1)


def samples(h: int, w: int, ctype: int, depth: int, seed: int, noise: float) -> np.ndarray:
    """uint16 [h, w, channels] samples of the given depth: the photo in grey / RGB, a ramp for alpha, random indices."""
    top = (1 << depth) - 1
    rng = np.random.default_rng(seed)
    img = photo(h, w, seed, noise)
    if ctype == 3:
        return rng.integers(0, top + 1, (h, w, 1)).astype(np.uint16)
    grey = img.mean(axis=2, keepdims=True)
    alpha = (np.arange(w)[None, :, None] / max(w - 1, 1)).repeat(h, axis=0)
    chans = {0: [grey], 2: [img], 4: [grey, alpha], 6: [img, alpha]}[ctype]
    return np.round(np.concatenate(chans, axis=2) * top).astype(np.uint16)


def pack_rows(s: np.ndarray, depth: int) -> np.ndarray:
    """uint8 [h, bytes per row]: samples packed MSB first (16 bits big-endian)."""
    h = s.shape[0]
    flat = s.reshape(h, -1)
    if depth == 16:
        return np.stack([flat >> 8, flat & 255], axis=2).reshape(h, -1).astype(np.uint8)
    if depth == 8:
        return flat.astype(np.uint8)
    per = 8 // depth
    n = flat.shape[1]
    pad = np.zeros((h, -(-n // per) * per), np.uint16)
    pad[:, :n] = flat
    v = pad.reshape(h, -1, per)
    out = np.zeros(v.shape[:2], np.uint16)
    for k in range(per):
        out |= v[:, :, k] << (8 - depth * (k + 1))
    return out.astype(np.uint8)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(rows: np.ndarray, bpp: int, types) -> bytes:
    out = []
    prev = np.zeros(rows.shape[1], np.int32)
    for r, ft in zip(rows.astype(np.int32), types):
        left = np.concatenate([np.zeros(bpp, np.int32), r[:-bpp]]) if len(r) > bpp else np.zeros_like(r)
        ul = np.concatenate([np.zeros(bpp, np.int32), prev[:-bpp]]) if len(r) > bpp else np.zeros_like(r)
        pred = [0, left, prev, (left + prev) >> 1, _paeth(left, prev, ul)][ft]
        out.append(bytes([ft]) + ((r - pred) & 255).astype(np.uint8).tobytes())
        prev = r
    return b"".join(out)


def chunk(kind: bytes, body: bytes) -> bytes:
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))


def encode(h: int, w: int, ctype: int, depth: int, seed: int, filt=None, level: int = 6, strategy: str = "",
           npal: int = 0, idat: int = 8192, noise: float = 3.0) -> bytes:
    s = samples(h, w, ctype, depth, seed, noise)
    rows = pack_rows(s, depth)
    bpp = max(1, CHANNELS[ctype] * depth // 8)
    rng = np.random.default_rng(seed + 1)
    types = [filt] * h if filt is not None else rng.integers(0, 5, h).tolist()
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, STRATEGIES[strategy])
    z = c.compress(filter_rows(rows, bpp, types)) + c.flush()
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, 0))
    if ctype == 3:
        out += chunk(b"PLTE", rng.integers(0, 256, 3 * npal, dtype=np.uint8).tobytes())
    out += chunk(b"tEXt", b"Comment\0fixture")
    for p in range(0, len(z), idat):
        out += chunk(b"IDAT", z[p:p + idat])
    return out + chunk(b"IEND", b"")


def fixtures() -> dict:
    out = {}
    seed = 0
    for ctype, depths in DEPTHS.items():
        for depth in depths:
            for h, w in ((1, 1), (1, 17), (7, 9), (63, 65)):
                seed += 1
                npal = (1 << depth) if depth < 8 else 256
                for np_ in ((npal, max(1, npal // 2 - 1)) if ctype == 3 else (0,)):
                    name = f"photo_{h}x{w}_c{ctype}_d{depth}" + (f"_p{np_}" if ctype == 3 else "")
                    out[name] = encode(h, w, ctype, depth, seed, npal=np_)
    for ft in range(5):
        out[f"photo_223x225_c2_d8_f{ft}"] = encode(223, 225, 2, 8, 100 + ft, filt=ft)
        out[f"noise_23x25_c2_d8_f{ft}"] = encode(23, 25, 2, 8, 105 + ft, filt=ft, noise=80.0)
        out[f"photo_31x47_c0_d2_f{ft}"] = encode(31, 47, 0, 2, 110 + ft, filt=ft)
        out[f"photo_31x47_c6_d16_f{ft}"] = encode(31, 47, 6, 16, 120 + ft, filt=ft)
    for level in (0, 1, 9):
        out[f"photo_63x65_c2_d8_z{level}"] = encode(63, 65, 2, 8, 130 + level, level=level)
    for strat in ("fixed", "huff", "rle"):
        out[f"photo_63x65_c2_d8_z6{strat}"] = encode(63, 65, 2, 8, 140, strategy=strat)
        out[f"photo_63x65_c3_d8_z6{strat}_p256"] = encode(63, 65, 3, 8, 141, strategy=strat, npal=256)
    # Pillow's own writer (its IDAT chunk size and zlib settings), RGB and palette
    from PIL import Image
    img = (photo(60, 80, 160) * 255).astype(np.uint8)
    for mode in ("RGB", "P"):
        b = io.BytesIO()
        im = Image.fromarray(img)
        (im.quantize(200) if mode == "P" else im).save(b, format="PNG")
        out[f"pillow_60x80_{mode.lower()}"] = b.getvalue()
    return out


def main() -> int:
    OUT.mkdir(parents=True, exist_ok=True)
    for old in OUT.glob("*.png"):
        old.unlink()
    total = 0
    for name, data in fixtures().items():
        (OUT / f"{name}.png").write_bytes(data)
        total += len(data)
    print(f"wrote {len(list(OUT.glob('*.png')))} files, {total} bytes, to {OUT}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
