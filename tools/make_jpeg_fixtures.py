"""Write the JPEG fixtures of tests/golden/jpeg/ with Pillow, deterministically (seeded content, fixed encoder options).

    python tools/make_jpeg_fixtures.py            # (re)writes tests/golden/jpeg/*.jpg

The GPU tests read these files, so they need no Pillow.  Each name says what the file covers:
<content>_<h>x<w>_<subsampling>_q<quality>[_opt][_rb<blocks>|_rr<rows>][_meta].jpg.  Encoders other than this Pillow /
libjpeg-turbo may produce other bytes for the same options; the tests compare the GPU decode with the host restatement of
these bytes, so the files need not be reproduced exactly.
"""
from __future__ import annotations

import io
import sys
from pathlib import Path

import numpy as np

OUT = Path(__file__).resolve().parents[1] / "tests" / "golden" / "jpeg"
SUBS = {"444": 0, "422": 1, "420": 2, "gray": None}


def content(kind: str, h: int, w: int, seed: int) -> np.ndarray:
    """uint8 RGB: 'photo' (gradients, waves and some noise), 'zero', 'full' (255) or 'checker' (0 / 255 pixels)."""
    if kind == "zero":
        return np.zeros((h, w, 3), np.uint8)
    if kind == "full":
        return np.full((h, w, 3), 255, np.uint8)
    if kind == "checker":
        c = ((np.arange(h)[:, None] + np.arange(w)[None, :]) & 1) * 255
        return np.repeat(c[:, :, None], 3, axis=2).astype(np.uint8)
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([128 + 100 * np.sin(x / (7 + c * 5) + y / (11 + c * 3) + c) for c in range(3)], axis=2)
    img += 60 * (x / max(w - 1, 1) - 0.5)[..., None] + rng.normal(0, 12, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def encode(img: np.ndarray, sub: str, quality: int, **kw) -> bytes:
    from PIL import Image
    im = Image.fromarray(img)
    if sub == "gray":
        im = im.convert("L")
    else:
        kw["subsampling"] = SUBS[sub]
    b = io.BytesIO()
    im.save(b, "JPEG", quality=quality, **kw)
    return b.getvalue()


def fixtures():
    """(name, bytes) of every fixture."""
    out = []

    def add(kind, h, w, sub, q, seed=0, tag="", **kw):
        name = f"{kind}_{h}x{w}_{sub}_q{q}{tag}.jpg"
        out.append((name, encode(content(kind, h, w, seed), sub, q, **kw)))
    sizes = [(1, 1), (1, 17), (3, 5), (5, 4), (7, 9), (15, 17), (16, 16), (17, 33)]
    for i, (h, w) in enumerate(sizes):
        for sub in SUBS:
            add("photo", h, w, sub, (5, 50, 75, 95, 100)[(i + len(sub)) % 5], seed=i)
    for sub in SUBS:
        for q in (5, 50, 75, 95, 100):
            add("photo", 223, 225, sub, q, seed=q)
        add("photo", 223, 225, sub, 75, seed=7, tag="_opt", optimize=True)
        add("photo", 223, 225, sub, 75, seed=8, tag="_rb1", restart_marker_blocks=1)
        add("photo", 223, 225, sub, 90, seed=9, tag="_rb4", restart_marker_blocks=4)
        add("photo", 223, 225, sub, 50, seed=10, tag="_rr1", restart_marker_rows=1)
        for kind in ("zero", "full", "checker"):
            add(kind, 31, 47, sub, 95)
    add("photo", 480, 640, "420", 75, seed=11)
    add("photo", 480, 640, "422", 90, seed=12, tag="_rr1", restart_marker_rows=1)
    add("photo", 1080, 1920, "420", 50, seed=13)
    exif = b"Exif\0\0MM\0*\0\0\0\x08\0\0" + b"\0" * 40
    icc = b"\0\0\x01\x00ICC-fixture" + bytes(range(256)) * 2
    add("photo", 40, 60, "420", 75, seed=14, tag="_meta", exif=exif, icc_profile=icc, comment=b"a comment segment")
    return out


def main() -> None:
    OUT.mkdir(parents=True, exist_ok=True)
    for old in OUT.glob("*.jpg"):
        old.unlink()
    total = 0
    for name, data in fixtures():
        (OUT / name).write_bytes(data)
        total += len(data)
    print(f"{len(fixtures())} files, {total} bytes in {OUT}", file=sys.stderr)


if __name__ == "__main__":
    main()
