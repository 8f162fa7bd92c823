"""Write the progressive JPEG fixtures of tests/golden/jpeg_progressive/ with Pillow (``progressive=True``), deterministically.

    python tools/make_jpeg_progressive_fixtures.py      # (re)writes tests/golden/jpeg_progressive/*.jpg

The GPU tests read these files, so they need no Pillow.  Names follow tools/make_jpeg_fixtures.py:
<content>_<h>x<w>_<subsampling>_q<quality>[_opt][_rb<blocks>|_rr<rows>].jpg.  Sizes where a component's own block grid is
smaller than its MCU-padded one (a luma width or height of 8k+1..8k+8 under 4:2:x) are included.
"""
from __future__ import annotations

import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))

from make_jpeg_fixtures import content, encode  # noqa: E402

OUT = Path(__file__).resolve().parents[1] / "tests" / "golden" / "jpeg_progressive"


def fixtures():
    """(name, bytes) of every fixture."""
    out = []

    def add(kind, h, w, sub, q, seed=0, tag="", **kw):
        out.append((f"{kind}_{h}x{w}_{sub}_q{q}{tag}.jpg", encode(content(kind, h, w, seed), sub, q, progressive=True, **kw)))
    for i, (h, w) in enumerate([(1, 1), (7, 9), (15, 17), (17, 33), (24, 40)]):
        for sub in ("444", "422", "420", "gray"):
            add("photo", h, w, sub, (5, 50, 75, 95, 100)[(i + len(sub)) % 5], seed=i)
    for sub in ("444", "422", "420", "gray"):
        add("photo", 61, 75, sub, 75, seed=5)
        add("photo", 61, 75, sub, 90, seed=6, tag="_opt", optimize=True)
        add("photo", 61, 75, sub, 75, seed=7, tag="_rb1", restart_marker_blocks=1)
        add("photo", 61, 75, sub, 50, seed=8, tag="_rr1", restart_marker_rows=1)
    add("checker", 31, 47, "420", 95)
    add("photo", 223, 225, "420", 100, seed=9)
    add("photo", 480, 640, "420", 75, seed=11)
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
