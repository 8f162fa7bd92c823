"""PNG decode on the GPU: `defer_k_png_decode` time per 32 files (CUDA events, median of --reps after a warm-up) at
480x640 and 1080x1920, for a photo-like image (Sub-filtered rows, zlib level 6) and a synthetic-noise one
(applications.synthetic_image-like uniform noise, zlib level 6, which stores it), each in a slot of its own size; and the
adversarial stream of tests/png_craft.py (maximal dynamic headers on empty blocks) filling each slot.  Card name and power
limit are read in the same run.  One JSON line.

    python tools/png_bench.py [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import zlib
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import png  # noqa: E402
import png_craft as PC  # noqa: E402
from test_gpu_png import decode_dev, png_photo  # noqa: E402


def noise_png(h: int, w: int, seed: int = 0) -> bytes:
    rng = np.random.default_rng(seed)
    raw = b"".join(b"\0" + rng.integers(0, 256, 3 * w, dtype=np.uint8).tobytes() for _ in range(h))
    z = zlib.compress(raw, 6)
    return PC.png_file(w, h, 8, 2, z, idat_sizes=[8192] * (len(z) // 8192))


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    out = {"card": card, "files_per_call": 32, "ms_per_32": {}, "file_bytes": {}}
    for H, W in ((480, 640), (1080, 1920)):
        cases = {"photo": png_photo(H, W, 1), "noise": noise_png(H, W),
                 "adversarial": PC.adversarial(png.slot_bytes(H, W) - 70000, W, H)}
        for name, d in cases.items():
            key = f"{name}_{H}x{W}"
            want = png.decode_png(d) if name != "adversarial" else None
            (ws, raw_off, y), _ = decode_dev([d] * 32, H, W, timed=True)      # warm-up, and the result is checked
            if want is not None:
                assert np.array_equal(y[0][:H * W * 3].reshape(H, W, 3), want), key
            times = [decode_dev([d] * 32, H, W, timed=True)[1] for _ in range(a.reps if name != "adversarial" else 1)]
            out["ms_per_32"][key] = round(float(np.median(times)), 2)
            out["file_bytes"][key] = len(d)
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
