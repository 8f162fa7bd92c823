"""Cost of JPEG files at ingress: the GPU decode (DEFER(decode="jpeg")) against Pillow's decode on the host.

ResNet50, caffe mode, fp32 parity, one GPU, coalesce=32, depth=4, bilinear resize to 224 x 224.  The JPEGs are encoded
here with Pillow from seeded synthetic photos (gradients, waves and noise), 4:2:0.  It prints one JSON line with:

  decode_op_us        time_op of the JPEG_DECODE op per 32-item microbatch (L2 flushed, median of 3), per
                      (size, quality) for 480x640 and 1080x1920 at q75 and q90, with the mean file size
  pillow_decode_ms    Pillow's decode (Image.open(...).convert("RGB")) of one file, median, in this process
  feeder_us           the feeder's host time per item: marker parse (memoised tables), block packing and the submit call
  rates               end-to-end inferences/s through DEFER (median, min, max over --reps alternated rounds) for
                        jpeg   JPEG files on a full input queue, decode="jpeg", max_image_size=(1080, 1920)
                        u8     the same images decoded before the clock starts, uint8 items, max_image_size=(1080, 1920)
                        f32    the same images decoded, resized and preprocessed before the clock starts, float items
  card                the GPU's name and power limit (read-only nvidia-smi query)

    python tools/jpeg_bench.py --size 480x640 --items 640 --reps 3
    python tools/jpeg_bench.py --progressive ...    # the same with progressive files (Pillow progressive=True)
"""
from __future__ import annotations

import argparse
import io
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from defer_b200 import applications, jpeg  # noqa: E402
from defer_b200.node import StageRunner  # noqa: E402
from ingress_bench import Arm, card, parse_size  # noqa: E402
from make_jpeg_fixtures import content, encode  # noqa: E402

G = 32
BOUND = (1080, 1920)


def files(size, quality, n=G, progressive=False):
    return [encode(content("photo", size[0], size[1], seed=i), "420", quality, progressive=progressive) for i in range(n)]


def decode_op_times(model, items, iters):
    r = StageRunner.from_model(model, device=0, dtype="float32", max_batch=G, depth=1, preprocess="caffe",
                               max_image_size=BOUND, interpolation="bilinear", decode="jpeg")
    try:
        r.predict_jpegs(items)
        ts = [r.time_op(0, iters=iters, flush_l2=True) for _ in range(3)]
        return {"us": round(statistics.median(ts), 1), "spread_us": round(max(ts) - min(ts), 1),
                "mean_file_bytes": int(np.mean([len(d) for d in items])), "kernel": r.op_info(0)["kernel"]}
    finally:
        r.close()


def pillow_ms(items):
    from PIL import Image
    ts = []
    for d in items:
        t = time.perf_counter()
        np.asarray(Image.open(io.BytesIO(d)).convert("RGB"))
        ts.append(time.perf_counter() - t)
    return round(1e3 * statistics.median(ts), 3)


def feeder_us(model, items, reps=20):
    r = StageRunner.from_model(model, device=0, dtype="float32", max_batch=G, depth=2, preprocess="caffe",
                               max_image_size=BOUND, interpolation="bilinear", decode="jpeg")
    try:
        r.submit_jpegs(0, 0, items)                         # memoises the tables
        r.sync()
        t = time.perf_counter()
        for k in range(reps):
            r.submit_jpegs(k, 0, items)
            r.sync()
        return round(1e6 * (time.perf_counter() - t) / (reps * len(items)), 1)
    finally:
        r.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--size", default="480x640", help="HxW of the images of the end-to-end arms")
    ap.add_argument("--quality", type=int, default=90)
    ap.add_argument("--items", type=int, default=640)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--op-iters", type=int, default=20)
    ap.add_argument("--progressive", action="store_true", help="encode every file progressive")
    args = ap.parse_args()
    model = applications.ResNet50()
    out = {"card": card(), "model": "resnet50", "mode": "caffe", "microbatch": G, "progressive": args.progressive,
           "decode_op_us": {}}
    for size in ((480, 640), (1080, 1920)):
        for q in (75, 90):
            items = files(size, q, progressive=args.progressive)
            key = f"{size[0]}x{size[1]}_q{q}"
            out["decode_op_us"][key] = decode_op_times(model, items, args.op_iters)
            out.setdefault("pillow_decode_ms", {})[key] = pillow_ms(items[:8])
            out.setdefault("feeder_us", {})[key] = feeder_us(model, items)
    size = parse_size(args.size)
    base = files(size, args.quality, n=64, progressive=args.progressive)
    jp = [base[i % len(base)] for i in range(args.items)]
    u8 = [jpeg.decode_jpeg(d)[None] for d in base]
    f32 = [applications.preprocess_input(applications.resize_image(x, (224, 224), "bilinear").astype(np.float32))
           for x in u8]
    arms = {"jpeg": (Arm(model, "caffe", None, max_image_size=BOUND, interpolation="bilinear", decode="jpeg"), jp),
            "u8": (Arm(model, "caffe", None, max_image_size=BOUND, interpolation="bilinear"),
                   [u8[i % len(u8)] for i in range(args.items)]),
            "f32": (Arm(model, None, None), [f32[i % len(f32)] for i in range(args.items)])}
    rates = {k: [] for k in arms}
    try:
        for k, (arm, items) in arms.items():                # warm-up round
            arm.rate(items)
        for _ in range(args.reps):
            for k, (arm, items) in arms.items():
                rates[k].append(arm.rate(items))
    finally:
        for arm, _ in arms.values():
            arm.close()
    own = {"jpeg": int(np.mean([len(d) for d in base])), "u8": size[0] * size[1] * 3,  # only the item's own bytes
           "f32": arms["f32"][0].h2d_per_item}
    out["rates"] = {k: {"median": round(statistics.median(v)), "min": round(min(v)), "max": round(max(v)),
                        "h2d_bytes_per_item": own[k]} for k, v in rates.items()}
    out["rates"]["images"] = f"{size[0]}x{size[1]} q{args.quality} 4:2:0"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
