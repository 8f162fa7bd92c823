"""Ingress cost of Keras preprocessing: host fp32 items vs uint8 items preprocessed on the GPU.

One GPU, ResNet50 in caffe mode or ResNet50V2 in tf mode (224 x 224, synthetic weights, fp32 parity), DEFER.run_defer
with coalesce=32 and depth=4.  Three arms, each a live pipeline, timed in alternation (--reps rounds after one warm-up
round):

  a  fp32 items, already preprocessed before the clock starts, put on a full input queue
  b  uint8 items, the host preprocessing function in the feeding thread (what a reference-style driver does):
     applications.preprocess_input (caffe) or applications.resnet_v2_preprocess_input (tf)
  c  uint8 items on a full input queue, DEFER(preprocess=mode): the first stage preprocesses on the GPU

With --image-size HxW (and --interpolation NAME, default nearest) the items are uint8 frames of that size, as a camera
gives them, and two more arms run in the same alternation:

  d  uint8 frames, Pillow's Image.resize to 224 x 224 in the feeding thread (Keras load_img's resize, what a
     reference-style driver does), DEFER(preprocess=mode)
  e  uint8 frames on a full input queue, DEFER(preprocess=mode, image_size=..., interpolation=...): the first stage
     resizes and preprocesses on the GPU

With --mixed-sizes HxW,HxW,... one more arm runs in the alternation:

  f  uint8 frames cycling through those sizes on a full input queue, DEFER(preprocess=mode, max_image_size=the largest,
     interpolation=...): each frame is resized on the GPU from its own size, frames of different sizes share a microbatch

It prints one JSON line: end-to-end inferences/s per arm (median, min, max over the rounds), H2D bytes per item, the
device time of the fp32 fused stem, the uint8 fused stem of the mode and its standalone preprocessing kernel (time_op,
L2 flushed), the host time of one preprocessing call, and the card's name and power limit (read-only nvidia-smi query);
with --image-size also the host time of one Pillow resize and the time_op of each RESIZE op at 32 frames; with
--mixed-sizes the time_op of the two per-sample RESIZE ops at 32 mixed frames and at 32 frames of the first size (under
a bound of that size), and arm f's H2D bytes per item (the image's own bytes plus its table block).  With --crop-sizes
HxW,HxW,... the time_op of each RESIZE op at 32 frames of each size, with keep_aspect_ratio off and on (the crop arm).

    python tools/ingress_bench.py [--model resnet50 --preprocess caffe] [--items 640] [--reps 3]
    python tools/ingress_bench.py --model resnet50v2 --preprocess tf
    python tools/ingress_bench.py --image-size 480x640 --interpolation bilinear
    python tools/ingress_bench.py --image-size 480x640 --mixed-sizes 480x640,720x1280,1080x1920
    python tools/ingress_bench.py --crop-sizes 480x640,640x480,1080x1920,1920x1080 --interpolation bilinear
"""
from __future__ import annotations

import argparse
import json
import os
import queue
import statistics
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from defer_b200 import applications  # noqa: E402
from defer_b200.dispatcher import DEFER  # noqa: E402
from defer_b200.node import StageRunner  # noqa: E402
from defer_b200.resize import frame_block_ints  # noqa: E402

G, DEPTH = 32, 4
MODELS = {"resnet50": applications.ResNet50, "resnet50v2": applications.ResNet50V2}
HOST_PREPROCESS = {"caffe": applications.preprocess_input, "tf": applications.resnet_v2_preprocess_input}
# mode -> (fused uint8 stem kernel, standalone preprocessing kernel)
KERNELS = {"caffe": ("conv_stem_u8_kernel", "preprocess_kernel"), "tf": ("conv_stem_u8tf_kernel", "preprocess_tf_kernel")}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = out[0].rsplit(",", 1)
        return {"gpu": name.strip(), "power_limit": power.strip()}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": f"unknown ({e})"}


class Arm:
    def __init__(self, model, preprocess, host_preprocess, **defer_kw):
        self.host_preprocess = host_preprocess
        self.defer = DEFER([0], depth=DEPTH, coalesce=G, linger_us=2000, preprocess=preprocess, **defer_kw)
        self.in_q, self.out_q = queue.Queue(), queue.Queue()
        self.err = []
        self.thread = threading.Thread(target=self._run, args=(model,), daemon=True)
        self.thread.start()
        if not self.defer.wait_ready(600) or self.err:
            raise RuntimeError(f"pipeline did not come up: {self.err}")
        st = self.defer.stages[0]
        self.h2d_per_item = st.io_bytes()[0] // st.batch

    def _run(self, model):
        try:
            self.defer.run_defer(model, [], self.in_q, self.out_q)
        except BaseException as e:  # noqa: BLE001
            self.err.append(e)

    def rate(self, items, host_preprocess=False):
        """Inferences/s from the first put to the last result."""
        t0 = time.perf_counter()
        if host_preprocess:
            def feed():
                for x in items:
                    self.in_q.put(self.host_preprocess(x))
            f = threading.Thread(target=feed, daemon=True)
            f.start()
        else:
            for x in items:
                self.in_q.put(x)
        for _ in items:
            self.out_q.get(timeout=300)
        dt = time.perf_counter() - t0
        if host_preprocess:
            f.join()
        if self.err:
            raise RuntimeError(self.err)
        return len(items) / dt

    def close(self):
        self.defer.close()
        self.thread.join(timeout=60)


def stem_times(model, mode, iters):
    """time_op (us) of the three stem kernels at the benchmarked microbatch (32 images)."""
    out = {}
    stem_u8, pre_kernel = KERNELS[mode]
    for key, env, pre, op in (("conv_stem_kernel_f32_us", None, None, 0), (f"{stem_u8}_us", None, mode, 1),
                              (f"{pre_kernel}_us", "0", mode, 0)):
        old = os.environ.pop("DEFER_STEM_FUSED", None)
        if env is not None:
            os.environ["DEFER_STEM_FUSED"] = env
        try:
            r = StageRunner.from_model(model, device=0, dtype="float32", max_batch=G, depth=1, preprocess=pre)
        finally:
            os.environ.pop("DEFER_STEM_FUSED", None)
            if old is not None:
                os.environ["DEFER_STEM_FUSED"] = old
        try:
            kernel = r.op_info(op)["kernel"]
            if key != "conv_stem_kernel_f32_us" and kernel != key[:-3]:
                raise RuntimeError(f"{key}: op {op} runs {kernel}")
            r.predict(applications.synthetic_image(G, seed=1) if pre else applications.synthetic_input(G, seed=1))
            ts = [r.time_op(op, iters=iters, flush_l2=True) for _ in range(3)]
            out[key] = {"kernel": kernel, "us": round(statistics.median(ts), 2), "spread_us": round(max(ts) - min(ts), 2)}
        finally:
            r.close()
    return out


def pillow_resize(size, interpolation):
    """Keras load_img's resize of one (1, h, w, 3) uint8 item to ``size`` through Pillow, as a feeding thread does it."""
    from PIL import Image
    method = getattr(Image, interpolation.upper())

    def fn(x):
        return np.asarray(Image.fromarray(x[0]).resize((size[1], size[0]), method))[None]
    return fn


def resize_times(model, mode, image_size, interpolation, iters, keep_aspect_ratio=False):
    """time_op (us) of each RESIZE op at the benchmarked microbatch (32 frames), L2 flushed."""
    r = StageRunner.from_model(model, device=0, dtype="float32", max_batch=G, depth=1, preprocess=mode,
                               image_size=image_size, interpolation=interpolation, keep_aspect_ratio=keep_aspect_ratio)
    out = {}
    try:
        r.predict(applications.synthetic_image(G, image_size + (3,), seed=1))
        for i, op in enumerate(r.plan.ops):
            if r.op_info(i)["kernel"] != "resize_u8_kernel":
                continue
            ts = [r.time_op(i, iters=iters, flush_l2=True) for _ in range(3)]
            out[op.layers[0]] = {"us": round(statistics.median(ts), 2), "spread_us": round(max(ts) - min(ts), 2),
                                 "alg_bytes": r.op_info(i)["alg_bytes"]}
    finally:
        r.close()
    return out


def frames_times(model, mode, bound, sizes, interpolation, iters):
    """time_op (us) of the two per-sample RESIZE ops at 32 frames cycling through ``sizes`` under ``bound``, L2 flushed."""
    r = StageRunner.from_model(model, device=0, dtype="float32", max_batch=G, depth=1, preprocess=mode,
                               max_image_size=bound, interpolation=interpolation)
    out = {"bound": list(bound), "sizes": [list(v) for v in sizes]}
    try:
        r.predict_frames([applications.synthetic_image(1, sizes[i % len(sizes)] + (3,), seed=i) for i in range(G)])
        for i, op in enumerate(r.plan.ops[:2]):
            ts = [r.time_op(i, iters=iters, flush_l2=True) for _ in range(3)]
            out[op.layers[0]] = {"kernel": r.op_info(i)["kernel"], "us": round(statistics.median(ts), 2),
                                 "spread_us": round(max(ts) - min(ts), 2), "alg_bytes_bound": r.op_info(i)["alg_bytes"]}
    finally:
        r.close()
    return out


def parse_size(text):
    h, w = (int(v) for v in text.lower().split("x"))
    if min(h, w) < 1:
        raise ValueError(text)
    return h, w


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--items", type=int, default=640, help="queue items per timed round (batch-1 images)")
    ap.add_argument("--reps", type=int, default=3, help="timed rounds per arm (alternated), >= 3")
    ap.add_argument("--op-iters", type=int, default=50)
    ap.add_argument("--model", choices=sorted(MODELS), default="resnet50")
    ap.add_argument("--preprocess", choices=sorted(HOST_PREPROCESS), default="caffe",
                    help="Keras preprocessing mode (the model's own: caffe for resnet50, tf for resnet50v2)")
    ap.add_argument("--image-size", default=None, help="HxW of uint8 frames for arms d and e, e.g. 480x640")
    ap.add_argument("--interpolation", choices=applications.INTERPOLATIONS, default="nearest")
    ap.add_argument("--mixed-sizes", default=None, help="HxW,HxW,... of uint8 frames for arm f, e.g. 480x640,720x1280")
    ap.add_argument("--crop-sizes", default=None,
                    help="HxW,HxW,...: time the RESIZE ops of each size with keep_aspect_ratio off and on, then exit")
    args = ap.parse_args()
    if args.reps < 3:
        ap.error("--reps must be >= 3")
    image_size = None
    if args.image_size:
        try:
            image_size = tuple(int(v) for v in args.image_size.lower().split("x"))
            assert len(image_size) == 2 and min(image_size) >= 1
        except (ValueError, AssertionError):
            ap.error(f"--image-size {args.image_size!r}: expected HxW, e.g. 480x640")
    mixed = None
    if args.mixed_sizes:
        try:
            mixed = [parse_size(v) for v in args.mixed_sizes.split(",")]
        except ValueError:
            ap.error(f"--mixed-sizes {args.mixed_sizes!r}: expected HxW,HxW,..., e.g. 480x640,720x1280")
        bound = (max(h for h, _ in mixed), max(w for _, w in mixed))

    model = MODELS[args.model]()
    if args.crop_sizes:
        try:
            crops = [parse_size(v) for v in args.crop_sizes.split(",")]
        except ValueError:
            ap.error(f"--crop-sizes {args.crop_sizes!r}: expected HxW,HxW,..., e.g. 480x640,1080x1920")
        res = {"metric": f"{args.model}_resize_time_op_us", "preprocess": args.preprocess, "frames": G,
               "interpolation": args.interpolation,
               "crop_time_op": {f"{h}x{w}": {k: resize_times(model, args.preprocess, (h, w), args.interpolation,
                                                             args.op_iters, keep_aspect_ratio=keep)
                                             for k, keep in (("off", False), ("keep_aspect_ratio", True))}
                                for h, w in crops}}
        res.update(card())
        print(json.dumps(res), flush=True)
        return
    host_fn = HOST_PREPROCESS[args.preprocess]
    imgs = [applications.synthetic_image(1, seed=i) for i in range(args.items)]
    pre = [host_fn(x) for x in imgs]

    t0 = time.perf_counter()
    n_host = 200
    for i in range(n_host):
        host_fn(imgs[i % len(imgs)])
    host_us = (time.perf_counter() - t0) / n_host * 1e6

    arms = {"a_f32_items": Arm(model, None, host_fn), "b_u8_host_preprocess": Arm(model, None, host_fn),
            "c_u8_gpu_preprocess": Arm(model, args.preprocess, host_fn)}
    feeds = {"a_f32_items": (pre, False), "b_u8_host_preprocess": (imgs, True), "c_u8_gpu_preprocess": (imgs, False)}
    if image_size is not None:
        frames = [applications.synthetic_image(1, image_size + (3,), seed=i) for i in range(args.items)]
        resize_fn = pillow_resize((224, 224), args.interpolation)
        t0 = time.perf_counter()
        for i in range(n_host):
            resize_fn(frames[i % len(frames)])
        resize_us = (time.perf_counter() - t0) / n_host * 1e6
        arms["d_u8_host_resize"] = Arm(model, args.preprocess, resize_fn)
        arms["e_u8_gpu_resize"] = Arm(model, args.preprocess, None, image_size=image_size, interpolation=args.interpolation)
        feeds["d_u8_host_resize"] = (frames, True)
        feeds["e_u8_gpu_resize"] = (frames, False)
    if mixed is not None:
        mixed_frames = [applications.synthetic_image(1, mixed[i % len(mixed)] + (3,), seed=i) for i in range(args.items)]
        arms["f_u8_gpu_resize_mixed"] = Arm(model, args.preprocess, None, max_image_size=bound,
                                            interpolation=args.interpolation)
        feeds["f_u8_gpu_resize_mixed"] = (mixed_frames, False)
    rates = {k: [] for k in arms}
    try:
        for rnd in range(args.reps + 1):
            for k, arm in arms.items():
                items, host = feeds[k]
                r = arm.rate(items, host_preprocess=host)
                if rnd > 0:                                   # round 0 warms every shape up
                    rates[k].append(r)
        h2d = {k: arm.h2d_per_item for k, arm in arms.items()}
        if mixed is not None:                                 # only the image's own bytes cross, plus its block
            plan = arms["f_u8_gpu_resize_mixed"].defer.stages[0].plan.frames
            block = frame_block_ints(plan["target"], plan["kw"]) * 4
            h2d["f_u8_gpu_resize_mixed"] = round(statistics.mean(x.nbytes for x in mixed_frames) + block, 1)
    finally:
        for arm in arms.values():
            arm.close()

    res = {
        "metric": f"{args.model}_ingress_inferences_per_s", "preprocess": args.preprocess,
        "coalesce": G, "depth": DEPTH, "items_per_round": args.items, "rounds": args.reps,
        "arms": {k: {"median": round(statistics.median(v), 1), "min": round(min(v), 1), "max": round(max(v), 1),
                     "all": [round(x, 1) for x in v], "h2d_bytes_per_item": h2d[k]} for k, v in rates.items()},
        "host_preprocess_input_us": round(host_us, 1),
        "stem_time_op": stem_times(model, args.preprocess, args.op_iters),
    }
    if image_size is not None:
        res.update({"image_size": list(image_size), "interpolation": args.interpolation,
                    "host_pillow_resize_us": round(resize_us, 1),
                    "resize_time_op": resize_times(model, args.preprocess, image_size, args.interpolation, args.op_iters)})
    if mixed is not None:
        res.update({"mixed_sizes": [list(v) for v in mixed], "max_image_size": list(bound),
                    "frames_time_op": {"mixed": frames_times(model, args.preprocess, bound, mixed, args.interpolation,
                                                             args.op_iters),
                                       "uniform": frames_times(model, args.preprocess, mixed[0], mixed[:1],
                                                               args.interpolation, args.op_iters)}})
        if image_size is None:
            res["interpolation"] = args.interpolation
    res.update(card())
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
