"""Step time of one model on one GPU, with the AFFINE fold on and off (DEFER_FOLD_AFFINE), by bench.py's flooded window.

One single-stage pipeline per arm (224 x 224, synthetic weights, --batch images per launch, --depth lanes), the inputs
resident in the stage's slots.  Each round steps every arm in turn: pre-flood 2 x depth microbatches, --warmup more,
then --steps timed ones between CUDA events recorded behind microbatch warmup-1 and warmup+steps-1, then a tail of depth
microbatches so the lanes stay busy past the window.  The folded and unfolded arms of one model and dtype are alive
together and alternated over --reps rounds; the JSON line reports the
median, min and max ms per microbatch of each arm, the images/s of the median, and the card's name and power limit.

Arms: ResNet50 (V1, nothing to fold) and ResNet50V2 / ResNet152V2 folded and unfolded, fp32 parity and bf16.

    python tools/model_bench.py [--models ResNet50,ResNet50V2,ResNet152V2] [--batch 32] [--steps 40] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from defer_b200 import applications  # noqa: E402
from defer_b200.node import StageRunner  # noqa: E402
from ingress_bench import card  # noqa: E402


def flooded_ms(r, x, depth, warmup, steps, seq0):
    """ms per microbatch of `steps` back-to-back microbatches, at most `depth` in flight, inputs already resident."""
    P, T = 2 * depth, depth
    total = P + warmup + steps + T
    r.mark_after(seq0 + P + warmup - 1, 0)
    r.mark_after(seq0 + P + warmup + steps - 1, 1)
    out = np.empty(r.out_shape, np.float32)
    for s in range(seq0, seq0 + total):
        if s - seq0 >= depth:
            r.result(s - depth, out)
        r.step(s)
    for s in range(seq0 + total - depth, seq0 + total):
        r.result(s, out)
    r.status()
    return r.mark_elapsed_ms() / steps, seq0 + total


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--models", default="ResNet50,ResNet50V2,ResNet152V2")
    ap.add_argument("--dtypes", default="float32,bfloat16")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--depth", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    x = applications.synthetic_input(args.batch, seed=1)
    res = {}
    for name in args.models.split(","):
        model = getattr(applications, name)()
        for dtype in args.dtypes.split(","):
            arms = {}                                              # the arms of one model and dtype are alive together
            for fold in ((1,) if not name.endswith("V2") else (1, 0)):
                os.environ["DEFER_FOLD_AFFINE"] = str(fold)        # read when the stage is created
                r = StageRunner.from_model(model, device=0, dtype=dtype, max_batch=args.batch, depth=args.depth)
                folded = sum(r.op_info(i)["kernel"].startswith("affine (fused") for i in range(len(r.plan.ops)))
                for d in range(args.depth):
                    r.submit(d, x)                                 # slot d % depth, stays there
                r.sync()
                arms[f"{name}/{dtype}/fold{fold}"] = {"runner": r, "seq": args.depth, "ms": [], "folded_ops": folded,
                                                      "kernels_per_step": r.num_kernels()}
            os.environ.pop("DEFER_FOLD_AFFINE", None)
            for rep in range(args.reps + 1):                       # round 0 warms every arm up and is not recorded
                for a in arms.values():
                    ms, a["seq"] = flooded_ms(a["runner"], x, args.depth, args.warmup, args.steps, a["seq"])
                    if rep:
                        a["ms"].append(ms)
            for k, a in arms.items():
                med = statistics.median(a["ms"])
                res[k] = {"ms_per_step_median": round(med, 4), "ms_min": round(min(a["ms"]), 4),
                          "ms_max": round(max(a["ms"]), 4), "images_per_s": round(args.batch * 1000.0 / med, 1),
                          "folded_affine_ops": a["folded_ops"], "kernels_per_step": a["kernels_per_step"]}
                a["runner"].close()
    print(json.dumps({"metric": "flooded step time, one GPU, one stage", "batch": args.batch, "depth": args.depth,
                      "steps": args.steps, "reps": args.reps, **card(), "arms": res}))


if __name__ == "__main__":
    main()
