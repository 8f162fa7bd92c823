"""SHA-256 fingerprints of what the resize options produce at their defaults: `resize_tables` over a sweep of sizes,
`pack_frame_tables` blocks, and whole `plan_stage` plans (ops, buffers, weights) with `image_size=`, `max_image_size=` and
`decode="jpeg"`.  Only the API that existed before `keep_aspect_ratio` is used, so the same code fingerprints an older
tree: `tests/golden/resize_default_fingerprints.json` holds the fingerprints of the tree before `keep_aspect_ratio` was
added, and `test_resize_keep_aspect_host.py` checks that the defaults still give them.

    python tests/resize_fingerprints.py OUT.json     # with the tree to fingerprint first on PYTHONPATH
"""
import hashlib
import json
import sys

import numpy as np

TABLE_IN = [1, 2, 3, 5, 7, 31, 100, 223, 224, 225, 299, 480, 640, 1080, 1920]
TABLE_OUT = [1, 3, 32, 224, 299]
BLOCK_SIZES = [(480, 640), (300, 200), (224, 224), (224, 500), (100, 224), (7, 3), (1, 1), (480, 1), (1, 640)]
PLAN_CONFIGS = [
    {"image_size": (48, 40), "interpolation": "bilinear"},
    {"image_size": (32, 100)},
    {"image_size": (7, 32), "interpolation": "box"},
    {"image_size": (32, 32), "interpolation": "lanczos"},
    {"image_size": (1080, 1920), "interpolation": "bicubic"},
    {"max_image_size": (48, 40), "interpolation": "bicubic"},
    {"max_image_size": (32, 32)},
    {"max_image_size": (480, 640), "interpolation": "hamming", "decode": "jpeg"},
]


def _digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(f"{a.dtype.str}{a.shape}".encode())
        h.update(a.tobytes())
    return h.hexdigest()


def _plan_digest(plan) -> str:
    ops = [(o.kind, o.in0, o.in1, o.out, o.kh, o.kw, o.sh, o.sw, tuple(o.pads), o.flags, o.w_kernel, o.w_scale, o.w_shift,
            o.mode, tuple(o.layers)) for o in plan.ops]
    frames = None if plan.frames is None else sorted((k, repr(v)) for k, v in plan.frames.items())
    head = repr((plan.bufs, ops, plan.input_buf, plan.output_buf, tuple(plan.input_shape), tuple(plan.output_shape),
                 sorted(plan.tensor_buf.items()), frames, plan.decode)).encode()
    return hashlib.sha256(head + _digest(*plan.weights).encode()).hexdigest()


def fingerprints() -> dict:
    from defer_b200 import applications
    from defer_b200.planner import plan_stage
    from defer_b200.resize import INTERPOLATIONS, kcap, pack_frame_tables, resize_tables
    out = {}
    for interpolation in INTERPOLATIONS:
        for n_in in TABLE_IN:
            for n_out in TABLE_OUT:
                out[f"tables/{interpolation}/{n_in}->{n_out}"] = _digest(*resize_tables(n_in, n_out, interpolation))
        for bound, target in (((480, 640), (224, 224)), ((1080, 1920), (224, 224)), ((40, 50), (32, 32))):
            kw = (kcap(bound[1], target[1], interpolation), kcap(bound[0], target[0], interpolation))
            hws = [(min(h, bound[0]), min(w, bound[1])) for h, w in BLOCK_SIZES]
            out[f"blocks/{interpolation}/{bound}->{target}"] = _digest(pack_frame_tables(hws, target, kw, interpolation))
    model = applications.ResNet50(input_shape=(32, 32, 3))
    for cfg in PLAN_CONFIGS:
        out[f"plan/{sorted(cfg.items())}"] = _plan_digest(plan_stage(model, True, True, preprocess="caffe", **cfg))
    return out


if __name__ == "__main__":
    with open(sys.argv[1], "w") as f:
        json.dump(fingerprints(), f, indent=1, sort_keys=True)
        f.write("\n")
