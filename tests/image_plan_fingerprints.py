"""SHA-256 fingerprints of the `plan_stage` plans that `decode="image"` sits beside: `decode="jpeg"`, `decode="png"` and
`max_image_size=` alone, over bounds, interpolations, `keep_aspect_ratio`, both preprocessing modes (ResNet50 and
ResNet50V2) and a cut.  Only the API that existed before `decode="image"` is used, so the same code fingerprints an older
tree:
`tests/golden/image_plan_fingerprints.json` holds the fingerprints of the tree before `decode="image"` was added, and
`test_image_host.py` checks that these plans still give them.

    python tests/image_plan_fingerprints.py OUT.json     # with the tree to fingerprint first on PYTHONPATH
"""
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
from resize_fingerprints import _plan_digest  # noqa: E402

PLAN_CONFIGS = [
    {"max_image_size": (480, 640)},
    {"max_image_size": (480, 640), "decode": "jpeg"},
    {"max_image_size": (480, 640), "decode": "png"},
    {"max_image_size": (1080, 1920), "interpolation": "bilinear", "decode": "jpeg"},
    {"max_image_size": (1080, 1920), "interpolation": "bilinear", "decode": "png"},
    {"max_image_size": (40, 50), "interpolation": "bicubic", "keep_aspect_ratio": True, "decode": "jpeg"},
    {"max_image_size": (40, 50), "interpolation": "bicubic", "keep_aspect_ratio": True, "decode": "png"},
    {"max_image_size": (40, 50), "interpolation": "lanczos", "keep_aspect_ratio": True},
]


def fingerprints() -> dict:
    from defer_b200 import applications, dag_util
    from defer_b200.planner import plan_stage
    model = applications.ResNet50(input_shape=(32, 32, 3))
    head = dag_util.construct_model(model, "input_1", "add_1", part_name="s1")
    v2 = applications.ResNet50V2(input_shape=(32, 32, 3))
    out = {}
    for cfg in PLAN_CONFIGS:
        out[f"plan/caffe/{sorted(cfg.items())}"] = _plan_digest(plan_stage(model, True, True, preprocess="caffe", **cfg))
        out[f"cut/caffe/{sorted(cfg.items())}"] = _plan_digest(plan_stage(head, True, False, preprocess="caffe", **cfg))
        out[f"plan/tf/{sorted(cfg.items())}"] = _plan_digest(plan_stage(v2, True, True, preprocess="tf", **cfg))
    return out


if __name__ == "__main__":
    with open(sys.argv[1], "w") as f:
        json.dump(fingerprints(), f, indent=1, sort_keys=True)
        f.write("\n")
