"""The one-process-per-GPU configurations of tests/test_gpu_dist.py, and the launcher of their torchrun runs (not a test
module).

Each case is one torchrun launch of tests/dist_hop_worker.py: every rank runs `Node.run` on its own stage (CUDA-IPC link
tokens, hops into a slot mapped from another process, the result ring in shared memory, `DistContext.shutdown`), and rank
0 is also the dispatcher.  CUDA IPC works between processes on one device, so the ranks need not have a GPU each: rank r
runs on visible GPU r % n (`rank_layout`), and ranks that share a GPU use a gloo group, as NCCL refuses two ranks on one
device.  The protocol is the one of distinct GPUs; only the NVLink transport is left out.

`CASES` is a pairwise-covering set of the values in `COVERAGE` (tests/test_dist_cases_host.py checks that every value is
reached).  Four of them are the earlier two-GPU runs, under their names: `hop-parity-g1` and `hop-parity-g4` (ResNet50
over two ranks, 14 float items, coalesce 1 and 4), `image-size` (10 frames of 480 x 640, bilinear) and `max-image-size`
(10 frames of mixed sizes up to 720 x 1280).  The items of a case (`make_items`) are distinct per item: seeded inputs, and
for JPEG the committed fixtures, baseline and progressive.
"""
import json
import os
import signal
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
WORKER = ROOT / "tests" / "dist_hop_worker.py"
CASE_ENV = "DEFER_DIST_CASE"          # the case, as JSON, for the worker
OUT_ENV = "DEFER_DIST_OUT"            # the directory rank 0 writes item_<i>.npy to, and every rank rank<r>.done
OUT_ELEMS = 1000                      # every case's model ends in a 1000-class head
WAIT_TIMEOUT_MS = 20000               # ranks that time-slice one GPU wait longer for their input than ranks with a GPU each
TOL = {"float32": 1e-3, "bfloat16": 6e-2}
# every knob a case may set; the launch clears the rest, as the reference run in the test process does
KNOBS = ("DEFER_STREAM", "DEFER_STREAM_MIN_TILES", "DEFER_STREAM_BN", "DEFER_PERSIST_MIN_TILES", "DEFER_UMMA_BN",
         "DEFER_UMMA_SPLITK", "DEFER_UMMA_CLUSTER", "DEFER_UMMA_FORCE_SPLITS", "DEFER_UMMA_FORCE_CSPLIT", "DEFER_MEGA",
         "DEFER_FOLD_AFFINE", "DEFER_HOP")

MIXED = [(480, 640), (224, 224), (300, 200), (1, 1), (720, 1280), (719, 1001), (224, 500)]
# baseline and progressive files in one queue, every one a different image (a baseline and a progressive file of one
# image at one quality decode to the same pixels, and their references would not be distinct)
JPEGS = [("jpeg_progressive", "photo_480x640_420_q75.jpg"), ("jpeg", "photo_223x225_444_q95.jpg"),
         ("jpeg_progressive", "photo_61x75_444_q90_opt.jpg"), ("jpeg", "photo_223x225_gray_q75_rb1.jpg"),
         ("jpeg_progressive", "photo_223x225_420_q100.jpg"), ("jpeg", "photo_480x640_422_q90_rr1.jpg"),
         ("jpeg_progressive", "photo_24x40_gray_q95.jpg"), ("jpeg", "photo_17x33_422_q5.jpg"),
         ("jpeg_progressive", "photo_61x75_422_q50_rr1.jpg"), ("jpeg", "photo_1x1_420_q95.jpg")]


def _case(id, model="ResNet50", ranks=2, cuts=None, dtype="float32", depth=3, coalesce=1, items=14, ring=64, hop="copy",
          env=None, ingress="float", interpolation="nearest"):
    """ingress: "float" (preprocessed float32 items), "caffe" / "tf" (uint8 224 x 224 images, preprocessed on the GPU),
    "image_size" (uint8 480 x 640 frames), "max_image_size" (uint8 frames of the sizes in MIXED), "jpeg" (the files of
    JPEGS, decoded with keep_aspect_ratio=True).  cuts None: `applications.default_cuts(model, ranks)`."""
    return dict(id=id, model=model, ranks=ranks, cuts=cuts, dtype=dtype, depth=depth, coalesce=coalesce, items=items,
                ring=ring, hop=hop, env=dict(env or {}), ingress=ingress, interpolation=interpolation)


CASES = [
    _case("hop-parity-g1", ring=4),                                          # 14 results through a ring of 4
    _case("hop-parity-g4", coalesce=4),                                      # groups of 4, 4, 4 and 2
    _case("r50-3r-tma-bf16-d1", ranks=3, dtype="bfloat16", depth=1, hop="tma", items=10, ring=3),
    _case("r50-4r-direct-d4-g4", ranks=4, depth=4, coalesce=4, hop="direct", items=18, ring=2),
    _case("r50v2-fold-preact-direct-tf", model="ResNet50V2", ranks=3, dtype="bfloat16", coalesce=2, items=7, hop="direct",
          cuts=["conv3_block1_preact_relu", "conv5_block1_preact_relu"], env={"DEFER_FOLD_AFFINE": 1}, ingress="tf"),
    _case("vgg16-conv-cut-tma-d1-caffe", model="VGG16", cuts=["block3_conv2"], depth=1, hop="tma", items=8, ring=3,
          ingress="caffe"),
    _case("image-size", coalesce=4, items=10, ingress="image_size", interpolation="bilinear"),
    _case("max-image-size", coalesce=4, items=10, ingress="max_image_size", interpolation="bilinear"),
    _case("jpeg-keep-aspect-4r-tma", ranks=4, coalesce=4, items=len(JPEGS), hop="tma", ingress="jpeg",
          interpolation="bilinear"),
]

# what the cases must reach between them
COVERAGE = {
    "ranks": {2, 3, 4},
    "hop": {"copy", "tma", "direct"},
    "dtype": {"float32", "bfloat16"},
    "ingress": {"float", "caffe", "tf", "image_size", "max_image_size", "jpeg"},
    "model": {"ResNet50", "ResNet50V2", "VGG16"},
}


def by_id(case_id):
    return next(c for c in CASES if c["id"] == case_id)


def n_groups(case):
    return -(-case["items"] // case["coalesce"])


# ------------------------------------------------------------------------------------------------ what a case runs
# The synthetic weights keep the softmax unsaturated for N(0, 1) inputs (`applications.synthetic_input`).  Images in caffe
# mode are some 70x larger, and ResNet50 and VGG16 then give a one-hot output: different images share its bits, and a stale
# slot would pass.  Their cases scale the last Dense down by this much more (logits of std ~2 again).
CAFFE_LOGIT_STD = 0.03


def build_model(case):
    from defer_b200 import applications
    if defer_kwargs(case).get("preprocess") != "caffe":
        return getattr(applications, case["model"])()
    model = getattr(applications, case["model"])(weights=None)
    applications.synthetic_weights(model, seed=1, logit_std=CAFFE_LOGIT_STD)   # the default draws, the head scaled
    return model


def cuts(case, model):
    from defer_b200 import applications
    return list(case["cuts"]) if case["cuts"] is not None else applications.default_cuts(model, case["ranks"])


def defer_kwargs(case):
    """The DEFER options of the case, the same in the torchrun run and in its one-process reference."""
    kw = dict(dtype=case["dtype"], depth=case["depth"], coalesce=case["coalesce"], linger_us=2000,
              wait_timeout_ms=WAIT_TIMEOUT_MS, interpolation=case["interpolation"])
    ing = case["ingress"]
    if ing != "float":
        kw["preprocess"] = "tf" if ing == "tf" else "caffe"
    if ing == "image_size":
        kw["image_size"] = (480, 640)
    elif ing == "max_image_size":
        kw["max_image_size"] = (720, 1280)
    elif ing == "jpeg":
        kw.update(max_image_size=(480, 640), decode="jpeg", keep_aspect_ratio=True)
    return kw


def make_items(case):
    """One distinct queue item per item of the case."""
    import numpy as np
    from defer_b200 import applications
    sys.path.insert(0, str(ROOT / "tests"))
    from test_resize_host import saturated_image
    n, ing = case["items"], case["ingress"]
    if ing == "float":
        return [applications.synthetic_input(1, seed=100 + i) for i in range(n)]
    if ing in ("caffe", "tf"):
        return [saturated_image(224, 224, seed=200 + i)[None] for i in range(n)]
    if ing == "image_size":
        return [saturated_image(480, 640, seed=51 + i)[None] for i in range(n)]
    if ing == "max_image_size":
        return [saturated_image(*MIXED[i % len(MIXED)], seed=51 + i)[None] for i in range(n)]
    if ing == "jpeg":
        assert n <= len(JPEGS)
        return [(GOLDEN / d / name).read_bytes() for d, name in JPEGS[:n]]
    raise ValueError(f"unknown ingress {ing!r}")


def knob_env(case):
    env = {"DEFER_HOP": case["hop"]}
    env.update({k: str(v) for k, v in case["env"].items()})
    return env


# ------------------------------------------------------------------------------------------------ placement
def rank_layout(world, n_visible):
    """(device, DistContext backend) of each rank: rank r on visible GPU r % n_visible; a gloo group when ranks share a
    GPU, NCCL for the GPUs otherwise."""
    if n_visible < 1:
        raise ValueError("no GPU visible")
    backend = "gloo" if world > n_visible else "cpu:gloo,cuda:nccl"
    return [(r % n_visible, backend) for r in range(world)]


# ------------------------------------------------------------------------------------------------ launching
def launch_env(case, out_dir, base=None):
    """The environment of the torchrun launch: `base` (default: this process's) with the case and its knobs.  GPU
    visibility (CUDA_VISIBLE_DEVICES) is passed on as given: the ranks use the GPUs this process may use, and no others."""
    env = dict(os.environ if base is None else base)
    for k in KNOBS:
        env.pop(k, None)
    env.update(knob_env(case))
    env[CASE_ENV] = json.dumps(case)
    env[OUT_ENV] = str(out_dir)
    return env


def torchrun_cmd(nproc, port, script=WORKER):
    """Loopback rendezvous only."""
    return [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
            "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)]


def free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _kill_group(proc, grace=10.0):
    """SIGTERM the process group `proc` leads (torchrun passes it on to its workers), wait up to `grace` seconds for the
    leader, then SIGKILL whatever of the group is left."""
    for sig in (signal.SIGTERM, signal.SIGKILL):
        try:
            os.killpg(proc.pid, sig)
        except ProcessLookupError:
            return
        try:
            proc.wait(timeout=grace)
        except subprocess.TimeoutExpired:
            pass
        try:
            os.killpg(proc.pid, 0)
        except ProcessLookupError:
            return


def run_group(cmd, env=None, cwd=None, timeout=900.0):
    """Run `cmd` in a session of its own, its output collected.  Returns (exit code, output, seconds); the exit code is None
    when `timeout` ran out.  On a timeout, or when this process is interrupted, the whole process group is killed (the
    torchrun agent and every worker and child it started), not just `cmd`, and the leader is reaped.  The output is read
    until every process holding it has exited, so a normal return leaves no process of the group behind either."""
    t0 = time.perf_counter()
    p = subprocess.Popen(cmd, env=env, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         start_new_session=True)
    try:
        out, _ = p.communicate(timeout=timeout)
        return p.returncode, out, time.perf_counter() - t0
    except subprocess.TimeoutExpired:
        _kill_group(p)
        out, _ = p.communicate()
        return None, out, time.perf_counter() - t0
    except BaseException:
        _kill_group(p)
        p.wait()
        raise
