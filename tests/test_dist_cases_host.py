"""The cases and the launcher of tests/test_gpu_dist.py, on the host: the cases reach every value they are there for, each
one can be built, ranks map onto devices and backends as documented, the launch passes GPU visibility on as given, and a
launch that runs out of time leaves no process behind."""
import os
import sys
import time
from pathlib import Path

import numpy as np
import pytest

import dist_cases as D
from defer_b200 import applications

CASES = D.CASES


def _values(key):
    return {c[key] for c in CASES}


def test_cases_cover_every_value():
    assert 8 <= len(CASES) <= 10
    assert len({c["id"] for c in CASES}) == len(CASES)
    for key, want in D.COVERAGE.items():
        assert want <= _values(key), (key, want - _values(key))
    depths = _values("depth")
    assert 1 in depths and max(depths) >= 3
    assert 1 in _values("coalesce")
    assert any(c["coalesce"] == 4 and c["items"] % 4 for c in CASES)                 # a partial last group
    assert any(D.n_groups(c) >= 3 * c["ring"] for c in CASES)                        # the result ring wraps several times
    assert any(c["model"] == "ResNet50" and c["cuts"] is None for c in CASES)        # its default cuts
    # ResNet50V2 with the affine fold, cut at a first block's pre-activation ReLU, with a hop that stores into the slot
    assert any(c["model"] == "ResNet50V2" and c["env"].get("DEFER_FOLD_AFFINE") == 1 and c["hop"] in ("tma", "direct")
               and any(k.endswith("_block1_preact_relu") for k in c["cuts"]) for c in CASES)
    assert any(c["model"] == "VGG16" and all("_conv" in k for k in c["cuts"]) for c in CASES)   # a post-ReLU hand-over


def test_mixed_sizes_and_both_jpeg_kinds_share_a_microbatch():
    frames = D.by_id("max-image-size")
    sizes = [x.shape[1:3] for x in D.make_items(frames)[:frames["coalesce"]]]
    assert len(set(sizes)) == len(sizes) > 1
    jp = next(c for c in CASES if c["ingress"] == "jpeg")
    assert D.defer_kwargs(jp)["keep_aspect_ratio"] is True
    kinds = [d for d, _ in D.JPEGS[:jp["items"]]]
    for g in range(0, jp["items"], jp["coalesce"]):
        assert set(kinds[g:g + jp["coalesce"]]) == {"jpeg", "jpeg_progressive"}
    from defer_b200.jpeg import check_jpeg
    infos = [check_jpeg(x, D.defer_kwargs(jp)["max_image_size"])[1] for x in D.make_items(jp)]
    assert {i.progressive for i in infos} == {False, True}


def test_folded_runs_keep_their_parameters():
    """The earlier two-GPU runs, as cases: ResNet50 over two ranks at their default cuts, fp32, depth 3."""
    for cid, coalesce, items, ingress in [("hop-parity-g1", 1, 14, "float"), ("hop-parity-g4", 4, 14, "float"),
                                          ("image-size", 4, 10, "image_size"), ("max-image-size", 4, 10, "max_image_size")]:
        c = D.by_id(cid)
        assert (c["model"], c["ranks"], c["cuts"], c["dtype"], c["depth"]) == ("ResNet50", 2, None, "float32", 3), cid
        assert (c["coalesce"], c["items"], c["ingress"]) == (coalesce, items, ingress), cid
    assert D.defer_kwargs(D.by_id("image-size"))["image_size"] == (480, 640)
    assert D.defer_kwargs(D.by_id("max-image-size"))["max_image_size"] == (720, 1280)


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_case_builds(case):
    from defer_b200.dispatcher import DEFER
    DEFER([0] * case["ranks"], **D.defer_kwargs(case))                  # the options are accepted together
    model = getattr(applications, case["model"])(weights=None)
    cuts = D.cuts(case, model)
    assert len(cuts) == case["ranks"] - 1
    names = {l.name for l, _ in model.iter_nodes()}
    assert set(cuts) <= names, set(cuts) - names
    assert case["ranks"] * case["depth"] <= 28       # the one-process reference holds every stage's lanes on one GPU
    items = D.make_items(case)
    assert len(items) == case["items"]
    raw = [bytes(x) if isinstance(x, bytes) else x.tobytes() for x in items]
    assert len(set(raw)) == len(raw)                                     # one distinct item each
    if case["ingress"] == "float":
        assert all(x.dtype == np.float32 and x.shape == (1, 224, 224, 3) for x in items)
    elif case["ingress"] != "jpeg":
        assert all(x.dtype == np.uint8 and x.ndim == 4 for x in items)
    assert D.knob_env(case)["DEFER_HOP"] == case["hop"]


@pytest.mark.parametrize("n_visible", [1, 2, 8])
def test_rank_layout(n_visible):
    for world in (2, 3, 4):
        layout = D.rank_layout(world, n_visible)
        assert [d for d, _ in layout] == [r % n_visible for r in range(world)]
        shared = world > n_visible                   # NCCL refuses two ranks on one device
        assert {b for _, b in layout} == {"gloo" if shared else "cpu:gloo,cuda:nccl"}
    with pytest.raises(ValueError):
        D.rank_layout(2, 0)


@pytest.mark.parametrize("visible", [None, "", "3", "1,0"])
def test_launch_env_keeps_gpu_visibility(visible, tmp_path):
    import json
    base = {"PATH": "/bin", "DEFER_MEGA": "1", "DEFER_HOP": "direct"}
    if visible is not None:
        base["CUDA_VISIBLE_DEVICES"] = visible
    case = D.by_id("r50v2-fold-preact-direct-tf")
    env = D.launch_env(case, tmp_path, base=base)
    assert env.get("CUDA_VISIBLE_DEVICES") == visible
    assert "DEFER_MEGA" not in env                   # knobs the case does not set are cleared
    assert env["DEFER_HOP"] == "direct" and env["DEFER_FOLD_AFFINE"] == "1"
    assert json.loads(env[D.CASE_ENV]) == case and env[D.OUT_ENV] == str(tmp_path)
    assert base.get("DEFER_MEGA") == "1"             # the caller's mapping is not changed


def test_torchrun_rendezvous_is_loopback():
    cmd = D.torchrun_cmd(3, 12345)
    assert cmd[cmd.index("--master-addr") + 1] == "127.0.0.1"
    assert cmd[cmd.index("--nproc-per-node") + 1] == "3" and cmd[-1] == str(D.WORKER)


def _gone(pid):
    """The process has exited (a zombie not yet reaped by whoever adopted it counts as gone)."""
    try:
        stat = Path(f"/proc/{pid}/stat").read_text()
    except FileNotFoundError:
        return True
    return stat.rsplit(")", 1)[1].split()[0] in ("Z", "X")


@pytest.mark.timeout(60)
def test_timeout_kills_the_whole_group():
    script = ("import subprocess, sys, time\n"
              "p = subprocess.Popen([sys.executable, '-c', 'import time; time.sleep(120)'])\n"
              "print(p.pid, flush=True)\n"
              "time.sleep(120)\n")
    t0 = time.perf_counter()
    code, out, secs = D.run_group([sys.executable, "-c", script], timeout=2.0)
    assert code is None and 2.0 <= secs < 30 and time.perf_counter() - t0 < 30
    grandchild = int(out.split()[0])
    deadline = time.time() + 10
    while not _gone(grandchild) and time.time() < deadline:
        time.sleep(0.05)
    assert _gone(grandchild), f"grandchild {grandchild} outlived the launch"


def test_run_group_returns_code_and_output():
    code, out, _ = D.run_group([sys.executable, "-c", "import sys; print('hello'); sys.exit(3)"],
                               env=dict(os.environ), timeout=60)
    assert code == 3 and out.strip() == "hello"
