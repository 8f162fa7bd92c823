"""A standalone AFFINE(+ReLU) folded into the epilogue of the wgmma conv that writes its input, and the Keras ResNet V2
models it exists for.

* every wgmma executor with the fold (DEFER_FOLD_AFFINE=1) against the same stage with the standalone eltwise kernel
  (the default): the same bits in every buffer both runs write, with and without a residual, with
  and without the conv's own store, in BF16X2 and BF16;
* ResNet50V2 / 101V2 / 152V2 against the oracle folded and unfolded, folded against the default, partitions (including a cut at
  a `_preact_relu`) against one stage, in every DEFER_HOP mode, and coalesced items against their own batch-1 answers."""
import queue
import re
import threading

import numpy as np
import pytest

import handover_check as H
from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200 import keras_like as K
from defer_b200.node import StageRunner

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

KNOBS = ("DEFER_STREAM", "DEFER_STREAM_MIN_TILES", "DEFER_STREAM_BN", "DEFER_PERSIST_MIN_TILES", "DEFER_UMMA_BN",
         "DEFER_UMMA_SPLITK", "DEFER_UMMA_CLUSTER", "DEFER_UMMA_FORCE_SPLITS", "DEFER_UMMA_FORCE_CSPLIT", "DEFER_MEGA",
         "DEFER_FOLD_AFFINE", "DEFER_HOP")


def _knobs(monkeypatch, **env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


# executor -> (knobs, conv kernel, what describe() must show for that conv)
NO_STREAM = {"DEFER_STREAM_MIN_TILES": 10 ** 9}
EXECUTORS = {
    "one_tile": (dict(NO_STREAM, DEFER_UMMA_SPLITK=0), "conv_umma_aff_kernel", "x k-splits 1,"),
    "split_k": (dict(NO_STREAM, DEFER_UMMA_FORCE_SPLITS=2), "conv_umma_aff_kernel", "x k-splits 2,"),
    "cluster": (dict(NO_STREAM, DEFER_UMMA_CLUSTER=1, DEFER_UMMA_FORCE_CSPLIT=2), "conv_umma_aff_kernel",
                "x k-splits 2 (cluster, DSMEM reduce)"),
    "stream64": ({"DEFER_STREAM_MIN_TILES": 1, "DEFER_STREAM_BN": 64}, "conv_stream_aff_kernel", "(BN 64)"),
    "stream128": ({"DEFER_STREAM_MIN_TILES": 1, "DEFER_STREAM_BN": 128}, "conv_stream_aff_kernel", "(BN 128)"),
    "grid": ({"DEFER_STREAM": 0, "DEFER_PERSIST_MIN_TILES": 1}, "conv_stream_aff_kernel(grid)", "(BN 64)"),
    # conv_mega_kernel has no second output: the conv carrying the fold ends the run and runs on its own
    "mega": ({"DEFER_MEGA": 1}, None, "megakernel group: ops"),
}


def _fold_model(residual, keep_store, relu):
    """relu(input) -> conv_a (128 -> 64) -> conv (64 -> 128) -> [+ relu(input) | ReLU] -> BN [-> ReLU].
    The residual (or the conv's ReLU) keeps the planner from folding the BN into the conv's scale/shift.
    keep_store: the conv output is also the model output's second addend, so its own store must stay."""
    K.clear_session()
    inp = K.Input(shape=(28, 28, 128))
    x = K.Activation("relu", name="head")(inp)
    a = K.Conv2D(64, 3, padding="same", name="conv_a")(x)
    y = K.Conv2D(128, 3, padding="same", activation=None if residual else "relu", name="conv")(a)
    if residual:
        y = K.Add(name="sum")([y, x])
    z = K.BatchNormalization(name="bn")(y)
    if relu:
        z = K.Activation("relu", name="bn_relu")(z)
    if keep_store:
        z = K.Add(name="out")([z, y])
    m = K.Model(inp, z, name="fold")
    applications.synthetic_weights(m, seed=3)
    return m


def _run(m, x, dtype):
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=x.shape[0], depth=1)
    try:
        y = r.predict(x)
        bufs = {}
        for i in range(len(r.plan.bufs)):
            try:
                bufs[i] = r.read_buffer(i)
            except A.DeferError as e:
                bufs[i] = str(e)
        return y, bufs, r.describe(), [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))], r.plan
    finally:
        r.close()


def _tiles_line(desc, i):
    """The `wgmma tiles:` line describe() prints under op i."""
    lines = desc.splitlines()
    k = next(j for j, l in enumerate(lines) if re.match(rf"\s*\[\s*{i}\]", l))
    assert "wgmma tiles:" in lines[k + 1], lines[k:k + 2]
    return lines[k + 1]


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("residual,keep_store,relu", [(True, False, True), (False, True, False), (True, True, False),
                                                      (False, False, True), (True, False, False)])
@pytest.mark.parametrize("executor", list(EXECUTORS))
def test_folded_equals_unfolded_bitwise(executor, residual, keep_store, relu, dtype, monkeypatch):
    env, kernel, shown = EXECUTORS[executor]
    m = _fold_model(residual, keep_store, relu)
    x = applications.synthetic_input(2, (28, 28, 128), seed=11)
    _knobs(monkeypatch, **env)
    y0, bufs0, desc0, kern0, plan = _run(m, x, dtype)
    _knobs(monkeypatch, DEFER_FOLD_AFFINE=1, **env)
    y1, bufs1, desc1, kern1, _ = _run(m, x, dtype)
    ai = next(i for i, op in enumerate(plan.ops) if op.kind == A.OP_AFFINE)
    ci = next(i for i, op in enumerate(plan.ops) if op.out == plan.ops[ai].in0)
    assert plan.ops[ci].layers[0] == "conv" and bool(plan.ops[ci].flags & A.FLAG_RESIDUAL) == residual
    assert kern0[ai] == "eltwise_kernel" and "_aff_" not in kern0[ci], kern0
    want = kernel or "conv_umma_aff_kernel"
    assert kern1[ci] == want and kern1[ai] == f"affine (fused into {want})", (kern1, desc1)
    if executor != "mega":
        assert shown in _tiles_line(desc1, ci), desc1
    if executor == "mega":
        assert shown in desc0, desc0
        first, last = map(int, re.search(r"megakernel group: ops (\d+)\.\.(\d+)", desc0).groups())
        assert last >= ci, desc0                        # unfolded: the conv runs inside the group
        assert not re.search(rf"megakernel group: ops \d+\.\.{ci}\b", desc1) and "conv_mega_kernel" not in kern1[ci]
    assert np.array_equal(y0, y1)
    conv_out = plan.ops[ci].out
    for i, b in bufs0.items():
        if i == conv_out and not keep_store:
            assert "never written" in bufs1[i] and "folded into it" in bufs1[i], bufs1[i]
            continue
        assert np.array_equal(b, bufs1[i]), (executor, "buffer", i)
    with pytest.raises(A.DeferError, match="launches nothing"):
        r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=2, depth=1)
        try:
            r.time_op(ai, iters=1)
        finally:
            r.close()


def test_simt_path_keeps_the_standalone_affine(monkeypatch):
    _knobs(monkeypatch, DEFER_FOLD_AFFINE=1)
    m = _fold_model(True, False, True)
    x = applications.synthetic_input(1, (28, 28, 128), seed=2)
    y0, _, _, kern, plan = _run(m, x, "float32_simt")
    ai = next(i for i, op in enumerate(plan.ops) if op.kind == A.OP_AFFINE)
    assert kern[ai] == "eltwise_kernel"


# ------------------------------------------------------------------------------------------------ ResNet V2
V2 = ["ResNet50V2", "ResNet101V2", "ResNet152V2"]


@pytest.fixture(scope="module")
def v2_models():
    return {n: getattr(applications, n)() for n in V2}


def _oracle(m, x):
    from oracle import keras_ref
    return keras_ref.predict(m.to_json(), m.get_weights(), x)


def _rel(a, b):
    from oracle.keras_ref import rel_err
    return rel_err(a, b)


@pytest.mark.parametrize("name", V2)
@pytest.mark.parametrize("fold", [0, 1])
def test_resnet_v2_against_oracle(v2_models, name, fold, monkeypatch):
    _knobs(monkeypatch, DEFER_FOLD_AFFINE=fold)
    m = v2_models[name]
    x = applications.synthetic_input(2, seed=21)
    ref = _oracle(m, x)
    n_blocks = len(applications.residual_add_names(m))
    for dtype, tol in (("float32", 1e-3), ("bfloat16", 6e-2)):
        r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=2, depth=1)
        try:
            y = r.predict(x)
            kernels = [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))]
        finally:
            r.close()
        # folded: every _preact_bn but the first (it reads the max-pool) and post_bn ride on the conv writing the block
        # output; unfolded: all n_blocks + 1 run eltwise_kernel
        assert sum(k.startswith("affine (fused into conv_") for k in kernels) == fold * n_blocks, kernels
        assert kernels.count("eltwise_kernel") == 1 + (1 - fold) * n_blocks, kernels
        assert _rel(y, ref) <= tol, (name, dtype, fold, _rel(y, ref))


def test_folded_equals_default_bitwise(v2_models, monkeypatch):
    """DEFER_FOLD_AFFINE=1 against the default (and DEFER_FOLD_AFFINE=0, the same standalone kernels)."""
    m = v2_models["ResNet50V2"]
    x = applications.synthetic_input(4, seed=5)
    outs = {}
    for fold in (None, 0, 1):
        _knobs(monkeypatch, **({} if fold is None else {"DEFER_FOLD_AFFINE": fold}))
        r = StageRunner.from_model(m, device=0, dtype="float32", max_batch=4, depth=1)
        try:
            outs[fold] = r.predict(x), r.num_kernels()
        finally:
            r.close()
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[None][0], outs[1][0])
    assert outs[None][1] == outs[0][1] and outs[0][1] - outs[1][1] == 16


@pytest.mark.parametrize("hop", ["copy", "tma", "direct"])
def test_partitions_equal_one_stage_bitwise(v2_models, hop, monkeypatch):
    """Cuts at `_preact_relu` (the stage output IS a folded affine op's output) and at `_out` Adds."""
    _knobs(monkeypatch, DEFER_HOP=hop, DEFER_FOLD_AFFINE=1)
    m = v2_models["ResNet50V2"]
    xs = [applications.synthetic_input(2, seed=9 + i) for i in range(4)]
    r = StageRunner.from_model(m, device=0, dtype="float32", max_batch=2, depth=1)
    try:
        whole = [r.predict(x) for x in xs]
    finally:
        r.close()
    cuts = ["conv3_block1_preact_relu", "conv3_block4_out", "conv5_block1_preact_relu", "conv5_block2_out"]
    run = H.run_chain(m, cuts, xs, depth=2)
    assert any(k.startswith("affine (fused into") for ks in run["kernels"] for k in ks), run["kernels"]
    assert run["status"] == ["ok"] * 5
    H.check_results(run["results"], whole, depth=2)


def test_coalesced_items_position_independent(v2_models, monkeypatch):
    """Three images repeat on purpose: an item's result must not depend on its position in a coalesced group."""
    from defer_b200 import DEFER
    _knobs(monkeypatch, DEFER_FOLD_AFFINE=1)
    m = v2_models["ResNet50V2"]
    xs = [applications.synthetic_input(1, seed=30 + i) for i in range(3)]
    defer = DEFER([0, 0], dtype="float32", depth=2, coalesce=4, linger_us=3000, wait_timeout_ms=5000)
    in_q, out_q = queue.Queue(), queue.Queue()
    t = threading.Thread(target=defer.run_defer, args=(m, applications.default_cuts(m, 2), in_q, out_q), daemon=True)
    t.start()
    try:
        assert defer.wait_ready(300)
        n = 11
        for i in range(n):
            in_q.put(xs[i % 3])
        outs = [out_q.get(timeout=120) for _ in range(n)]
    finally:
        defer.close()
        t.join(timeout=30)
    assert not t.is_alive()
    for i in range(n):
        assert _rel(outs[i], _oracle(m, xs[i % 3])) <= 1e-3, i
        assert np.array_equal(outs[i], outs[i % 3]), i
