"""The hand-over between microbatches on the GPU: input slots, ready / free flags, the hop, per-lane output buffers.

Every microbatch gets its own seeded input, so a stale, overwritten, swapped or torn slot changes a result (the reasons are in
tests/handover_check.py, whose checker is exercised on the CPU by tests/test_handover_host.py).  Each configuration runs
3·depth + 2 microbatches through a same-process chain in one step order and requires:
  * the references (one stage of the same model, dtype, batch and knobs, depth 1; for cuts that split a conv from its BN,
    the same chain at depth 1) pairwise distinct, bitwise and by > 1e-3;
  * each result bitwise equal to its own reference, and every stage's status clean;
  * copy hop: every consumer input slot equal to its producer's output buffer, lane by lane;
  * one item per model within the parity bar of the fp64 oracle.
Then the public queue API with coalesced ingress of distinct fp32 and uint8 items, and defer_stage_result's refusal of a
microbatch its lane no longer holds."""
import queue
import threading
import time

import numpy as np
import pytest

import handover_check as H
from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200 import keras_like as K
from defer_b200.node import StageRunner
from test_gpu_fold_affine import _knobs

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

TOL = {"float32": 1e-3, "bfloat16": 6e-2}


def _cfg(id, model="ResNet50", cuts=("default", 4), dtype="float32", batch=1, depth=3, hop="copy", order="dispatcher",
         pin=False, use_graph=True, env=None, oracle=False, serial_ref=False):
    return pytest.param(dict(model=model, cuts=cuts, dtype=dtype, batch=batch, depth=depth, hop=hop, order=order, pin=pin,
                             use_graph=use_graph, env=env or {}, oracle=oracle, serial_ref=serial_ref), id=id)


CONFIGS = (
    # 8 stages, hand-over before the ReLU of add_2k
    [_cfg(f"r50-test-cuts-{hop}", cuts=applications.RESNET50_TEST_CUTS, hop=hop, oracle=hop == "copy")
     for hop in ("copy", "tma", "direct")]
    + [_cfg(f"r50-4stage-d{d}-{order}", depth=d, order=order)
       for order in ("stage_major", "consumer_first") for d in (1, 2, 4)]
    # batch 4 runs the streaming wgmma executors
    + [_cfg("r50-2stage-b4-copy-pinned", cuts=("default", 2), batch=4, depth=4, pin=True),
       _cfg("r50-2stage-b4-direct-pinned", cuts=("default", 2), batch=4, depth=4, hop="direct", pin=True),
       _cfg("r50-2stage-b4-copy-eager", cuts=("default", 2), batch=4, depth=4, pin=True, use_graph=False)]
    # output writer and last input reader inside megakernel group spans
    + [_cfg("r50-4stage-mega-tma", depth=2, hop="tma", order="stage_major",
            env={"DEFER_MEGA": 1, "DEFER_UMMA_SPLITK": 0})]
    # standalone AFFINE / RELU / PAD ops write the stage outputs.  The cut at conv1 stores the conv output before its BN, which
    # one stage keeps in the conv's fp32 epilogue, so the reference is this chain at depth 1, one microbatch at a time
    + [_cfg("r50-unfused-cuts-direct", cuts=["conv1", "activation_9", "avg_pool"], hop="direct", order="consumer_first",
            oracle=True, serial_ref=True)]
    + [_cfg("r50-4stage-bf16", dtype="bfloat16", oracle=True)]
    # the stage output is a folded affine op's output
    + [_cfg("r50v2-fold-tma", model="ResNet50V2", batch=2, hop="tma", env={"DEFER_FOLD_AFFINE": 1}, oracle=True,
            cuts=["conv3_block1_preact_relu", "conv3_block4_out", "conv5_block1_preact_relu"])]
)


@pytest.fixture(scope="module")
def models():
    return {}


def _model(models, name):
    if name not in models:
        models.clear()                      # one model's weights at a time
        models[name] = getattr(applications, name)()
    return models[name]


_REFS = {}      # (model, dtype, batch, knobs, seed) -> single-stage output
_ORACLE = {}    # (model, batch, seed) -> oracle output


def _inputs(batch, n, seed0=1000):
    return [applications.synthetic_input(batch, seed=seed0 + i) for i in range(n)]


def _references(model, dtype, batch, env, seeds, xs):
    """Single-stage depth-1 results of xs (seeded by seeds), built with the knobs currently set (env: all but DEFER_HOP)."""
    key = (model.name, dtype, batch, tuple(sorted(env.items())))
    missing = [i for i, s in enumerate(seeds) if key + (s,) not in _REFS]
    if missing:
        r = StageRunner.from_model(model, device=0, dtype=dtype, max_batch=batch, depth=1)
        try:
            for i in missing:
                _REFS[key + (seeds[i],)] = r.predict(xs[i])
        finally:
            r.close()
    return [_REFS[key + (s,)] for s in seeds]


def _oracle(model, x, seed):
    from oracle import keras_ref
    key = (model.name, x.shape[0], seed)
    if key not in _ORACLE:
        _ORACLE[key] = keras_ref.predict(model.to_json(), model.get_weights(), x)
    return _ORACLE[key]


@pytest.mark.parametrize("cfg", CONFIGS)
def test_handover(models, cfg, monkeypatch, request):
    m = _model(models, cfg["model"])
    cuts = cfg["cuts"]
    if isinstance(cuts, tuple):
        cuts = applications.default_cuts(m, cuts[1])
    depth, n_stages = cfg["depth"], len(cuts) + 1
    assert n_stages * depth <= 28                     # the lane streams one device may hold (node.MAX_STREAMS_PER_DEVICE)
    n = 3 * depth + 2
    seeds = [1000 + i for i in range(n)]
    xs = _inputs(cfg["batch"], n)
    _knobs(monkeypatch, DEFER_HOP=cfg["hop"], **cfg["env"])
    if cfg["serial_ref"]:
        refs = H.run_chain(m, cuts, xs, dtype=cfg["dtype"], depth=1)["results"]
    else:
        refs = _references(m, cfg["dtype"], cfg["batch"], cfg["env"], seeds, xs)
    distinct = H.n_distinct(refs)
    t0 = time.perf_counter()
    run = H.run_chain(m, cuts, xs, dtype=cfg["dtype"], depth=depth, pin=cfg["pin"], use_graph=cfg["use_graph"],
                      order=cfg["order"])
    print(f"{request.node.callspec.id}: {n_stages} stages, depth {depth}, {cfg['order']}, {n} items, {distinct} distinct "
          f"references, status {run['status']}, {time.perf_counter() - t0:.1f} s")
    assert distinct == n, "the references must be pairwise distinct, or a stale slot would pass"
    H.check_results(run["results"], refs, depth)
    assert run["status"] == ["ok"] * n_stages
    if cfg["hop"] == "copy":
        assert len(run["links"]) == n_stages - 1
        for k, link in enumerate(run["links"]):
            for lane, (prod, cons) in enumerate(link):
                assert np.array_equal(prod, cons), (f"link {k}", f"lane {lane}")
    else:
        assert run["links"] is None
    if cfg["oracle"]:
        from oracle.keras_ref import rel_err
        e = rel_err(run["results"][0], _oracle(m, xs[0], seeds[0]))
        print(f"  item 0 against the oracle: rel err {e:.3e}")
        assert e <= TOL[cfg["dtype"]]


# ------------------------------------------------------------------------------------------------ the queue API
def _run_defer(model, cuts, depth, items, **kw):
    """Feed `items` to DEFER on GPU 0 with coalesce = 4, pausing after every 7th so partial groups also go out mid-stream;
    return what comes out, and check that nothing more does."""
    from defer_b200 import DEFER
    devices = [0] * (len(cuts) + 1)
    defer = DEFER(devices, dtype="float32", depth=depth, coalesce=4, linger_us=3000, wait_timeout_ms=20000, **kw)
    in_q, out_q = queue.Queue(), queue.Queue()
    t = threading.Thread(target=defer.run_defer, args=(model, cuts, in_q, out_q), daemon=True)
    t.start()
    try:
        while not defer.wait_ready(0.5):
            assert t.is_alive(), f"run_defer died: {defer._error!r}"
        for i, x in enumerate(items):
            in_q.put(x)
            if i % 7 == 6:
                time.sleep(0.05)
        outs = [out_q.get(timeout=120) for _ in items]
        with pytest.raises(queue.Empty):
            out_q.get(timeout=0.5)
    finally:
        defer.close()
        t.join(timeout=30)
    assert not t.is_alive()
    return outs


def _batch4_references(model, items, **kw):
    """Item i's result at some position of a single-stage batch-4 run (an item's result does not depend on its position)."""
    r = StageRunner.from_model(model, device=0, dtype="float32", max_batch=4, depth=1, **kw)
    try:
        refs = []
        for g in range(0, len(items), 4):
            group = items[g:g + 4]
            y = r.predict(np.concatenate(group + [group[0]] * (4 - len(group)), axis=0))
            refs += [y[i:i + 1].copy() for i in range(len(group))]
        return refs
    finally:
        r.close()


@pytest.mark.parametrize("depth", [2, 3])
@pytest.mark.parametrize("devices", [[0], [0, 0]], ids=["1stage", "2stage"])
def test_coalesced_distinct_items(resnet50, devices, depth, monkeypatch):
    _knobs(monkeypatch)
    n = 4 * depth * 2 + 3
    xs = [applications.synthetic_input(1, seed=3000 + i) for i in range(n)]
    refs = _batch4_references(resnet50, xs)
    assert H.n_distinct(refs) == n
    outs = _run_defer(resnet50, applications.default_cuts(resnet50, len(devices)), depth, xs)
    print(f"coalesce 4, {len(devices)} stage(s), depth {depth}: {n} distinct items in FIFO order")
    assert all(y.shape == (1, 1000) for y in outs)
    H.check_results(outs, refs, 4 * depth)


def test_coalesced_distinct_uint8_items(monkeypatch):
    """uint8 images minus the ImageNet mean are ~100x the synthetic weights' input scale and saturate the softmax, so the
    items' probabilities need not differ: the model ends at the pooled features.  It is cut from a fresh ResNet50: after
    DEFER has partitioned a model, a new Model over that model's tensors no longer finds its input layer."""
    from test_gpu_preprocess import _image
    _knobs(monkeypatch)
    resnet50 = applications.ResNet50()
    features = K.Model(resnet50.input, resnet50.get_layer("avg_pool").output, name="features")
    depth = 2
    n = 4 * depth * 2 + 3
    xs = [_image(1, 224, 224, seed=4000 + i) for i in range(n)]
    refs = _batch4_references(features, xs, preprocess="caffe")
    assert H.n_distinct(refs) == n
    outs = _run_defer(features, applications.default_cuts(resnet50, 2), depth, xs, preprocess="caffe")
    H.check_results(outs, refs, 4 * depth)


# ------------------------------------------------------------------------------------------------ result() state
def _small_model():
    K.clear_session()
    inp = K.Input(shape=(16, 16, 32))
    a = K.Conv2D(32, 3, padding="same", activation="relu", name="c1")(inp)
    m = K.Model(inp, K.Conv2D(64, 3, padding="same", name="c2")(a), name="small")
    applications.synthetic_weights(m, seed=4)
    return m


def _refused(r, seq, why):
    with pytest.raises(A.DeferError, match=why) as ei:
        r.result(seq)
    assert ei.value.code == A.ERR_STATE


def test_result_refuses_a_microbatch_its_lane_no_longer_holds():
    """At depth 2, after steps 0, 1, 2: result(0) would copy microbatch 2's output; result(7) was never stepped."""
    m = _small_model()
    xs = [applications.synthetic_input(1, (16, 16, 32), seed=50 + i) for i in range(3)]
    r = StageRunner.from_model(m, device=0, dtype="float32", max_batch=1, depth=1)
    try:
        refs = [r.predict(x) for x in xs]
    finally:
        r.close()
    assert H.n_distinct(refs) == 3
    r = StageRunner.from_model(m, device=0, dtype="float32", max_batch=1, depth=2)
    try:
        _refused(r, 0, "never stepped")
        for seq in range(3):
            r.submit(seq, xs[seq])
            r.step(seq)
        _refused(r, 0, "lane 0 has since run microbatch 2")
        assert np.array_equal(r.result(2), refs[2]) and np.array_equal(r.result(1), refs[1])
        _refused(r, 7, "never stepped")
        for _ in range(2):
            for x, ref in zip(xs, refs):
                assert np.array_equal(r.predict(x), ref)
    finally:
        r.close()
    with H.open_chain(m, ["c1"], depth=2) as (first, last):
        _refused(last, 0, "never stepped")
        for seq in range(3):
            first.submit(seq, xs[seq])
            first.step(seq)
            last.step(seq)
        _refused(last, 0, "lane 0 has since run microbatch 2")
        assert np.array_equal(last.result(2), refs[2]) and np.array_equal(last.result(1), refs[1])
        _refused(last, 7, "never stepped")
