"""GPU parity of whole models and pipelines against the oracle (through the C-ABI)."""
import os
import queue
import threading

import numpy as np
import pytest

import handover_check as H
from defer_b200 import _cabi as A
from defer_b200 import applications, dag_util
from defer_b200.node import StageRunner

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

# parity bar of BASELINE.json: max|y - ref| / max|ref| <= 1e-3 for the fp32 configs
TOL = {"float32": 1e-3, "float32_simt": 1e-4, "bfloat16": 6e-2}


def _oracle(model, x, **kw):
    from oracle import keras_ref
    return keras_ref.predict(model.to_json(), model.get_weights(), x, **kw)


def _rel(y, ref):
    from oracle.keras_ref import rel_err
    return rel_err(y, ref)


@pytest.mark.parametrize("dtype", ["float32_simt", "float32", "bfloat16"])
def test_resnet50_single_stage(resnet50, x224, dtype):
    r = StageRunner.from_model(resnet50, device=0, dtype=dtype, max_batch=1, depth=1)
    try:
        y = r.predict(x224)
        ref_all = _oracle(resnet50, x224, return_all=True)
        ref = ref_all["fc1000"]
        # layer-granular report first (helps localise a bad kernel), then the end-to-end bar
        worst = 0.0
        for name in ["activation", "max_pooling2d", "activation_3", "activation_9", "activation_21", "activation_39",
                     "activation_48", "avg_pool"]:
            got = r.read_layer(name)
            e = _rel(got.reshape(ref_all[name].shape), ref_all[name])
            worst = max(worst, e)
            print(f"{dtype:13s} {name:16s} rel={e:.3e}")
        e_prob = _rel(y, ref)
        print(f"{dtype:13s} probabilities    rel={e_prob:.3e}  kernels/step={r.num_kernels()}")
        assert y.shape == (1, 1000)
        assert abs(float(y.sum()) - 1.0) < 1e-3
        assert e_prob <= TOL[dtype], (dtype, e_prob)
        assert worst <= TOL[dtype] * (1 if dtype != "bfloat16" else 2)
        if dtype != "bfloat16":
            assert int(np.argmax(y)) == int(np.argmax(ref))
    finally:
        r.close()


def test_megakernel_and_per_op_paths_agree_bitwise(resnet50, x224, monkeypatch):
    """The cluster megakernel (one launch per run of convs) and the per-op kernels compute the same tiles
    with the same K order: results must be identical, and both must meet the parity bar."""
    outs = {}
    monkeypatch.setenv("DEFER_UMMA_SPLITK", "0")     # split-K would change the summation order of the per-op plan
    for mega in ("1", "0"):
        monkeypatch.setenv("DEFER_MEGA", mega)
        r = StageRunner.from_model(resnet50, device=0, dtype="float32", max_batch=1, depth=1)
        try:
            outs[mega] = r.predict(x224)
            n_kernels = r.num_kernels()
            assert ("megakernel group" in r.describe()) == (mega == "1")
            # per-op: 53 convs (the RGB stem is ONE fused kernel since round 2) + max-pool + GAP + dense + softmax
            assert n_kernels == (6 if mega == "1" else 57), n_kernels
        finally:
            r.close()
    ref = _oracle(resnet50, x224)
    assert _rel(outs["1"], ref) <= 1e-3 and _rel(outs["0"], ref) <= 1e-3
    # per-op plans pick BN=128 tiles and other executors: different tile shapes, the same K order per output
    assert np.array_equal(outs["1"], outs["0"])


def _items(n, seed0, batch=1):
    """One seeded input per microbatch: with the same input on every lane a stale or swapped slot gives the right answer."""
    return [applications.synthetic_input(batch, seed=seed0 + i) for i in range(n)]


def _single_stage(model, xs, dtype="float32"):
    r = StageRunner.from_model(model, device=0, dtype=dtype, max_batch=xs[0].shape[0], depth=1)
    try:
        return [r.predict(x) for x in xs]
    finally:
        r.close()


@pytest.mark.parametrize("n_stages", [2, 8])
def test_resnet50_pipeline_same_gpu(resnet50, n_stages):
    cuts = applications.default_cuts(resnet50, n_stages)
    xs = _items(5, 100)
    run = H.run_chain(resnet50, cuts, xs, depth=2)
    assert run["status"] == ["ok"] * n_stages
    assert _rel(run["results"][0], _oracle(resnet50, xs[0])) <= 1e-3
    # the hop is lossless: every item gives the answer of one stage on its own input
    H.check_results(run["results"], _single_stage(resnet50, xs), depth=2)


def test_pipeline_equals_single_stage_bitwise(resnet50):
    """Partitioning must not change results at all (reference hop = lossless codec, src/node.py:76-79)."""
    xs = _items(4, 200)
    run = H.run_chain(resnet50, applications.RESNET50_TEST_CUTS, xs, depth=2)
    H.check_results(run["results"], _single_stage(resnet50, xs), depth=2)


def test_defer_api_queues(resnet50):
    """The reference's own usage pattern (test/test.py:39-49): run_defer in a daemon thread, queues in/out; a distinct
    input per item, each result bitwise the single-stage answer, in FIFO order."""
    from defer_b200 import DEFER
    n_dev = A.device_count()
    cuts = applications.default_cuts(resnet50, 4)
    defer = DEFER([i % n_dev for i in range(4)], dtype="float32", depth=3, wait_timeout_ms=2000)
    in_q, out_q = queue.Queue(10), queue.Queue(10)
    t = threading.Thread(target=defer.run_defer, args=(resnet50, cuts, in_q, out_q), daemon=True)
    t.start()
    try:
        n = 12
        xs = _items(n, 300)
        for x in xs:
            in_q.put(x)
        refs = _single_stage(resnet50, xs)
        assert _rel(refs[0], _oracle(resnet50, xs[0])) <= 1e-3
        outs = []
        for i in range(n):
            for _ in range(240):
                try:
                    res = out_q.get(timeout=0.5)
                    break
                except queue.Empty:
                    assert t.is_alive(), f"run_defer died: {defer._error!r}"
            else:
                raise AssertionError("no result within 120 s")
            assert res.shape == (1, 1000)
            outs.append(res)
    finally:
        defer.close()
        t.join(timeout=30)
    assert not t.is_alive()
    H.check_results(outs, refs, depth=3)


def test_batch4_matches_batch1(resnet50):
    x = applications.synthetic_input(4, seed=3)
    r = StageRunner.from_model(resnet50, device=0, dtype="float32", max_batch=4, depth=1)
    try:
        y = r.predict(x)
    finally:
        r.close()
    ref = _oracle(resnet50, x)
    assert _rel(y, ref) <= 1e-3


def test_vgg16_single_stage():
    m = applications.VGG16()
    x = applications.synthetic_input(1, seed=5)
    r = StageRunner.from_model(m, device=0, dtype="float32", max_batch=1, depth=1)
    try:
        y = r.predict(x)
    finally:
        r.close()
    ref = _oracle(m, x)
    assert _rel(y, ref) <= 1e-3


def test_resnet152_8_stage_bf16_same_gpu():
    """BASELINE config 5 shape on one GPU: ResNet152, 8 stages (cuts after blocks 5,11,...,41), bf16."""
    m = applications.ResNet152()
    xs = _items(3, 11)
    cuts = applications.default_cuts(m, 8)
    outs = H.run_chain(m, cuts, xs, "bfloat16", depth=2)["results"]
    ref = _oracle(m, xs[0])
    assert _rel(outs[0], ref) <= 8e-2         # bf16 storage over 152 layers; fp32 path is checked at 1e-3 below
    H.check_results(outs, _single_stage(m, xs, "bfloat16"), depth=2)
    outs32 = H.run_chain(m, cuts, xs[:2], "float32", depth=2)["results"]
    for x, y in zip(xs, outs32):
        assert _rel(y, _oracle(m, x)) <= 1e-3


def test_vgg16_4_stage_both_cut_lists():
    """BASELINE config 4: VGG16, 4 stages - pool cuts and the MAC-balanced conv cuts (post-ReLU hand-over)."""
    m = applications.VGG16()
    xs = _items(3, 12)
    refs = [_oracle(m, x) for x in xs]
    for cuts in (["block1_pool", "block2_pool", "block3_pool"], ["block2_conv1", "block3_conv2", "block4_conv2"]):
        outs = H.run_chain(m, cuts, xs, depth=2)["results"]
        for i, (y, ref) in enumerate(zip(outs, refs)):
            assert _rel(y, ref) <= 1e-3, (cuts, i)


def test_unfused_cut_points_on_gpu(resnet50):
    """Cuts that break the conv+BN+ReLU fusion exercise the standalone AFFINE / RELU / PAD kernels."""
    cuts = ["conv1", "activation_9", "avg_pool"]
    xs = _items(3, 500)
    outs = H.run_chain(resnet50, cuts, xs, depth=2)["results"]
    for x, y in zip(xs, outs):
        assert _rel(y, _oracle(resnet50, x)) <= 1e-3


def test_stalled_upstream_poisons_the_chain(resnet50, x224):
    """A stage whose input never arrives times out on the device; the failure must travel down the chain with the
    ready flags (poison bit) so the LAST stage's result call reports it instead of delivering garbage."""
    cuts = applications.default_cuts(resnet50, 4)[:2]
    names = ["input_1"] + cuts + [resnet50.output._keras_history[0].name]
    parts = [dag_util.construct_model(resnet50, names[i], names[i + 1], part_name=f"part{i+1}") for i in range(3)]
    runners = [StageRunner.from_wire(p.to_json(), p.get_weights(), device=0, dtype="float32", max_batch=1, depth=2,
                                     is_first=(i == 0), is_last=(i == 2), finalize=False, wait_timeout_ms=300)
               for i, p in enumerate(parts)]
    try:
        for i in range(2):
            runners[i].link_to(runners[i + 1])
        for r in runners:
            r.finalize()
        # healthy microbatch first
        runners[0].submit(0, x224)
        for r in runners:
            r.step(0)
        y = runners[2].result(0)
        assert _rel(y, _oracle(resnet50, x224)) <= 1e-3
        # now the first stage "dies": only stages 1 and 2 are stepped
        runners[1].step(1)
        runners[2].step(1)
        with pytest.raises(A.DeferError) as ei:
            runners[2].result(1)
        assert ei.value.code == A.ERR_TIMEOUT
        with pytest.raises(A.DeferError):
            runners[1].status()
        with pytest.raises(A.DeferError):
            runners[2].status()
        runners[0].status()          # the stage that was never stepped has nothing to report
    finally:
        for r in runners:
            try:
                r.sync()
            except Exception:
                pass
        for r in runners:
            r.unlink()
        for r in runners:
            r.close()


@pytest.mark.parametrize("coalesce", [4, 8])
def test_defer_coalesced_items_fifo_and_parity(resnet50, x224, coalesce):
    """Coalesced ingress on the GPU: single-image queue items, `coalesce` of them per launch, per-item results in FIFO
    order, each within the parity bar; an item's answer does not depend on its position inside the group.  Asserts
    position independence, so three images repeat on purpose; distinct items are in tests/test_gpu_handover.py."""
    from defer_b200 import DEFER
    n_dev = A.device_count()
    cuts = applications.default_cuts(resnet50, 2)
    defer = DEFER([i % n_dev for i in range(2)], dtype="float32", depth=2, coalesce=coalesce, linger_us=3000,
                  wait_timeout_ms=5000)
    in_q, out_q = queue.Queue(), queue.Queue()
    t = threading.Thread(target=defer.run_defer, args=(resnet50, cuts, in_q, out_q), daemon=True)
    t.start()
    try:
        assert defer.wait_ready(300)
        xs = [x224 * np.float32(1.0 + 0.1 * i) for i in range(3)]
        refs = [_oracle(resnet50, x) for x in xs]
        n = 3 * coalesce + 5                      # the last group is partial
        for i in range(n):
            in_q.put(xs[i % 3])
        outs = [out_q.get(timeout=120) for _ in range(n)]
        for i, y in enumerate(outs):
            assert y.shape == (1, 1000)
            assert _rel(y, refs[i % 3]) <= 1e-3, i
        for i in range(3, n):                     # same image => same bits wherever it sat in its group
            assert np.array_equal(outs[i], outs[i % 3]), i
    finally:
        defer.close()
        t.join(timeout=30)
    assert not t.is_alive()


def test_batch8_stream_kernel_vs_oracle_and_round1_executor(resnet50, monkeypatch):
    """A coalesced microbatch of 8 different images runs most convs on conv_stream_kernel: parity with the oracle per
    image, and the same bits as the round-1 persistent executor (DEFER_STREAM=0): same K order per output."""
    x = applications.synthetic_input(8, seed=17)
    x *= np.linspace(0.7, 1.3, 8, dtype=np.float32).reshape(8, 1, 1, 1)
    outs = {}
    monkeypatch.setenv("DEFER_UMMA_SPLITK", "0")     # split-K would change the summation order of small per-op plans
    for stream in ("1", "0"):
        monkeypatch.setenv("DEFER_STREAM", stream)
        r = StageRunner.from_model(resnet50, device=0, dtype="float32", max_batch=8, depth=1)
        try:
            outs[stream] = r.predict(x)
            assert ("conv_stream_kernel" in r.describe()) == (stream == "1")
        finally:
            r.close()
    ref = _oracle(resnet50, x)
    for i in range(8):
        assert _rel(outs["1"][i], ref[i]) <= 1e-3, i
    assert np.array_equal(outs["1"], outs["0"])


def test_balanced_cuts_pipeline_on_gpu(resnet50):
    """SURVEY 8f rank 1 on the GPU: cut layers chosen by defer_b200.autocut from per-op times MEASURED on the device give a
    legal pipeline with the same answer as the reference cut list (bitwise) and the oracle (<= 1e-3)."""
    from defer_b200 import autocut
    probe = StageRunner.from_model(resnet50, device=0, dtype="float32", max_batch=1, depth=1)
    try:
        op_us = [max(1.0, probe.time_op(i, iters=5, flush_l2=False)) for i in range(len(probe.plan.ops))]
    finally:
        probe.close()
    cuts, stage_us = autocut.balanced_cuts(resnet50, 4, op_costs=op_us)
    assert len(cuts) == 3 and len(stage_us) == 4
    assert max(stage_us) <= 0.5 * sum(stage_us)          # no stage holds more than half of the measured work
    xs = _items(3, 600)
    outs = H.run_chain(resnet50, cuts, xs, depth=2)["results"]
    ref_cuts = H.run_chain(resnet50, applications.default_cuts(resnet50, 4), xs, depth=2)["results"]
    assert _rel(outs[0], _oracle(resnet50, xs[0])) <= 1e-3
    H.check_results(outs, ref_cuts, depth=2)
