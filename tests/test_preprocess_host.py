"""Host side of uint8 ingress with Keras caffe preprocessing (no GPU): `applications.preprocess_input` against known
answers and an independent restatement, the planner's PREPROCESS op, the dispatcher's feeder, and the option's path to
rank 0 of a one-process-per-GPU pipeline."""
import os
import queue
import socket
import sys
import threading
from pathlib import Path

import numpy as np
import pytest

from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200 import keras_like as K
from defer_b200.dispatcher import DEFER
from defer_b200.planner import plan_stage

ROOT = Path(__file__).resolve().parents[1]
MEAN_BGR = (103.939, 116.779, 123.68)


def keras_caffe(x):
    """keras_applications.imagenet_utils._preprocess_numpy_input, mode='caffe', channels_last, restated step by step:
    cast non-float input to float32, 'RGB'->'BGR', then zero-center each channel by the ImageNet mean in float32."""
    if not np.issubdtype(x.dtype, np.floating):
        x = x.astype(np.float32)
    x = np.array(x[..., ::-1], dtype=np.float32)
    for c in range(3):
        x[..., c] = x[..., c] - np.float32(MEAN_BGR[c])
    return x


# ------------------------------------------------------------------------------------------------ preprocess_input
def test_known_answer():
    px = np.array([[[[255, 0, 10]]]], np.uint8)                   # (R, G, B)
    y = applications.preprocess_input(px)
    want = np.array([np.float32(10) - np.float32(103.939), np.float32(0) - np.float32(116.779),
                     np.float32(255) - np.float32(123.68)], np.float32)
    assert y.dtype == np.float32 and y.shape == (1, 1, 1, 3)
    assert np.array_equal(y.reshape(3).view(np.uint32), want.view(np.uint32))


def test_uint8_and_float32_inputs_give_the_same_bits_and_leave_the_input_alone():
    img = applications.synthetic_image(2, (5, 7, 3), seed=3)
    before = img.copy()
    a = applications.preprocess_input(img)
    f = img.astype(np.float32)
    f_before = f.copy()
    b = applications.preprocess_input(f)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.array_equal(img, before) and np.array_equal(f, f_before)
    assert a is not f and not np.shares_memory(a, f)


def test_matches_independent_restatement_bitwise():
    img = np.random.default_rng(11).integers(0, 256, (2, 37, 53, 3), dtype=np.uint8)
    y = applications.preprocess_input(img)
    assert np.array_equal(y.view(np.uint32), keras_caffe(img).view(np.uint32))
    # the device form: flip, then one fp32 add of -mean
    dev = img[..., ::-1].astype(np.float32) + applications.caffe_shift()
    assert np.array_equal(y.view(np.uint32), dev.view(np.uint32))


def test_only_caffe_mode():
    with pytest.raises(ValueError, match="caffe"):
        applications.preprocess_input(np.zeros((1, 2, 2, 3), np.uint8), mode="tf")
    with pytest.raises(ValueError, match="caffe"):
        DEFER([0], preprocess="torch")
    with pytest.raises(ValueError):
        applications.preprocess_input(np.zeros((1, 2, 2, 4), np.uint8))


def test_synthetic_image():
    a = applications.synthetic_image(4, (32, 32, 3), seed=5)
    assert a.dtype == np.uint8 and a.shape == (4, 32, 32, 3)
    assert a.min() == 0 and a.max() == 255
    assert np.array_equal(a, applications.synthetic_image(4, (32, 32, 3), seed=5))
    assert not np.array_equal(a, applications.synthetic_image(4, (32, 32, 3), seed=6))


# ------------------------------------------------------------------------------------------------ planner
def _plan_key(p, shift=0):
    ops = [(o.kind, o.in0 - shift, o.out - shift, o.in1 - shift if o.in1 >= 0 else -1, o.kh, o.kw, o.sh, o.sw, o.pads,
            o.flags, o.layers) for o in p.ops]
    return ops, p.bufs, p.input_buf, p.output_buf, p.input_shape, p.output_shape


def _small_resnet():
    return applications.ResNet50(input_shape=(32, 32, 3))


def test_caffe_plan_starts_with_u8_input_and_preprocess():
    m = _small_resnet()
    plain = plan_stage(m, is_first=True, is_last=True)
    pp = plan_stage(m, is_first=True, is_last=True, preprocess="caffe")
    assert pp.bufs[pp.input_buf] == (32, 32, 3, A.BUF_U8) and pp.input_buf == 0
    op = pp.ops[0]
    assert op.kind == A.OP_PREPROCESS and op.in0 == pp.input_buf and op.in1 == -1
    assert pp.bufs[op.out] == (32, 32, 3, A.BUF_F32)
    assert pp.weights[op.w_shift].dtype == np.float32
    assert np.array_equal(pp.weights[op.w_shift], -np.float32([103.939, 116.779, 123.68]))
    assert op.w_kernel == -1 and op.w_scale == -1
    # the rest is the plain plan reading the preprocessed image: same ops, same weights
    first_conv = pp.ops[1]
    assert first_conv.kind == A.OP_CONV and first_conv.in0 == op.out
    assert [(o.kind, o.layers, o.flags, o.pads) for o in pp.ops[1:]] == [(o.kind, o.layers, o.flags, o.pads) for o in plain.ops]
    assert pp.bufs[2:] == plain.bufs[1:]
    w_pp = [pp.weights[i] for i in range(len(pp.weights)) if i != op.w_shift]
    assert len(w_pp) == len(plain.weights) and all(np.array_equal(a, b) for a, b in zip(w_pp, plain.weights))
    assert pp.output_shape == plain.output_shape


def test_caffe_plan_rejects_misuse():
    m = _small_resnet()
    with pytest.raises(ValueError, match="first stage"):
        plan_stage(m, is_first=False, is_last=True, preprocess="caffe")
    with pytest.raises(ValueError, match="caffe"):
        plan_stage(m, is_first=True, is_last=True, preprocess="tf")
    K.clear_session()
    inp = K.Input(shape=(8, 8, 4))
    x = K.Conv2D(8, (3, 3), name="c")(inp)
    with pytest.raises(ValueError, match="RGB"):
        plan_stage(K.Model(inp, x, name="c4"), is_first=True, is_last=True, preprocess="caffe")


def test_none_plan_is_the_plain_plan():
    m = _small_resnet()
    a = plan_stage(m, is_first=True, is_last=True)
    b = plan_stage(m, is_first=True, is_last=True, preprocess=None)
    assert _plan_key(a) == _plan_key(b)
    assert len(a.weights) == len(b.weights) and all(np.array_equal(x, y) for x, y in zip(a.weights, b.weights))
    assert a.bufs[a.input_buf] == (32, 32, 3, A.BUF_F32)
    assert all(o.kind != A.OP_PREPROCESS for o in a.ops)


# ------------------------------------------------------------------------------------------------ dispatcher feeder
class FakeStage:
    """Stands in for StageRunner: records the dtype of every item handed to submit_items; y = per-sample mean."""

    def __init__(self, batch, depth):
        self.batch, self.depth = batch, depth
        self.out_shape = (batch, 5)
        self.slots = [np.zeros((batch, 2, 2, 3), np.float64) for _ in range(depth)]
        self.outs, self.dtypes = {}, []

    def submit_items(self, seq, items):
        for i, x in enumerate(items):
            self.dtypes.append(x.dtype)
            self.slots[seq % self.depth][i:i + 1] = x

    def step(self, seq):
        x = self.slots[seq % self.depth]
        self.outs[seq] = np.repeat(x.reshape(self.batch, -1).mean(axis=1, keepdims=True), 5, axis=1).astype(np.float32)

    def result(self, seq, out=None):
        return self.outs.pop(seq)

    def sync(self):
        pass

    def unlink(self):
        pass

    def close(self):
        pass


class FakeDefer(DEFER):
    def _partition(self, model, layer_parts):
        return [None]

    def _dispatchModels(self, models, nodeIPs):
        self.stages = [FakeStage(self.engine_batch, self.depth)]


def _feed(defer, items):
    in_q, out_q = queue.Queue(), queue.Queue()
    err = []

    def run():
        try:
            defer.run_defer(None, [], in_q, out_q)
        except BaseException as e:  # noqa: BLE001
            err.append(e)
    t = threading.Thread(target=run, daemon=True)
    t.start()
    assert defer.wait_ready(10)
    stage = defer.stages[0]
    got = []
    for x in items:
        in_q.put(x)
    try:
        for _ in items:
            got.append(out_q.get(timeout=5))
    except queue.Empty:
        pass
    defer.close()
    t.join(timeout=10)
    assert not t.is_alive()
    return got, stage, err


def test_feeder_keeps_uint8_items_uint8():
    items = [np.full((1, 2, 2, 3), i, np.uint8) for i in range(9)]
    got, stage, err = _feed(FakeDefer([0], depth=2, coalesce=4, linger_us=2000, preprocess="caffe"), items)
    assert not err
    assert stage.dtypes == [np.dtype(np.uint8)] * 9
    assert [float(g[0, 0]) for g in got] == [float(i) for i in range(9)]


def test_feeder_rejects_float_items_with_a_hint():
    items = [np.zeros((1, 2, 2, 3), np.float32)]
    got, stage, err = _feed(FakeDefer([0], depth=2, coalesce=4, linger_us=2000, preprocess="caffe"), items)
    assert not got and not stage.dtypes
    assert len(err) == 1 and isinstance(err[0], TypeError)
    assert "uint8" in str(err[0]) and "astype(np.uint8)" in str(err[0])


def test_feeder_without_option_casts_uint8_to_float32():
    items = [np.full((1, 2, 2, 3), i, np.uint8) for i in range(5)]
    got, stage, err = _feed(FakeDefer([0], depth=2, coalesce=2, linger_us=2000), items)
    assert not err
    assert stage.dtypes == [np.dtype(np.float32)] * 5
    assert [float(g[0, 0]) for g in got] == [float(i) for i in range(5)]


# ------------------------------------------------------------------------------------------------ gloo world 2
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class _HostStage:
    """StageRunner stand-in (as in test_dist_gloo): records the preprocess option each rank's from_wire receives."""
    made = []

    def __init__(self, batch, depth, rank, world):
        self.batch, self.depth, self.rank, self.world = batch, depth, rank, world
        self.out_shape = (batch, 4)
        self.links, self.steps, self.items = {}, [], []
        self.finalized = self.closed = self.unlinked = False

    @classmethod
    def from_wire(cls, model_json, weights, device=0, dtype="float32", max_batch=1, depth=1, is_first=True, is_last=True,
                  finalize=True, **kw):
        r = cls(max_batch, depth, int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]))
        r.is_first, r.is_last, r.kw = is_first, is_last, dict(kw)
        cls.made.append(r)
        return r

    def export_link(self, role):
        return f"tok-r{self.rank}-role{role}".encode()

    def import_link(self, role, token):
        self.links[role] = bytes(token)

    def finalize(self):
        self.finalized = True

    def submit_items(self, seq, items):
        self.items.append((seq, [x.dtype.name for x in items]))

    def step(self, seq):
        self.steps.append(seq)

    def result(self, seq, out=None):
        if out is None:
            out = np.empty(self.out_shape, np.float32)
        out[...] = (seq * self.batch + np.arange(self.batch, dtype=np.float32))[:, None]
        return out

    def sync(self):
        pass

    def unlink(self):
        self.unlinked = True

    def close(self):
        self.closed = True


def _worker_defer(rank, world, port, q):
    sys.path.insert(0, str(ROOT))
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import queue as pyqueue
    import defer_b200.node as node_mod
    from defer_b200 import applications
    from defer_b200.dispatcher import DEFER
    from defer_b200.dist import DistContext
    node_mod.StageRunner = _HostStage
    G = 2
    ctx = DistContext(backend="gloo", ring=8, out_elems=4, batch=G)
    try:
        node = node_mod.Node(dist_ctx=ctx, device=rank, poll_s=1e-4)
        nt = threading.Thread(target=node.run, daemon=True)
        nt.start()
        if rank == 0:
            model = applications.ResNet50(input_shape=(32, 32, 3))
            defer = DEFER(list(range(world)), depth=2, coalesce=G, linger_us=200000, dist=ctx, preprocess="caffe")
            in_q, out_q = pyqueue.Queue(), pyqueue.Queue()
            t = threading.Thread(target=defer.run_defer, args=(model, applications.default_cuts(model, world), in_q, out_q),
                                 daemon=True)
            t.start()
            assert defer.wait_ready(60), "pipeline did not come up"
            for i in range(4):
                in_q.put(np.full((1, 32, 32, 3), i, np.uint8))
            got = [out_q.get(timeout=60) for _ in range(4)]
            assert [float(g[0, 0]) for g in got] == [0.0, 1.0, 2.0, 3.0]
            defer.close()
            t.join(timeout=30)
            assert not t.is_alive()
        ctx.shutdown(nt)
        stage = _HostStage.made[0]
        assert "preprocess" in stage.kw
        assert stage.kw["preprocess"] == ("caffe" if rank == 0 else None), stage.kw
        if rank == 0:
            assert [d for _, ds in stage.items for d in ds] == ["uint8"] * 4
        q.put((rank, "ok"))
    except BaseException:  # noqa: BLE001
        import traceback
        q.put((rank, "fail: " + traceback.format_exc()))
        try:
            ctx.close()
        except Exception:
            pass


@pytest.mark.timeout(240)
def test_preprocess_reaches_rank0_only_world2():
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    mpctx = mp.get_context("spawn")
    q = mpctx.Queue()
    procs = [mpctx.Process(target=_worker_defer, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(world):
        r, s = q.get(timeout=200)
        res[r] = s
    for p in procs:
        p.join(timeout=30)
    assert res == {0: "ok", 1: "ok"}, res
