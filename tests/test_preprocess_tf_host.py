"""Host side of uint8 ingress with Keras tf-mode preprocessing (ResNet V2; no GPU): `resnet_v2_preprocess_input`
against an independent restatement and exact rational arithmetic over every byte value, an exact emulation of the
division-free sequence the device runs, the planner's tf PREPROCESS op and the model-mode check, the dispatcher's feeder,
and the option's path to rank 0 of a one-process-per-GPU pipeline."""
import os
import queue
import sys
import threading
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200 import keras_like as K
from defer_b200.dispatcher import DEFER
from defer_b200.planner import plan_stage
from test_preprocess_host import FakeDefer, _feed, _free_port

ROOT = Path(__file__).resolve().parents[1]
BYTES = np.arange(256, dtype=np.uint8)


def keras_tf(x):
    """keras_applications.imagenet_utils._preprocess_numpy_input, mode='tf', restated step by step: cast non-float input
    to float32, then `x /= 127.5; x -= 1.` in place."""
    if not np.issubdtype(x.dtype, np.floating):
        x = x.astype(np.float32)
    x = np.array(x, dtype=np.float32)
    x /= 127.5
    x -= 1.
    return x


def r32(x: Fraction) -> Fraction:
    """`x` rounded to the nearest fp32 value, ties to even (normal range: every value below is 0 or above 2^-40)."""
    if x == 0:
        return Fraction(0)
    sign, a = (-1 if x < 0 else 1), abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    ulp = Fraction(2) ** (e - 23)
    m = a / ulp                                   # in [2^23, 2^24)
    fl = m.numerator // m.denominator
    rem = m - fl
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
        fl += 1
    return sign * fl * ulp


def _frac(v) -> Fraction:
    return Fraction(float(np.float32(v)))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ------------------------------------------------------------------------------------------------ the host transform
def test_every_byte_matches_keras_and_exact_arithmetic():
    exact = [r32(r32(Fraction(b) / Fraction(255, 2)) - 1) for b in range(256)]
    for x in (BYTES, BYTES.astype(np.float32)):
        before = x.copy()
        y = applications.resnet_v2_preprocess_input(x)
        assert y.dtype == np.float32 and y.shape == (256,)
        assert np.array_equal(_bits(y), _bits(keras_tf(x)))
        assert [_frac(v) for v in y] == exact
        assert np.array_equal(x, before) and not np.shares_memory(x, y)
    assert applications.resnet_v2_preprocess_input(np.uint8(0)) == np.float32(-1)
    assert applications.resnet_v2_preprocess_input(np.uint8(255)) == np.float32(1)


def test_images_match_keras_bitwise_and_leave_the_input_alone():
    img = applications.synthetic_image(2, (37, 53, 3), seed=12)
    before = img.copy()
    y = applications.resnet_v2_preprocess_input(img)
    assert y.shape == img.shape and y.dtype == np.float32
    assert np.array_equal(_bits(y), _bits(keras_tf(img)))
    assert np.array_equal(_bits(y), _bits(applications.resnet_v2_preprocess_input(img.astype(np.float32))))
    assert np.array_equal(img, before)
    # tf mode keeps the channel order: a pure-red pixel stays red
    px = applications.resnet_v2_preprocess_input(np.array([[[[255, 0, 0]]]], np.uint8))
    assert px.reshape(3).tolist() == [1.0, -1.0, -1.0]


# ------------------------------------------------------------------------------------------------ the device sequence
R_BITS = 0x3C008081


def _device_sequence(b: int) -> Fraction:
    """keras_tf_preprocess (csrc/common.cuh), one round to fp32 per _rn intrinsic; FMA rounds once."""
    B, r = Fraction(b), r32(Fraction(2, 255))
    q = r32(B * r)                                  # __fmul_rn(b, r)
    e = r32(B - q * Fraction(255, 2))               # __fmaf_rn(-q, 127.5f, b)
    q = r32(q + e * r)                              # __fmaf_rn(e, r, q)
    return r32(q - 1)                               # __fsub_rn(q, 1.0f)


def test_device_constant_is_the_rounded_reciprocal():
    r = np.array([R_BITS], np.uint32).view(np.float32)[0]
    assert _frac(r) == r32(Fraction(2, 255))
    assert np.float32(127.5) == 127.5                # exact in fp32


def test_device_sequence_is_exact_for_every_byte():
    keras = [_frac(v) for v in keras_tf(BYTES)]
    assert [_device_sequence(b) for b in range(256)] == keras
    # the negative controls: the reciprocal product alone, with a separate and with a contracted (FMA) subtraction,
    # is wrong for many bytes - so the correction step above is what makes the sequence exact
    r = r32(Fraction(2, 255))
    mul_sub = sum(r32(r32(Fraction(b) * r) - 1) != keras[b] for b in range(256))
    fma = sum(r32(Fraction(b) * r - 1) != keras[b] for b in range(256))
    assert mul_sub == 111 and fma == 205, (mul_sub, fma)


# ------------------------------------------------------------------------------------------------ modes on the models
def test_builders_record_their_keras_mode():
    small = dict(input_shape=(32, 32, 3))
    for name in ("ResNet50", "ResNet101", "ResNet152"):
        assert getattr(applications, name)(**small).preprocess_mode == "caffe", name
    assert applications.VGG16(input_shape=(32, 32, 3)).preprocess_mode == "caffe"
    for name in ("ResNet50V2", "ResNet101V2", "ResNet152V2"):
        assert getattr(applications, name)(**small).preprocess_mode == "tf", name
    assert applications.ResNet50V2(weights=None, input_shape=(32, 32, 3)).preprocess_mode == "tf"


def test_mode_names():
    assert applications.PREPROCESS_MODES == ("caffe", "tf")
    with pytest.raises(ValueError, match="'caffe'.*'tf'"):
        applications.check_preprocess("torch")
    with pytest.raises(ValueError, match="resnet_v2_preprocess_input"):
        applications.preprocess_input(np.zeros((1, 2, 2, 3), np.uint8), mode="tf")
    DEFER([0], preprocess="tf")


# ------------------------------------------------------------------------------------------------ planner
def _small_v2():
    return applications.ResNet50V2(input_shape=(32, 32, 3))


def _op_keys(ops, shift=0):
    return [(o.kind, o.in0 - shift, o.out - shift, o.in1 - shift if o.in1 >= 0 else -1, o.kh, o.kw, o.sh, o.sw, o.pads,
             o.flags, o.w_kernel, o.w_scale, o.w_shift, o.layers) for o in ops]


def test_tf_plan_starts_with_u8_input_and_a_weightless_preprocess():
    m = _small_v2()
    plain = plan_stage(m, is_first=True, is_last=True)
    pp = plan_stage(m, is_first=True, is_last=True, preprocess="tf")
    assert pp.bufs[pp.input_buf] == (32, 32, 3, A.BUF_U8) and pp.input_buf == 0
    op = pp.ops[0]
    assert op.kind == A.OP_PREPROCESS and op.mode == A.PRE_TF == 1
    assert op.in0 == pp.input_buf and op.in1 == -1 and pp.bufs[op.out] == (32, 32, 3, A.BUF_F32)
    assert op.w_kernel == op.w_scale == op.w_shift == -1
    assert op.layers == ["preprocess_input(tf)"]
    # the rest is the plain plan reading the preprocessed image: buffer ids shift by one, the weights are the same list
    assert pp.ops[1].in0 == op.out
    assert _op_keys(pp.ops[1:], shift=1) == _op_keys(plain.ops)
    assert pp.bufs[op.out] == plain.bufs[plain.input_buf] and pp.bufs[2:] == plain.bufs[1:]
    assert pp.output_buf == plain.output_buf + 1 and pp.output_shape == plain.output_shape
    assert len(pp.weights) == len(plain.weights) and all(np.array_equal(a, b) for a, b in zip(pp.weights, plain.weights))
    assert all(o.mode == 0 for o in pp.ops[1:])


def test_caffe_plan_carries_mode_zero():
    for m in (applications.ResNet50(input_shape=(32, 32, 3)), _small_v2()):
        pp = plan_stage(m, is_first=True, is_last=True, preprocess="caffe")
        assert pp.ops[0].kind == A.OP_PREPROCESS and pp.ops[0].mode == A.PRE_CAFFE == 0
        assert pp.ops[0].w_shift >= 0
        assert all(o.mode == 0 for o in pp.ops)


def test_tf_refused_on_caffe_models_only():
    for m in (applications.ResNet50(input_shape=(32, 32, 3)), applications.ResNet152(input_shape=(32, 32, 3)),
              applications.VGG16(input_shape=(32, 32, 3))):
        with pytest.raises(ValueError, match="'caffe'"):
            plan_stage(m, is_first=True, is_last=True, preprocess="tf")
    m = _small_v2()
    plan_stage(m, is_first=True, is_last=True, preprocess="tf")
    plan_stage(m, is_first=True, is_last=True, preprocess="caffe")     # unchanged: caffe is accepted for every model
    with pytest.raises(ValueError, match="first stage"):
        plan_stage(m, is_first=False, is_last=True, preprocess="tf")
    # a model without the record (a partition, or a model rebuilt from JSON) is not checked
    K.clear_session()
    inp = K.Input(shape=(8, 8, 3))
    x = K.Conv2D(8, (3, 3), name="c")(inp)
    assert plan_stage(K.Model(inp, x, name="c3"), is_first=True, is_last=True, preprocess="tf").ops[0].mode == A.PRE_TF


def test_defer_refuses_tf_for_a_caffe_model_before_partitioning():
    m = applications.ResNet50(input_shape=(32, 32, 3))
    d = DEFER([0, 0], depth=2, preprocess="tf")
    with pytest.raises(ValueError, match="'caffe'"):
        d.run_defer(m, applications.default_cuts(m, 2), queue.Queue(), queue.Queue())
    assert not d.stages and not d._threads


# ------------------------------------------------------------------------------------------------ dispatcher feeder
def test_feeder_keeps_uint8_items_uint8():
    items = [np.full((1, 2, 2, 3), i, np.uint8) for i in range(9)]
    got, stage, err = _feed(FakeDefer([0], depth=2, coalesce=4, linger_us=2000, preprocess="tf"), items)
    assert not err
    assert stage.dtypes == [np.dtype(np.uint8)] * 9
    assert [float(g[0, 0]) for g in got] == [float(i) for i in range(9)]


def test_feeder_rejects_float_items_naming_the_mode():
    items = [applications.resnet_v2_preprocess_input(np.zeros((1, 2, 2, 3), np.uint8))]
    got, stage, err = _feed(FakeDefer([0], depth=2, coalesce=4, linger_us=2000, preprocess="tf"), items)
    assert not got and not stage.dtypes
    assert len(err) == 1 and isinstance(err[0], TypeError)
    assert "preprocess='tf'" in str(err[0]) and "astype(np.uint8)" in str(err[0])


# ------------------------------------------------------------------------------------------------ gloo world 2
def _worker_tf(rank, world, port, q):
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "tests"))
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import queue as pyqueue
    import defer_b200.node as node_mod
    from defer_b200 import applications
    from defer_b200.dispatcher import DEFER
    from defer_b200.dist import DistContext
    from test_preprocess_host import _HostStage as Stage
    node_mod.StageRunner = Stage
    G = 2
    ctx = DistContext(backend="gloo", ring=8, out_elems=4, batch=G)
    try:
        node = node_mod.Node(dist_ctx=ctx, device=rank, poll_s=1e-4)
        nt = threading.Thread(target=node.run, daemon=True)
        nt.start()
        if rank == 0:
            model = applications.ResNet50V2(input_shape=(32, 32, 3))
            defer = DEFER(list(range(world)), depth=2, coalesce=G, linger_us=200000, dist=ctx, preprocess="tf")
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
        stage = Stage.made[0]
        assert stage.kw["preprocess"] == ("tf" if rank == 0 else None), stage.kw
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
def test_tf_reaches_rank0_only_world2():
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    mpctx = mp.get_context("spawn")
    q = mpctx.Queue()
    procs = [mpctx.Process(target=_worker_tf, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(world):
        r, s = q.get(timeout=200)
        res[r] = s
    for p in procs:
        p.join(timeout=30)
    assert res == {0: "ok", 1: "ok"}, res
