"""Keras load_img's resize on the host (no GPU): `applications.resize_image` against Pillow byte for byte, the per-axis
tables the library validates, the planner's RESIZE ops, and the refusals of `image_size=` / `interpolation=`."""
import numpy as np
import pytest

from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200.planner import plan_stage
from defer_b200.resize import INTERPOLATIONS, PRECISION_BITS, resize_tables

SIZES = [((480, 640), (224, 224)), ((720, 1280), (224, 224)), ((1080, 1920), (224, 224)), ((7, 5), (32, 32)),
         ((1000, 333), (224, 224)), ((224, 300), (224, 224)), ((3, 3), (224, 224)), ((17, 1000), (224, 3)),
         ((1, 1), (224, 224)), ((299, 299), (224, 224))]


def saturated_image(h, w, seed=0):
    """Uniform bytes with blocks of 0 and 255 and a one-pixel checkerboard: the negative lobes of bicubic and lanczos
    overshoot on the edges between them and hit both ends of the clamp."""
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    x[: h // 3] = 0
    x[h // 3: h // 2, : w // 2] = 255
    yy, xx = np.mgrid[:h, :w]
    cb = (yy + xx) % 2 == 0
    band = (yy >= h // 2) & (yy < 2 * h // 3)
    x[band & cb] = 255
    x[band & ~cb] = 0
    return x


@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
@pytest.mark.parametrize("src,dst", SIZES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in SIZES])
def test_resize_image_is_pillow(src, dst, interpolation):
    Image = pytest.importorskip("PIL.Image")
    x = saturated_image(*src, seed=src[0] + src[1])
    ref = np.asarray(Image.fromarray(x).resize((dst[1], dst[0]), getattr(Image, interpolation.upper())))
    got = applications.resize_image(x, dst, interpolation)
    assert got.dtype == np.uint8 and got.shape == ref.shape
    assert np.array_equal(got, ref), int((got != ref).sum())


def test_resize_image_batch_and_no_op():
    x = np.stack([saturated_image(30, 50, seed=s) for s in range(3)])
    y = applications.resize_image(x, (20, 24), "bicubic")
    assert y.shape == (3, 20, 24, 3)
    for i in range(3):
        assert np.array_equal(y[i], applications.resize_image(x[i], (20, 24), "bicubic"))
    same = applications.resize_image(x, (30, 50), "lanczos")
    assert np.array_equal(same, x) and same is not x                 # no resize at target_size, as in Keras


@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
@pytest.mark.parametrize("n_in,n_out", [(640, 224), (480, 224), (1920, 224), (5, 32), (1, 224), (3, 224), (1000, 3),
                                        (224, 224), (333, 224), (299, 224), (224, 4000)])
def test_tables_satisfy_the_library_bounds(n_in, n_out, interpolation):
    first, count, coef = resize_tables(n_in, n_out, interpolation)
    assert first.dtype == count.dtype == coef.dtype == np.int32
    assert first.shape == count.shape == (n_out,) and coef.shape[0] == n_out
    ksize = coef.shape[1]
    assert (first >= 0).all() and (count >= 1).all() and (count <= ksize).all() and (first + count <= n_in).all()
    for i in range(n_out):
        assert not coef[i, count[i]:].any()                          # no weight past `count`
    sums = coef.astype(np.int64).sum(axis=1)                        # normalised: each row sums to ~1.0
    assert np.abs(sums - (1 << PRECISION_BITS)).max() <= ksize
    if interpolation == "nearest":
        assert ksize == 1 and (coef == 1 << PRECISION_BITS).all()


def test_nearest_accumulates_like_pillow():
    """The nearest index comes from an accumulated position, not the closed form: they differ at 640 -> 224."""
    first, _, _ = resize_tables(640, 224, "nearest")
    closed = np.floor((np.arange(224) + 0.5) * 640 / 224).astype(np.int32)
    assert not np.array_equal(first, closed)


# ------------------------------------------------------------------------------------------------ planner
@pytest.fixture(scope="module")
def model():
    return applications.ResNet50(input_shape=(32, 32, 3))


def _ops(plan):
    return [(o.kind, o.in0, o.in1, o.out, o.kh, o.kw, o.sh, o.sw, o.pads, o.flags, o.w_kernel, o.w_scale, o.w_shift,
             o.mode, tuple(o.layers)) for o in plan.ops]


def _same_plan(a, b):
    assert a.bufs == b.bufs and _ops(a) == _ops(b)
    assert a.input_buf == b.input_buf and a.output_buf == b.output_buf
    assert a.input_shape == b.input_shape and a.output_shape == b.output_shape and a.tensor_buf == b.tensor_buf
    assert len(a.weights) == len(b.weights)
    for x, y in zip(a.weights, b.weights):
        assert x.dtype == y.dtype and np.array_equal(x, y)


@pytest.mark.parametrize("interpolation", ["nearest", "bilinear", "lanczos"])
def test_planner_emits_width_then_height_then_preprocess(model, interpolation):
    base = plan_stage(model, True, True, preprocess="caffe")
    p = plan_stage(model, True, True, preprocess="caffe", image_size=(48, 40), interpolation=interpolation)
    assert [o.kind for o in p.ops[:3]] == [A.OP_RESIZE, A.OP_RESIZE, A.OP_PREPROCESS]
    rw, rh, pre = p.ops[:3]
    assert p.input_buf == rw.in0 and p.bufs[rw.in0] == (48, 40, 3, A.BUF_U8)
    assert rh.in0 == rw.out and p.bufs[rw.out] == (48, 32, 3, A.BUF_U8)
    assert pre.in0 == rh.out and p.bufs[rh.out] == (32, 32, 3, A.BUF_U8)
    assert p.bufs[pre.out] == (32, 32, 3, A.BUF_F32)
    assert p.input_shape == (48, 40, 3) and p.output_shape == base.output_shape
    for op, n_in in ((rw, 40), (rh, 48)):
        first, count, coef = resize_tables(n_in, 32, interpolation)
        assert op.kw == coef.shape[1] and op.w_shift == -1 and op.flags == 0 and op.mode == 0
        assert p.weights[op.w_scale].dtype == np.int32 and np.array_equal(p.weights[op.w_scale], np.stack([first, count], 1))
        assert p.weights[op.w_kernel].dtype == np.int32 and np.array_equal(p.weights[op.w_kernel], coef)
    # everything from PREPROCESS on is the plan without image_size, shifted by the two new buffers and four tables
    assert [(o.kind, o.layers, o.flags) for o in p.ops[2:]] == [(o.kind, o.layers, o.flags) for o in base.ops]
    assert p.bufs[3:] == base.bufs[1:]
    assert all(np.array_equal(x, y) for x, y in zip(p.weights[4:], base.weights))


def test_planner_resizes_only_the_axis_that_changes(model):
    p = plan_stage(model, True, True, preprocess="caffe", image_size=(32, 100))
    assert [o.kind for o in p.ops[:2]] == [A.OP_RESIZE, A.OP_PREPROCESS]
    assert p.bufs[p.ops[0].in0][:2] == (32, 100) and p.bufs[p.ops[0].out][:2] == (32, 32)
    assert p.ops[0].layers == ["load_img(width 100->32, nearest)"]
    p = plan_stage(model, True, True, preprocess="caffe", image_size=(7, 32), interpolation="box")
    assert [o.kind for o in p.ops[:2]] == [A.OP_RESIZE, A.OP_PREPROCESS]
    assert p.bufs[p.ops[0].in0][:2] == (7, 32) and p.bufs[p.ops[0].out][:2] == (32, 32)
    assert p.ops[0].layers == ["load_img(height 7->32, box)"]


@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
def test_image_size_of_the_model_input_changes_nothing(model, interpolation):
    base = plan_stage(model, True, True, preprocess="caffe")
    _same_plan(plan_stage(model, True, True, preprocess="caffe", image_size=(32, 32), interpolation=interpolation), base)
    _same_plan(plan_stage(model, True, True, preprocess="caffe", image_size=[32, 32]), base)


def test_resnet_v2_tf_plan():
    m = applications.ResNet50V2(input_shape=(32, 32, 3))
    p = plan_stage(m, True, True, preprocess="tf", image_size=(64, 48), interpolation="bilinear")
    assert [o.kind for o in p.ops[:3]] == [A.OP_RESIZE, A.OP_RESIZE, A.OP_PREPROCESS]
    assert p.ops[2].mode == A.PRE_TF


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(model):
    from defer_b200.dispatcher import DEFER
    with pytest.raises(ValueError, match="needs preprocess"):
        plan_stage(model, True, True, image_size=(48, 40))
    with pytest.raises(ValueError, match="needs preprocess"):
        DEFER([0], image_size=(48, 40))
    for bad in ("linear", "NEAREST", "antialias", None):
        with pytest.raises(ValueError, match="interpolation"):
            plan_stage(model, True, True, preprocess="caffe", image_size=(48, 40), interpolation=bad)
        with pytest.raises(ValueError, match="interpolation"):
            DEFER([0], preprocess="caffe", image_size=(48, 40), interpolation=bad)
        with pytest.raises(ValueError, match="interpolation"):
            applications.resize_image(saturated_image(4, 4), (2, 2), bad)
    for bad in ((0, 40), (48, -1), (48,), (48, 40, 3), (48.5, 40), "48x40", 48):
        with pytest.raises(ValueError, match="image_size"):
            plan_stage(model, True, True, preprocess="caffe", image_size=bad)
        with pytest.raises(ValueError, match="image_size"):
            DEFER([0], preprocess="caffe", image_size=bad)
        with pytest.raises(ValueError, match="target_size"):
            applications.resize_image(saturated_image(4, 4), bad)
    with pytest.raises(ValueError, match="uint8 RGB"):
        applications.resize_image(saturated_image(4, 4).astype(np.float32), (2, 2))
    with pytest.raises(ValueError, match="uint8 RGB"):
        applications.resize_image(np.zeros((4, 4), np.uint8), (2, 2))
    with pytest.raises(ValueError, match="first stage"):
        plan_stage(model, False, True, preprocess="caffe", image_size=(48, 40))
