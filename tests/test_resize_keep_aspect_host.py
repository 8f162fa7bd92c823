"""Keras load_img(keep_aspect_ratio=True) on the host (no GPU): `resize_image` against Pillow's `Image.resize(box=...)`
byte for byte, `keras_crop_box` against a restatement of Keras, box tables, the planner's ops, the per-sample blocks
through the restatement of the GPU kernel, the defaults fingerprinted against the tree before the option, and the
refusals."""
import json
from pathlib import Path

import numpy as np
import pytest

from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200.dispatcher import DEFER
from defer_b200.planner import plan_stage
from defer_b200.resize import (INTERPOLATIONS, axis_tables, crop_boxes, frame_block_ints, kcap, keras_crop_box,
                               pack_frame_tables, resize_axis, resize_tables)
from frames_check import pack_slots, resize_frames_host
from resize_fingerprints import fingerprints
from test_resize_host import saturated_image

GOLDEN = Path(__file__).resolve().parent / "golden" / "resize_default_fingerprints.json"


def keras_box(img_size, target_size):
    """Keras' keep_aspect_ratio arithmetic as written in keras.utils.load_img: `img_size` is PIL's (width, height),
    `target_size` Keras' (height, width); the box is PIL's [left, upper, right, lower]."""
    width, height = img_size
    target_width, target_height = target_size[1], target_size[0]
    crop_height = (width * target_height) // target_width
    crop_width = (height * target_width) // target_height
    crop_height = min(height, crop_height)
    crop_width = min(width, crop_width)
    crop_box_hstart = int(float(height - crop_height) / 2)
    crop_box_wstart = int(float(width - crop_width) / 2)
    crop_box_wend = crop_box_wstart + crop_width
    crop_box_hend = crop_box_hstart + crop_height
    return [crop_box_wstart, crop_box_hstart, crop_box_wend, crop_box_hend]


def pillow_load_img(x, target, interpolation):
    """What load_img(target_size=target, interpolation=..., keep_aspect_ratio=True) does to the decoded image `x`."""
    Image = pytest.importorskip("PIL.Image")
    img = Image.fromarray(x)
    if img.size == (target[1], target[0]):
        return x.copy()
    return np.asarray(img.resize((target[1], target[0]), getattr(Image, interpolation.upper()),
                                 box=keras_box(img.size, target)))


# (source (h, w), target (h, w)): landscape, portrait and square sources; downscales from 1080x1920 and 480x640 both ways
# round; upscales; 1xN and Nx1 sources with crops of zero rows or columns; odd differences where the centring floors;
# an axis at the target length under a partial box; and a source already at the target
SHAPES = [((1080, 1920), (224, 224)), ((1920, 1080), (224, 224)), ((480, 640), (224, 224)), ((640, 480), (224, 224)),
          ((300, 300), (224, 224)), ((300, 300), (224, 160)), ((480, 640), (299, 299)), ((1080, 1920), (240, 320)),
          ((7, 5), (32, 32)), ((5, 9), (224, 300)), ((33, 17), (10, 7)), ((1, 1), (3, 5)),
          ((1, 1000), (224, 448)), ((1000, 1), (448, 224)), ((1, 1000), (224, 224)), ((1000, 1), (224, 224)),
          ((2, 1000), (224, 224)), ((1, 7), (224, 224)), ((481, 643), (224, 224)), ((643, 481), (225, 223)),
          ((100, 224), (224, 224)), ((224, 100), (224, 224)), ((224, 999), (224, 224)), ((999, 224), (224, 224)),
          ((224, 224), (224, 224)), ((299, 299), (299, 299))]


@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
@pytest.mark.parametrize("src,dst", SHAPES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in SHAPES])
def test_resize_image_is_pillow_with_box(src, dst, interpolation):
    x = saturated_image(*src, seed=src[0] * 3 + src[1])
    ref = pillow_load_img(x, dst, interpolation)
    got = applications.resize_image(x, dst, interpolation, keep_aspect_ratio=True)
    assert got.dtype == np.uint8 and got.shape == ref.shape
    assert np.array_equal(got, ref), int((got != ref).sum())


def test_shapes_cover_the_edge_cases():
    boxes = {(s, d): keras_crop_box(*s, d) for s, d in SHAPES}
    assert any(b[0] == b[2] or b[1] == b[3] for b in boxes.values())                     # zero-size crops
    assert any((b[2] - b[0]) % 2 != src[1] % 2 for (src, _), b in boxes.items())         # the centring floors
    assert any(s[1] == d[1] and (b[0], b[2]) != (0, s[1]) for (s, d), b in boxes.items())   # width at target, cropped
    assert any(s[0] == d[0] and (b[1], b[3]) != (0, s[0]) for (s, d), b in boxes.items())   # height at target, cropped


def test_keras_crop_box_is_keras():
    rng = np.random.default_rng(0)
    sizes = [(h, w) for h in (1, 2, 3, 7, 223, 224, 225, 480, 1080) for w in (1, 2, 5, 224, 640, 1920)]
    sizes += [tuple(int(v) for v in rng.integers(1, 5000, 2)) for _ in range(300)]
    targets = [(224, 224), (299, 299), (224, 448), (448, 224), (1, 1), (3, 7), (331, 17)]
    for h, w in sizes:
        for t in targets:
            assert list(keras_crop_box(h, w, t)) == keras_box((w, h), t), (h, w, t)


def test_batch_equals_each_image():
    x = np.stack([saturated_image(30, 50, seed=s) for s in range(3)])
    y = applications.resize_image(x, (20, 24), "bicubic", keep_aspect_ratio=True)
    assert y.shape == (3, 20, 24, 3)
    for i in range(3):
        assert np.array_equal(y[i], applications.resize_image(x[i], (20, 24), "bicubic", keep_aspect_ratio=True))
    same = applications.resize_image(x, (30, 50), "lanczos", keep_aspect_ratio=True)
    assert np.array_equal(same, x) and same is not x


# ------------------------------------------------------------------------------------------------ tables
@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
def test_whole_axis_box_is_no_box(interpolation):
    for n_in in (1, 3, 224, 480, 640, 1920):
        for n_out in (1, 7, 224):
            want = resize_tables(n_in, n_out, interpolation)
            for got in (resize_tables(n_in, n_out, interpolation, None), resize_tables(n_in, n_out, interpolation,
                                                                                       (0, n_in))):
                assert all(a.dtype == b.dtype and np.array_equal(a, b) for a, b in zip(got, want)), (n_in, n_out)


@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
@pytest.mark.parametrize("n_in,n_out,box", [(640, 224, (80, 560)), (1920, 224, (420, 1500)), (224, 224, (62, 162)),
                                            (1000, 224, (499, 500)), (1000, 448, (500, 500)), (1, 224, (0, 0)),
                                            (5, 32, (0, 5)), (9, 300, (1, 7)), (17, 7, (0, 17))])
def test_box_tables_satisfy_the_library_bounds(n_in, n_out, box, interpolation):
    first, count, coef = resize_tables(n_in, n_out, interpolation, box)
    assert first.dtype == count.dtype == coef.dtype == np.int32 and first.shape == count.shape == (n_out,)
    assert (first >= 0).all() and (count >= 1).all() and (count <= coef.shape[1]).all() and (first + count <= n_in).all()
    assert coef.shape[1] <= kcap(n_in, n_out, interpolation)                # a box never needs more taps than its axis
    for i in range(n_out):
        assert not coef[i, count[i]:].any()


def test_box_taps_reach_outside_the_box():
    """Pillow clamps the taps to the image, not the box: a box resize is not a crop then a resize."""
    first, count, _ = resize_tables(640, 224, "lanczos", (80, 560))
    assert first[0] < 80 and first[-1] + count[-1] > 560
    x = saturated_image(4, 640, seed=1)
    boxed = resize_axis(x, 1, *resize_tables(640, 224, "lanczos", (80, 560)))
    cropped = resize_axis(np.ascontiguousarray(x[:, 80:560]), 1, *resize_tables(480, 224, "lanczos"))
    assert not np.array_equal(boxed, cropped)


def test_bad_boxes_are_refused():
    for box in ((-1, 5), (3, 2), (0, 11), (10, 10), (0.5, 3), (1,), "ab", 3):
        with pytest.raises(ValueError, match="box"):
            resize_tables(10, 4, "bilinear", box)


def test_axis_tables_memoise_on_the_box():
    a = axis_tables(224, 224, "bilinear", (62, 162))
    assert axis_tables(224, 224, "bilinear", (62, 162)) is a
    assert axis_tables(224, 224, "bilinear", (61, 161)) is not a
    assert all(np.array_equal(x, y) for x, y in zip(a, resize_tables(224, 224, "bilinear", (62, 162))))
    assert not any(x.flags.writeable for x in a)
    ident = axis_tables(224, 224, "bilinear")
    assert (ident[1] == 1).all() and not np.array_equal(a[0], ident[0])


def test_crop_boxes():
    assert crop_boxes(480, 640, (224, 224), False) == (None, None)
    assert crop_boxes(480, 640, (224, 224), True) == ((80, 560), None)
    assert crop_boxes(640, 480, (224, 224), True) == (None, (80, 560))
    assert crop_boxes(100, 224, (224, 224), True) == ((62, 162), None)
    assert crop_boxes(224, 224, (224, 224), True) == (None, None)
    assert crop_boxes(300, 300, (224, 224), True) == (None, None)


# ------------------------------------------------------------------------------------------------ the defaults
def test_defaults_match_the_tree_before_the_option():
    """`resize_tables` over a sweep of sizes, `pack_frame_tables` blocks and whole plans (ops, buffers, weights) with
    `image_size`, `max_image_size` and `decode="jpeg"` are byte for byte what they were before `keep_aspect_ratio`."""
    want = json.loads(GOLDEN.read_text())
    got = fingerprints()
    assert sorted(got) == sorted(want)
    assert [k for k in want if got[k] != want[k]] == []


# ------------------------------------------------------------------------------------------------ per-sample blocks
BOUND, TARGET = (480, 640), (224, 224)
FRAME_SIZES = [(480, 640), (480, 360), (300, 200), (224, 224), (224, 500), (100, 224), (224, 100), (7, 3),
               (1, 1), (480, 1), (1, 640), (251, 303), (2, 640)]


def _blocks(hws, interpolation, keep, bound=BOUND, target=TARGET):
    kw = (kcap(bound[1], target[1], interpolation), kcap(bound[0], target[0], interpolation))
    return pack_frame_tables(hws, target, kw, interpolation, keep), kw


@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
def test_blocks_give_resize_image_with_the_crop(interpolation):
    images = [saturated_image(h, w, seed=h * 5 + w) for h, w in FRAME_SIZES]
    blocks, kw = _blocks(FRAME_SIZES, interpolation, True)
    assert blocks.shape == (len(FRAME_SIZES), frame_block_ints(TARGET, kw))
    mid, out = resize_frames_host(pack_slots(images, *BOUND), blocks, TARGET, kw)
    for i, (im, (h, w)) in enumerate(zip(images, FRAME_SIZES)):
        assert np.array_equal(out[i], applications.resize_image(im, TARGET, interpolation, keep_aspect_ratio=True)), (h, w)
        box_w, _ = crop_boxes(h, w, TARGET, True)
        want_mid = im if (w == TARGET[1] and box_w is None) else resize_axis(im, 1, *resize_tables(w, TARGET[1],
                                                                                                   interpolation, box_w))
        assert np.array_equal(mid[i, :h], want_mid), (h, w)


def test_block_identity_only_for_a_whole_box():
    blocks, kw = _blocks([(100, 224), (300, 224)], "bilinear", True)
    w_out = TARGET[1]
    for b, identity in zip(blocks, (False, True)):
        bw = b[2:2 + 2 * w_out].reshape(w_out, 2)
        assert (np.array_equal(bw[:, 0], np.arange(w_out)) and (bw[:, 1] == 1).all()) == identity


def test_blocks_without_the_option_are_unchanged():
    for interpolation in INTERPOLATIONS:
        a, _ = _blocks(FRAME_SIZES, interpolation, False)
        b = pack_frame_tables(FRAME_SIZES, TARGET, _blocks([(1, 1)], interpolation, False)[1], interpolation)
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ planner
@pytest.fixture(scope="module")
def model():
    return applications.ResNet50(input_shape=(32, 32, 3))


def _ops(plan):
    return [(o.kind, o.in0, o.in1, o.out, o.kh, o.kw, o.sh, o.sw, o.pads, o.flags, o.w_kernel, o.w_scale, o.w_shift,
             o.mode, tuple(o.layers)) for o in plan.ops]


@pytest.mark.parametrize("interpolation", ["nearest", "bilinear", "lanczos"])
def test_planner_emits_box_tables(model, interpolation):
    p = plan_stage(model, True, True, preprocess="caffe", image_size=(48, 64), interpolation=interpolation,
                   keep_aspect_ratio=True)
    rw, rh, pre = p.ops[:3]
    assert [o.kind for o in (rw, rh, pre)] == [A.OP_RESIZE, A.OP_RESIZE, A.OP_PREPROCESS]
    assert (rw.mode, rh.mode) == (0, 0)
    assert rw.layers == [f"load_img(width 64->32 box 8..56, {interpolation})"]
    assert rh.layers == [f"load_img(height 48->32, {interpolation})"]
    for op, n_in, box in ((rw, 64, (8, 56)), (rh, 48, None)):
        first, count, coef = resize_tables(n_in, 32, interpolation, box)
        assert op.kw == coef.shape[1]
        assert np.array_equal(p.weights[op.w_scale], np.stack([first, count], 1))
        assert np.array_equal(p.weights[op.w_kernel], coef)
    base = plan_stage(model, True, True, preprocess="caffe", image_size=(48, 64), interpolation=interpolation)
    assert [(o.kind, o.layers) for o in p.ops[2:]] == [(o.kind, o.layers) for o in base.ops[2:]]
    assert p.bufs == base.bufs and p.frames is None


@pytest.mark.parametrize("image_size,axis", [((16, 32), "width"), ((32, 16), "height")])
def test_planner_resamples_an_axis_at_the_target_under_a_box(model, image_size, axis):
    """A 16x32 image to 32x32 keeps its width but crops it to 8..24: that axis is resampled, by an op naming it."""
    p = plan_stage(model, True, True, preprocess="caffe", image_size=image_size, interpolation="bicubic",
                   keep_aspect_ratio=True)
    rw, rh = p.ops[:2]
    assert [o.kind for o in p.ops[:3]] == [A.OP_RESIZE, A.OP_RESIZE, A.OP_PREPROCESS]
    h, w = image_size
    assert p.bufs[rw.out][:2] == (h, 32) and p.bufs[rh.out][:2] == (32, 32)
    if axis == "width":
        assert (rw.mode, rh.mode) == (A.RESIZE_W, 0)
        assert rw.layers == ["load_img(width 32->32 box 8..24, bicubic)"]
        first, count, coef = resize_tables(32, 32, "bicubic", (8, 24))
        op = rw
    else:
        assert (rw.mode, rh.mode) == (0, A.RESIZE_H)
        assert rh.layers == ["load_img(height 32->32 box 8..24, bicubic)"]
        first, count, coef = resize_tables(32, 32, "bicubic", (8, 24))
        op = rh
    assert np.array_equal(p.weights[op.w_scale], np.stack([first, count], 1))
    assert np.array_equal(p.weights[op.w_kernel], coef)


@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
def test_image_size_of_the_model_input_still_plans_no_resize(model, interpolation):
    base = plan_stage(model, True, True, preprocess="caffe")
    p = plan_stage(model, True, True, preprocess="caffe", image_size=(32, 32), interpolation=interpolation,
                   keep_aspect_ratio=True)
    assert p.bufs == base.bufs and _ops(p) == _ops(base) and len(p.weights) == len(base.weights)
    # a square image is cropped by nothing either: the plan is the one without the option
    q = plan_stage(model, True, True, preprocess="caffe", image_size=(48, 48), interpolation=interpolation,
                   keep_aspect_ratio=True)
    q0 = plan_stage(model, True, True, preprocess="caffe", image_size=(48, 48), interpolation=interpolation)
    assert _ops(q) == _ops(q0) and all(np.array_equal(a, b) for a, b in zip(q.weights, q0.weights))


@pytest.mark.parametrize("decode", [None, "jpeg"])
def test_planner_records_the_option_for_the_feeder(model, decode):
    p = plan_stage(model, True, True, preprocess="caffe", max_image_size=(48, 40), interpolation="bicubic",
                   keep_aspect_ratio=True, decode=decode)
    base = plan_stage(model, True, True, preprocess="caffe", max_image_size=(48, 40), interpolation="bicubic",
                      decode=decode)
    assert p.frames == dict(base.frames, keep_aspect_ratio=True)
    assert "keep_aspect_ratio" not in base.frames
    assert p.bufs == base.bufs and [o.mode for o in p.ops] == [o.mode for o in base.ops]
    assert [o.kw for o in p.ops] == [o.kw for o in base.ops]
    n = 1 if decode else 0
    assert p.ops[n].layers == ["load_img(width <=40->32, bicubic, keep_aspect_ratio)"]
    assert p.ops[n + 1].layers == ["load_img(height <=48->32, bicubic, keep_aspect_ratio)"]


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(model):
    from defer_b200.node import StageRunner
    makers = (lambda **kw: plan_stage(model, True, True, **kw), lambda **kw: DEFER([0], **kw),
              lambda **kw: StageRunner.from_model(model, **kw))
    for make in makers:
        for kw in ({}, {"preprocess": "caffe"}):
            with pytest.raises(ValueError, match=r"keep_aspect_ratio=True .*needs image_size= or max_image_size="):
                make(keep_aspect_ratio=True, **kw)
        for bad in (1, 0, "True", None, 1.0, [True]):
            with pytest.raises(ValueError, match=r"keep_aspect_ratio=.*expected True or False"):
                make(preprocess="caffe", image_size=(48, 40), keep_aspect_ratio=bad)
            with pytest.raises(ValueError, match=r"keep_aspect_ratio=.*expected True or False"):
                make(preprocess="caffe", max_image_size=(48, 40), keep_aspect_ratio=bad)
    for bad in (1, "yes", None):
        with pytest.raises(ValueError, match=r"keep_aspect_ratio=.*expected True or False"):
            applications.resize_image(saturated_image(4, 4), (2, 2), keep_aspect_ratio=bad)
    # the other refusals keep their reasons when the option is on
    with pytest.raises(ValueError, match="needs preprocess"):
        plan_stage(model, True, True, image_size=(48, 40), keep_aspect_ratio=True)
    with pytest.raises(ValueError, match="first stage"):
        plan_stage(model, False, True, preprocess="caffe", image_size=(48, 40), keep_aspect_ratio=True)
    # numpy's bool is a bool
    p = plan_stage(model, True, True, preprocess="caffe", image_size=(48, 40), keep_aspect_ratio=np.bool_(True))
    assert "box" in p.ops[1].layers[0]


# ------------------------------------------------------------------------------------------------ dispatch
class _FakeDist:
    def __init__(self):
        self.msgs = {}

    def send_stage(self, i, msg):
        self.msgs[i] = msg

    def wait_all_ready(self):
        pass


@pytest.mark.parametrize("keep", [False, True])
def test_stage_messages_carry_the_option_to_the_first_stage(keep):
    d = DEFER([0, 1], preprocess="caffe", max_image_size=(48, 40), keep_aspect_ratio=keep, dist=_FakeDist())
    m = applications.ResNet50(input_shape=(32, 32, 3))
    d._dispatchModels(d._partition(m, applications.default_cuts(m, 2)), [0, 1])
    assert [d.dist.msgs[i]["keep_aspect_ratio"] for i in (0, 1)] == [keep, False]
    assert d.dist.msgs[0]["max_image_size"] == (48, 40) and d.dist.msgs[1]["max_image_size"] is None


def test_feeder_coalesces_mixed_sizes_with_the_option():
    from test_resize_frames_host import FakeFrameDefer, _start
    d = FakeFrameDefer([0], depth=2, coalesce=4, linger_us=200000, preprocess="caffe", max_image_size=(60, 80),
                       keep_aspect_ratio=True)
    assert d.keep_aspect_ratio is True
    in_q, out_q, t, err = _start(d)
    items = [np.full((1,) + s + (3,), i, np.uint8) for i, s in enumerate([(60, 80), (1, 1), (30, 80), (60, 7)])]
    for x in items:
        in_q.put(x)
    try:
        got = [out_q.get(timeout=10) for _ in items]
    finally:
        d.close()
        t.join(timeout=10)
    assert not err, err
    assert [float(g[0, 0]) for g in got] == [0.0, 1.0, 2.0, 3.0]
