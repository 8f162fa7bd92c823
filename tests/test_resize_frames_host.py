"""Images of mixed sizes on the host (no GPU): the per-sample table blocks of `max_image_size=`, run through a restatement
of the GPU kernel with its clamps, equal `resize_image` from each image's own size; `kcap` bounds every table; the memo,
the planner's ops, the refusals, and the feeder coalescing items of different sizes in FIFO order."""
import queue
import threading

import numpy as np
import pytest

from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200.dispatcher import DEFER
from defer_b200.planner import plan_stage
from defer_b200.resize import (INTERPOLATIONS, axis_tables, frame_block_ints, kcap, pack_frame_tables, resize_axis,
                               resize_tables)
from frames_check import pack_slots, resize_frames_host
from test_resize_host import saturated_image

BOUND, TARGET = (480, 640), (224, 224)
# mixed downscales, the bound itself, one axis or no axis at the target, upscales, one pixel, one row, one column
SIZES = [(480, 640), (300, 200), (224, 224), (224, 500), (100, 224), (7, 3), (1, 1), (480, 1), (1, 640), (250, 300)]


def _blocks(hws, interpolation, bound=BOUND, target=TARGET):
    kw = (kcap(bound[1], target[1], interpolation), kcap(bound[0], target[0], interpolation))
    return pack_frame_tables(hws, target, kw, interpolation), kw


@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
def test_blocks_give_resize_image_from_each_size(interpolation):
    images = [saturated_image(h, w, seed=h * 7 + w) for h, w in SIZES]
    blocks, kw = _blocks(SIZES, interpolation)
    assert blocks.dtype == np.int32 and blocks.shape == (len(SIZES), frame_block_ints(TARGET, kw))
    mid, out = resize_frames_host(pack_slots(images, *BOUND), blocks, TARGET, kw)
    for i, (im, (h, w)) in enumerate(zip(images, SIZES)):
        assert np.array_equal(out[i], applications.resize_image(im, TARGET, interpolation)), (h, w)
        want_mid = im if w == TARGET[1] else resize_axis(im, 1, *resize_tables(w, TARGET[1], interpolation))
        assert np.array_equal(mid[i, :h], want_mid), (h, w)


def test_block_layout():
    blocks, kw = _blocks([(300, 224)], "bicubic")
    b = blocks[0]
    assert (b[0], b[1]) == (300, 224)
    w_out, h_out = TARGET[1], TARGET[0]
    bw = b[2:2 + 2 * w_out].reshape(w_out, 2)
    assert np.array_equal(bw[:, 0], np.arange(w_out)) and (bw[:, 1] == 1).all()           # width 224: identity
    tw = b[2 + 2 * w_out:2 + w_out * (2 + kw[0])].reshape(w_out, kw[0])
    assert (tw[:, 0] == 1 << 22).all() and not tw[:, 1:].any()
    off = 2 + w_out * (2 + kw[0])
    first, count, coef = resize_tables(300, h_out, "bicubic")
    bh = b[off:off + 2 * h_out].reshape(h_out, 2)
    th = b[off + 2 * h_out:].reshape(h_out, kw[1])
    assert np.array_equal(bh[:, 0], first) and np.array_equal(bh[:, 1], count)
    assert np.array_equal(th[:, :coef.shape[1]], coef) and not th[:, coef.shape[1]:].any()


@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
@pytest.mark.parametrize("max_len,out_len", [(1, 224), (7, 5), (300, 224), (300, 5), (260, 64)])
def test_kcap_bounds_every_length(max_len, out_len, interpolation):
    cap = kcap(max_len, out_len, interpolation)
    widest = 0
    for n in range(1, max_len + 1):
        first, count, coef = resize_tables(n, out_len, interpolation)
        assert coef.shape[1] <= cap and (count <= cap).all(), n
        widest = max(widest, coef.shape[1])
    assert widest == cap                                          # tight: the bound's own ksize
    assert axis_tables(out_len, out_len, interpolation)[1].max() <= cap


def test_identity_axis_is_a_copy():
    x = saturated_image(37, 224, seed=3)
    for interpolation in INTERPOLATIONS:
        first, count, coef = axis_tables(224, 224, interpolation)
        assert np.array_equal(first, np.arange(224)) and (count == 1).all() and (coef == 1 << 22).all()
        assert np.array_equal(resize_axis(x, 1, first, count, coef), x)


def test_memo_returns_the_same_tables():
    a = axis_tables(640, 224, "bilinear")
    assert axis_tables(640, 224, "bilinear") is a
    assert all(np.array_equal(x, y) for x, y in zip(a, resize_tables(640, 224, "bilinear")))
    assert not any(x.flags.writeable for x in a)
    assert axis_tables(640, 224, "bicubic") is not a


@pytest.mark.parametrize("interpolation", ["nearest", "bilinear", "lanczos"])
def test_corrupt_or_zero_blocks_stay_in_bounds(interpolation):
    bound, target = (40, 50), (32, 32)
    images = [saturated_image(h, w, seed=h) for h, w in ((40, 50), (3, 9), (17, 1))]
    slots = pack_slots(images, *bound)
    blocks, kw = _blocks([im.shape[:2] for im in images], interpolation, bound, target)
    _, out = resize_frames_host(slots, np.zeros_like(blocks), target, kw)        # never-written samples
    assert not out.any()
    rng = np.random.default_rng(0)
    for trial in range(20):
        bad = blocks.copy()
        if trial % 2:
            bad[:] = rng.integers(-2 ** 31, 2 ** 31, bad.shape, dtype=np.int64).astype(np.int32)
        else:                                                      # plausible tables, hostile headers and bounds
            bad[:, :2] = rng.choice([-5, 0, 1, 39, 40, 41, 10 ** 9], (len(bad), 2))
            idx = rng.integers(2, bad.shape[1], 50)
            bad[:, idx] = rng.choice([-(2 ** 31), -1, 0, 7, 60, 2 ** 31 - 1], (len(bad), 50))
        mid, out = resize_frames_host(slots, bad, target, kw)
        assert out.shape == (3, 32, 32, 3) and mid.shape == (3, 40, 32, 3)


def test_pack_refuses_a_narrow_block():
    with pytest.raises(ValueError, match="taps"):
        pack_frame_tables([(480, 640)], TARGET, (1, 1), "bilinear")


# ------------------------------------------------------------------------------------------------ planner
@pytest.fixture(scope="module")
def model():
    return applications.ResNet50(input_shape=(32, 32, 3))


@pytest.mark.parametrize("bound", [(48, 40), (32, 32), (32, 100), (7, 3)])
def test_planner_emits_both_passes(model, bound):
    base = plan_stage(model, True, True, preprocess="caffe")
    p = plan_stage(model, True, True, preprocess="caffe", max_image_size=bound, interpolation="bicubic")
    rw, rh, pre = p.ops[:3]
    H, W = bound
    assert [(o.kind, o.mode) for o in (rw, rh)] == [(A.OP_RESIZE, A.RESIZE_SAMPLE_W), (A.OP_RESIZE, A.RESIZE_SAMPLE_H)]
    assert pre.kind == A.OP_PREPROCESS and pre.in0 == rh.out
    assert rw.in0 == p.input_buf and p.bufs[p.input_buf] == (H, W, 3, A.BUF_U8)
    assert rh.in0 == rw.out and p.bufs[rw.out] == (H, 32, 3, A.BUF_U8) and p.bufs[rh.out] == (32, 32, 3, A.BUF_U8)
    assert (rw.kw, rh.kw) == (kcap(W, 32, "bicubic"), kcap(H, 32, "bicubic"))
    assert all(o.w_kernel == o.w_scale == o.w_shift == -1 and o.flags == 0 for o in (rw, rh))
    assert p.input_shape == (H, W, 3) and p.output_shape == base.output_shape
    assert p.frames == {"max_image_size": bound, "target": (32, 32), "kw": (rw.kw, rh.kw), "interpolation": "bicubic"}
    assert [(o.kind, o.layers, o.flags) for o in p.ops[2:]] == [(o.kind, o.layers, o.flags) for o in base.ops]
    assert len(p.weights) == len(base.weights)                    # no tables in the plan: they come with each image
    assert base.frames is None


def test_refusals(model):
    for make in (lambda **kw: plan_stage(model, True, True, **kw), lambda **kw: DEFER([0], **kw)):
        with pytest.raises(ValueError, match=r"max_image_size=\(48, 40\).*needs preprocess"):
            make(max_image_size=(48, 40))
        with pytest.raises(ValueError, match=r"max_image_size=\(48, 40\) and image_size"):
            make(preprocess="caffe", max_image_size=(48, 40), image_size=(48, 40))
        for bad in ((0, 40), (48,), "48x40", (48.5, 40)):
            with pytest.raises(ValueError, match="max_image_size"):
                make(preprocess="caffe", max_image_size=bad)
        with pytest.raises(ValueError, match="interpolation"):
            make(preprocess="caffe", max_image_size=(48, 40), interpolation="linear")
    with pytest.raises(ValueError, match="first stage"):
        plan_stage(model, False, True, preprocess="caffe", max_image_size=(48, 40))


# ------------------------------------------------------------------------------------------------ feeder
class FakeFrameStage:
    """Stands in for a max_image_size StageRunner: records each group's item shapes; y[i] = the item's first byte."""

    def __init__(self, batch, depth):
        self.batch, self.depth = batch, depth
        self.out_shape = (batch, 5)
        self.groups, self.pending, self.outs = [], {}, {}

    def submit_frames(self, seq, index, frames):
        assert index == 0
        self.pending[seq] = [f.shape for f in frames]
        self.outs[seq] = np.zeros(self.out_shape, np.float32)
        for i, f in enumerate(frames):
            self.outs[seq][i] = f.reshape(-1)[0]

    def step(self, seq):
        self.groups.append(self.pending.pop(seq))

    def result(self, seq, out=None):
        return self.outs.pop(seq)

    def sync(self):
        pass

    def unlink(self):
        pass

    def close(self):
        pass


class FakeFrameDefer(DEFER):
    def _partition(self, model, layer_parts):
        return [None]

    def _dispatchModels(self, models, nodeIPs):
        self.stages = [FakeFrameStage(self.engine_batch, self.depth)]


def _start(d):
    in_q, out_q = queue.Queue(), queue.Queue()
    err = []

    def run():
        try:
            d.run_defer(None, [], in_q, out_q)
        except BaseException as e:  # noqa: BLE001
            err.append(e)
    t = threading.Thread(target=run, daemon=True)
    t.start()
    assert d.wait_ready(10)
    return in_q, out_q, t, err


def test_mixed_sizes_coalesce_in_fifo_order():
    d = FakeFrameDefer([0], depth=2, coalesce=8, linger_us=200000, preprocess="caffe", max_image_size=(60, 80))
    in_q, out_q, t, err = _start(d)
    sizes = [(60, 80), (1, 1), (30, 80), (60, 7), (12, 13)]
    items = [np.full((1,) + sizes[i % len(sizes)] + (3,), i, np.uint8) for i in range(20)]
    for x in items:
        in_q.put(x)
    try:
        got = [out_q.get(timeout=10) for _ in items]
    finally:
        stage = d.stages[0]
        d.close()
        t.join(timeout=10)
    assert not err, err
    assert [float(g[0, 0]) for g in got] == [float(i) for i in range(20)]
    assert [len(g) for g in stage.groups] == [8, 8, 4]
    assert stage.groups[0] == [x.shape for x in items[:8]]                 # one microbatch of different sizes


@pytest.mark.parametrize("bad,match", [(np.zeros((1, 61, 80, 3), np.uint8), r"outside max_image_size=\(60, 80\)"),
                                       (np.zeros((1, 60, 81, 3), np.uint8), r"outside max_image_size=\(60, 80\)"),
                                       (np.zeros((1, 0, 5, 3), np.uint8), r"outside max_image_size=\(60, 80\)"),
                                       (np.zeros((1, 3, 60, 80), np.uint8), r"channels-last.*max_image_size=\(60, 80\)"),
                                       (np.zeros((1, 60, 80, 3), np.float32), r"max_image_size=\(60, 80\) takes uint8"),
                                       (np.zeros((1, 60, 80, 3), np.int32), r"max_image_size=\(60, 80\) takes uint8")])
def test_feeder_refuses(bad, match):
    d = FakeFrameDefer([0], depth=2, coalesce=4, linger_us=2000, preprocess="caffe", max_image_size=(60, 80))
    in_q, out_q, t, err = _start(d)
    in_q.put(np.zeros((1, 5, 5, 3), np.uint8))
    in_q.put(bad)
    t.join(timeout=10)
    assert not t.is_alive()
    d.close()
    assert len(err) == 1 and isinstance(err[0], ValueError), err
    assert err[0].args and __import__("re").search(match, str(err[0])), str(err[0])


def test_other_configurations_keep_the_same_shape_rule():
    from test_coalesce_host import FakeDefer
    d = FakeDefer([0], depth=2, coalesce=4, linger_us=200000)
    in_q, out_q, t, err = _start(d)
    in_q.put(np.zeros((1, 2, 2, 1), np.float32))
    in_q.put(np.zeros((1, 2, 3, 1), np.float32))
    t.join(timeout=10)
    d.close()
    assert len(err) == 1 and "differ in shape" in str(err[0])
