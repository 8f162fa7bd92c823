"""Images of mixed sizes (`max_image_size=`) on the GPU, bit for bit against the host.

The contract: each uint8 image of its own size up to the bound gives exactly `applications.resize_image(image, model
input, interpolation)` fed to the same pipeline without the option - for `defer_k_resize_frames` against the numpy
restatement of the kernel, for the two per-sample RESIZE ops of a stage in both preprocessing modes, dtypes and stem paths,
after re-use of a lane, and for `DEFER` end to end over one and two stages (one process per GPU: the `max-image-size` case
of tests/test_gpu_dist.py)."""
import copy
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from defer_b200 import _cabi as A  # noqa: E402
from defer_b200 import applications  # noqa: E402
from defer_b200.resize import INTERPOLATIONS, kcap, pack_frame_tables, resize_axis, resize_tables  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

resize_image = applications.resize_image


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _image(h, w, seed):
    from test_resize_host import saturated_image
    return saturated_image(h, w, seed=seed)


def _kw(bound, target, interpolation):
    return kcap(bound[1], target[1], interpolation), kcap(bound[0], target[0], interpolation)


# ------------------------------------------------------------------------------------------------ the kernel
KERNEL_BOUND, KERNEL_TARGET = (240, 320), (224, 224)
KERNEL_SIZES = [(240, 320), (224, 224), (1, 1), (100, 300), (240, 17), (3, 224), (224, 5)]


@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
def test_k_resize_frames_matches_host(interpolation, offset):
    import torch
    from frames_check import pack_slots, resize_frames_host
    lib = A.load()
    (H, W), (Ho, Wo) = KERNEL_BOUND, KERNEL_TARGET
    kw = _kw(KERNEL_BOUND, KERNEL_TARGET, interpolation)
    n = len(KERNEL_SIZES)
    slots = pack_slots([_image(h, w, seed=h + 3 * w) for h, w in KERNEL_SIZES], H, W)
    blocks = pack_frame_tables(KERNEL_SIZES, KERNEL_TARGET, kw, interpolation)
    mid_ref, out_ref = resize_frames_host(slots, blocks, KERNEL_TARGET, kw)

    def dev(nbytes, fill=0):                                       # offset 1: one byte off any alignment
        return torch.full((nbytes + offset,), fill, dtype=torch.uint8, device="cuda")[offset:]
    x = dev(slots.size)
    x.copy_(torch.from_numpy(slots.reshape(-1)))
    mid, out = dev(n * H * Wo * 3, 77), dev(n * Ho * Wo * 3, 77)
    tables = torch.from_numpy(blocks.reshape(-1)).cuda()
    geo = (n, H, W, Ho, Wo, *kw)
    A.check(lib.defer_k_resize_frames(A.RESIZE_SAMPLE_W, x.data_ptr(), mid.data_ptr(), tables.data_ptr(), *geo, 3, None))
    A.check(lib.defer_k_resize_frames(A.RESIZE_SAMPLE_H, mid.data_ptr(), out.data_ptr(), tables.data_ptr(), *geo, 3, None))
    torch.cuda.synchronize()
    mid_got = mid.cpu().numpy().reshape(n, H, Wo, 3)
    assert np.array_equal(out.cpu().numpy().reshape(out_ref.shape), out_ref)
    for i, (h, w) in enumerate(KERNEL_SIZES):
        assert np.array_equal(mid_got[i, :h], mid_ref[i, :h]), (h, w)
        assert (mid_got[i, h:] == 77).all(), (h, w)                   # rows past the image's height are not written
        assert np.array_equal(out_ref[i], resize_image(slots[i].reshape(-1)[:h * w * 3].reshape(h, w, 3), KERNEL_TARGET,
                                                       interpolation))
    args = (x.data_ptr(), mid.data_ptr(), tables.data_ptr(), *geo)
    assert lib.defer_k_resize_frames(A.RESIZE_SAMPLE_W, *args, 4, None) == A.ERR_INVALID
    assert lib.defer_k_resize_frames(0, *args, 3, None) == A.ERR_INVALID


# ------------------------------------------------------------------------------------------------ stage level
BOUND = (1080, 1920)
FRAME_SIZES = [(480, 640), (224, 224), (1, 1), (300, 200), (1080, 1920)]


def _stem(seed):
    from test_gpu_conv_paths import STEMS, _stem_model
    b, h, w, cin, cout, k, s, pad = STEMS["resnet_b1"]
    return _stem_model(h, w, cin, cout, k, s, pad, seed=seed)


def _frames(sizes, seed):
    return [_image(h, w, seed=seed + i)[None] for i, (h, w) in enumerate(sizes)]


@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("mode,interpolation", [("caffe", "nearest"), ("caffe", "bicubic"), ("tf", "bilinear"),
                                                ("tf", "lanczos")])
def test_stage_resize_frames(mode, interpolation, dtype, path, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch, **({"DEFER_STREAM_MIN_TILES": 1} if path == "fused" else {"DEFER_STEM_FUSED": 0}))
    m = _stem(seed=len(mode + interpolation))
    n = len(FRAME_SIZES)
    items = _frames(FRAME_SIZES, seed=5)
    fin = np.concatenate([resize_image(x, (224, 224), interpolation) for x in items])
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode, max_image_size=BOUND,
                               interpolation=interpolation)
    r0 = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode)
    try:
        y = r.predict_frames(items)
        y0 = r0.predict(fin)
        kernels = [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))]
        kernels0 = [r0.op_info(i)["kernel"] for i in range(len(r0.plan.ops))]
        assert kernels == ["resize_frames_u8_kernel"] * 2 + kernels0, r.describe()
        assert r.num_kernels() == r0.num_kernels() + 2
        mid = r.read_buffer(r.plan.ops[0].out)
        for i, (x, (h, w)) in enumerate(zip(items, FRAME_SIZES)):
            want = x[0] if w == 224 else resize_axis(x[0], 1, *resize_tables(w, 224, interpolation))
            assert np.array_equal(mid[i, :h], want.astype(np.float32)), (h, w)
        assert np.array_equal(r.read_buffer(r.plan.ops[1].out), fin.astype(np.float32))
        assert np.array_equal(_bits(r.read_layer("relu")), _bits(r0.read_layer("relu")))
        assert np.array_equal(_bits(y), _bits(y0))
        kw = r.plan.frames["kw"]
        for i, (n_in, n_out, out_len) in enumerate(((n * 1080 * 1920 * 3, n * 1080 * 224 * 3, 224),
                                                    (n * 1080 * 224 * 3, n * 224 * 224 * 3, 224))):
            assert r.op_info(i)["alg_bytes"] == n_in + n_out + n * (2 + out_len * (2 + kw[i])) * 4
            assert r.time_op(i, iters=3) > 0
        assert r.io_bytes()[0] == n * 1080 * 1920 * 3
    finally:
        r.close()
        r0.close()


def test_lane_reuse_and_never_written_samples(monkeypatch):
    """Depth 1: a small group after a large one runs on the same slots and blocks.  Its samples past the group and the
    bytes past each small image are stale; the results show none of them is read.  A fresh stage's never-written
    samples read zeroed blocks: a 1x1 image of weight 0, all-zero output."""
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch)
    m = _stem(seed=2)
    r = StageRunner.from_model(m, device=0, max_batch=4, depth=1, preprocess="caffe", max_image_size=(720, 1280),
                               interpolation="bilinear")
    r0 = StageRunner.from_model(m, device=0, max_batch=4, depth=1, preprocess="caffe")
    try:
        one = _frames([(5, 9)], seed=40)
        y = r.predict_frames(one)
        assert y.shape == (1, 112, 112, 64)
        assert not r.read_buffer(r.plan.ops[1].out)[1:].any()
        want = r0.predict(np.concatenate([resize_image(one[0], (224, 224), "bilinear")] + [np.zeros((3, 224, 224, 3),
                                                                                                    np.uint8)]))
        assert np.array_equal(_bits(r.result(0)), _bits(want))
        big = _frames([(720, 1280), (700, 1000), (719, 3), (600, 1280)], seed=41)
        small = _frames([(2, 3), (50, 40)], seed=45)
        for group in (big, small, big[:3], small[1:]):
            y = r.predict_frames(group)
            fin = np.concatenate([resize_image(x, (224, 224), "bilinear") for x in group])
            full = np.concatenate([fin, np.zeros((4 - len(group), 224, 224, 3), np.uint8)])
            assert np.array_equal(r.read_buffer(r.plan.ops[1].out)[:len(group)], fin.astype(np.float32))
            assert np.array_equal(_bits(y), _bits(r0.predict(full)[:len(group)]))
    finally:
        r.close()
        r0.close()


def test_submit_frames_refusals_copy_nothing(monkeypatch):
    import torch  # noqa: F401  (initialises the device like the other tests)
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch)
    r = StageRunner.from_model(_stem(seed=3), device=0, max_batch=2, depth=1, preprocess="caffe", max_image_size=(40, 50))
    fixed = StageRunner.from_model(_stem(seed=3), device=0, max_batch=2, depth=1, preprocess="caffe")
    lib = r.lib
    try:
        kw = r.plan.frames["kw"]
        img = _image(40, 50, seed=1)

        def call(hw, header, table_bytes_delta=0, stage=r):
            blocks = pack_frame_tables([(40, 50)], (224, 224), kw, "nearest")
            blocks[0, :2] = header
            hw = np.array([hw], np.int32)
            ptrs = (C.c_void_p * 1)(img.ctypes.data)
            return lib.defer_stage_submit_frames(stage.handle, 0, 0, 1, ptrs, hw.ctypes.data, blocks.ctypes.data,
                                                 blocks.nbytes + table_bytes_delta)
        assert call((41, 50), (41, 50)) == A.ERR_INVALID                     # over the bound
        assert call((40, 51), (40, 51)) == A.ERR_INVALID
        assert call((0, 5), (0, 5)) == A.ERR_INVALID
        assert call((40, 50), (40, 49)) == A.ERR_INVALID                     # header and hw disagree
        assert call((40, 50), (40, 50), table_bytes_delta=4) == A.ERR_INVALID
        assert call((40, 50), (40, 50), table_bytes_delta=-4) == A.ERR_INVALID
        assert call((40, 50), (40, 50), stage=fixed) == A.ERR_INVALID         # a fixed-size stage
        r.sync()
        assert not r.read_buffer(r.plan.input_buf).any()                    # nothing was copied
        with pytest.raises(ValueError, match="submit_frames"):
            r.predict(np.zeros((2, 40, 50, 3), np.uint8))
        with pytest.raises(ValueError, match=r"max_image_size=\(40, 50\)"):
            r.submit_frames(0, 0, [np.zeros((1, 41, 50, 3), np.uint8)])
        with pytest.raises(ValueError, match="do not fit"):
            r.submit_frames(0, 1, [np.zeros((2, 4, 5, 3), np.uint8)])
        assert call((40, 50), (40, 50)) == A.OK
        r.sync()
        assert np.array_equal(r.read_buffer(r.plan.input_buf)[0], img.astype(np.float32))
    finally:
        r.close()
        fixed.close()


def test_stage_create_rejects_bad_frame_ops():
    from defer_b200.node import StageRunner
    from defer_b200.planner import plan_stage
    base = plan_stage(applications.ResNet50(input_shape=(32, 32, 3)), True, True, preprocess="caffe",
                      max_image_size=(40, 48), interpolation="bilinear")

    def create(plan):
        with pytest.raises(A.DeferError) as e:
            StageRunner(plan, device=0, batch=1, depth=1)
        assert e.value.code == A.ERR_INVALID
        return str(e.value)
    for i in (0, 1):
        p = copy.deepcopy(base)
        p.ops[i].kw = 0
        assert "kw" in create(p)
        p = copy.deepcopy(base)
        p.ops[i].kw = 1000
        assert "kw" in create(p)
    p = copy.deepcopy(base)                                  # the width pass changing the height
    p.bufs[p.ops[0].out] = (41, 32, 3, A.BUF_U8)
    assert "SAMPLE_W maps" in create(p)
    p = copy.deepcopy(base)                                  # two width passes
    p.ops[1].mode = A.RESIZE_SAMPLE_W
    assert "SAMPLE_W maps" in create(p)
    p = copy.deepcopy(base)                                  # a width pass alone
    p.ops[1].mode = 0
    assert "resize" in create(p)
    p = copy.deepcopy(base)
    p.ops[1].mode = 3
    assert "unknown mode" in create(p)
    p = copy.deepcopy(base)                                  # weights on a per-sample op
    p.ops[0].w_shift = 0
    assert "no weights" in create(p)


# ------------------------------------------------------------------------------------------------ DEFER end to end
MIXED = [(480, 640), (224, 224), (300, 200), (1, 1), (720, 1280), (719, 1001), (224, 500)]


def _items(n, seed):
    return _frames([MIXED[i % len(MIXED)] for i in range(n)], seed)


@pytest.mark.parametrize("n_stages", [1, 2])
def test_resnet50_defer_mixed_frames(resnet50, n_stages, monkeypatch):
    from oracle import keras_ref
    from test_gpu_conv_paths import _knobs
    from test_gpu_resize import _run_defer
    _knobs(monkeypatch)
    items = _items(40, seed=31)                                # one full group of 32 and a partial one
    y, io, kernels = _run_defer(resnet50, items, n_stages, preprocess="caffe", max_image_size=(720, 1280))
    resized = [resize_image(x, (224, 224)) for x in items]
    y0, io0, _ = _run_defer(resnet50, resized, n_stages, preprocess="caffe")
    assert kernels == ["resize_frames_u8_kernel", "resize_frames_u8_kernel", "preprocess (fused into conv_stem_u8_kernel)",
                       "conv_stem_u8_kernel"], kernels
    assert y.shape == (40, 1000)
    assert np.array_equal(_bits(y), _bits(y0))                # FIFO order and every bit
    assert io[0] == 32 * 720 * 1280 * 3 and io[1] == io0[1]
    ref = keras_ref.predict(resnet50.to_json(), resnet50.get_weights(),
                            applications.preprocess_input(np.concatenate([resized[0], resized[39]])))
    for j, p in enumerate((0, 39)):
        assert keras_ref.rel_err(y[p], ref[j]) <= 1e-3, p


def test_resnet50v2_defer_mixed_frames_tf_bilinear(monkeypatch):
    from test_gpu_conv_paths import _knobs
    from test_gpu_resize import _run_defer
    _knobs(monkeypatch)
    m = applications.ResNet50V2()
    items = _items(9, seed=41)
    y, _, kernels = _run_defer(m, items, 1, preprocess="tf", max_image_size=(720, 1280), interpolation="bilinear")
    y0, _, _ = _run_defer(m, [resize_image(x, (224, 224), "bilinear") for x in items], 1, preprocess="tf")
    assert kernels[:2] == ["resize_frames_u8_kernel"] * 2
    assert np.array_equal(_bits(y), _bits(y0))
