"""Keras load_img(keep_aspect_ratio=True) on the GPU, bit for bit against the host.

The contract: an item in a `keep_aspect_ratio=True` pipeline gives exactly what `applications.resize_image(item, model
input, interpolation, keep_aspect_ratio=True)` gives fed to the same pipeline without resizing - with `image_size=`
(landscape, portrait, and an axis at the model input's length that its crop box resamples), with `max_image_size=` and
items of mixed sizes in one microbatch, and with `decode="jpeg"` on the committed fixtures and on landscape and portrait
encodes; in both preprocessing modes, dtypes and stem paths, after lane re-use, and through `DEFER` over one and two
stages."""
import copy
import functools
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests", ROOT / "tools"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import _cabi as A  # noqa: E402
from defer_b200 import applications  # noqa: E402
from defer_b200 import jpeg  # noqa: E402
from defer_b200.resize import crop_boxes, resize_axis, resize_tables  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

TARGET = (224, 224)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _image(h, w, seed):
    from test_resize_host import saturated_image
    return saturated_image(h, w, seed=seed)


def _keep(x, interpolation):
    return applications.resize_image(x, TARGET, interpolation, keep_aspect_ratio=True)


def _stem(seed):
    from test_gpu_conv_paths import STEMS, _stem_model
    b, h, w, cin, cout, k, s, pad = STEMS["resnet_b1"]
    return _stem_model(h, w, cin, cout, k, s, pad, seed=seed)


PATHS = [{"DEFER_STREAM_MIN_TILES": 1}, {"DEFER_STEM_FUSED": 0}]
MODES = [("caffe", "nearest"), ("caffe", "bicubic"), ("tf", "bilinear"), ("tf", "lanczos")]


# ------------------------------------------------------------------------------------------------ image_size
@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("mode,interpolation", MODES)
@pytest.mark.parametrize("image_size", [(480, 640), (640, 480), (100, 224), (224, 1000)])
def test_stage_image_size(image_size, mode, interpolation, dtype, path, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch, **PATHS[path == "unfused"])
    m = _stem(seed=len(mode + interpolation))
    h, w = image_size
    x = np.stack([_image(h, w, seed=7 + i) for i in range(2)])
    fin = _keep(x, interpolation)
    box_w, _ = crop_boxes(h, w, TARGET, True)
    mid = resize_axis(x, 2, *resize_tables(w, 224, interpolation, box_w))
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=2, depth=1, preprocess=mode, image_size=image_size,
                               interpolation=interpolation, keep_aspect_ratio=True)
    r0 = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=2, depth=1, preprocess=mode)
    try:
        y = r.predict(x)
        y0 = r0.predict(fin)
        # (224, 1000): the height is at the model input's and its box is whole, so only the width is resized
        n_resize = 1 if image_size == (224, 1000) else 2
        assert [r.op_info(i)["kernel"] for i in range(n_resize)] == ["resize_u8_kernel"] * n_resize, r.describe()
        assert r.num_kernels() == r0.num_kernels() + n_resize
        # (100, 224): the width keeps its length and is resampled under its box, by an op that names the axis
        assert r.plan.ops[0].mode == (A.RESIZE_W if w == 224 else 0)
        assert np.array_equal(r.read_buffer(r.plan.ops[0].out), mid.astype(np.float32))
        assert np.array_equal(r.read_buffer(r.plan.ops[n_resize - 1].out), fin.astype(np.float32))
        assert np.array_equal(_bits(r.read_layer("relu")), _bits(r0.read_layer("relu")))
        assert np.array_equal(_bits(y), _bits(y0))
        assert r.io_bytes()[0] == 2 * h * w * 3
    finally:
        r.close()
        r0.close()


def test_stage_create_checks_the_named_axis():
    from defer_b200.node import StageRunner
    from defer_b200.planner import plan_stage
    base = plan_stage(applications.ResNet50(input_shape=(32, 32, 3)), True, True, preprocess="caffe", image_size=(16, 32),
                      interpolation="bilinear", keep_aspect_ratio=True)
    assert [o.mode for o in base.ops[:2]] == [A.RESIZE_W, 0]

    def create(plan):
        with pytest.raises(A.DeferError) as e:
            StageRunner(plan, device=0, batch=1, depth=1)
        assert e.value.code == A.ERR_INVALID
        return str(e.value)
    p = copy.deepcopy(base)                                   # mode 0 cannot tell the axis of a 16x32 -> 16x32 pass
    p.ops[0].mode = 0
    assert "exactly one axis" in create(p)
    p = copy.deepcopy(base)                                   # the height pass named as a width pass
    p.ops[1].mode = A.RESIZE_W
    assert "mode W / H" in create(p)
    p = copy.deepcopy(base)                                   # its tables must fit the named axis
    p.weights[base.ops[0].w_scale][-1, 0] = 32
    assert "first + count" in create(p)
    r = StageRunner(base, device=0, batch=1, depth=1)
    r.close()


# ------------------------------------------------------------------------------------------------ max_image_size
BOUND = (1080, 1920)
FRAME_SIZES = [(480, 640), (640, 480), (1080, 1920), (1080, 607), (100, 224), (224, 1000), (1, 1), (1, 1000), (1000, 1)]


def _frames(sizes, seed):
    return [_image(h, w, seed=seed + i)[None] for i, (h, w) in enumerate(sizes)]


@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("mode,interpolation", MODES)
def test_stage_mixed_sizes(mode, interpolation, dtype, path, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch, **PATHS[path == "unfused"])
    m = _stem(seed=len(mode + interpolation))
    n = len(FRAME_SIZES)
    items = _frames(FRAME_SIZES, seed=5)
    fin = np.concatenate([_keep(x, interpolation) for x in items])
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode, max_image_size=BOUND,
                               interpolation=interpolation, keep_aspect_ratio=True)
    r0 = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode)
    try:
        y = r.predict_frames(items)
        y0 = r0.predict(fin)
        assert [r.op_info(i)["kernel"] for i in range(2)] == ["resize_frames_u8_kernel"] * 2, r.describe()
        mid = r.read_buffer(r.plan.ops[0].out)
        for i, (x, (h, w)) in enumerate(zip(items, FRAME_SIZES)):
            box_w, _ = crop_boxes(h, w, TARGET, True)
            want = x[0] if (w == 224 and box_w is None) else resize_axis(x[0], 1, *resize_tables(w, 224, interpolation,
                                                                                                 box_w))
            assert np.array_equal(mid[i, :h], want.astype(np.float32)), (h, w)
        assert np.array_equal(r.read_buffer(r.plan.ops[1].out), fin.astype(np.float32))
        assert np.array_equal(_bits(y), _bits(y0))
    finally:
        r.close()
        r0.close()


def test_lane_reuse_after_larger_items(monkeypatch):
    """Depth 1: small groups after large ones run on the same slots and blocks; stale bytes and tables are never read."""
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch)
    m = _stem(seed=2)
    r = StageRunner.from_model(m, device=0, max_batch=4, depth=1, preprocess="caffe", max_image_size=(720, 1280),
                               interpolation="bilinear", keep_aspect_ratio=True)
    r0 = StageRunner.from_model(m, device=0, max_batch=4, depth=1, preprocess="caffe")
    try:
        big = _frames([(720, 1280), (1280 // 2, 1000), (719, 3), (600, 1280)], seed=41)
        small = _frames([(2, 3), (50, 40), (224, 100)], seed=45)
        for group in (big, small, big[:3], small[1:], big):
            y = r.predict_frames(group)
            fin = np.concatenate([_keep(x, "bilinear") for x in group])
            full = np.concatenate([fin, np.zeros((4 - len(group), 224, 224, 3), np.uint8)])
            assert np.array_equal(r.read_buffer(r.plan.ops[1].out)[:len(group)], fin.astype(np.float32))
            assert np.array_equal(_bits(y), _bits(r0.predict(full)[:len(group)]))
    finally:
        r.close()
        r0.close()


# ------------------------------------------------------------------------------------------------ decode="jpeg"
JPEG_GOLDEN = ROOT / "tests" / "golden"
FIXTURES = ["jpeg/photo_480x640_420_q75.jpg", "jpeg/photo_1080x1920_420_q50.jpg", "jpeg/photo_5x4_444_q50.jpg",
            "jpeg/photo_223x225_422_q50_rr1.jpg", "jpeg/photo_1x17_gray_q5.jpg", "jpeg/checker_31x47_420_q95.jpg",
            "jpeg_progressive/photo_480x640_420_q75.jpg", "jpeg_progressive/photo_17x33_444_q50.jpg"]


@functools.lru_cache(maxsize=None)
def _jpeg_files():
    """The fixtures, then landscape and portrait encodes, baseline and progressive, up to 1920 on a side."""
    from make_jpeg_fixtures import content, encode
    files = [(JPEG_GOLDEN / nm).read_bytes() for nm in FIXTURES]
    for i, (h, w, sub, prog) in enumerate([(640, 480, "420", False), (1920, 1080, "422", False), (1080, 1920, "444", True),
                                           (1000, 300, "gray", True), (300, 1001, "420", False)]):
        files.append(encode(content("photo", h, w, seed=60 + i), sub, 80, progressive=prog))
    return tuple(files)


@functools.lru_cache(maxsize=None)
def _decoded(i):
    return jpeg.decode_jpeg(_jpeg_files()[i])


@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("mode,interpolation", [("caffe", "nearest"), ("tf", "bilinear"), ("caffe", "lanczos")])
def test_stage_jpeg(mode, interpolation, dtype, path, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch, **PATHS[path == "unfused"])
    m = _stem(seed=len(mode + interpolation))
    files = list(_jpeg_files())
    n = len(files)
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode, max_image_size=(1920, 1920),
                               interpolation=interpolation, decode="jpeg", keep_aspect_ratio=True)
    r0 = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode)
    try:
        y = r.predict_jpegs(files)
        fin = np.concatenate([_keep(_decoded(i), interpolation)[None] for i in range(n)])
        assert np.array_equal(r.read_buffer(r.plan.ops[2].out), fin.astype(np.float32))
        assert np.array_equal(_bits(y), _bits(r0.predict(fin)))
        # the small files after the large ones, on the same slots
        y = r.predict_jpegs(files[2:6])
        assert np.array_equal(_bits(y), _bits(r0.predict(np.concatenate([fin[2:6], fin[:n - 4]]))[:4]))
    finally:
        r.close()
        r0.close()


# ------------------------------------------------------------------------------------------------ DEFER end to end
def _ingress(kind, n):
    if kind == "image_size":
        frames = np.stack([_image(640, 480, seed=31 + i) for i in range(n)])
        return [frames[i:i + 1] for i in range(n)], {"image_size": (640, 480)}
    if kind == "max_image_size":
        return _frames([FRAME_SIZES[i % len(FRAME_SIZES)] for i in range(n)], seed=31), {"max_image_size": BOUND}
    files = _jpeg_files()
    return [files[i % len(files)] for i in range(n)], {"max_image_size": (1920, 1920), "decode": "jpeg"}


@pytest.mark.parametrize("kind", ["image_size", "max_image_size", "jpeg"])
@pytest.mark.parametrize("n_stages", [1, 2])
def test_resnet50_defer(resnet50, n_stages, kind, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from test_gpu_resize import _run_defer
    _knobs(monkeypatch)
    n = 40 if kind == "max_image_size" else 12                 # 40: one full group of 32 and a partial one
    items, kw = _ingress(kind, n)
    y, io, kernels = _run_defer(resnet50, items, n_stages, preprocess="caffe", interpolation="bilinear",
                                keep_aspect_ratio=True, **kw)
    images = [_decoded(i % len(_jpeg_files())) for i in range(n)] if kind == "jpeg" else items
    resized = [_keep(x, "bilinear").reshape(1, 224, 224, 3) for x in images]
    y0, io0, _ = _run_defer(resnet50, resized, n_stages, preprocess="caffe")
    assert "resize" in " ".join(kernels), kernels
    assert y.shape == (n, 1000)
    assert np.array_equal(_bits(y), _bits(y0))                # FIFO order and every bit
    assert io[1] == io0[1]
