"""Keras load_img's resize on the GPU (`image_size=`, `interpolation=`), bit for bit against the host.

The contract: a uint8 image of `image_size` in a resizing pipeline gives exactly the result of
`applications.resize_image(image, model input, interpolation)` in the same pipeline without the option - for
`defer_k_resize` alone, for the `RESIZE` ops of a stage in both preprocessing modes, dtypes and stem paths, and for
`DEFER` end to end over one and two stages (one process per GPU: the `image-size` case of tests/test_gpu_dist.py)."""
import queue
import sys
import threading
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from defer_b200 import _cabi as A  # noqa: E402
from defer_b200 import applications  # noqa: E402
from defer_b200.resize import INTERPOLATIONS, resize_axis, resize_tables  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

resize_image = applications.resize_image
PRE = {"caffe": applications.preprocess_input, "tf": applications.resnet_v2_preprocess_input}


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _frames(n, h, w, seed):
    """Uniform bytes with saturated blocks and a checkerboard band (the clamp is hit at both ends), per image."""
    from test_resize_host import saturated_image
    return np.stack([saturated_image(h, w, seed=seed + i) for i in range(n)])


# ------------------------------------------------------------------------------------------------ the kernel
# (axis, source h, source w, resized length): downscale, upscale, from one pixel, to three
KERNEL_CASES = [("w", 9, 640, 224), ("w", 5, 5, 32), ("w", 4, 1, 7), ("w", 2, 1000, 3),
                ("h", 480, 11, 224), ("h", 5, 5, 32), ("h", 1, 4, 7), ("h", 1000, 2, 3)]


@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("interpolation", INTERPOLATIONS)
@pytest.mark.parametrize("case", KERNEL_CASES, ids=[f"{a}-{h}x{w}-{n}" for a, h, w, n in KERNEL_CASES])
def test_k_resize_matches_host(case, interpolation, offset):
    lib = A.load()
    import torch
    axis, h, w, n_out = case
    ax = 2 if axis == "w" else 1
    x = _frames(3, h, w, seed=h + w)
    first, count, coef = resize_tables(x.shape[ax], n_out, interpolation)
    ref = resize_axis(x, ax, first, count, coef)
    # offset 1: input and output one byte off any alignment
    xd = torch.zeros(x.size + offset, dtype=torch.uint8, device="cuda")[offset:]
    xd.copy_(torch.from_numpy(x.reshape(-1)))
    y = torch.full((ref.size + offset,), 77, dtype=torch.uint8, device="cuda")[offset:]
    bounds = torch.from_numpy(np.stack([first, count], 1).reshape(-1)).cuda()
    taps = torch.from_numpy(coef.reshape(-1)).cuda()
    _, ho, wo, _ = ref.shape
    args = (xd.data_ptr(), y.data_ptr(), bounds.data_ptr(), taps.data_ptr(), coef.shape[1], 3, h, w, ho, wo)
    A.check(lib.defer_k_resize(*args, 3, None))
    torch.cuda.synchronize()
    assert np.array_equal(y.cpu().numpy().reshape(ref.shape), ref)
    assert lib.defer_k_resize(*args, 4, None) == A.ERR_INVALID
    both = (ho + 1, wo) if axis == "w" else (ho, wo + 1)                                 # two axes change
    assert lib.defer_k_resize(*args[:8], *both, 3, None) == A.ERR_INVALID


# ------------------------------------------------------------------------------------------------ stage level
def _stem(seed):
    from test_gpu_conv_paths import STEMS, _stem_model
    b, h, w, cin, cout, k, s, pad = STEMS["resnet_b1"]
    return _stem_model(h, w, cin, cout, k, s, pad, seed=seed)


@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("mode,interpolation", [("caffe", "nearest"), ("caffe", "bicubic"), ("tf", "bilinear"),
                                                ("tf", "lanczos")])
def test_stage_resize(mode, interpolation, dtype, path, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch, **({"DEFER_STREAM_MIN_TILES": 1} if path == "fused" else {"DEFER_STEM_FUSED": 0}))
    m = _stem(seed=len(mode + interpolation))
    x = _frames(2, 480, 640, seed=5)
    mid = resize_axis(x, 2, *resize_tables(640, 224, interpolation))              # width first, as Pillow
    fin = resize_image(x, (224, 224), interpolation)
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=2, depth=1, preprocess=mode, image_size=(480, 640),
                               interpolation=interpolation)
    r0 = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=2, depth=1, preprocess=mode)
    try:
        y = r.predict(x)
        y0 = r0.predict(fin)
        kernels = [r.op_info(i)["kernel"] for i in range(4)]
        assert kernels[:2] == ["resize_u8_kernel"] * 2, r.describe()
        if path == "fused":
            stem = "conv_stem_u8tf_kernel" if mode == "tf" else "conv_stem_u8_kernel"
            assert kernels[2:] == [f"preprocess (fused into {stem})", stem], r.describe()
        else:
            assert kernels[2] == ("preprocess_tf_kernel" if mode == "tf" else "preprocess_kernel"), r.describe()
        assert r.num_kernels() == r0.num_kernels() + 2
        assert np.array_equal(r.read_buffer(r.plan.ops[0].out), mid.astype(np.float32))
        assert np.array_equal(r.read_buffer(r.plan.ops[1].out), fin.astype(np.float32))
        assert np.array_equal(r.read_buffer(r.plan.input_buf), x.astype(np.float32))
        assert np.array_equal(_bits(r.read_layer("relu")), _bits(r0.read_layer("relu")))
        assert np.array_equal(_bits(y), _bits(y0))
        for i in (0, 1):
            op = r.plan.ops[i]
            tables = r.plan.weights[op.w_scale].nbytes + r.plan.weights[op.w_kernel].nbytes
            n_in, n_out = (2 * 480 * 640 * 3, 2 * 480 * 224 * 3) if i == 0 else (2 * 480 * 224 * 3, 2 * 224 * 224 * 3)
            assert r.op_info(i)["alg_bytes"] == n_in + n_out + tables
            assert r.time_op(i, iters=3) > 0
        assert r.io_bytes()[0] == 2 * 480 * 640 * 3
    finally:
        r.close()
        r0.close()


def test_stage_checks_the_item_size(monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch)
    r = StageRunner.from_model(_stem(seed=1), device=0, max_batch=1, depth=1, preprocess="caffe", image_size=(300, 400))
    try:
        for bad in (np.zeros((1, 224, 224, 3), np.uint8), np.zeros((1, 400, 300, 3), np.uint8),
                    np.zeros((1, 3, 300, 400), np.uint8)):
            with pytest.raises(ValueError, match="image_size=\\(300, 400\\)"):
                r.predict(bad)
        assert r.predict(np.zeros((1, 300, 400, 3), np.uint8)).shape == (1, 112, 112, 64)
    finally:
        r.close()


def test_stage_create_rejects_bad_tables():
    import copy
    from defer_b200.node import StageRunner
    from defer_b200.planner import plan_stage
    base = plan_stage(applications.ResNet50(input_shape=(32, 32, 3)), True, True, preprocess="caffe", image_size=(40, 48),
                      interpolation="bilinear")

    def create(plan):
        with pytest.raises(A.DeferError) as e:
            StageRunner(plan, device=0, batch=1, depth=1)
        assert e.value.code == A.ERR_INVALID
        return str(e.value)

    op = base.ops[0]
    p = copy.deepcopy(base)                                  # taps of the wrong size
    p.weights[op.w_kernel] = p.weights[op.w_kernel][:, :-1].copy()
    assert "w_kernel" in create(p)
    p = copy.deepcopy(base)                                  # bounds of the wrong size
    p.weights[op.w_scale] = p.weights[op.w_scale][:-1].copy()
    assert "w_scale" in create(p)
    p = copy.deepcopy(base)                                  # reads past the end of the row
    p.weights[op.w_scale][-1, 0] = 48 - p.weights[op.w_scale][-1, 1] + 1
    assert "first + count" in create(p)
    p = copy.deepcopy(base)                                  # more taps than the table holds
    p.weights[op.w_scale][5, 1] = op.kw + 1
    assert "count" in create(p)
    p = copy.deepcopy(base)                                  # a negative first
    p.weights[op.w_scale][0, 0] = -1
    assert "0 <= first" in create(p)
    p = copy.deepcopy(base)                                  # both axes in one op
    p.ops[1].in0 = p.input_buf
    assert "exactly one axis" in create(p)
    p = copy.deepcopy(base)                                  # a resize writing fp32
    p.bufs[op.out] = p.bufs[op.out][:3] + (A.BUF_F32,)
    assert "U8" in create(p)
    p = copy.deepcopy(base)                                  # a conv reading the resized image
    p.ops[3].in0 = p.ops[1].out
    assert "PREPROCESS" in create(p)


# ------------------------------------------------------------------------------------------------ DEFER end to end
def _run_defer(model, items, n_stages, **kw):
    from defer_b200.dispatcher import DEFER
    d = DEFER([0] * n_stages, depth=4, coalesce=32, linger_us=20000, **kw)
    in_q, out_q = queue.Queue(), queue.Queue()
    err = []

    def run():
        try:
            d.run_defer(model, applications.default_cuts(model, n_stages), in_q, out_q)
        except BaseException as e:  # noqa: BLE001
            err.append(e)
    t = threading.Thread(target=run, daemon=True)
    t.start()
    assert d.wait_ready(300)
    io = d.stages[0].io_bytes()
    kernels = [d.stages[0].op_info(i)["kernel"] for i in range(len(d.stages[0].plan.ops))][:4]
    for x in items:
        in_q.put(x)
    try:
        got = [out_q.get(timeout=120) for _ in items]
    finally:
        d.close()
        t.join(timeout=60)
    assert not err, err
    return np.concatenate(got), io, kernels


@pytest.mark.parametrize("n_stages", [1, 2])
def test_resnet50_defer_frames(resnet50, n_stages, monkeypatch):
    from oracle import keras_ref
    from test_gpu_conv_paths import _knobs
    _knobs(monkeypatch)
    frames = _frames(40, 480, 640, seed=31)                # one full group of 32 and a partial one
    items = [frames[i:i + 1] for i in range(len(frames))]
    y, io, kernels = _run_defer(resnet50, items, n_stages, preprocess="caffe", image_size=(480, 640))
    resized = [resize_image(x, (224, 224)) for x in items]
    y0, io0, _ = _run_defer(resnet50, resized, n_stages, preprocess="caffe")
    assert kernels == ["resize_u8_kernel", "resize_u8_kernel", "preprocess (fused into conv_stem_u8_kernel)",
                       "conv_stem_u8_kernel"], kernels
    assert y.shape == (40, 1000)
    assert np.array_equal(_bits(y), _bits(y0))                # FIFO order and every bit
    assert io[0] == 32 * 480 * 640 * 3 and io[1] == io0[1]
    ref = keras_ref.predict(resnet50.to_json(), resnet50.get_weights(),
                            applications.preprocess_input(np.concatenate([resized[0], resized[39]])))
    for j, p in enumerate((0, 39)):
        assert keras_ref.rel_err(y[p], ref[j]) <= 1e-3, p


def test_resnet50v2_defer_frames_tf_bilinear(monkeypatch):
    from test_gpu_conv_paths import _knobs
    _knobs(monkeypatch)
    m = applications.ResNet50V2()
    frames = _frames(9, 480, 640, seed=41)
    items = [frames[i:i + 1] for i in range(len(frames))]
    y, _, kernels = _run_defer(m, items, 1, preprocess="tf", image_size=(480, 640), interpolation="bilinear")
    y0, _, _ = _run_defer(m, [resize_image(x, (224, 224), "bilinear") for x in items], 1, preprocess="tf")
    assert kernels[:2] == ["resize_u8_kernel"] * 2
    assert np.array_equal(_bits(y), _bits(y0))
