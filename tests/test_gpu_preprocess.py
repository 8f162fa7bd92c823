"""uint8 ingress with Keras caffe preprocessing on the GPU (`preprocess="caffe"`), bit for bit against the host.

The contract: a uint8 image in a preprocessing pipeline gives exactly the result of `applications.preprocess_input(image)`
in the same pipeline without the option - on the standalone `preprocess_kernel`, on the fused stem that preprocesses
each tap as it builds its patch rows (`conv_stem_u8_kernel`), for every dtype, stem path, coalescing factor and stage
count."""
import queue
import threading

import numpy as np
import pytest

from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200 import keras_like as K
from defer_b200.dispatcher import DEFER
from defer_b200.node import StageRunner
from test_gpu_conv_paths import STEM_PATHS, STEMS, _knobs, _stem_model

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _image(b, h, w, seed):
    """Uniform 0..255 with saturated borders: 255 on the top row and left column, 0 on the bottom row and right column."""
    x = applications.synthetic_image(b, (h, w, 3), seed=seed)
    x[:, 0, :, :] = 255
    x[:, :, 0, :] = 255
    x[:, -1, :, :] = 0
    x[:, :, -1, :] = 0
    x[:, h // 2, w // 2, :] = (255, 0, 255)
    return x


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("shape", [(1, 224, 224), (3, 37, 53), (2, 1, 5), (1, 7, 1)])
@pytest.mark.parametrize("offset", [0, 1])
def test_k_preprocess_matches_host(shape, offset):
    lib = A.load()
    import torch
    n, h, w = shape
    x = _image(n, h, w, seed=h * w)
    ref = applications.preprocess_input(x)
    # offset 1: an unaligned image (the one-pixel-per-thread path)
    xd_store = torch.zeros(x.size + offset, dtype=torch.uint8, device="cuda")
    xd = xd_store[offset:]
    xd.copy_(torch.from_numpy(x.reshape(-1)))
    shift = torch.from_numpy(applications.caffe_shift()).cuda()
    y = torch.full((x.size + offset,), float("nan"), dtype=torch.float32, device="cuda")[offset:]
    A.check(lib.defer_k_preprocess(xd.data_ptr(), shift.data_ptr(), y.data_ptr(), n, h, w, 3, None))
    torch.cuda.synchronize()
    assert np.array_equal(_bits(y.cpu().numpy().reshape(ref.shape)), _bits(ref))
    assert lib.defer_k_preprocess(xd.data_ptr(), shift.data_ptr(), y.data_ptr(), n, h, w, 4, None) == A.ERR_INVALID


# ------------------------------------------------------------------------------------------------ stem paths at stage level
RGB_STEMS = [k for k in STEMS if STEMS[k][3] == 3]


def _pair(m, x, dtype, path, env, monkeypatch):
    """(u8 stage output, fp32 stage output on preprocess_input(x), kernels, launch counts) for one stem path."""
    _knobs(monkeypatch, **env)
    backend = 1 if path == "simt" else 0
    res = {}
    for mode in (None, "caffe"):
        r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=x.shape[0], depth=1, conv_backend=backend,
                                   preprocess=mode)
        try:
            r.predict(x if mode else applications.preprocess_input(x))
            res[mode] = (r.read_layer("relu"), [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))], r.num_kernels(),
                         r.describe())
        finally:
            r.close()
    return res["caffe"], res[None]


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("name", RGB_STEMS)
def test_stem_paths_u8(name, dtype, monkeypatch):
    b, h, w, cin, cout, k, s, pad = STEMS[name]
    m = _stem_model(h, w, cin, cout, k, s, pad, seed=len(name))
    x = _image(b, h, w, seed=len(name))
    for path, (kernel, env) in list(STEM_PATHS.items()) + [("simt", ("conv_simt_kernel", {}))]:
        (y8, k8, n8, d8), (y32, k32, n32, _) = _pair(m, x, dtype, path, env, monkeypatch)
        fused = path == "fused" and cout == 64
        if path == "fused" and cout != 64:
            kernel = "stem_im2col+conv_stream_kernel"
        assert k32[0] == kernel, (name, path, k32)
        if fused:
            assert k8[:2] == ["preprocess (fused into conv_stem_u8_kernel)", "conv_stem_u8_kernel"], (name, path, d8)
            assert n8 == n32, (name, path, d8)
        else:
            assert k8[:2] == ["preprocess_kernel", kernel], (name, path, d8)
            assert n8 == n32 + 1, (name, path, d8)
        assert np.array_equal(_bits(y8), _bits(y32)), (name, dtype, path)


def test_stem_u8_float32_simt(monkeypatch):
    b, h, w, cin, cout, k, s, pad = STEMS["straddle"]
    m = _stem_model(h, w, cin, cout, k, s, pad, seed=3)
    x = _image(b, h, w, seed=3)
    (y8, k8, n8, _), (y32, k32, n32, _) = _pair(m, x, "float32_simt", "simt", {}, monkeypatch)
    assert k8[:2] == ["preprocess_kernel", "conv_simt_kernel"] and k32[0] == "conv_simt_kernel"
    assert n8 == n32 + 1
    assert np.array_equal(_bits(y8), _bits(y32))


def test_fused_stage_introspection(monkeypatch):
    """The folded op launches nothing, cannot be timed, and its never-written F32 image cannot be read."""
    _knobs(monkeypatch)
    b, h, w, cin, cout, k, s, pad = STEMS["resnet_b1"]
    m = _stem_model(h, w, cin, cout, k, s, pad, seed=1)
    x = _image(b, h, w, seed=1)
    r = StageRunner.from_model(m, device=0, dtype="float32", max_batch=1, depth=1, preprocess="caffe")
    r32 = StageRunner.from_model(m, device=0, dtype="float32", max_batch=1, depth=1)
    try:
        r.predict(x)
        assert "preprocess (fused into conv_stem_u8_kernel)" in r.describe()
        with pytest.raises(A.DeferError, match="folded into op 1"):
            r.time_op(0)
        with pytest.raises(A.DeferError, match="never written"):
            r.read_buffer(r.plan.ops[0].out)
        assert np.array_equal(r.read_buffer(r.plan.input_buf), x.astype(np.float32))     # U8 reads back as 0..255
        assert r.time_op(1, iters=3) > 0
        conv8, conv32 = r.op_info(1), r32.op_info(0)
        assert conv32["alg_bytes"] - conv8["alg_bytes"] == 3 * x.size       # the image is read at 1 B/elem, not 4
        assert r.op_info(0)["alg_bytes"] == 0
        assert r.io_bytes()[0] * 4 == r32.io_bytes()[0]
    finally:
        r.close()
        r32.close()
    _knobs(monkeypatch, DEFER_STEM_FUSED=0, DEFER_STREAM_MIN_TILES=1)
    r = StageRunner.from_model(m, device=0, dtype="float32", max_batch=1, depth=1, preprocess="caffe")
    try:
        r.predict(x)
        assert r.op_info(0)["kernel"] == "preprocess_kernel"
        assert r.op_info(0)["alg_bytes"] == x.size * (1 + 4)
        assert r.time_op(0, iters=3) > 0
        assert np.array_equal(_bits(r.read_buffer(r.plan.ops[0].out)), _bits(applications.preprocess_input(x)))
    finally:
        r.close()


def test_first_op_not_a_conv(monkeypatch):
    _knobs(monkeypatch)
    K.clear_session()
    inp = K.Input(shape=(19, 23, 3))
    x = K.GlobalAveragePooling2D(name="gap")(inp)
    x = K.Dense(10, activation="softmax", name="fc")(x)
    m = K.Model(inp, x, name="gap_head")
    applications.synthetic_weights(m, seed=2)
    img = _image(2, 19, 23, seed=4)
    for dtype in ("float32", "bfloat16", "float32_simt"):
        outs = {}
        for mode in (None, "caffe"):
            r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=2, depth=1, preprocess=mode)
            try:
                outs[mode] = r.predict(img if mode else applications.preprocess_input(img))
                if mode:
                    assert r.op_info(0)["kernel"] == "preprocess_kernel"
            finally:
                r.close()
        assert np.array_equal(_bits(outs["caffe"]), _bits(outs[None])), dtype


# ------------------------------------------------------------------------------------------------ ResNet50 through DEFER
def _run_defer(model, items, n_stages, preprocess):
    d = DEFER([0] * n_stages, depth=4, coalesce=32, linger_us=20000, preprocess=preprocess)
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
    for x in items:
        in_q.put(x)
    try:
        got = [out_q.get(timeout=120) for _ in items]
    finally:
        d.close()
        t.join(timeout=60)
    assert not err, err
    return np.concatenate(got), io


@pytest.mark.parametrize("n_stages", [1, 2])
def test_resnet50_defer_u8_items(resnet50, n_stages, monkeypatch):
    from oracle import keras_ref
    _knobs(monkeypatch)
    imgs = _image(40, 224, 224, seed=17)                  # one full group of 32 and a partial one
    items8 = [imgs[i:i + 1] for i in range(len(imgs))]
    y8, io8 = _run_defer(resnet50, items8, n_stages, "caffe")
    y32, io32 = _run_defer(resnet50, [applications.preprocess_input(x) for x in items8], n_stages, None)
    assert y8.shape == (40, 1000)
    assert np.array_equal(_bits(y8), _bits(y32))              # FIFO order and every bit
    assert io8[0] * 4 == io32[0] and io8[1] == io32[1]
    ref = keras_ref.predict(resnet50.to_json(), resnet50.get_weights(), applications.preprocess_input(imgs[[0, 39]]))
    for j, p in enumerate((0, 39)):
        assert keras_ref.rel_err(y8[p], ref[j]) <= 1e-3, p


# ------------------------------------------------------------------------------------------------ misuse
def test_float_item_to_caffe_pipeline_is_an_error(monkeypatch):
    _knobs(monkeypatch)
    m = applications.ResNet50(input_shape=(32, 32, 3))
    d = DEFER([0], depth=2, coalesce=2, preprocess="caffe")
    in_q, out_q = queue.Queue(), queue.Queue()
    err = []
    t = threading.Thread(target=lambda: err.append(pytest.raises(TypeError, d.run_defer, m, [], in_q, out_q)), daemon=True)
    t.start()
    assert d.wait_ready(120)
    in_q.put(applications.preprocess_input(applications.synthetic_image(1, (32, 32, 3))))
    t.join(timeout=60)
    assert not t.is_alive() and err and "uint8" in str(err[0].value)
    d.close()
    r = StageRunner.from_model(m, device=0, max_batch=1, depth=1, preprocess="caffe")
    try:
        with pytest.raises(TypeError, match="astype"):
            r.predict(np.zeros((1, 32, 32, 3), np.float32))
        chw = np.zeros((1, 3, 32, 32), np.uint8)                # channels-first: the same byte count, the wrong image
        with pytest.raises(ValueError, match="channels-last"):
            r.predict(chw)
        with pytest.raises(ValueError, match="channels-last"):
            r.submit_items(0, [chw])
        with pytest.raises(ValueError, match="channels-last"):
            r.submit_part(0, 0, chw)
        r.predict(np.zeros((1, 32, 32, 3), np.uint8))
    finally:
        r.close()


def test_stage_create_rejects_u8_misuse():
    m = applications.ResNet50(input_shape=(32, 32, 3))
    from defer_b200.planner import plan_stage
    import copy

    def create(plan, **kw):
        with pytest.raises(A.DeferError) as e:
            StageRunner(plan, device=0, batch=1, depth=1, **kw)
        assert e.value.code == A.ERR_INVALID
        return str(e.value)

    base = plan_stage(m, is_first=True, is_last=True, preprocess="caffe")
    p = copy.deepcopy(base)                                  # U8 on a buffer that is not the stage input
    h, w, c, _ = p.bufs[3]
    p.bufs[3] = (h, w, c, A.BUF_U8)
    assert "U8" in create(p)
    assert "U8" in create(copy.deepcopy(base), is_first=False)   # U8 input of a stage that is not first
    p = copy.deepcopy(base)                                  # PREPROCESS writing an ACT buffer
    p.bufs[p.ops[0].out] = p.bufs[p.ops[0].out][:3] + (A.BUF_ACT,)
    assert "F32" in create(p)
    p = copy.deepcopy(base)                                  # wrong shift size
    p.weights[p.ops[0].w_shift] = np.zeros(4, np.float32)
    assert "3 fp32" in create(p)
    p = copy.deepcopy(base)                                  # PREPROCESS over 4 channels
    p.bufs[0] = p.bufs[0][:2] + (4, A.BUF_U8)
    p.bufs[1] = p.bufs[1][:2] + (4, A.BUF_F32)
    assert "3 channels" in create(p)
    p = copy.deepcopy(base)                                  # a conv reading the U8 image directly
    p.ops[1].in0 = p.input_buf
    assert "PREPROCESS" in create(p)
