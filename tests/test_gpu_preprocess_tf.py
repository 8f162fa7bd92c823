"""uint8 ingress with Keras tf-mode preprocessing on the GPU (`preprocess="tf"`, the ResNet V2 family), bit for bit
against the host.

The contract: a uint8 image in a tf-preprocessing pipeline gives exactly the result of
`applications.resnet_v2_preprocess_input(image)` in the same pipeline without the option - on the standalone
`preprocess_tf_kernel`, on the fused stem that preprocesses each tap as it builds its patch rows
(`conv_stem_u8tf_kernel`), for every dtype, stem path, coalescing factor and stage count."""
import copy
import queue
import threading

import numpy as np
import pytest

from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200.dispatcher import DEFER
from defer_b200.node import StageRunner
from defer_b200.planner import plan_stage
from test_gpu_conv_paths import STEM_PATHS, STEMS, _knobs, _stem_model
from test_gpu_preprocess import _bits, _image

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

pre_tf = applications.resnet_v2_preprocess_input


def _every_byte_image():
    """(1, 16, 16, 3): each channel holds all 256 byte values, in a different order per channel."""
    v = np.arange(256, dtype=np.uint8)
    return np.stack([v, v[::-1], np.roll(v, 85)], axis=-1).reshape(1, 16, 16, 3)


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("shape", [None, (1, 224, 224), (3, 37, 53), (2, 1, 5), (1, 7, 1)])
@pytest.mark.parametrize("offset", [0, 1])
def test_k_preprocess_tf_matches_host(shape, offset):
    lib = A.load()
    import torch
    x = _every_byte_image() if shape is None else _image(*shape, seed=shape[1] * shape[2])
    n, h, w, _ = x.shape
    ref = pre_tf(x)
    # offset 1: an unaligned image (the one-pixel-per-thread path)
    xd = torch.zeros(x.size + offset, dtype=torch.uint8, device="cuda")[offset:]
    xd.copy_(torch.from_numpy(x.reshape(-1)))
    y = torch.full((x.size + offset,), float("nan"), dtype=torch.float32, device="cuda")[offset:]
    A.check(lib.defer_k_preprocess_tf(xd.data_ptr(), y.data_ptr(), n, h, w, 3, None))
    torch.cuda.synchronize()
    assert np.array_equal(_bits(y.cpu().numpy().reshape(ref.shape)), _bits(ref))
    assert lib.defer_k_preprocess_tf(xd.data_ptr(), y.data_ptr(), n, h, w, 4, None) == A.ERR_INVALID


# ------------------------------------------------------------------------------------------------ stem paths at stage level
RGB_STEMS = [k for k in STEMS if STEMS[k][3] == 3]


def _pair(m, x, dtype, path, env, monkeypatch):
    """(u8 tf stage output, fp32 stage output on resnet_v2_preprocess_input(x), kernels, launch counts) for one path."""
    _knobs(monkeypatch, **env)
    backend = 1 if path == "simt" else 0
    res = {}
    for mode in (None, "tf"):
        r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=x.shape[0], depth=1, conv_backend=backend,
                                   preprocess=mode)
        try:
            r.predict(x if mode else pre_tf(x))
            res[mode] = (r.read_layer("relu"), [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))], r.num_kernels(),
                         r.describe())
        finally:
            r.close()
    return res["tf"], res[None]


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("name", RGB_STEMS)
def test_stem_paths_u8_tf(name, dtype, monkeypatch):
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
            assert k8[:2] == ["preprocess (fused into conv_stem_u8tf_kernel)", "conv_stem_u8tf_kernel"], (name, path, d8)
            assert n8 == n32, (name, path, d8)
        else:
            assert k8[:2] == ["preprocess_tf_kernel", kernel], (name, path, d8)
            assert n8 == n32 + 1, (name, path, d8)
        assert np.array_equal(_bits(y8), _bits(y32)), (name, dtype, path)


def test_stem_u8_tf_float32_simt(monkeypatch):
    b, h, w, cin, cout, k, s, pad = STEMS["straddle"]
    m = _stem_model(h, w, cin, cout, k, s, pad, seed=3)
    x = _image(b, h, w, seed=3)
    (y8, k8, n8, _), (y32, k32, n32, _) = _pair(m, x, "float32_simt", "simt", {}, monkeypatch)
    assert k8[:2] == ["preprocess_tf_kernel", "conv_simt_kernel"] and k32[0] == "conv_simt_kernel"
    assert n8 == n32 + 1
    assert np.array_equal(_bits(y8), _bits(y32))


def test_fused_tf_stage_introspection(monkeypatch):
    """The folded op launches nothing and cannot be timed; unfolded, its image is the host's, bit for bit."""
    _knobs(monkeypatch)
    b, h, w, cin, cout, k, s, pad = STEMS["resnet_b1"]
    m = _stem_model(h, w, cin, cout, k, s, pad, seed=1)
    x = _image(b, h, w, seed=1)
    r = StageRunner.from_model(m, device=0, dtype="float32", max_batch=1, depth=1, preprocess="tf")
    try:
        r.predict(x)
        assert "preprocess (fused into conv_stem_u8tf_kernel)" in r.describe()
        with pytest.raises(A.DeferError, match="folded into op 1"):
            r.time_op(0)
        with pytest.raises(A.DeferError, match="never written"):
            r.read_buffer(r.plan.ops[0].out)
        assert r.time_op(1, iters=3) > 0
    finally:
        r.close()
    _knobs(monkeypatch, DEFER_STEM_FUSED=0, DEFER_STREAM_MIN_TILES=1)
    r = StageRunner.from_model(m, device=0, dtype="float32", max_batch=1, depth=1, preprocess="tf")
    try:
        r.predict(x)
        assert r.op_info(0)["kernel"] == "preprocess_tf_kernel"
        assert r.time_op(0, iters=3) > 0
        assert np.array_equal(_bits(r.read_buffer(r.plan.ops[0].out)), _bits(pre_tf(x)))
    finally:
        r.close()


# ------------------------------------------------------------------------------------------------ ResNet50V2 through DEFER
@pytest.fixture(scope="module")
def resnet50v2():
    return applications.ResNet50V2()


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
    kernels = [d.stages[0].op_info(i)["kernel"] for i in range(2)]
    for x in items:
        in_q.put(x)
    try:
        got = [out_q.get(timeout=120) for _ in items]
    finally:
        d.close()
        t.join(timeout=60)
    assert not err, err
    return np.concatenate(got), kernels


@pytest.mark.parametrize("n_stages,fold", [(1, 0), (2, 0), (2, 1)])
def test_resnet50v2_defer_u8_tf_items(resnet50v2, n_stages, fold, monkeypatch):
    from oracle import keras_ref
    _knobs(monkeypatch)
    monkeypatch.setenv("DEFER_FOLD_AFFINE", str(fold))
    imgs = _image(40, 224, 224, seed=23)                  # one full group of 32 and a partial one
    items8 = [imgs[i:i + 1] for i in range(len(imgs))]
    y8, k8 = _run_defer(resnet50v2, items8, n_stages, "tf")
    y32, _ = _run_defer(resnet50v2, [pre_tf(x) for x in items8], n_stages, None)
    assert k8 == ["preprocess (fused into conv_stem_u8tf_kernel)", "conv_stem_u8tf_kernel"], k8
    assert y8.shape == (40, 1000)
    assert np.array_equal(_bits(y8), _bits(y32))              # FIFO order and every bit
    ref = keras_ref.predict(resnet50v2.to_json(), resnet50v2.get_weights(), pre_tf(imgs[[0, 39]]))
    for j, p in enumerate((0, 39)):
        assert keras_ref.rel_err(y8[p], ref[j]) <= 1e-3, p


# ------------------------------------------------------------------------------------------------ misuse
def test_float_item_to_tf_pipeline_is_an_error(monkeypatch):
    _knobs(monkeypatch)
    m = applications.ResNet50V2(input_shape=(32, 32, 3))
    d = DEFER([0], depth=2, coalesce=2, preprocess="tf")
    in_q, out_q = queue.Queue(), queue.Queue()
    err = []
    t = threading.Thread(target=lambda: err.append(pytest.raises(TypeError, d.run_defer, m, [], in_q, out_q)), daemon=True)
    t.start()
    assert d.wait_ready(120)
    in_q.put(pre_tf(applications.synthetic_image(1, (32, 32, 3))))
    t.join(timeout=60)
    assert not t.is_alive() and err and "preprocess='tf'" in str(err[0].value)
    d.close()
    r = StageRunner.from_model(m, device=0, max_batch=1, depth=1, preprocess="tf")
    try:
        with pytest.raises(TypeError, match="preprocess='tf'"):
            r.predict(np.zeros((1, 32, 32, 3), np.float32))
        r.predict(np.zeros((1, 32, 32, 3), np.uint8))
    finally:
        r.close()


def test_tf_on_a_caffe_model_is_refused():
    m = applications.ResNet50(input_shape=(32, 32, 3))
    with pytest.raises(ValueError, match="'caffe'"):
        StageRunner.from_model(m, device=0, max_batch=1, depth=1, preprocess="tf")
    d = DEFER([0], depth=2, preprocess="tf")
    with pytest.raises(ValueError, match="'caffe'"):
        d.run_defer(m, [], queue.Queue(), queue.Queue())
    assert not d.stages


def test_stage_create_rejects_mode_misuse():
    def create(plan):
        with pytest.raises(A.DeferError) as e:
            StageRunner(plan, device=0, batch=1, depth=1)
        assert e.value.code == A.ERR_INVALID
        return str(e.value)

    base = plan_stage(applications.ResNet50V2(input_shape=(32, 32, 3)), is_first=True, is_last=True, preprocess="tf")
    p = copy.deepcopy(base)                                  # tf takes no weights
    p.weights.append(np.zeros(3, np.float32))
    p.ops[0].w_shift = len(p.weights) - 1
    assert "no weights" in create(p)
    p = copy.deepcopy(base)                                  # an unknown mode
    p.ops[0].mode = 2
    assert "unknown mode" in create(p)
    p = copy.deepcopy(base)                                  # a mode on an op that is not PREPROCESS
    p.ops[1].mode = A.PRE_TF
    assert "mode" in create(p)
