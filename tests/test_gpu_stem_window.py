"""The fused RGB stem's image window on the GPU: conv_stem_kernel (fp32 image), conv_stem_u8_kernel (uint8, Keras caffe)
and conv_stem_u8tf_kernel (uint8, Keras tf) against stem_im2col + conv_stream_kernel, bit for bit, in fp32 parity and
in bf16.  The maps are small enough that tiles are ragged in both directions and windows cross every image border (top,
bottom, left, right and the corners); batch 3, with the middle image also run alone.  A stem whose window does not fit
the kernel's window buffer (32 input channels, only an fp32 image can have them) stays on the im2col path."""
import numpy as np
import pytest

from defer_b200 import applications
from defer_b200.node import StageRunner
from test_gpu_conv_paths import _knobs, _stem_model
from test_gpu_preprocess import _bits, _image

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

FUSED = {None: "conv_stem_kernel", "caffe": "conv_stem_u8_kernel", "tf": "conv_stem_u8tf_kernel"}
IM2COL = "stem_im2col+conv_stream_kernel"

# batch, h, w, cin, k, s, padding
SHAPES = {
    # 19 x 23 outputs: tiles of 8 x 16, the last row of tiles 3 high and the last column 7 wide
    "ragged_7x7s2": (3, 37, 45, 3, 7, 2, ((3, 3), (3, 3))),
    # asymmetric padding, 18 x 21 outputs
    "asym_7x7s2": (3, 39, 43, 3, 7, 2, ((2, 3), (1, 4))),
    # 3x3/1 'same' (VGG), 21 x 35 outputs
    "same_3x3s1": (3, 21, 35, 3, 3, 1, "same"),
}


def _run(m, x, dtype, preprocess, env, monkeypatch):
    _knobs(monkeypatch, **env)
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=x.shape[0], depth=1, preprocess=preprocess)
    try:
        kernels = [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))]
        r.predict(x)
        return r.read_layer("relu"), kernels
    finally:
        r.close()


def _input(b, h, w, cin, preprocess, seed):
    if preprocess is None:
        return applications.synthetic_input(b, (h, w, cin), seed=seed)
    return _image(b, h, w, seed=seed)


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("preprocess", [None, "caffe", "tf"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_fused_stem_matches_im2col(name, preprocess, dtype, monkeypatch):
    b, h, w, cin, k, s, pad = SHAPES[name]
    m = _stem_model(h, w, cin, 64, k, s, pad, seed=len(name))
    x = _input(b, h, w, cin, preprocess, seed=len(name))
    conv = 0 if preprocess is None else 1          # a folded PREPROCESS op comes first
    y, kf = _run(m, x, dtype, preprocess, {"DEFER_STREAM_MIN_TILES": 1}, monkeypatch)
    assert kf[conv] == FUSED[preprocess], kf
    y_ref, kr = _run(m, x, dtype, preprocess, {"DEFER_STEM_FUSED": 0, "DEFER_STREAM_MIN_TILES": 1}, monkeypatch)
    assert kr[conv] == IM2COL, kr
    assert np.array_equal(_bits(y), _bits(y_ref)), (name, preprocess, dtype)
    # the middle image alone: the same bits as in the batch of 3
    y1, k1 = _run(m, x[1:2], dtype, preprocess, {"DEFER_STREAM_MIN_TILES": 1}, monkeypatch)
    assert k1[conv] == FUSED[preprocess], k1
    assert np.array_equal(_bits(y1[0]), _bits(y[1])), (name, preprocess, dtype)


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
def test_window_over_budget_stays_on_im2col(dtype, monkeypatch):
    # 32 channels, 2x2/2: a 16 x 1024-value window (64 KB) > the 24 KB buffer
    b, h, w, cin = 3, 40, 40, 32
    m = _stem_model(h, w, cin, 64, 2, 2, "same", seed=7)
    x = applications.synthetic_input(b, (h, w, cin), seed=7)
    y, kf = _run(m, x, dtype, None, {"DEFER_STREAM_MIN_TILES": 1}, monkeypatch)
    assert kf[0] == IM2COL, kf
    y_ref, kr = _run(m, x, dtype, None, {"DEFER_STEM_FUSED": 0, "DEFER_STREAM_MIN_TILES": 1}, monkeypatch)
    assert kr[0] == IM2COL, kr
    assert np.array_equal(_bits(y), _bits(y_ref))
