"""Per-kernel GPU parity through the C-ABI entry points (defer_k_*), torch tensors as containers only.

Tests named `test_conv_tcgen05_*` keep the names they had when the tensor-core convolution targeted Blackwell; they
exercise the sm_90a wgmma kernels (defer_k_conv backends 2-7) - there is no Blackwell path in this library."""
import numpy as np
import pytest

from conv_check import FMTS, TOL, _alloc_act, _conv_case, _decode, _encode, _ptr, _quantise, ConvCase, check_executors
from defer_b200 import _cabi as A

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


@pytest.fixture(scope="module")
def torch_cuda():
    lib = A.load()          # sets CUDA_DEVICE_MAX_CONNECTIONS before torch touches CUDA
    import torch
    assert torch.cuda.is_available()
    return torch, lib


# most of ResNet50's distinct conv shapes at batch 1 (SURVEY.md 8d; not res4a_branch1) + batch / edge variants.  The
# complete list of the applications' conv geometries, derived from their plans, is tests/app_convs.py
RESNET_SHAPES = [
    # n, h, w, cin, cout, k, s, pad
    (1, 56, 56, 64, 64, 1, 1, 0), (1, 56, 56, 64, 64, 3, 1, 1), (1, 56, 56, 64, 256, 1, 1, 0),
    (1, 56, 56, 256, 64, 1, 1, 0), (1, 56, 56, 256, 128, 1, 2, 0), (1, 28, 28, 128, 128, 3, 1, 1),
    (1, 28, 28, 128, 512, 1, 1, 0), (1, 56, 56, 256, 512, 1, 2, 0), (1, 28, 28, 512, 128, 1, 1, 0),
    (1, 28, 28, 512, 256, 1, 2, 0), (1, 14, 14, 256, 256, 3, 1, 1), (1, 14, 14, 256, 1024, 1, 1, 0),
    (1, 14, 14, 1024, 256, 1, 1, 0), (1, 14, 14, 1024, 512, 1, 2, 0), (1, 7, 7, 512, 512, 3, 1, 1),
    (1, 7, 7, 512, 2048, 1, 1, 0), (1, 7, 7, 2048, 512, 1, 1, 0), (1, 14, 14, 1024, 2048, 1, 2, 0),
    (3, 7, 7, 512, 512, 3, 1, 1), (2, 28, 28, 128, 128, 3, 1, 1), (5, 14, 14, 256, 256, 3, 1, 1),
    # tile geometry outside ResNet50 (umma_conv_prepare): VGG-wide rows (wo > 128: two 112-wide parts), a ragged
    # tile_w (131 = 66 + 65), odd input at stride 2, 5x5 and 7x7 over 64 channels, tile_n = 2 with a ragged batch,
    # a 2x2 map with odd channel-block counts (3 in, 5 out), a 1x1 map, padding larger than k - 1, 288 k-blocks
    (1, 224, 224, 64, 64, 3, 1, 1), (1, 130, 131, 64, 128, 3, 1, 1), (3, 57, 57, 64, 128, 3, 2, 1),
    (1, 28, 28, 64, 64, 5, 1, 2), (1, 14, 14, 64, 64, 7, 1, 3), (5, 7, 7, 512, 512, 3, 1, 1),
    (4, 2, 2, 192, 320, 3, 1, 1), (1, 1, 1, 64, 64, 1, 1, 0), (2, 9, 9, 64, 64, 3, 1, 3),
    (1, 14, 14, 2048, 512, 3, 1, 1),
]


@pytest.mark.parametrize("fmt_name", ["f32", "bf16x2", "bf16"])
def test_conv_simt_shapes(torch_cuda, fmt_name):
    torch, lib = torch_cuda
    for i, (n, h, w, cin, cout, k, s, pad) in enumerate(RESNET_SHAPES[:8] + [(1, 230, 230, 3, 64, 7, 2, 0), (2, 9, 11, 8, 12, 3, 2, 1)]):
        err, _, _ = _conv_case(torch, lib, fmt_name, 1, n, h, w, cin, cout, k, s, pad, relu=(i % 2 == 0), residual=(i % 3 == 0), seed=i)
        assert err <= TOL[fmt_name], (fmt_name, (n, h, w, cin, cout, k, s, pad), err)


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("shape", RESNET_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_conv_tcgen05_shapes(torch_cuda, fmt_name, shape, monkeypatch):
    """Every wgmma executor against the oracle (global and per-channel error), bit-identical to each other."""
    torch, lib = torch_cuda
    n, h, w, cin, cout, k, s, pad = shape
    i = RESNET_SHAPES.index(shape)
    case = ConvCase(fmt_name, (n, h, w, cin, cout, k, k, s, s, pad, pad, pad, pad), relu=(i % 2 == 0), residual=(i % 3 == 0),
                    seed=i)
    check_executors(torch, lib, case, monkeypatch)


def test_conv_tcgen05_vs_simt_same_inputs(torch_cuda):
    """The two backends see identical quantised inputs; bf16x2 results agree to ~1e-5."""
    torch, lib = torch_cuda
    e1, y1, _ = _conv_case(torch, lib, "bf16x2", 1, 1, 28, 28, 128, 128, 3, 1, 1, True, True, seed=42)
    e2, y2, _ = _conv_case(torch, lib, "bf16x2", 2, 1, 28, 28, 128, 128, 3, 1, 1, True, True, seed=42)
    from oracle.keras_ref import rel_err
    assert rel_err(y2, y1) <= 1e-4


@pytest.mark.parametrize("fmt_name", ["f32", "bf16x2", "bf16"])
def test_maxpool_gap_dense_softmax(torch_cuda, fmt_name):
    from oracle import keras_ref as R
    torch, lib = torch_cuda
    fmt = FMTS[fmt_name]
    rng = np.random.default_rng(7)
    # max-pool 3x3/2 with fused ZeroPadding2D(1) - negative inputs exercise the "pad value is 0" rule
    x = rng.standard_normal((2, 112, 112, 64), dtype=np.float32)
    xq = _quantise(x, fmt)
    ref = R.maxpool2d(R.zeropad2d(xq, ((1, 1), (1, 1))), (3, 3), (2, 2))
    xd = _encode(torch, lib, x, fmt)
    yd = _alloc_act(torch, fmt, ref.size)
    A.check(lib.defer_k_maxpool(fmt, _ptr(xd), _ptr(yd), 2, 112, 112, 64, 3, 3, 2, 2, 1, 1, 1, 1, None))
    y = _decode(torch, lib, yd, fmt, ref.shape)
    assert np.array_equal(y, ref)          # max of representable values is exact in every format
    # global average pool
    x = rng.standard_normal((3, 7, 7, 2048), dtype=np.float32)
    xq = _quantise(x, fmt)
    ref = xq.astype(np.float64).mean(axis=(1, 2))
    xd = _encode(torch, lib, x, fmt)
    yd = _alloc_act(torch, fmt, ref.size)
    A.check(lib.defer_k_gap(fmt, _ptr(xd), _ptr(yd), 3, 7, 7, 2048, None))
    y = _decode(torch, lib, yd, fmt, ref.shape)
    assert R.rel_err(y, ref) <= (1e-2 if fmt_name == "bf16" else 1e-5)
    # dense 2048 -> 1000 (+ bias), fp32 logits out, then softmax
    x = rng.standard_normal((3, 2048), dtype=np.float32)
    wk = (rng.standard_normal((2048, 1000)) * 0.03).astype(np.float32)
    b = (rng.standard_normal(1000) * 0.1).astype(np.float32)
    xq = _quantise(x, fmt)
    ref = xq.astype(np.float64) @ wk.astype(np.float64) + b
    xd = _encode(torch, lib, x, fmt)
    wd, bd = torch.from_numpy(wk).cuda(), torch.from_numpy(b).cuda()
    yd = torch.empty(3 * 1000, dtype=torch.float32, device="cuda")
    A.check(lib.defer_k_dense(fmt, _ptr(xd), _ptr(wd), _ptr(bd), _ptr(yd), 1, 3, 2048, 1000, 0, None))
    y = yd.cpu().numpy().reshape(3, 1000)
    assert R.rel_err(y, ref) <= 1e-5
    pd = torch.empty_like(yd)
    A.check(lib.defer_k_softmax(_ptr(yd), _ptr(pd), 3, 1000, None))
    p = pd.cpu().numpy().reshape(3, 1000)
    assert R.rel_err(p, R.softmax(y.astype(np.float64))) <= 1e-5
    assert np.allclose(p.sum(axis=1), 1.0, atol=1e-5)


@pytest.mark.parametrize("fmt_name", ["f32", "bf16x2", "bf16"])
def test_dense_fused_single_launch(torch_cuda, fmt_name):
    """Fused dense (weight stream + split reduction by the last-arriving CTA + bias/ReLU in one launch): batch chunks
    beyond 8 rows, ReLU, ragged K splits, the units % 4 != 0 fallback, and run-to-run determinism."""
    from oracle import keras_ref as R
    torch, lib = torch_cuda
    fmt = FMTS[fmt_name]
    rng = np.random.default_rng(11)
    for n, F, U, relu in [(1, 2048, 1000, False), (3, 4096, 512, True), (9, 520, 1000, False), (2, 1000, 1002, True),
                          (2, 4096, 1000, False), (1, 4096, 4096, True)]:
        x = rng.standard_normal((n, F), dtype=np.float32)
        wk = (rng.standard_normal((F, U)) * 0.03).astype(np.float32)
        b = (rng.standard_normal(U) * 0.1).astype(np.float32)
        ref = _quantise(x, fmt).astype(np.float64) @ wk.astype(np.float64) + b
        if relu:
            ref = np.maximum(ref, 0)
        xd = _encode(torch, lib, x, fmt)
        wd, bd = torch.from_numpy(wk).cuda(), torch.from_numpy(b).cuda()
        outs = []
        for _ in range(2):
            yd = torch.empty(n * U, dtype=torch.float32, device="cuda")
            A.check(lib.defer_k_dense(fmt, _ptr(xd), _ptr(wd), _ptr(bd), _ptr(yd), 1, n, F, U, A.FLAG_RELU if relu else 0, None))
            outs.append(yd.cpu().numpy().reshape(n, U))
        assert R.rel_err(outs[0], ref) <= 1e-5, (n, F, U, R.rel_err(outs[0], ref))
        assert np.array_equal(outs[0], outs[1])


@pytest.mark.parametrize("fmt_name", ["f32", "bf16x2", "bf16"])
def test_eltwise(torch_cuda, fmt_name):
    torch, lib = torch_cuda
    fmt = FMTS[fmt_name]
    rng = np.random.default_rng(9)
    a = rng.standard_normal((2, 14, 14, 256), dtype=np.float32)
    b = rng.standard_normal((2, 14, 14, 256), dtype=np.float32)
    sc = rng.uniform(0.5, 1.5, 256).astype(np.float32)
    sf = rng.standard_normal(256).astype(np.float32)
    aq, bq = _quantise(a, fmt), _quantise(b, fmt)
    ad, bd = _encode(torch, lib, a, fmt), _encode(torch, lib, b, fmt)
    sd, fd = torch.from_numpy(sc).cuda(), torch.from_numpy(sf).cuda()
    tol = 1e-2 if fmt_name == "bf16" else 1e-5
    from oracle.keras_ref import rel_err
    for kind, ref in [(A.OP_RELU, np.maximum(aq, 0)), (A.OP_ADD, aq + bq), (A.OP_AFFINE, aq * sc + sf)]:
        yd = _alloc_act(torch, fmt, a.size)
        A.check(lib.defer_k_eltwise(fmt, kind, _ptr(ad), _ptr(bd), _ptr(sd), _ptr(fd), _ptr(yd), 2, 14, 14, 256, 0, None))
        y = _decode(torch, lib, yd, fmt, a.shape)
        assert rel_err(y, ref) <= tol, (kind, rel_err(y, ref))


def test_encode_decode_roundtrip(torch_cuda):
    torch, lib = torch_cuda
    x = np.random.default_rng(1).standard_normal(10007).astype(np.float32) * 37.0
    for name, fmt in FMTS.items():
        y = _decode(torch, lib, _encode(torch, lib, x, fmt), fmt, x.shape)
        assert np.array_equal(y, _quantise(x, fmt)), name
        if name == "bf16x2":
            assert np.max(np.abs(y - x) / np.abs(x)) < 2.0 ** -15


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
def test_conv_tcgen05_forced_split_k(torch_cuda, fmt_name, monkeypatch):
    """Deterministic split-K (fixed-order reduction by the last CTA) on small-M, deep-K layers, with residual."""
    torch, lib = torch_cuda
    monkeypatch.setenv("DEFER_UMMA_FORCE_SPLITS", "3")
    for i, shape in enumerate([(1, 7, 7, 512, 512, 3, 1, 1), (2, 14, 14, 1024, 256, 1, 1, 0), (1, 7, 7, 2048, 512, 1, 1, 0)]):
        n, h, w, cin, cout, k, s, pad = shape
        e1, y1, _ = _conv_case(torch, lib, fmt_name, 2, n, h, w, cin, cout, k, s, pad, relu=True, residual=(i != 1), seed=i)
        e2, y2, _ = _conv_case(torch, lib, fmt_name, 2, n, h, w, cin, cout, k, s, pad, relu=True, residual=(i != 1), seed=i)
        assert e1 <= TOL[fmt_name], (shape, e1)
        assert np.array_equal(y1, y2)            # run-to-run deterministic


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("csplit", [2, 4, 8])
@pytest.mark.parametrize("bn", [64, 128])
def test_conv_tcgen05_cluster_split_k(torch_cuda, fmt_name, csplit, bn, monkeypatch):
    """Cluster split-K: the S CTAs of a tile reduce their partial tiles through distributed shared memory and
    share the epilogue (rows j, j+S, ...).  Every cluster size x N-tile width, ragged M tiles, residual / ReLU,
    uneven k-block ranges (9 k-blocks over 2 / 4 / 8 CTAs), run-to-run determinism."""
    torch, lib = torch_cuda
    monkeypatch.setenv("DEFER_UMMA_FORCE_CSPLIT", str(csplit))
    monkeypatch.setenv("DEFER_UMMA_BN", str(bn))
    shapes = [(1, 7, 7, 512, 512, 3, 1, 1), (1, 14, 14, 1024, 256, 1, 1, 0), (1, 56, 56, 64, 64, 3, 1, 1),
              (2, 14, 14, 1024, 512, 1, 2, 0), (1, 28, 28, 512, 128, 1, 1, 0), (3, 7, 7, 512, 2048, 1, 1, 0)]
    for i, shape in enumerate(shapes):
        n, h, w, cin, cout, k, s, pad = shape
        e1, y1, _ = _conv_case(torch, lib, fmt_name, 2, n, h, w, cin, cout, k, s, pad, relu=(i % 2 == 0), residual=(i % 3 != 1), seed=i)
        e2, y2, _ = _conv_case(torch, lib, fmt_name, 2, n, h, w, cin, cout, k, s, pad, relu=(i % 2 == 0), residual=(i % 3 != 1), seed=i)
        assert e1 <= TOL[fmt_name], (shape, csplit, bn, e1)
        assert np.array_equal(y1, y2)


def test_conv_tcgen05_cluster_matches_single_cta(torch_cuda, monkeypatch):
    """Same inputs through the cluster path and the one-CTA-per-tile path agree to fp32 summation-order noise."""
    torch, lib = torch_cuda
    from oracle.keras_ref import rel_err
    shape = (1, 14, 14, 256, 256, 3, 1, 1)
    monkeypatch.setenv("DEFER_UMMA_CLUSTER", "0")
    _, y0, _ = _conv_case(torch, lib, "bf16x2", 2, *shape, True, True, seed=5)
    monkeypatch.setenv("DEFER_UMMA_CLUSTER", "1")
    _, y1, _ = _conv_case(torch, lib, "bf16x2", 2, *shape, True, True, seed=5)
    assert rel_err(y1, y0) <= 1e-5


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("mode", ["ring2", "ring_deep", "staged_bn64"])
def test_conv_tcgen05_epilogue_variants(torch_cuda, fmt_name, mode, monkeypatch):
    """The one-tile-per-CTA kernel with the shallowest operand ring (two stages: every fill waits for the previous k-block), a deep ring and
    64-wide N tiles gives the same answers as the default plan - bitwise, the K order per output is the same."""
    torch, lib = torch_cuda
    monkeypatch.setenv("DEFER_UMMA_SPLITK", "0")       # split-K would change the summation order
    shapes = [(1, 56, 56, 64, 256, 1, 1, 0), (1, 28, 28, 128, 128, 3, 1, 1), (2, 14, 14, 256, 1024, 1, 1, 0),
              (1, 7, 7, 512, 2048, 1, 1, 0), (1, 56, 56, 256, 512, 1, 2, 0)]
    ref_y = []
    for i, shape in enumerate(shapes):
        _, y, _ = _conv_case(torch, lib, fmt_name, 2, *shape, relu=True, residual=(i != 1), seed=10 + i)
        ref_y.append(y)
    if mode == "ring2":
        monkeypatch.setenv("DEFER_UMMA_STAGES", "2")
    elif mode == "ring_deep":
        monkeypatch.setenv("DEFER_UMMA_STAGES", "8")
    else:
        monkeypatch.setenv("DEFER_UMMA_BN", "64")
    for i, shape in enumerate(shapes):
        err, y, _ = _conv_case(torch, lib, fmt_name, 2, *shape, relu=True, residual=(i != 1), seed=10 + i)
        assert err <= TOL[fmt_name], (mode, shape, err)
        assert np.array_equal(y, ref_y[i]), (mode, shape)


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
def test_conv_persistent_grid_kernel(torch_cuda, fmt_name):
    """backend 3: the persistent grid with 64-wide N tiles (each CTA walks many tiles through one operand ring)."""
    torch, lib = torch_cuda
    for i, shape in enumerate([(8, 56, 56, 64, 256, 1, 1, 0), (4, 56, 56, 64, 64, 3, 1, 1), (8, 28, 28, 256, 512, 1, 2, 0),
                               (3, 14, 14, 256, 256, 3, 1, 1)]):
        n, h, w, cin, cout, k, s, pad = shape
        err, _, _ = _conv_case(torch, lib, fmt_name, 3, n, h, w, cin, cout, k, s, pad, relu=(i % 2 == 0), residual=(i % 2 == 1), seed=i)
        assert err <= TOL[fmt_name], (shape, err)


def test_stem_kernel_f32_input(torch_cuda):
    """The dedicated 7x7/2 RGB stem kernel (fp32 image in, stage format out) against the oracle."""
    from oracle import keras_ref as R
    torch, lib = torch_cuda
    rng = np.random.default_rng(3)
    for fmt_name in ("f32", "bf16x2", "bf16"):
        fmt = FMTS[fmt_name]
        x = rng.standard_normal((2, 224, 224, 3), dtype=np.float32)
        wk = (rng.standard_normal((7, 7, 3, 64)) * 0.1).astype(np.float32)
        sc = rng.uniform(0.5, 1.5, 64).astype(np.float32)
        sf = rng.standard_normal(64).astype(np.float32)
        ref = np.maximum(R.conv2d(np.pad(x.astype(np.float64), ((0, 0), (3, 3), (3, 3), (0, 0))), wk.astype(np.float64), None, (2, 2), "valid") * sc + sf, 0)
        xd, wd = torch.from_numpy(x).cuda(), torch.from_numpy(wk).cuda()
        sd, fd = torch.from_numpy(sc).cuda(), torch.from_numpy(sf).cuda()
        yd = _alloc_act(torch, fmt, ref.size)
        A.check(lib.defer_k_conv(fmt, 1, _ptr(xd), 1, _ptr(wd), _ptr(sd), _ptr(fd), None, _ptr(yd), 2, 224, 224, 3, 64, 7, 7, 2, 2,
                                 3, 3, 3, 3, A.FLAG_RELU, None))
        y = _decode(torch, lib, yd, fmt, ref.shape)
        assert R.rel_err(y, ref) <= (5e-3 if fmt_name == "bf16" else 2e-5), fmt_name


@pytest.mark.parametrize("backend", [3, 4, 5])
def test_conv_persistent_executors_match_one_tile_per_cta(torch_cuda, backend, monkeypatch):
    """The persistent grid (64- and 128-wide N tiles, each CTA walking many tiles through one operand ring) and the
    one-tile-per-CTA grid compute every output with the same K order: results must be bit-identical."""
    torch, lib = torch_cuda
    monkeypatch.setenv("DEFER_UMMA_SPLITK", "0")
    shapes = [(1, 56, 56, 64, 256, 1, 1, 0), (1, 14, 14, 256, 256, 3, 1, 1), (1, 7, 7, 2048, 512, 1, 1, 0),
              (4, 28, 28, 128, 128, 3, 1, 1)]
    for i, sh in enumerate(shapes):
        _, ref, _ = _conv_case(torch, lib, "bf16x2", 2, *sh, relu=True, residual=(i != 1), seed=20 + i)
        err, y, _ = _conv_case(torch, lib, "bf16x2", backend, *sh, relu=True, residual=(i != 1), seed=20 + i)
        assert err <= TOL["bf16x2"] and np.array_equal(y, ref), (backend, sh)


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
def test_conv_tcgen05_1x1_with_bottom_right_padding(torch_cuda, fmt_name):
    """A fused asymmetric ZeroPadding2D(((0, 1), (0, 2))) in front of a 1x1 'valid' conv: pad_t == pad_l == 0 but the
    output grid is larger than the input grid, so the flat [M, C] fast path must NOT be taken (ADVICE round 1)."""
    torch, lib = torch_cuda
    from oracle import keras_ref as R
    fmt = FMTS[fmt_name]
    rng = np.random.default_rng(31)
    n, h, w, cin, cout = 2, 13, 14, 64, 128
    pb, pr = 1, 2
    x = rng.standard_normal((n, h, w, cin), dtype=np.float32)
    wk = rng.standard_normal((1, 1, cin, cout), dtype=np.float32) * np.float32(np.sqrt(2.0 / cin))
    shift = (rng.standard_normal(cout) * 0.2).astype(np.float32)
    xq, wq = _quantise(x, fmt), _quantise(wk, fmt)
    ref = R.conv2d(np.pad(xq.astype(np.float64), ((0, 0), (0, pb), (0, pr), (0, 0))), wq.astype(np.float64), None, (1, 1), "valid")
    ref = ref + shift.astype(np.float64)
    xd = _encode(torch, lib, x, fmt)
    wd, fd = torch.from_numpy(wk).cuda(), torch.from_numpy(shift).cuda()
    yd = _alloc_act(torch, fmt, ref.size)
    A.check(lib.defer_k_conv(fmt, 2, _ptr(xd), 0, _ptr(wd), None, _ptr(fd), None, _ptr(yd), n, h, w, cin, cout, 1, 1, 1, 1,
                             0, 0, pb, pr, 0, None))
    torch.cuda.synchronize()
    y = _decode(torch, lib, yd, fmt, ref.shape)
    assert R.rel_err(y, ref) <= TOL[fmt_name]
    assert np.allclose(y[:, h:, :, :], shift, atol=1e-2)      # the padded rows / columns see only the shift


STREAM_SHAPES = [
    # n, h, w, cin, cout, k, s, pad
    (8, 56, 56, 64, 256, 1, 1, 0),      # flat, one k-block per tile, 4 / 2 column blocks
    (4, 56, 56, 64, 64, 3, 1, 1),       # 3x3, N = 64 only, 112-row tiles
    (8, 28, 28, 256, 512, 1, 2, 0),     # stride 2 through TMA element strides
    (3, 14, 14, 256, 256, 3, 1, 1),     # 98-row tiles, K-heavy (36 k-blocks)
    (16, 7, 7, 512, 512, 3, 1, 1),      # two images per tile, 72 k-blocks
    (5, 14, 14, 1024, 256, 1, 1, 0),    # flat, ragged last M tile (980 rows), 16 k-blocks
    (2, 28, 28, 128, 128, 3, 1, 1),
    (1, 56, 56, 256, 64, 1, 1, 0),
    (9, 7, 7, 2048, 512, 1, 1, 0),      # 441 rows: 4 tiles, 32 k-blocks
]


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("shape", STREAM_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_conv_stream_kernel(torch_cuda, fmt_name, shape):
    """conv_stream_kernel (deep operand ring, in-place chunked epilogue): 64- and 128-wide N tiles, staged (TMA) and
    per-thread (peer-capable) epilogues, with and without residual / ReLU - against the fp64 oracle, and bit-identical
    across tile widths and epilogue kinds (same K order per output)."""
    torch, lib = torch_cuda
    n, h, w, cin, cout, k, s, pad = shape
    i = STREAM_SHAPES.index(shape)
    outs = {}
    for backend in (4, 5, 6, 7):
        for residual in (False, True):
            err, y, _ = _conv_case(torch, lib, fmt_name, backend, n, h, w, cin, cout, k, s, pad, relu=(i % 2 == 0),
                                   residual=residual, seed=100 + i)
            assert err <= TOL[fmt_name], (fmt_name, shape, backend, residual, err)
            outs[(backend, residual)] = y
    for residual in (False, True):
        for backend in (5, 6, 7):
            assert np.array_equal(outs[(backend, residual)], outs[(4, residual)]), (shape, backend, residual)


@pytest.mark.parametrize("fmt_name,stages", [("bf16x2", 2), ("bf16x2", 3), ("bf16x2", 4), ("bf16", 2), ("bf16", 6),
                                             ("bf16", 8)])
def test_conv_stream_kernel_ring_depths(torch_cuda, fmt_name, stages, monkeypatch):
    """Every operand-ring depth of the persistent kernel (the host clamps it to what fits in 227 KB) must give the same
    bits, including rings shallower than a tile's K loop, where the producer refills stages mid-tile."""
    torch, lib = torch_cuda
    shapes = [(4, 56, 56, 64, 256, 1, 1, 0), (3, 14, 14, 256, 256, 3, 1, 1)]
    ref = [_conv_case(torch, lib, fmt_name, 5, *sh, relu=True, residual=True, seed=7 + j)[1] for j, sh in enumerate(shapes)]
    monkeypatch.setenv("DEFER_STREAM_STAGES", str(stages))
    for j, sh in enumerate(shapes):
        for backend in (4, 5):
            err, y, _ = _conv_case(torch, lib, fmt_name, backend, *sh, relu=True, residual=True, seed=7 + j)
            assert err <= TOL[fmt_name] and np.array_equal(y, ref[j]), (stages, sh, backend)
