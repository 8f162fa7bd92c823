"""The SIMT kernels other than the convolutions (max-pool, GAP, dense, softmax, the element-wise ops, ZeroPadding2D,
format copies) against float64 references op by op: through their `defer_k_*` entry points at the shapes the models
produce, in stages that run paths with no entry point (bf16 dense weights, activation-format dense outputs, standalone
pad / add), and at every op of cut-point pipelines, read back from the GPU's own input and output buffers.

Exact ops (max-pool, pad, ReLU, copy, and the element-wise ops against host fp32 arithmetic plus the format's store
rule) must match bit for bit; the reductions are held to per-element bars (tests/simt_bars.py, checked against wrong
arithmetic by tests/test_simt_bars_host.py).  Each test prints the fraction of its bars it used."""
import numpy as np
import pytest

import handover_check as H
import simt_bars as S
from conv_check import FMTS, TOL, _alloc_act, _decode, _encode, _ptr, _quantise, conv_errors, conv_oracle
from defer_b200 import _cabi as A
from defer_b200 import applications, keras_like as K
from defer_b200.node import StageRunner
from plan_interp import run_op

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

FMT_LIST = ["f32", "bf16x2", "bf16"]
DTYPE_FMT_NAME = {"float32": "bf16x2", "bfloat16": "bf16", "float32_simt": "f32"}


@pytest.fixture(scope="module")
def torch_cuda():
    lib = A.load()          # sets CUDA_DEVICE_MAX_CONNECTIONS before torch touches CUDA
    import torch
    assert torch.cuda.is_available()
    return torch, lib


def _report(what, used):
    print(f"bar {what}: {used:.3g} of the bar")
    assert used <= 1.0, (what, used)
    return used


def _raw(torch, t):
    """Raw bits of a device activation tensor: int16 planes (bf16 formats) or uint32 words (f32)."""
    if t.dtype == torch.float32:
        return t.cpu().numpy().view(np.uint32)
    return t.view(torch.int16).cpu().numpy()


# ================================================================================================ 1. per-kernel matrix
# (n, h, w, c, pool, stride, (pad_t, pad_l, pad_b, pad_r))
MAXPOOL_CASES = (
    [(1, 112, 112, c, 3, 2, (1, 1, 1, 1)) for c in (64, 12, 20)] + [(2, 112, 112, 64, 3, 2, (1, 1, 1, 1))]
    # VGG: 2x2/2 unpadded
    + [(1, 224, 224, 64, 2, 2, (0, 0, 0, 0)), (1, 112, 112, 128, 2, 2, (0, 0, 0, 0)), (1, 56, 56, 256, 2, 2, (0, 0, 0, 0)),
       (1, 28, 28, 512, 2, 2, (0, 0, 0, 0)), (32, 14, 14, 512, 2, 2, (0, 0, 0, 0)), (1, 28, 28, 12, 2, 2, (0, 0, 0, 0)),
       (32, 14, 14, 20, 2, 2, (0, 0, 0, 0))]
    # ResNet V2 shortcut: MaxPooling2D(1, strides=2), at an odd 7 -> 4 too
    + [(1, 56, 56, 256, 1, 2, (0, 0, 0, 0)), (32, 28, 28, 64, 1, 2, (0, 0, 0, 0)), (1, 14, 14, 2048, 1, 2, (0, 0, 0, 0)),
       (32, 7, 7, 2048, 1, 2, (0, 0, 0, 0)), (1, 7, 7, 12, 1, 2, (0, 0, 0, 0)), (1, 7, 7, 20, 1, 2, (0, 0, 0, 0))]
    # TF 'same' at odd sizes: the extra row / column goes after
    + [(1, 7, 7, 2048, 2, 2, (0, 0, 1, 1)), (32, 13, 13, 64, 2, 2, (0, 0, 1, 1)), (1, 15, 15, 20, 2, 2, (0, 0, 1, 1)),
       (1, 13, 13, 12, 2, 2, (0, 0, 1, 1))]
)


def test_maxpool_cases_take_both_kernels():
    """In the bf16 formats c % 8 == 0 selects maxpool8_kernel and c % 8 == 4 the 4-channel maxpool_kernel: both occur,
    at every pool geometry."""
    for geom in {(k, s, p) for _, _, _, _, k, s, p in MAXPOOL_CASES}:
        cs = {c % 8 == 0 for _, _, _, c, k, s, p in MAXPOOL_CASES if (k, s, p) == geom}
        assert cs == {True, False}, geom
    assert {n for n, *_ in MAXPOOL_CASES} == {1, 2, 32}


def _maxpool(torch, lib, fmt, x, k, s, pads):
    n, h, w, c = x.shape
    t, l, b, r = pads
    ho, wo = (h + t + b - k) // s + 1, (w + l + r - k) // s + 1
    xd = _encode(torch, lib, x, fmt)
    yd = _alloc_act(torch, fmt, n * ho * wo * c)
    A.check(lib.defer_k_maxpool(fmt, _ptr(xd), _ptr(yd), n, h, w, c, k, k, s, s, t, l, b, r, None))
    return yd, (n, ho, wo, c)


@pytest.mark.parametrize("fmt_name", FMT_LIST)
def test_maxpool_exact(torch_cuda, fmt_name):
    """Max of representable values is exact: decoded output == max over the zero-padded decoded input.  All inputs are
    negative, so every window that reaches into the padding must return 0."""
    from oracle import keras_ref as R
    torch, lib = torch_cuda
    fmt = FMTS[fmt_name]
    rng = np.random.default_rng(1)
    for n, h, w, c, k, s, pads in MAXPOOL_CASES:
        x = -np.abs(rng.standard_normal((n, h, w, c), dtype=np.float32)) - np.float32(0.01)
        t, l, b, r = pads
        ref = R.maxpool2d(np.pad(_quantise(x, fmt), ((0, 0), (t, b), (l, r), (0, 0))), (k, k), (s, s))
        yd, shape = _maxpool(torch, lib, fmt, x, k, s, pads)
        y = _decode(torch, lib, yd, fmt, shape)
        assert np.array_equal(y, ref), (fmt_name, (n, h, w, c, k, s, pads))
        if any(pads):
            assert (y == 0).any()
    with pytest.raises(A.DeferError) as ei:          # argument check before any launch
        lib_x = _encode(torch, lib, np.zeros((1, 4, 4, 6), np.float32), fmt)
        A.check(lib.defer_k_maxpool(fmt, _ptr(lib_x), _ptr(lib_x), 1, 4, 4, 6, 2, 2, 2, 2, 0, 0, 0, 0, None))
    assert ei.value.code == A.ERR_INVALID


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
def test_maxpool8_and_maxpool4_same_bits(torch_cuda, fmt_name):
    """maxpool8_kernel (c = 24) and the 4-channel kernel (c = 20) on the same values write identical planes."""
    torch, lib = torch_cuda
    fmt = FMTS[fmt_name]
    x24 = np.random.default_rng(2).standard_normal((2, 57, 57, 24), dtype=np.float32)
    x20 = np.ascontiguousarray(x24[..., :20])
    planes = 2 if fmt_name == "bf16x2" else 1
    for k, s, pads in [(3, 2, (1, 1, 1, 1)), (2, 2, (0, 0, 1, 1)), (1, 2, (0, 0, 0, 0))]:
        y24, sh24 = _maxpool(torch, lib, fmt, x24, k, s, pads)
        y20, sh20 = _maxpool(torch, lib, fmt, x20, k, s, pads)
        a = _raw(torch, y24).reshape((planes,) + sh24)[..., :20]
        b = _raw(torch, y20).reshape((planes,) + sh20)
        assert np.array_equal(a, b), (fmt_name, k, s, pads)


GAP_SHAPES = [(1, 1, 1, 64), (2, 2, 3, 100), (3, 7, 7, 2048), (32, 7, 7, 2048), (1, 14, 14, 1000), (1, 56, 56, 36)]


@pytest.mark.parametrize("fmt_name", FMT_LIST)
def test_gap_per_element_bound(torch_cuda, fmt_name):
    torch, lib = torch_cuda
    fmt = FMTS[fmt_name]
    assert any(c % 32 for *_, c in GAP_SHAPES) and any(h * w < 8 for _, h, w, _ in GAP_SHAPES)
    rng = np.random.default_rng(3)
    worst = 0.0
    for n, h, w, c in GAP_SHAPES:
        x = rng.standard_normal((n, h, w, c), dtype=np.float32) + np.float32(0.5)
        ref, mag = S.gap_ref(_quantise(x, fmt))
        xd = _encode(torch, lib, x, fmt)
        yd = _alloc_act(torch, fmt, n * c)
        A.check(lib.defer_k_gap(fmt, _ptr(xd), _ptr(yd), n, h, w, c, None))
        y = _decode(torch, lib, yd, fmt, (n, c))
        if h * w == 1:
            assert np.array_equal(y, _quantise(x.reshape(n, c), fmt))     # the mean of one pixel is the pixel
        worst = max(worst, S.bar_used(y, ref, mag, S.A_GAP, S.C_FMT[fmt_name]))
    _report(f"gap {fmt_name}", worst)


DENSE_CASES = [(1, 25088, 4096), (8, 25088, 4096), (32, 4096, 1000), (17, 2048, 1000), (1, 1, 8), (3, 63, 12),
               (2, 65, 1000), (9, 4096, 1002), (1, 520, 7)]


def test_dense_cases_take_both_kernels():
    """units % 4 == 0 runs dense_fused_kernel, otherwise dense_partial_kernel + dense_reduce_kernel."""
    assert {u % 4 == 0 for *_, u in DENSE_CASES} == {True, False}


@pytest.mark.parametrize("case", DENSE_CASES, ids=lambda c: "x".join(map(str, c)))
def test_dense_per_element_bound(torch_cuda, case):
    """defer_k_dense with fp32 weights, every format, bias or none, ReLU or not, fp32 or stage-format output; two
    launches give identical bits."""
    torch, lib = torch_cuda
    n, F, U = case
    rng = np.random.default_rng(F + U)
    x = rng.standard_normal((n, F), dtype=np.float32)
    wk = (rng.standard_normal((F, U), dtype=np.float32) * np.float32(np.sqrt(2.0 / F)))
    b = (rng.standard_normal(U) * 0.1).astype(np.float32)
    wd, bd = torch.from_numpy(wk).cuda(), torch.from_numpy(b).cuda()
    w64 = wk.astype(np.float64)
    aw64 = np.abs(w64)
    for fmt_name in FMT_LIST:
        fmt = FMTS[fmt_name]
        xq = _quantise(x, fmt).astype(np.float64)
        base, base_mag = xq @ w64, np.abs(xq) @ aw64
        xd = _encode(torch, lib, x, fmt)
        worst = {1: 0.0, 0: 0.0}
        for bias in (None, b):
            for relu in (False, True):
                ref = base + (0 if bias is None else bias.astype(np.float64))
                mag = base_mag + (0 if bias is None else np.abs(bias.astype(np.float64)))
                if relu:
                    ref = np.maximum(ref, 0)
                for y_f32 in (1, 0):
                    outs = []
                    for _ in range(2):
                        yd = (torch.empty(n * U, dtype=torch.float32, device="cuda") if y_f32
                              else _alloc_act(torch, fmt, n * U))
                        A.check(lib.defer_k_dense(fmt, _ptr(xd), _ptr(wd), _ptr(bd if bias is not None else None), _ptr(yd),
                                                  y_f32, n, F, U, A.FLAG_RELU if relu else 0, None))
                        outs.append(yd)
                    assert torch.equal(outs[0], outs[1]), (case, fmt_name, bias is None, relu, y_f32)
                    y = outs[0].cpu().numpy() if y_f32 else _decode(torch, lib, outs[0], fmt, (n, U))
                    c = 0.0 if y_f32 else S.C_FMT[fmt_name]
                    worst[y_f32] = max(worst[y_f32], S.bar_used(y, ref, mag, S.A_DENSE, c))
        _report(f"dense {case} {fmt_name} fp32-out", worst[1])
        _report(f"dense {case} {fmt_name} {fmt_name}-out", worst[0])


@pytest.mark.parametrize("n", [1, 32])
def test_softmax_per_element_bound(torch_cuda, n):
    torch, lib = torch_cuda
    worst = 0.0
    for c in (1, 7, 255, 256, 257, 1000, 1001, 4097):
        rows = np.concatenate([S.softmax_rows(c, seed=k) for k in range(7)])[:max(n, 5)]
        groups = [rows[i:i + 1] for i in range(5)] if n == 1 else [rows[:n]]
        for x in groups:
            xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
            pd = torch.empty_like(xd)
            A.check(lib.defer_k_softmax(_ptr(xd), _ptr(pd), x.shape[0], c, None))
            p = pd.cpu().numpy()
            assert np.all(np.isfinite(p)), c
            if c == 1:
                assert np.all(p == 1)
            worst = max(worst, S.softmax_bar_used(p, x))
    _report(f"softmax n={n}", worst)


ELT_SHAPES = [(1, 1, 1, 4), (3, 7, 7, 52)]     # 3*7*7*52/4 = 1911 threads: not a multiple of 256


@pytest.mark.parametrize("fmt_name", FMT_LIST)
def test_eltwise_bits(torch_cuda, fmt_name):
    """AFFINE (scale and shift, either one NULL) / ADD, with and without FLAG_RELU, and RELU: the output planes equal
    the store rule applied to host fp32 arithmetic on the decoded operands (fmaf for AFFINE).  BF16X2 RELU keeps or
    zeroes the input planes (relu_planes_kernel)."""
    torch, lib = torch_cuda
    fmt = FMTS[fmt_name]
    rng = np.random.default_rng(4)
    for n, h, w, c in ELT_SHAPES:
        a = rng.standard_normal((n, h, w, c), dtype=np.float32)
        b = rng.standard_normal((n, h, w, c), dtype=np.float32)
        sc = rng.uniform(0.5, 1.5, c).astype(np.float32)
        sf = rng.standard_normal(c).astype(np.float32)
        ad, bd = _encode(torch, lib, a, fmt), _encode(torch, lib, b, fmt)
        aq, bq = _decode(torch, lib, ad, fmt, a.shape), _decode(torch, lib, bd, fmt, b.shape)
        sd, fd = torch.from_numpy(sc).cuda(), torch.from_numpy(sf).cuda()
        cases = []
        for relu in (0, A.FLAG_RELU):
            for s_, f_ in ((sc, sf), (None, sf), (sc, None)):
                v = S.fma32(aq, np.float32(1) if s_ is None else s_, np.float32(0) if f_ is None else f_)
                cases.append((A.OP_AFFINE, relu, s_ is not None, f_ is not None, v))
            cases.append((A.OP_ADD, relu, False, False, aq + bq))
        cases.append((A.OP_RELU, 0, False, False, aq))
        for kind, flags, has_s, has_f, v in cases:
            if flags or kind == A.OP_RELU:
                v = np.maximum(v, np.float32(0))
            yd = _alloc_act(torch, fmt, a.size)
            A.check(lib.defer_k_eltwise(fmt, kind, _ptr(ad), _ptr(bd if kind == A.OP_ADD else None),
                                        _ptr(sd if has_s else None), _ptr(fd if has_f else None), _ptr(yd),
                                        n, h, w, c, flags, None))
            got = _raw(torch, yd)
            if fmt_name == "bf16x2" and kind == A.OP_RELU:
                planes = _raw(torch, ad).reshape(2, -1)
                want = np.where(planes[0] > 0, planes, 0).reshape(-1)
            else:
                want = S.store_planes(v, fmt_name)
            assert np.array_equal(got, want), (fmt_name, (n, h, w, c), kind, flags, has_s, has_f)
    with pytest.raises(A.DeferError) as ei:          # argument check before any launch
        A.check(lib.defer_k_eltwise(fmt, A.OP_RELU, _ptr(ad), None, None, None, _ptr(ad), 1, 1, 1, 6, 0, None))
    assert ei.value.code == A.ERR_INVALID


def test_preprocess_rejects_non_rgb(torch_cuda):
    torch, lib = torch_cuda
    x = torch.zeros(64, dtype=torch.uint8, device="cuda")
    sh = torch.zeros(4, dtype=torch.float32, device="cuda")
    y = torch.zeros(64, dtype=torch.float32, device="cuda")
    with pytest.raises(A.DeferError) as ei:
        A.check(lib.defer_k_preprocess(_ptr(x), _ptr(sh), _ptr(y), 1, 4, 4, 4, None))
    assert ei.value.code == A.ERR_INVALID


def test_relu_planes_bit_rule(torch_cuda):
    """BF16X2 ReLU works on the planes: (hi, lo) passes untouched where hi > 0 and becomes (0, 0) elsewhere - never a
    re-split of hi + lo, so the bits do not depend on where the model is cut."""
    torch, lib = torch_cuda
    special_hi = [0x0000, 0x8000, 0x3F80, 0x3F80, 0xBF80, 0xBF80, 0x0080, 0x8080, 0x0001, 0x8001, 0x007F, 0x3F81, 0xC2F7]
    special_lo = [0x3000, 0x3000, 0xB700, 0x3700, 0x3700, 0xB700, 0x0001, 0x0001, 0x8000, 0x0000, 0x8001, 0xB780, 0x3F00]
    rng = np.random.default_rng(5)
    m = 4096
    hi = np.concatenate([special_hi, rng.integers(0, 0x10000, m - len(special_hi))]).astype(np.uint16)
    lo = np.concatenate([special_lo, rng.integers(0, 0x10000, m - len(special_lo))]).astype(np.uint16)
    finite = (hi & 0x7F80) != 0x7F80                       # no inf / NaN patterns in the random part
    hi, lo = np.where(finite, hi, hi & 0x807F), np.where((lo & 0x7F80) != 0x7F80, lo, lo & 0x807F)
    planes = np.concatenate([hi, lo]).view(np.int16)
    xd = torch.from_numpy(planes.copy()).cuda().view(torch.bfloat16)
    yd = torch.empty_like(xd)
    A.check(lib.defer_k_eltwise(A.FMT_BF16X2, A.OP_RELU, _ptr(xd), None, None, None, _ptr(yd), 1, 1, m // 4, 4, 0, None))
    got = yd.view(torch.int16).cpu().numpy().reshape(2, m)
    keep = ((hi & 0x8000) == 0) & ((hi & 0x7FFF) != 0)
    want = np.where(keep, planes.reshape(2, m), 0)
    assert np.array_equal(got, want)
    assert keep[[2, 3, 6, 8, 10, 11]].all() and not keep[[0, 1, 4, 5, 7, 9, 12]].any()


# ================================================================================================ op-by-op checker
def check_stage_ops(r, fmt_name, lane=0, label=""):
    """Every op of stage `r` that launches a kernel, against `run_op` / the exact rules on the GPU's own input
    buffers (lane `lane`).  Returns {op kind: fraction of its bar used} (0 for exact ops)."""
    plan = r.plan
    fmt = FMTS[fmt_name]
    cache = {}

    def buf(i):
        if i not in cache:
            cache[i] = r.read_buffer(i, lane)
        return cache[i]

    used = {}
    for i, op in enumerate(plan.ops):
        kname = r.op_info(i)["kernel"]
        if "fused into" in kname:
            continue
        x, y = buf(op.in0), buf(op.out)
        in_f32 = plan.bufs[op.in0][3] == A.BUF_F32
        out_f32 = plan.bufs[op.out][3] == A.BUF_F32
        what = (label, i, A.OP_NAMES[op.kind], kname, fmt_name)
        W = plan.weights
        u = 0.0
        if op.kind == A.OP_COPY:
            want = _quantise(x, fmt) if (in_f32 and not out_f32) else x
            assert np.array_equal(y, want), what
        elif op.kind in (A.OP_PAD, A.OP_MAXPOOL, A.OP_RELU):
            assert np.array_equal(y, run_op(plan, op, {op.in0: x}, W)), what
        elif op.kind in (A.OP_AFFINE, A.OP_ADD):
            v = (S.fma32(x, W[op.w_scale], W[op.w_shift]) if op.kind == A.OP_AFFINE else x + buf(op.in1))
            if op.flags & A.FLAG_RELU:
                v = np.maximum(v, np.float32(0))
            assert np.array_equal(y, _quantise(v, fmt)), what
        elif op.kind == A.OP_GAP:
            ref, mag = S.gap_ref(x)
            u = S.bar_used(y.reshape(ref.shape), ref, mag, S.A_GAP, S.C_FMT[fmt_name])
        elif op.kind == A.OP_DENSE:
            wk = S.bf16_rne(W[op.w_kernel]) if fmt == A.FMT_BF16 else W[op.w_kernel]
            ref, mag = S.dense_ref(x, wk, W[op.w_shift] if op.w_shift >= 0 else None, op.flags & A.FLAG_RELU)
            u = S.bar_used(y.reshape(ref.shape), ref, mag, S.A_DENSE, 0.0 if out_f32 else S.C_FMT[fmt_name])
        elif op.kind == A.OP_SOFTMAX:
            u = S.softmax_bar_used(y.reshape(len(y), -1), x.reshape(len(x), -1))
        elif op.kind == A.OP_CONV:
            tc = "simt" not in kname                         # the wgmma kernels read bf16 planes of weights (and image)
            wk = _quantise(W[op.w_kernel], fmt) if tc else W[op.w_kernel]
            xin = _quantise(x, fmt) if (tc and in_f32) else x
            res = buf(op.in1) if op.flags & A.FLAG_RESIDUAL else None
            ref = np.concatenate([conv_oracle(xin[j:j + 1], wk, W[op.w_scale] if op.w_scale >= 0 else None,
                                              W[op.w_shift] if op.w_shift >= 0 else None,
                                              None if res is None else res[j:j + 1], (op.sh, op.sw), op.pads,
                                              op.flags & A.FLAG_RELU) for j in range(len(x))])
            # the global measure of conv_check at the stage format's bar.  Its per-channel measure is calibrated on random
            # convolutions; folded BN scales of a model leave channels whose outputs are far below their dot products
            # (2.3e-3 seen in ResNet50 at fp32 parity), and the conv kernels are held to it by the conv tests.
            g, ch = conv_errors(y, ref)
            assert g <= TOL[fmt_name], (what, g, ch)
        else:
            raise AssertionError(f"no check for op kind {op.kind}")
        assert u <= 1.0, (what, u)
        used[op.kind] = max(used.get(op.kind, 0.0), u)
    return used


def _print_used(label, used):
    print(label + ": " + ", ".join(f"{A.OP_NAMES[k]} {v:.3g}" for k, v in sorted(used.items())))


# ================================================================================================ 2. stage-level paths
def _dense_model(in_shape, units, seed, activation=None):
    rng = np.random.default_rng(seed)
    inp = K.Input(shape=in_shape)
    y = K.Flatten()(inp)
    d = K.Dense(units, activation=activation)
    y = d(y)
    F = int(np.prod(in_shape))
    d.set_weights([rng.standard_normal((F, units), dtype=np.float32) * np.float32(np.sqrt(2.0 / F)),
                   (rng.standard_normal(units) * 0.1).astype(np.float32)])
    return K.Model(inp, y)


def test_stage_dense_both_kernels_both_weight_types():
    """Flatten -> Dense in bfloat16 stages (bf16-RNE weights, converted at stage creation) and float32 stages (fp32
    weights): U = 1000 runs dense_fused_kernel, U = 1002 dense_partial_kernel, at batch 1 and 32, activation-format
    output.  The bar rejects the same GPU output against weights swapped within each 4-unit group."""
    ran = set()
    for dtype in ("bfloat16", "float32"):
        fmt_name = DTYPE_FMT_NAME[dtype]
        for U in (1000, 1002):
            m = _dense_model((2, 2, 512), U, seed=U, activation="relu")
            for batch in (1, 32):
                x = np.random.default_rng(batch).standard_normal((batch, 2, 2, 512), dtype=np.float32)
                r = StageRunner.from_model(m, dtype=dtype, max_batch=batch, depth=1)
                try:
                    r.predict(x)
                    i = next(i for i, o in enumerate(r.plan.ops) if o.kind == A.OP_DENSE)
                    kname = r.op_info(i)["kernel"]
                    assert kname == ("dense_fused_kernel" if U % 4 == 0 else "dense_partial_kernel")
                    ran.add((kname, "bf16" if dtype == "bfloat16" else "fp32"))
                    used = check_stage_ops(r, fmt_name, label=f"dense U={U} n={batch}")
                    _print_used(f"stage dense {dtype} U={U} n={batch}", used)
                    if dtype == "bfloat16" and U == 1000 and batch == 32:
                        op = r.plan.ops[i]
                        wq = S.bf16_rne(r.plan.weights[op.w_kernel])
                        perm = np.arange(U).reshape(-1, 4)[:, [1, 0, 3, 2]].reshape(-1)
                        ref, mag = S.dense_ref(r.read_buffer(op.in0), wq[:, perm], r.plan.weights[op.w_shift], True)
                        y = r.read_buffer(op.out).reshape(batch, U)
                        assert S.bar_used(y, ref, mag, S.A_DENSE, S.C_FMT["bf16"]) > 1
                finally:
                    r.close()
    assert ran == {(k, t) for k in ("dense_fused_kernel", "dense_partial_kernel") for t in ("bf16", "fp32")}


@pytest.fixture(scope="module")
def vgg_head():
    """(7, 7, 512) -> Flatten -> Dense(4096, relu) -> Dense(4096, relu) -> Dense(1000, softmax), seeded weights."""
    rng = np.random.default_rng(16)
    inp = K.Input(shape=(7, 7, 512))
    y = K.Flatten()(inp)
    layers = [K.Dense(4096, activation="relu"), K.Dense(4096, activation="relu"), K.Dense(1000, activation="softmax")]
    F = 25088
    for d in layers:
        y = d(y)
        d.set_weights([rng.standard_normal((F, d.units), dtype=np.float32) * np.float32(np.sqrt(2.0 / F)),
                       (rng.standard_normal(d.units) * 0.05).astype(np.float32)])
        F = d.units
    return K.Model(inp, y)


@pytest.mark.parametrize("dtype", ["float32", "bfloat16", "float32_simt"])
def test_vgg_head_steps_and_lanes(vgg_head, dtype):
    """Three dense layers with 32, 32 and 8 column blocks share one lane workspace: six steps over two lanes give
    identical bits (the fused kernel's arrival counters re-arm across ops, steps and lanes), and every op of both lanes
    passes its bar against run_op on the lane's own input buffer.  The input repeats on purpose: the test asserts that
    steps and lanes do not change the bits."""
    fmt_name = DTYPE_FMT_NAME[dtype]
    for batch in (1, 8, 32):
        x = np.random.default_rng(batch).standard_normal((batch, 7, 7, 512), dtype=np.float32)
        x = np.maximum(x, 0)
        r = StageRunner.from_model(vgg_head, dtype=dtype, max_batch=batch, depth=2)
        try:
            kinds = [o.kind for o in r.plan.ops]
            assert kinds == [A.OP_COPY, A.OP_DENSE, A.OP_DENSE, A.OP_DENSE, A.OP_SOFTMAX]
            assert [r.op_info(i)["kernel"] for i in (1, 2, 3)] == ["dense_fused_kernel"] * 3
            outs = []
            for seq in range(6):
                r.submit(seq, x)
                r.step(seq)
                if seq >= 1:
                    outs.append(r.result(seq - 1))
            outs.append(r.result(5))
            for y in outs[1:]:
                assert np.array_equal(y, outs[0]), (dtype, batch)
            lanes = [[r.read_buffer(b, lane) for b in range(len(r.plan.bufs))] for lane in (0, 1)]
            for b0, b1 in zip(*lanes):
                assert np.array_equal(b0, b1)
            used = check_stage_ops(r, fmt_name, lane=1, label=f"vgg head n={batch}")
            _print_used(f"vgg head {dtype} n={batch}", used)
        finally:
            r.close()


@pytest.mark.parametrize("dtype", ["float32", "bfloat16", "float32_simt"])
def test_standalone_zero_padding(dtype):
    """A stage whose output is ZeroPadding2D(((1, 2), (3, 0))) runs pad_kernel: decoded output == np.pad of the decoded
    input, bit for bit."""
    inp = K.Input(shape=(5, 6, 12))
    m = K.Model(inp, K.ZeroPadding2D(((1, 2), (3, 0)))(inp))
    x = np.random.default_rng(7).standard_normal((2, 5, 6, 12), dtype=np.float32)
    r = StageRunner.from_model(m, dtype=dtype, max_batch=2, depth=1)
    try:
        y = r.predict(x)
        i = next(i for i, o in enumerate(r.plan.ops) if o.kind == A.OP_PAD)
        assert r.op_info(i)["kernel"] == "pad_kernel" and r.plan.ops[i].pads == (1, 3, 2, 0)
        check_stage_ops(r, DTYPE_FMT_NAME[dtype], label="pad")
        assert np.array_equal(y, np.pad(_quantise(x, FMTS[DTYPE_FMT_NAME[dtype]]), ((0, 0), (1, 2), (3, 0), (0, 0))))
    finally:
        r.close()


def _add_model():
    """relu(bn1(x)) + bn2(x), then ReLU (folds into the ADD); a three-input Add of that, relu(bn1(x)) and bn2(x) (two
    chained ADD ops)."""
    rng = np.random.default_rng(8)
    inp = K.Input(shape=(7, 7, 52))
    bns = [K.BatchNormalization(), K.BatchNormalization()]
    outs = [b(inp) for b in bns]
    for b in bns:
        b.set_weights([rng.uniform(0.5, 1.5, 52).astype(np.float32), rng.standard_normal(52).astype(np.float32) * 0.3,
                       rng.standard_normal(52).astype(np.float32) * 0.3, rng.uniform(0.5, 2, 52).astype(np.float32)])
    a = K.Activation("relu")(outs[0])
    s = K.Activation("relu")(K.Add()([a, outs[1]]))
    return K.Model(inp, K.Add()([s, a, outs[1]]))


@pytest.mark.parametrize("dtype", ["float32", "bfloat16", "float32_simt"])
def test_standalone_add(dtype):
    m = _add_model()
    x = np.random.default_rng(9).standard_normal((3, 7, 7, 52), dtype=np.float32)
    r = StageRunner.from_model(m, dtype=dtype, max_batch=3, depth=1)
    try:
        r.predict(x)
        adds = [o for o in r.plan.ops if o.kind == A.OP_ADD]
        assert len(adds) == 3 and adds[0].flags == A.FLAG_RELU
        assert adds[2].in0 == adds[1].out                     # the three-input Add: two chained ADD ops
        assert sum(1 for o in r.plan.ops if o.kind == A.OP_AFFINE and o.flags & A.FLAG_RELU) == 1
        used = check_stage_ops(r, DTYPE_FMT_NAME[dtype], label="add")
        assert {A.OP_COPY, A.OP_AFFINE, A.OP_ADD} <= set(used)
    finally:
        r.close()


# ================================================================================================ 3. cut-point pipelines
PIPELINES = {
    # stage 1: fp32 image cast to the stage format (COPY) + PAD; 2: the 7x7/2 conv on a padded activation input;
    # 3: a standalone AFFINE; 4: RELU + PAD; 5: an unpadded max-pool first; 6: a RELU first; 7: DENSE + SOFTMAX
    "ResNet50": (["conv1_pad", "conv1", "bn_conv1", "pool1_pad", "add_2", "avg_pool"],
                 {A.OP_COPY, A.OP_PAD, A.OP_CONV, A.OP_AFFINE, A.OP_RELU, A.OP_MAXPOOL, A.OP_GAP, A.OP_DENSE,
                  A.OP_SOFTMAX}),
    # the 1x1/2 max-pool shortcuts inside stages; the last stage starts with a standalone RELU
    "ResNet50V2": (["conv2_block1_preact_relu", "conv3_block1_out", "post_bn"],
                   {A.OP_CONV, A.OP_MAXPOOL, A.OP_AFFINE, A.OP_RELU, A.OP_GAP, A.OP_DENSE, A.OP_SOFTMAX}),
    # DENSE with an activation-format output and ReLU at a stage boundary
    "VGG16": (["block1_pool", "block5_pool", "fc1"],
              {A.OP_CONV, A.OP_MAXPOOL, A.OP_DENSE, A.OP_SOFTMAX}),
}


def test_pipeline_op_kinds_cover_every_kind():
    """Together with the standalone ADD stage, the pipelines run every op kind but PREPROCESS."""
    kinds = set().union(*(k for _, k in PIPELINES.values())) | {A.OP_ADD}
    assert kinds == set(A.OP_NAMES) - {A.OP_PREPROCESS}


@pytest.fixture(scope="module")
def models():
    return {}


@pytest.mark.parametrize("batch", [1, 8])
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("name", list(PIPELINES))
def test_pipeline_every_op(models, name, dtype, batch):
    """Every op of every stage against run_op on the operands it read.  Both lanes get the same input on purpose: their
    results must be identical (lane independence); the hand-over with distinct inputs is in tests/test_gpu_handover.py."""
    if name not in models:
        models.clear()                                          # one model's weights at a time
        models[name] = getattr(applications, name)()
    model = models[name]
    cuts, want_kinds = PIPELINES[name]
    x = applications.synthetic_input(batch, seed=20 + batch)
    if batch > 1:
        x *= np.linspace(0.7, 1.3, batch, dtype=np.float32).reshape(batch, 1, 1, 1)
    depth = 2
    with H.open_chain(model, cuts, dtype=dtype, batch=batch, depth=depth, wait_timeout_ms=5000) as runners:
        for seq in range(depth):
            runners[0].submit(seq, x)
            for r in runners:
                r.step(seq)
        outs = [runners[-1].result(seq) for seq in range(depth)]
        for r in runners:
            r.status()
        assert np.array_equal(outs[0], outs[1])
        seen = {}
        for i, r in enumerate(runners):
            used = check_stage_ops(r, DTYPE_FMT_NAME[dtype], lane=0, label=f"{name} stage {i + 1}")
            for k, v in used.items():
                seen[k] = max(seen.get(k, 0.0), v)
        _print_used(f"pipeline {name} {dtype} n={batch}", seen)
        assert set(seen) == want_kinds, (sorted(A.OP_NAMES[k] for k in set(seen) ^ want_kinds))
        if name == "VGG16":
            fc1 = runners[2].plan.ops[0]
            assert fc1.kind == A.OP_DENSE and fc1.flags == A.FLAG_RELU and runners[2].plan.bufs[fc1.out][3] == A.BUF_ACT
