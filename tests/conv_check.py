"""Shared helpers of the convolution tests (not a test module).

Stage-format encode / decode through the C-ABI, quantisation to what a format can represent, one convolution through
`defer_k_conv` against the fp64 oracle (`oracle.keras_ref.conv2d` on the quantised operands), and the error measures
every convolution check asserts on:

* `rel_err`: max|y - ref| / max|ref| over the whole output;
* per-output-channel: max over c of max|y_c - ref_c| / max|ref_c|.  An epilogue error confined to channels with small
  outputs (a wrong shift, scale or residual plane for a few channels) hides under the global max norm; it does not
  hide here.

These bars are the precision check for random operands.  Every executor is also checked bit for bit against exact
expected bits on exactly summable operands (tests/exact_conv.py, tests/test_gpu_conv_exact.py), which one wrong term fails.
"""
import ctypes as C

import numpy as np

from defer_b200 import _cabi as A

FMTS = {"f32": A.FMT_F32, "bf16x2": A.FMT_BF16X2, "bf16": A.FMT_BF16}

# Tolerances of the two measures per stage format, for a kernel fed exactly the operands the oracle sees.  Worst cases
# observed on an H100 (700 W) over tests/test_gpu_kernels.py::test_conv_tcgen05_shapes and tests/test_gpu_conv_paths.py:
#   bf16x2 (fp32 parity: hi*hi + lo*hi + hi*lo into the fp32 wgmma accumulator, hi/lo split of the output): rel_err
#     6.3e-5, at K = 18432 (3x3 over 2048 channels); it grows about linearly with K (5e-6 at K = 1024).  Per-channel
#     4.3e-4, in a post-ReLU channel of a 7x7 map whose largest output is small against its dot products.  Bars: ~3x
#     that.  A dropped cross term or a missing residual lo plane costs ~2^-9 = 2e-3.
#   bf16 (one plane, bf16 rounding of the output, half an ulp = 2^-9 of a value): rel_err 3.7e-3, per-channel 3.9e-3.
#     Bars: 1e-2.
#   f32 (SIMT, exact-order fp32): the SIMT kernels' bar.
TOL = {"f32": 2e-5, "bf16x2": 2e-4, "bf16": 1e-2}
TOL_CH = {"f32": 2e-5, "bf16x2": 1.5e-3, "bf16": 1e-2}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _encode(torch, lib, x_np, fmt):
    x = torch.from_numpy(np.ascontiguousarray(x_np, np.float32)).cuda()
    if fmt == A.FMT_F32:
        return x
    n = x.numel()
    planes = 2 if fmt == A.FMT_BF16X2 else 1
    y = torch.empty(planes * n, dtype=torch.bfloat16, device="cuda")
    A.check(lib.defer_k_encode(fmt, _ptr(x), _ptr(y), n, None))
    return y


def _decode(torch, lib, y, fmt, shape):
    if fmt == A.FMT_F32:
        return y.cpu().numpy().reshape(shape)
    n = int(np.prod(shape))
    out = torch.empty(n, dtype=torch.float32, device="cuda")
    A.check(lib.defer_k_decode(fmt, _ptr(y), _ptr(out), n, None))
    return out.cpu().numpy().reshape(shape)


def _alloc_act(torch, fmt, n_elems):
    if fmt == A.FMT_F32:
        return torch.zeros(n_elems, dtype=torch.float32, device="cuda")
    return torch.zeros((2 if fmt == A.FMT_BF16X2 else 1) * n_elems, dtype=torch.bfloat16, device="cuda")


def _quantise(x, fmt):
    """What the stage format can represent (so the oracle sees the same inputs the kernel does)."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(x, np.float32))
    if fmt == A.FMT_F32:
        return np.asarray(x, np.float32)
    hi = t.to(torch.bfloat16)
    if fmt == A.FMT_BF16:
        return hi.float().numpy()
    lo = (t - hi.float()).to(torch.bfloat16)
    return (hi.float() + lo.float()).numpy()


# ------------------------------------------------------------------------------------------------ error measures
def conv_errors(y, ref):
    """(rel_err, per-output-channel rel_err) of an NHWC (or [..., C]) output; a channel whose reference is all zero is
    measured against a floor of 1e-6 * max|ref|."""
    y = np.asarray(y, np.float64)
    ref = np.asarray(ref, np.float64)
    c = ref.shape[-1]
    d = np.abs(y - ref).reshape(-1, c).max(axis=0)
    m = np.abs(ref).reshape(-1, c).max(axis=0)
    top = max(float(m.max()), 1e-30)
    return float(d.max() / top), float((d / np.maximum(m, 1e-6 * top)).max())


def assert_conv(y, ref, fmt_name, what=""):
    """Both measures within the format's bars; returns them."""
    g, ch = conv_errors(y, ref)
    assert g <= TOL[fmt_name] and ch <= TOL_CH[fmt_name], (what, fmt_name, f"rel_err {g:.3e}", f"per-channel {ch:.3e}")
    return g, ch


# ------------------------------------------------------------------------------------------------ one conv
def conv_oracle(x, wk, scale, shift, res, strides, pads, relu):
    """fp64 conv2d of already-quantised operands, then scale / shift / residual / ReLU (None = absent)."""
    from oracle import keras_ref as R
    t, l, b, r = pads
    ref = R.conv2d(np.pad(np.asarray(x, np.float64), ((0, 0), (t, b), (l, r), (0, 0))), np.asarray(wk, np.float64), None,
                   strides, "valid")
    if scale is not None:
        ref = ref * np.asarray(scale, np.float64)
    if shift is not None:
        ref = ref + np.asarray(shift, np.float64)
    if res is not None:
        ref = ref + np.asarray(res, np.float64)
    if relu:
        ref = np.maximum(ref, 0)
    return ref


class ConvCase:
    """Seeded inputs of one convolution and their fp64 oracle.  `geom` = (n, h, w, cin, cout, kh, kw, sh, sw, pad_t,
    pad_l, pad_b, pad_r); `quantise_w`: the tensor-core backends (>= 2) see bf16 weight planes, SIMT the fp32 weights."""

    def __init__(self, fmt_name, geom, relu, residual, seed=0, scale=True, shift=True, quantise_w=True):
        n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = geom
        self.fmt_name, self.fmt, self.geom, self.relu = fmt_name, FMTS[fmt_name], tuple(geom), relu
        rng = np.random.default_rng(seed)
        self.x = rng.standard_normal((n, h, w, cin), dtype=np.float32)
        self.wk = rng.standard_normal((kh, kw, cin, cout), dtype=np.float32) * np.float32(np.sqrt(2.0 / (kh * kw * cin)))
        sc = rng.uniform(0.5, 1.5, cout).astype(np.float32)
        sf = (rng.standard_normal(cout) * 0.2).astype(np.float32)
        self.scale, self.shift = (sc if scale else None), (sf if shift else None)
        self.ho = (h + pt + pb - kh) // sh + 1
        self.wo = (w + pl + pr - kw) // sw + 1
        self.res = rng.standard_normal((n, self.ho, self.wo, cout), dtype=np.float32) if residual else None
        wq = _quantise(self.wk, self.fmt) if quantise_w else self.wk
        self.ref = conv_oracle(_quantise(self.x, self.fmt), wq, self.scale, self.shift,
                               None if self.res is None else _quantise(self.res, self.fmt), (sh, sw), (pt, pl, pb, pr), relu)

    def run(self, torch, lib, backend):
        """The kernel's output (decoded to fp32) through defer_k_conv `backend`."""
        n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = self.geom
        fmt = self.fmt
        dev = lambda a: torch.from_numpy(a).cuda() if a is not None else None   # noqa: E731
        xd = _encode(torch, lib, self.x, fmt)
        rd = _encode(torch, lib, self.res, fmt) if self.res is not None else None
        wd, sd, fd = dev(self.wk), dev(self.scale), dev(self.shift)
        yd = _alloc_act(torch, fmt, n * self.ho * self.wo * cout)
        A.check(lib.defer_k_conv(fmt, backend, _ptr(xd), 0, _ptr(wd), _ptr(sd), _ptr(fd), _ptr(rd), _ptr(yd),
                                 n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr, A.FLAG_RELU if self.relu else 0, None))
        torch.cuda.synchronize()
        return _decode(torch, lib, yd, fmt, (n, self.ho, self.wo, cout))


def _conv_case(torch, lib, fmt_name, backend, n, h, w, cin, cout, k, s, pad, relu, residual, seed=0):
    """Square kernel, equal strides and symmetric padding: (rel_err, y, ref) of one run of `backend`."""
    from oracle import keras_ref as R
    case = ConvCase(fmt_name, (n, h, w, cin, cout, k, k, s, s, pad, pad, pad, pad), relu, residual, seed,
                    quantise_w=backend >= 2)
    y = case.run(torch, lib, backend)
    return R.rel_err(y, case.ref), y, case.ref


def check_executors(torch, lib, case, monkeypatch):
    """Every wgmma executor on one case.  Backend 2 without split-K (one tile per CTA, BN 128 where C_out allows),
    3 (persistent grid, BN 64), 4 (streaming, BN 64) and 5 (streaming, BN 128, when C_out % 128 == 0) must each pass the
    oracle check and be bit-identical to each other: they share the K order of every output.  Backend 2 with its default
    plan (split-K where it triggers) is checked against the oracle only.  Returns the worst (rel_err, per-channel)."""
    cout = case.geom[4]
    worst = (0.0, 0.0)
    monkeypatch.setenv("DEFER_UMMA_SPLITK", "0")
    outs = {}
    for backend in (2, 3, 4) + ((5,) if cout % 128 == 0 else ()):
        outs[backend] = y = case.run(torch, lib, backend)
        worst = max(worst, assert_conv(y, case.ref, case.fmt_name, (case.geom, backend)))
    for backend, y in outs.items():
        assert np.array_equal(y, outs[2]), (case.geom, case.fmt_name, "backend", backend, "differs from backend 2")
    monkeypatch.delenv("DEFER_UMMA_SPLITK")
    y = case.run(torch, lib, 2)
    return max(worst, assert_conv(y, case.ref, case.fmt_name, (case.geom, "2 default plan")))
