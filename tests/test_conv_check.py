"""The convolution checker of tests/conv_check.py, without a GPU: it accepts a numpy emulation of the wgmma kernels'
arithmetic at the tolerances the GPU tests use, and rejects each of a set of subtly wrong variants of that emulation.

Emulated arithmetic (what conv_body + epi_pair compute, in the fixed K order of the kernel):
* bf16x2: operands split into bf16 hi / lo planes; per k the products hi*hi, lo*hi, hi*lo (exact in fp32) are added
  to an fp32 accumulator; epilogue fmaf(acc, scale, shift) + residual hi + residual lo, ReLU, hi / lo split;
* bf16: one plane, products summed in fp32, the same epilogue, bf16 rounding of the output.
"""
import numpy as np
import pytest

from conv_check import FMTS, TOL, TOL_CH, ConvCase, assert_conv, conv_errors


def _bf16(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).float().numpy()


def _planes(x, fmt_name):
    hi = _bf16(x)
    return (hi, _bf16(np.asarray(x, np.float32) - hi)) if fmt_name == "bf16x2" else (hi, None)


def _im2col(x, kh, kw, sh, sw, pads):
    """[M, K] patch matrix, k = (kernel row, kernel column, channel): the HWIO order of the filter bank."""
    t, l, b, r = pads
    xp = np.pad(x, ((0, 0), (t, b), (l, r), (0, 0)))
    n, h, w, c = xp.shape
    ho, wo = (h - kh) // sh + 1, (w - kw) // sw + 1
    s0, s1, s2, s3 = xp.strides
    p = np.lib.stride_tricks.as_strided(xp, (n, ho, wo, kh, kw, c), (s0, s1 * sh, s2 * sw, s1, s2, s3), writeable=False)
    return np.ascontiguousarray(p.reshape(n * ho * wo, kh * kw * c))


def emulate(case, drop_cross=False, res_hi_only=False, shift_from_neighbour=None, zero_last_tile=False,
            top_row_as_padding=False):
    """The kernel's output for `case`, optionally with one defect."""
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = case.geom
    f = case.fmt_name
    x = case.x.copy()
    if top_row_as_padding:          # stem patch builder testing ih > 0 instead of ih >= 0
        x[:, 0] = 0
    ah, al = _planes(_im2col(x, kh, kw, sh, sw, (pt, pl, pb, pr)), f)
    bh, bl = _planes(case.wk.reshape(kh * kw * cin, cout), f)
    acc = np.zeros((ah.shape[0], cout), np.float32)
    for k in range(ah.shape[1]):
        acc += np.outer(ah[:, k], bh[k])
        if f == "bf16x2":
            acc += np.outer(al[:, k], bh[k])
            if not drop_cross:
                acc += np.outer(ah[:, k], bl[k])
    shift = case.shift.copy()
    if shift_from_neighbour is not None:
        shift[shift_from_neighbour] = shift[shift_from_neighbour + 1]
    v = (acc.astype(np.float64) * case.scale + shift).astype(np.float32)      # fmaf: one rounding
    if case.res is not None:
        rh, rl = _planes(case.res.reshape(-1, cout), f)
        v = v + rh
        if rl is not None and not res_hi_only:
            v = v + rl
    if case.relu:
        v = np.maximum(v, 0)
    hi, lo = _planes(v, f)
    y = hi + lo if lo is not None else hi
    if zero_last_tile:              # the rows of the last, partial 128-row tile never stored
        y[y.shape[0] // 128 * 128:] = 0
    return y.reshape(case.ref.shape)


CASES = {
    # geometry (n, h, w, cin, cout, kh, kw, sh, sw, pad t, l, b, r), relu, residual
    "3x3": ((2, 7, 9, 64, 64, 3, 3, 1, 1, 1, 1, 1, 1), True, True),
    "deep_k": ((1, 5, 5, 256, 64, 3, 3, 1, 1, 1, 1, 1, 1), False, True),        # K = 2304
    "stem": ((2, 23, 19, 3, 64, 7, 7, 2, 2, 3, 3, 2, 2), True, False),          # 198 rows: one full, one ragged tile
}


def _case(name, fmt_name, **kw):
    geom, relu, residual = CASES[name]
    return ConvCase(fmt_name, geom, relu, residual, seed=len(name), **kw)


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("name", list(CASES))
def test_checker_accepts_emulated_kernel(name, fmt_name):
    case = _case(name, fmt_name)
    g, ch = assert_conv(emulate(case), case.ref, fmt_name, name)
    # the emulation is not the oracle: it carries the format's rounding, and the bars sit above it
    assert 0 < g and 0 < ch


@pytest.mark.parametrize("name", ["3x3", "deep_k"])
def test_checker_rejects_dropped_cross_term(name):
    case = _case(name, "bf16x2")
    with pytest.raises(AssertionError):
        assert_conv(emulate(case, drop_cross=True), case.ref, "bf16x2")


@pytest.mark.parametrize("name", ["3x3", "deep_k"])
def test_checker_rejects_residual_without_lo_plane(name):
    case = _case(name, "bf16x2")
    with pytest.raises(AssertionError):
        assert_conv(emulate(case, res_hi_only=True), case.ref, "bf16x2")


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
def test_checker_rejects_shift_of_the_neighbour_channel(fmt_name):
    case = _case("3x3", fmt_name)
    with pytest.raises(AssertionError):
        assert_conv(emulate(case, shift_from_neighbour=5), case.ref, fmt_name)


def test_per_channel_measure_sees_a_small_channel():
    """The same defect in a channel whose outputs are small (scale 0.01): the global max norm passes it in bf16, the
    per-channel measure does not."""
    case = _case("stem", "bf16")
    case.scale[5] = np.float32(0.01)
    case.shift[5:7] = np.float32([0.002, -0.004])
    case.ref = emulate(case).astype(np.float64)              # the defect-free kernel as the reference of this check
    g, ch = conv_errors(emulate(case, shift_from_neighbour=5), case.ref)
    assert g <= TOL["bf16"] and ch > TOL_CH["bf16"], (g, ch)


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
def test_checker_rejects_unstored_ragged_tile(fmt_name):
    case = _case("stem", fmt_name)
    with pytest.raises(AssertionError):
        assert_conv(emulate(case, zero_last_tile=True), case.ref, fmt_name)


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
def test_checker_rejects_top_image_row_as_padding(fmt_name):
    case = _case("stem", fmt_name)
    with pytest.raises(AssertionError):
        assert_conv(emulate(case, top_row_as_padding=True), case.ref, fmt_name)


def test_formats_and_bars():
    assert set(TOL) == set(TOL_CH) == set(FMTS)
    assert TOL["bf16x2"] < 2.0 ** -9 < TOL["bf16"]       # a dropped bf16x2 term (~2^-9) cannot pass
