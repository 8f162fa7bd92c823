"""The exact convolution check of tests/exact_conv.py, without a GPU.

* every defer_k_conv case tests/test_gpu_conv_exact.py runs satisfies the exactness precondition (the generators are
  seeded, so this is known before any GPU run);
* fp32 accumulation of the exact terms, in the kernel's K order, in random orders and in split-K groupings, gives the
  exact accumulator bit for bit at the deepest K of the suite (18432), for every operand family;
* deliberately wrong arithmetic changes the expected bits, while the norm bars of tests/conv_check.py accept some of
  it (in bf16): the gap this check closes."""
import numpy as np
import pytest

import exact_conv as X
import test_gpu_conv_exact as G
from conv_check import TOL, TOL_CH, conv_errors, conv_oracle
from simt_bars import store_planes


# ------------------------------------------------------------------------------------------------ 1. precondition
@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
def test_every_wgmma_case_is_exactly_summable(fmt_name):
    worst = 0.0
    for name in G.WGMMA_SHAPES:
        for case in G.wgmma_cases(name, fmt_name):
            worst = max(worst, X.assert_exactly_summable(case.pairs("wgmma"), case.geom, (name, case.family)))
    for name in G.RING_SHAPES:
        for case in G.ring_cases(name, fmt_name):
            worst = max(worst, X.assert_exactly_summable(case.pairs("wgmma"), case.geom, (name, case.family)))
    print(f"{fmt_name}: worst sum|terms| / g = 2^{np.log2(worst):.2f}")


@pytest.mark.parametrize("fmt_name", ["f32", "bf16x2", "bf16"])
def test_every_simt_and_stem_case_is_exactly_summable(fmt_name):
    for name in G.SIMT_SHAPES:
        for case in G.simt_cases(name, fmt_name):
            X.assert_exactly_summable(case.pairs("simt"), case.geom, (name, case.family))
    for name in G.STEM_SHAPES:
        for case in G.stem_cases(name, fmt_name):
            X.assert_exactly_summable(case.pairs("stem"), case.geom, (name, case.family))


def test_families_have_the_planes_they_claim():
    """F1: no lo plane; F2: lo in x only; F3: lo in w only; F4: both; every value has at most 16 significant bits."""
    for fam, (sx, sw) in X.FAMILIES.items():
        case = X.ExactCase("bf16x2", (1, 6, 6, 64, 64, 3, 3, 1, 1, 1, 1, 1, 1), fam, False, False, seed=1)
        for v, split in ((case.x, sx), (case.wk, sw)):
            hi, lo = X.bf16_planes(v)
            assert np.array_equal(hi + lo, v)                       # hi + lo reproduces every value exactly
            assert bool(np.any(lo != 0)) == split, fam


# ------------------------------------------------------------------------------------------------ 2. orders
def _im2col(x, geom):
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = geom
    xp = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    _, hp, wp, c = xp.shape
    ho, wo = (hp - kh) // sh + 1, (wp - kw) // sw + 1
    s0, s1, s2, s3 = xp.strides
    p = np.lib.stride_tricks.as_strided(xp, (n, ho, wo, kh, kw, c), (s0, s1 * sh, s2 * sw, s1, s2, s3), writeable=False)
    return p.reshape(n * ho * wo, kh * kw * c)


def _terms(case, kind, rows, cols):
    """[outputs, terms] fp32 products of the sampled outputs, in the kernel's K order (per k the products of the
    pairs, hi*hi first)."""
    pairs = case.pairs(kind)
    t = []
    for a, b in pairs:
        A_ = _im2col(a, case.geom)[rows].astype(np.float64)
        B_ = b.reshape(-1, b.shape[-1])[:, cols].T.astype(np.float64)
        t.append(A_ * B_)
    t = np.stack(t, axis=-1).reshape(len(rows), -1)
    assert np.array_equal(t.astype(np.float32).astype(np.float64), t)  # every product exact in fp32
    return t.astype(np.float32)


def _seq_sum(t):
    """Left-to-right fp32 sum of each row."""
    return np.add.accumulate(t, axis=1, dtype=np.float32)[:, -1]


@pytest.mark.parametrize("kind,fmt_name", [("wgmma", "bf16x2"), ("wgmma", "bf16"), ("simt", "f32")])
@pytest.mark.parametrize("family", list(X.FAMILIES))
def test_fp32_sums_are_exact_in_every_order(family, kind, fmt_name):
    geom = max(G.WGMMA_SHAPES.values(), key=lambda g: g[3] * g[5] * g[6])
    assert geom[5] * geom[6] * geom[3] == 18432              # 3x3 over 2048 channels
    case = X.ExactCase(fmt_name, geom, family, False, False, seed=7)
    exact = case.acc(kind).reshape(-1, geom[4])
    rng = np.random.default_rng(0)
    rows = rng.integers(0, exact.shape[0], 48)
    rows[:2] = (0, exact.shape[0] - 1)                       # the corners: taps in the padding
    cols = rng.integers(0, geom[4], 48)
    t = _terms(case, kind, rows, cols)
    want = exact[rows, cols]
    assert np.any(want != 0)
    assert np.array_equal(_seq_sum(t), want), "kernel K order"
    for _ in range(3):
        assert np.array_equal(_seq_sum(t[:, rng.permutation(t.shape[1])]), want), "random order"
    per_kb = 64 * (t.shape[1] // case.geom[3] // geom[5] // geom[6])      # terms per 64-channel k-block
    kbs = t.shape[1] // per_kb
    for splits in (2, 3, 8):                                 # k-block ranges (s * kbs) / S as split-K plans them
        parts = [_seq_sum(t[:, (s * kbs) // splits * per_kb:((s + 1) * kbs) // splits * per_kb]) for s in range(splits)]
        assert np.array_equal(_seq_sum(np.stack(parts, axis=1)), want), ("split order", splits)


# ------------------------------------------------------------------------------------------------ 3. mutants
MUT_GEOM = (1, 14, 14, 64, 64, 3, 3, 1, 1, 1, 1, 1, 1)


def _bars(v, case, kind):
    """Whether conv_check's norm bars accept the decoded output `v` against the fp64 oracle of the operands read."""
    hi, lo = X.bf16_planes(case.x)
    x = hi + lo if case.fmt_name == "bf16x2" else hi
    whi, wlo = X.bf16_planes(case.wk)
    w = whi + wlo if case.fmt_name == "bf16x2" else whi
    res = None if case.res is None else X.decode(case.res, case.fmt_name)
    ref = conv_oracle(x, w, case.scale, case.shift, res, case.geom[7:9], case.geom[9:], case.relu)
    g, ch = conv_errors(X.decode(v, case.fmt_name), ref)
    return g <= TOL[case.fmt_name] and ch <= TOL_CH[case.fmt_name], g, ch


def _report(name, case, v_mut, kind="wgmma"):
    want = case.expected_bits(kind)
    got = store_planes(v_mut, case.fmt_name)
    rejected = not np.array_equal(got, want)
    accepted, g, ch = _bars(v_mut, case, kind)
    print(f"{name:34s} {case.fmt_name:6s} {case.family}: norm bars {'ACCEPT' if accepted else 'reject'} "
          f"(rel {g:.2e}, per-channel {ch:.2e}); bitwise check {'rejects' if rejected else 'ACCEPTS'}")
    assert rejected, (name, case.fmt_name)
    return accepted


def _epi(case, acc, kind="wgmma", **kw):
    args = dict(scale=case.scale, shift=case.shift, res=case.res, relu=case.relu)
    args.update(kw)
    return X.replay(acc, args["scale"], args["shift"], args["res"], args["relu"], case.fmt_name, kind)


def _dropped_term(case):
    """The accumulator with one term missing at a border output: the smallest product at pixel (0, 0, 0) whose
    removal changes the stored bits."""
    acc = case.acc("wgmma")
    cols = _im2col(case.x, case.geom)[0].astype(np.float64)
    wk = case.wk.reshape(-1, case.geom[4]).astype(np.float64)
    want = case.expected_bits("wgmma")
    prod = cols[:, None] * wk
    for k, c in sorted(zip(*np.nonzero(prod)), key=lambda kc: abs(prod[kc])):
        a = acc.copy()
        a[0, 0, 0, c] = np.float32(acc[0, 0, 0, c] - prod[k, c])
        v = _epi(case, a)
        if not np.array_equal(store_planes(v, case.fmt_name), want):
            return v
    raise AssertionError("no single dropped term changes the bits")


def _split_partial(case, splits, s):
    cols = _im2col(case.x, case.geom).astype(np.float64)
    pairs = case.pairs("wgmma")
    kb = cols.shape[1] // 64
    lo_k, hi_k = (s * kb) // splits * 64, ((s + 1) * kb) // splits * 64
    part = 0
    for a, b in pairs:
        part = part + _im2col(a, case.geom)[:, lo_k:hi_k].astype(np.float64) @ b.reshape(-1, b.shape[-1])[lo_k:hi_k]
    return part.reshape(case.out_shape)


def test_bitwise_check_rejects_wrong_arithmetic():
    accepted_bf16 = []
    for fmt_name in ("bf16x2", "bf16"):
        dense = X.ExactCase(fmt_name, MUT_GEOM, "F1", False, True, seed=11)
        acc = dense.acc("wgmma")
        sf = dense.shift.copy()
        sf[[3, 4]] = sf[[4, 3]]
        # a tap off by one at the right border: the last output column reads one input column further right
        shifted = np.zeros_like(dense.x)
        shifted[:, :, :-1] = dense.x[:, :, 1:]
        off = acc.copy()
        off[:, :, -1] = X.exact_acc(X.product_pairs(shifted, dense.wk, fmt_name, "wgmma"), dense.geom)[:, :, -1]
        # one split's partial counted twice (split-K over 3)
        twice = (acc.astype(np.float64) + _split_partial(dense, 3, 1)).astype(np.float32)
        for name, v in (("one dropped term at (0, 0, 0)", _dropped_term(dense)),
                        ("shifts of channels 3 and 4 swapped", _epi(dense, acc, shift=sf)),
                        ("right-border tap off by one", _epi(dense, off)),
                        ("split 1 of 3 added twice", _epi(dense, twice))):
            accepted = _report(name, dense, v)
            if fmt_name == "bf16":
                accepted_bf16.append(accepted)
    # the three-product scheme, in fp32 parity: a fourth product (lo*lo), and lo*hi dropped
    f4 = X.ExactCase("bf16x2", MUT_GEOM, "F4", False, True, seed=12)
    xl, wl = X.bf16_planes(f4.x)[1], X.bf16_planes(f4.wk)[1]
    lolo = X.exact_acc([(xl, wl)], f4.geom)
    _report("four products (lo*lo added)", f4, _epi(f4, (f4.acc("wgmma").astype(np.float64) + lolo).astype(np.float32)))
    f2 = X.ExactCase("bf16x2", MUT_GEOM, "F2", False, True, seed=13)
    lohi = X.exact_acc([(X.bf16_planes(f2.x)[1], X.bf16_planes(f2.wk)[0])], f2.geom)
    _report("lo*hi dropped", f2, _epi(f2, (f2.acc("wgmma").astype(np.float64) - lohi).astype(np.float32)))
    # the residual as one fp32 add of hi + lo where the wgmma epilogue does two.  At an output whose accumulator is an
    # odd multiple m of the grid g (no scale, no shift), a residual of sign(m) (2^24 + 2) g makes v + res_hi a tie that
    # rounds to even; adding res_lo = 2g then lands on the other side of the tie that v + (res_hi + res_lo) rounds to.
    rc = X.ExactCase("bf16x2", MUT_GEOM, "F1", False, True, seed=14, scale=False, shift=False)
    g = 2.0 ** (X.EXP_X + X.EXP_W)
    m = rc.acc("wgmma").astype(np.float64) / g
    e = np.unravel_index(np.flatnonzero((m % 2 == 1) & (np.abs(m) < 250))[0], m.shape)
    rc.res[e] = np.float32(np.sign(m[e]) * (2 ** 24 + 2) * g)
    _report("residual added as hi + lo in one add", rc, X.replay(rc.acc("wgmma"), None, None, rc.res, False, "bf16x2", "simt"))
    assert any(accepted_bf16), "no bf16 mutant passes the norm bars: the demonstration lost its point"


def test_replay_matches_the_oracle_within_the_bars():
    """The expected bits themselves are right: decoded, they pass conv_check's bars against the fp64 oracle."""
    for fmt_name in ("bf16x2", "bf16"):
        for fam in X.FAMILIES:
            case = X.ExactCase(fmt_name, MUT_GEOM, fam, True, True, seed=21)
            accepted, g, ch = _bars(case.expected_value("wgmma"), case, "wgmma")
            assert accepted, (fmt_name, fam, g, ch)
