"""Exact expected bits of a convolution (not a test module).

A norm bar (tests/conv_check.py) cannot see one wrong term of a long dot product.  Here the operands are chosen so that
nothing is left to round in the accumulator: every product is a multiple of a grid g (the product of the finest grids of
the two operands), and the magnitudes of the products an output sums are at most BOUND * g.  Every fp32 partial sum is
then an exact multiple of g below 2^24 g, so the accumulator is the same in every K order, every split-K and every cluster
reduction, and equals the fp64 sum.  What follows the accumulator is a fixed sequence of fp32 operations, replayed here
as each kernel documents it; the expected output bits are the store rule applied to the replayed value.

The bound is 2^22, not 2^24: how wide the wgmma accumulator's internal alignment is on H100 has not been measured, and
two bits of margin keep the check from depending on it.  A case that violates it is a test-design error and fails on the
host (`assert_exactly_summable`), before any GPU run.

Executor kinds (the products each forms, per k):
* "wgmma": the tensor-core kernels (defer_k_conv backends 2-7, stems, megakernel).  BF16X2: hi*hi + lo*hi + hi*lo of the
  bf16 planes hi = rn(v), lo = rn(v - hi) of activations and weights (lo*lo is dropped, so the accumulator is
  sum(x*w - lo_x*lo_w)); BF16: hi*hi.  Epilogue (`epi_tile`): fmaf(acc, scale, shift), + res_hi, + res_lo (two fp32
  adds), ReLU, split.
* "simt": `conv_simt_kernel`: the decoded activation (hi + lo, hi, or fp32) times the fp32 weight.  Epilogue: fmaf, one
  add of the decoded residual, ReLU.
* "stem": `stem7x7s2_kernel` (fp32 image, fp32 weights): full products; fmaf, ReLU (it takes no residual).
An absent scale is 1 and an absent shift 0 in every epilogue (the kernels load 1.f / 0.f for a null pointer).
"""
import numpy as np

from simt_bars import fma32, store_planes

BOUND = 2 ** 22

# operand families: (activation has a non-zero lo plane, weight has a non-zero lo plane)
FAMILIES = {"F1": (False, False), "F2": (True, False), "F3": (False, True), "F4": (True, True)}
EXP_X, EXP_W = -4, -6           # power-of-two scales of the operands: accumulators of a few units, not integers
SPLIT_FRAC = 0.5                # share of the values of a lo-carrying operand that have a lo plane
MEAN_SMALL, MEAN_SPLIT = 4.0, 0.5 * 4.0 + 0.5 * 384.0
TARGET = 2 ** 19                # expected sum|terms| / g per output; the worst output must stay below BOUND


# ------------------------------------------------------------------------------------------------ planes and grids
def bf16_planes(v):
    """(hi, lo) as float32: hi = rn(v), lo = rn(v - hi), v - hi exact in fp32 (defer_k_encode, weight_transform_kernel,
    the stem's window split)."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(v, np.float32))
    hi = t.to(torch.bfloat16).float()
    lo = (t - hi).to(torch.bfloat16).float()
    return hi.numpy(), lo.numpy()


def quantum(*arrays):
    """The finest grid of the values: the smallest power of two that divides every non-zero value (1 if all are 0)."""
    v = np.concatenate([np.abs(np.asarray(a, np.float64)).ravel() for a in arrays])
    v = v[v != 0]
    if not v.size:
        return 1.0
    m, e = np.frexp(v)
    mi = (m * 2.0 ** 53).astype(np.int64)
    return float(np.min((mi & -mi).astype(np.float64) * np.exp2(e - 53)))


def values(rng, shape, split, density, exp):
    """Seeded operand: small integers 1..7 (at most 3 significant bits, lo = 0), and with `split` half of them 257..511 odd
    (9 bits: hi = rn(v) is even, lo = +-1), random signs, zeros at rate 1 - density, times 2^exp."""
    v = rng.integers(1, 8, shape).astype(np.float64)
    if split:
        big = 257 + 2 * rng.integers(0, 128, shape)
        v = np.where(rng.random(shape) < SPLIT_FRAC, big, v)
    v = v * rng.choice([-1.0, 1.0], shape) * (rng.random(shape) < density)
    return (v * 2.0 ** exp).astype(np.float32)


def density(family, K):
    """Density of both operands that puts the expected sum|terms| / g of an output at TARGET for depth K."""
    sx, sw = FAMILIES[family]
    m = (MEAN_SPLIT if sx else MEAN_SMALL) * (MEAN_SPLIT if sw else MEAN_SMALL)
    return float(min(1.0, np.sqrt(TARGET / (K * m))))


# ------------------------------------------------------------------------------------------------ one case
class ExactCase:
    """Seeded operands of one convolution drawn from `family`.  `geom` = (n, h, w, cin, cout, kh, kw, sh, sw, pad_t,
    pad_l, pad_b, pad_r).  Scale, shift and residual are arbitrary fp32 values (their rounding is replayed, not avoided)."""

    def __init__(self, fmt_name, geom, family, relu, residual, seed=0, scale=True, shift=True):
        n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = geom
        self.fmt_name, self.geom, self.family, self.relu = fmt_name, tuple(geom), family, relu
        rng = np.random.default_rng(seed)
        d = density(family, kh * kw * cin)
        sx, sw_ = FAMILIES[family]
        self.x = values(rng, (n, h, w, cin), sx, d, EXP_X)
        self.wk = values(rng, (kh, kw, cin, cout), sw_, d, EXP_W)
        self.scale = rng.uniform(0.5, 1.5, cout).astype(np.float32) if scale else None
        self.shift = (rng.standard_normal(cout) * 2).astype(np.float32) if shift else None
        self.ho = (h + pt + pb - kh) // sh + 1
        self.wo = (w + pl + pr - kw) // sw + 1
        self.res = (rng.standard_normal((n, self.ho, self.wo, cout)) * 4).astype(np.float32) if residual else None
        self._acc = {}

    @property
    def out_shape(self):
        return (self.geom[0], self.ho, self.wo, self.geom[4])

    def pairs(self, kind):
        return product_pairs(self.x, self.wk, self.fmt_name, kind)

    def acc(self, kind):
        """The exact accumulator of `kind` (float32), after asserting the precondition."""
        if kind not in self._acc:
            pairs = self.pairs(kind)
            assert_exactly_summable(pairs, self.geom, (self.family, self.fmt_name, kind))
            self._acc[kind] = exact_acc(pairs, self.geom)
        return self._acc[kind]

    def expected_value(self, kind):
        return replay(self.acc(kind), self.scale, self.shift, self.res, self.relu, self.fmt_name, kind)

    def expected_bits(self, kind):
        return store_planes(self.expected_value(kind), self.fmt_name)


def product_pairs(x, wk, fmt_name, kind):
    """[(activation operand, weight operand)] whose products the executor adds (float32 arrays, NHWC / HWIO)."""
    if kind == "stem" or (kind == "simt" and fmt_name == "f32"):
        return [(np.asarray(x, np.float32), np.asarray(wk, np.float32))]
    xh, xl = bf16_planes(x)
    if kind == "simt":                   # the decoded activation times the fp32 weight
        return [((xh + xl) if fmt_name == "bf16x2" else xh, np.asarray(wk, np.float32))]
    wh, wl = bf16_planes(wk)
    if fmt_name == "bf16":
        return [(xh, wh)]
    return [(xh, wh), (xl, wh), (xh, wl)]


def _conv64(x, wk, geom):
    from oracle import keras_ref as R
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = geom
    xp = np.pad(np.asarray(x, np.float64), ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    return R.conv2d(xp, np.asarray(wk, np.float64), None, (sh, sw), "valid")


def _pairs_conv64(pairs, geom, f=lambda a: a):
    """sum over the pairs of conv(f(a), f(b)): one conv of the pairs stacked along the input channels."""
    xs = np.concatenate([f(np.asarray(a, np.float64)) for a, _ in pairs], axis=-1)
    ws = np.concatenate([f(np.asarray(b, np.float64)) for _, b in pairs], axis=2)
    g = geom[:3] + (xs.shape[-1],) + geom[4:]
    return _conv64(xs, ws, g)


def mass(pairs, geom):
    """sum|terms| / g per output, g = (finest grid of the activation operands) * (finest grid of the weight operands)."""
    g = quantum(*[a for a, _ in pairs]) * quantum(*[b for _, b in pairs])
    return _pairs_conv64(pairs, geom, np.abs) / g


def assert_exactly_summable(pairs, geom, what=""):
    """Every output's products sum exactly in fp32, in any order and grouping: sum|terms| <= BOUND * g."""
    m = float(mass(pairs, geom).max())
    assert m <= BOUND, ("operands not exactly summable", what, geom, f"max sum|terms| / g = {m:.4g} > 2^22")
    return m


def exact_acc(pairs, geom):
    """The accumulator, exact in fp64 under the bound, as float32 (asserted exact)."""
    acc = _pairs_conv64(pairs, geom)
    acc32 = acc.astype(np.float32)
    assert np.array_equal(acc32.astype(np.float64), acc), "accumulator not representable in fp32"
    return acc32


# ------------------------------------------------------------------------------------------------ epilogues
def replay(acc, scale, shift, res, relu, fmt_name, kind):
    """The kernel's fp32 epilogue on the float32 accumulator, operation by operation."""
    cout = acc.shape[-1]
    sc = np.ones(cout, np.float32) if scale is None else np.asarray(scale, np.float32)
    sf = np.zeros(cout, np.float32) if shift is None else np.asarray(shift, np.float32)
    v = fma32(acc, sc, sf)
    if res is not None:
        assert kind != "stem", "stem7x7s2_kernel takes no residual"
        if fmt_name == "f32":
            v = v + np.asarray(res, np.float32)
        else:
            rh, rl = bf16_planes(res)
            if fmt_name == "bf16":
                v = v + rh
            elif kind == "wgmma":
                v = (v + rh) + rl
            else:
                v = v + (rh + rl)
    if relu:
        v = np.maximum(v, np.float32(0))
    return v.astype(np.float32)


def decode(v, fmt_name):
    """The value a reader of the stored `v` decodes: hi + lo, the bf16, or the fp32 word."""
    v = np.asarray(v, np.float32)
    if fmt_name == "f32":
        return v
    hi, lo = bf16_planes(v)
    return hi + lo if fmt_name == "bf16x2" else hi


def replay_affine(stored, scale2, shift2, relu2):
    """The folded affine op's second output: fmaf of the decoded stored value, then the optional ReLU."""
    u = fma32(stored, np.asarray(scale2, np.float32), np.asarray(shift2, np.float32))
    return np.maximum(u, np.float32(0)) if relu2 else u


# ------------------------------------------------------------------------------------------------ comparison
def raw_bits(torch, y, fmt_name):
    """The raw words of an output buffer: uint32 (F32) or the int16 planes [hi | lo] (BF16X2) / [hi] (BF16)."""
    if fmt_name == "f32":
        return y.view(torch.int32).cpu().numpy().view(np.uint32).copy()
    return y.view(torch.int16).cpu().numpy().copy()


def assert_bits(got, want, out_shape, fmt_name, what):
    """Raw output words equal the expected bits; else report the first mismatch as (plane, n, h, w, c), its flat
    output row and the 128-row x 64-column tile that holds it."""
    got, want = np.asarray(got).ravel(), np.asarray(want).ravel()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero(got != want)
    if not bad.size:
        return
    per_plane = int(np.prod(out_shape))
    i = int(bad[0])
    plane, e = divmod(i, per_plane)
    nhwc = tuple(int(v) for v in np.unravel_index(e, out_shape))
    row, c = divmod(e, out_shape[-1])
    to_f = ((lambda a: a.view(np.float32)) if fmt_name == "f32"
            else (lambda a: (a.view(np.uint16).astype(np.uint32) << 16).view(np.float32)))
    raise AssertionError(f"{what}: {bad.size} of {got.size} words differ; first at plane {plane} (n, h, w, c) = {nhwc}, "
                         f"row {row} (M tile {row // 128}, row {row % 128}), column group {c // 64}: "
                         f"got {to_f(got[i:i + 1])[0]!r}, want {to_f(want[i:i + 1])[0]!r}")
