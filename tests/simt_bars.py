"""Shared helpers of the SIMT-op tests (not a test module): fp64 references of the reductions (dense, global average
pool, softmax) with their per-element error bars, and host restatements of the kernels' exact rules (the split counts
of the dense kernels, fp32 fma, the activation formats' store rule).

A reduction bar is per element, `|y - ref| <= a * sum|terms| + c_fmt * |ref|`: `a` bounds fp32 accumulation against the
sum of the magnitudes that were added, `c_fmt` the rounding of the stored result.  A max-norm bar (max|y - ref| /
max|ref|) would let a single dropped term of a 25088-long dot product through; this one does not
(tests/test_simt_bars_host.py shows it on deliberately wrong arithmetic).
"""
import numpy as np

# rounding of a value stored in the stage format, relative to |value|: exact fp32; hi + lo (lo is rounded to 8
# significant bits of a remainder below 2^-8 |value|: 2^-16, bar 2^-15); one bf16 (unit roundoff 2^-8, reached just above
# a power of two - a bf16 output uses up to the whole of this term, by construction)
C_FMT = {"f32": 0.0, "bf16x2": 2.0 ** -15, "bf16": 2.0 ** -8}

# `a` of the reductions.  A chain of k fp32 additions is off by at most ~k * 2^-24 * sum|terms|; the kernels add at most
# a few hundred terms in one chain (a split's rows per warp, then 8 warps, then the splits; pixels per threadIdx.y row,
# then 8 rows), and rounding errors of independent terms mostly cancel.  Worst cases observed on an H100 (700 W) over
# tests/test_gpu_simt_ops.py with an fp32 output (so c_fmt = 0), as a fraction of the bar: dense 0.097 (at F = 1 and
# F = 65, where sum|terms| is smallest against the rounding of the result), gap 0.17.  A dropped term of the largest case
# (F = 25088) costs ~2e-4 * sum|terms| in the worst output unit, 200x the bar.
A_DENSE = 1e-6
A_GAP = 1e-6

# softmax: exp(x - m) * (1 / sum), element by element relative to the fp64 result.  expf is accurate to 2 ulp, the sum
# of up to 4097 terms in 256 strided chains plus a warp tree; x - m is rounded to fp32, which moves exp by up to
# |x - m| * 2^-24 relative (so that term is part of the bar).  Below FLT_MIN a float has fewer than 24 significant bits:
# those outputs are held to an absolute FLT_MIN.  Observed worst case on an H100: 0.53 of the bar.
SOFTMAX_RTOL = 3e-6
FLT_MIN = float(np.finfo(np.float32).tiny)
SOFTMAX_SUM_TOL = 1e-5


# ------------------------------------------------------------------------------------------------ host rules
def bf16_rne(x):
    """fp32 -> bf16 round-to-nearest-even, back as float32 (what `launch_f32_to_bf16` does to dense weights)."""
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).float().numpy()


def store_planes(v, fmt_name):
    """Raw bits the format's store rule writes for the float32 values `v`: the fp32 words (uint32), one bf16 plane
    (int16), or [hi plane | lo plane] with hi = rn(v) and lo = rn(v - hi), v - hi exact in fp32 (int16)."""
    import torch
    v = np.ascontiguousarray(v, np.float32).reshape(-1)
    if fmt_name == "f32":
        return v.view(np.uint32).copy()
    t = torch.from_numpy(v)
    hi = t.to(torch.bfloat16)
    if fmt_name == "bf16":
        return hi.view(torch.int16).numpy().copy()
    lo = (t - hi.float()).to(torch.bfloat16)
    return torch.cat([hi, lo]).view(torch.int16).numpy().copy()


def fma32(a, b, c):
    """Correctly rounded float32 fma(a, b, c) (fmaf).  a * b is exact in fp64 (24 + 24 bits); a + c in fp64 may round,
    and rounding that again to fp32 can land on the wrong side of a fp32 tie.  TwoSum gives the exact error e of the
    fp64 sum s; where s is exactly a tie between two floats and e != 0, the exact value lies on e's side of it."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)
    c = np.asarray(c, np.float64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    d = s - r.astype(np.float64)                              # s = r + d exactly
    up = np.nextafter(r, np.float32(np.inf))
    dn = np.nextafter(r, np.float32(-np.inf))
    tie = (d != 0) & ((2 * d == up.astype(np.float64) - r) | (2 * d == dn.astype(np.float64) - r))
    # at a tie r is the even neighbour; the exact value s + e is past the tie when e has d's sign, short of it otherwise
    away = np.where(d > 0, up, dn)
    tie_r = np.where(np.sign(e) == np.sign(d), away, r)
    # d == 0 (s representable) with e != 0 rounds to r; no tie: |e| < half an fp64 ulp cannot cross an fp32 boundary
    return np.where(tie & (e != 0), tie_r, r).astype(np.float32)


def dense_splits(n, F, U):
    """Restatement of `dense_splits` (kernels_simt.cu): K splits of the two-kernel dense path."""
    col_blocks = (U + 127) // 128
    want = (2 * 132 + col_blocks - 1) // col_blocks
    s = min(want, (F + 31) // 32)
    s = max(s, (F + 1023) // 1024)
    return max(s, 1)


def dense_fused_splits(n, F, U):
    """Restatement of `dense_fused_splits`: K splits of `dense_fused_kernel` (capped by the workspace's split count)."""
    col_blocks = (U + 127) // 128
    want = (2 * 132 + col_blocks - 1) // col_blocks
    s = min(want, max(F // 64, 1), dense_splits(n, F, U))
    s = max(s, (F + 1023) // 1024)
    return max(s, 1)


def split_rows(splits, F):
    """(rows per split, number of splits) after the launcher's rounding: the last split is ragged."""
    rows = (F + splits - 1) // splits
    return rows, (F + rows - 1) // rows


# ------------------------------------------------------------------------------------------------ references and bars
def dense_ref(x, w, bias, relu):
    """fp64 dense of the operands the kernel read, and sum|terms| per output ((n, U) each)."""
    x = np.asarray(x, np.float64).reshape(len(x), -1)
    w = np.asarray(w, np.float64)
    ref = x @ w
    mag = np.abs(x) @ np.abs(w)
    if bias is not None:
        ref = ref + np.asarray(bias, np.float64)
        mag = mag + np.abs(np.asarray(bias, np.float64))
    if relu:
        ref = np.maximum(ref, 0)
    return ref, mag


def gap_ref(x):
    """fp64 mean over (h, w) and the mean of |x| (sum|terms| of the mean) per (n, c)."""
    x = np.asarray(x, np.float64)
    return x.mean(axis=(1, 2)), np.abs(x).mean(axis=(1, 2))


def bar_used(y, ref, mag, a, c):
    """Largest |y - ref| / (a * mag + c * |ref|): the fraction of the bar used (<= 1 passes; NaN / inf -> inf)."""
    y = np.asarray(y, np.float64).reshape(ref.shape)
    err = np.abs(y - ref)
    lim = a * mag + c * np.abs(ref)
    r = np.where(err == 0, 0.0, err / np.maximum(lim, 1e-300))
    return float(np.inf) if not np.all(np.isfinite(y)) else float(r.max())


def softmax_ref(x):
    """fp64 softmax of the fp32 logits `x` ([n, c])."""
    x = np.asarray(x, np.float64)
    z = x - x.max(axis=-1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(axis=-1, keepdims=True)


def softmax_bar_used(p, x):
    """Fraction of the softmax bar used: per element relative to the fp64 result (with the fp32 rounding of x - m),
    the row sums, and argmax equality (inf if it differs or a value is not finite)."""
    x = np.asarray(x, np.float64)
    p = np.asarray(p, np.float64).reshape(x.shape)
    if not np.all(np.isfinite(p)):
        return float(np.inf)
    ref = softmax_ref(x)
    z = np.abs(x - x.max(axis=-1, keepdims=True))
    lim = (SOFTMAX_RTOL + z * 2.0 ** -24) * ref + FLT_MIN
    used = float((np.abs(p - ref) / lim).max())
    used = max(used, float(np.abs(p.sum(axis=-1) - 1).max()) / SOFTMAX_SUM_TOL)
    if not np.array_equal(p.argmax(axis=-1), ref.argmax(axis=-1)):
        return float(np.inf)
    return used


def softmax_rows(c, seed=0):
    """Softmax test rows of length c: logits at scale 1, at scale 100, spanning +-1e4, a constant row, one dominant
    entry (float32, [5, c])."""
    rng = np.random.default_rng(seed)
    return np.stack([rng.standard_normal(c), 100 * rng.standard_normal(c), rng.uniform(-1e4, 1e4, c),
                     np.full(c, 3.25), np.where(np.arange(c) == c // 2, 40.0, rng.standard_normal(c))]).astype(np.float32)
