"""Host-side checks of the error bars tests/test_gpu_simt_ops.py holds the SIMT kernels to (no GPU needed).

Each reduction bar must pass an fp32 computation in the kernel's own summation order and reject fp64 results of
deliberately wrong arithmetic on the same seeded inputs: a dropped K row at a split boundary, a bias added twice, a
permuted 4-unit group, ReLU before the bias (dense); a dropped pixel, division by hw - 1 (GAP); no max subtraction, a
missing term of the sum (softmax).  The restated host rules (fp32 fma, split counts) are pinned here too."""
import numpy as np
import pytest

import simt_bars as S

FMT_NAMES = ("f32", "bf16x2", "bf16")


# ------------------------------------------------------------------------------------------------ restated rules
def test_dense_fused_splits_at_vgg_fc1():
    """fc1 (F = 25088, U = 4096): 25 splits (min_split decides), 24 of 1004 rows and a ragged one of 992."""
    s = S.dense_fused_splits(1, 25088, 4096)
    rows, splits = S.split_rows(s, 25088)
    assert (s, rows, splits) == (25, 1004, 25)
    assert 25088 - (splits - 1) * rows == 992
    # 8 column blocks: 33 splits for two waves of 132 SMs, the last one 96 rows
    assert S.split_rows(S.dense_fused_splits(32, 4096, 1000), 4096) == (125, 33)
    assert S.split_rows(S.dense_splits(9, 4096, 1002), 4096) == (125, 33)


def test_fma32_rounds_once():
    """fp64 a*b + c rounded to fp32 double-rounds when the fp64 sum lands on a fp32 tie; fma32 does not."""
    a = np.float32(-(2.0 ** -24) * (1 + 2.0 ** -23))
    b = np.float32(1 - 2.0 ** -23)
    c = np.float32(1 + 2.0 ** -23)
    # exact: 1 + 2^-24 + 2^-70, just above the tie between 1 and 1 + 2^-23
    assert np.float32(np.float64(a) * np.float64(b) + np.float64(c)) == np.float32(1.0)
    assert S.fma32(a, b, c) == np.float32(1 + 2.0 ** -23)
    assert S.fma32(-a, b, np.float32(1.0)) == np.float32(1.0)            # 1 + 2^-24 - 2^-70: below the tie
    rng = np.random.default_rng(0)
    x, y, z = (rng.standard_normal(10000).astype(np.float32) for _ in range(3))
    ref = (x.astype(np.float64) * y + z).astype(np.float32)
    assert np.array_equal(S.fma32(x, y, z), ref)                          # no ties in random data


def test_store_planes_rule():
    v = np.array([1.0, 1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -3.3, 0.0], np.float32)
    hi = S.store_planes(v, "bf16")
    assert hi.dtype == np.int16 and hi[0] == 0x3F80 and hi[1] == 0x3F80 and hi[2] == 0x3F82   # ties to even
    p = S.store_planes(v, "bf16x2")
    assert np.array_equal(p[:5], hi)
    import torch
    dec = torch.from_numpy(p).view(torch.bfloat16).float().numpy()
    assert np.array_equal(dec[:3] + dec[5:8], v[:3])                      # 16 significant bits: exact here
    assert abs(dec[3] + dec[8] - v[3]) <= 2.0 ** -17 * abs(v[3]) and dec[3] == np.float32(-3.296875)


# ------------------------------------------------------------------------------------------------ dense
def _fused_order_fp32(x, w, bias, relu):
    """fp32 dense in dense_fused_kernel's order: per split, 8 warps take every 8th row, warps summed in order, splits
    summed in order, then bias and ReLU."""
    n, F = x.shape
    U = w.shape[1]
    rows, splits = S.split_rows(S.dense_fused_splits(n, F, U), F)
    total = np.zeros((n, U), np.float32)
    for k in range(splits):
        f0, f1 = k * rows, min(F, (k + 1) * rows)
        part = np.zeros((n, U), np.float32)
        for wq in range(8):
            acc = np.zeros((n, U), np.float32)
            for f in range(f0 + wq, f1, 8):
                acc = acc + x[:, f:f + 1] * w[f]
            part = part + acc
        total = total + part
    if bias is not None:
        total = total + bias
    return np.maximum(total, 0) if relu else total


@pytest.fixture(scope="module")
def dense_case():
    rng = np.random.default_rng(5)
    n, F, U = 2, 25088, 4096
    x = np.maximum(rng.standard_normal((n, F), dtype=np.float32), 0)       # post-ReLU features, as VGG's fc1 reads
    w = (rng.standard_normal((F, U), dtype=np.float32) * np.float32(0.01))
    b = (rng.standard_normal(U) * 0.1).astype(np.float32)
    return x, w, b


def test_dense_bar_passes_fp32_and_rejects_wrong_arithmetic(dense_case):
    x, w, b = dense_case
    n, F = x.shape
    ref, mag = S.dense_ref(x, w, b, relu=True)
    y32 = _fused_order_fp32(x, w, b, relu=True)
    for f in FMT_NAMES:
        assert S.bar_used(y32, ref, mag, S.A_DENSE, S.C_FMT[f]) <= 0.5, f
    rows, _ = S.split_rows(S.dense_fused_splits(n, F, w.shape[1]), F)
    x64, w64, b64 = x.astype(np.float64), w.astype(np.float64), b.astype(np.float64)
    # a row at a split boundary (last of one split or first of the next) that every batch row reads as non-zero
    f = next(f for k in range(1, F // rows + 1) for f in (k * rows - 1, k * rows) if np.abs(x[:, f]).min() > 0.5)
    keep = np.ones(F, bool)
    keep[f] = False
    wrong = {
        "dropped K row": np.maximum(x64[:, keep] @ w64[keep] + b64, 0),
        "bias twice": np.maximum(x64 @ w64 + 2 * b64, 0),
        "4-unit group permuted": ref.reshape(n, -1, 4)[:, :, [1, 0, 3, 2]].reshape(n, -1),
        "ReLU before bias": np.maximum(x64 @ w64, 0) + b64,
    }
    for name, y in wrong.items():
        for f in FMT_NAMES:
            assert S.bar_used(y, ref, mag, S.A_DENSE, S.C_FMT[f]) > 1, (name, f)


# ------------------------------------------------------------------------------------------------ gap
@pytest.mark.parametrize("shape", [(3, 7, 7, 2048), (1, 56, 56, 36), (2, 2, 3, 100)])
def test_gap_bar_passes_fp32_and_rejects_wrong_arithmetic(shape):
    n, h, w, c = shape
    hw = h * w
    x = np.random.default_rng(6).standard_normal(shape, dtype=np.float32).reshape(n, hw, c)
    ref, mag = S.gap_ref(x.reshape(shape))
    # gap_kernel's order: threadIdx.y row r sums pixels r, r + 8, ...; the 8 rows are summed in order, then / hw
    rows = [np.zeros((n, c), np.float32) for _ in range(8)]
    for p in range(hw):
        rows[p % 8] = rows[p % 8] + x[:, p]
    t = np.zeros((n, c), np.float32)
    for r in rows:
        t = t + r
    y32 = t / np.float32(hw)
    for f in FMT_NAMES:
        assert S.bar_used(y32, ref, mag, S.A_GAP, S.C_FMT[f]) <= 0.5, f
    x64 = x.astype(np.float64)
    wrong = {"dropped pixel": x64[:, 1:].sum(axis=1) / hw, "divided by hw - 1": x64.sum(axis=1) / (hw - 1)}
    for name, y in wrong.items():
        for f in FMT_NAMES:
            # a scaling by hw / (hw - 1) below the output format's rounding (bf16 at hw = 3136) is beyond any bar
            if name == "divided by hw - 1" and 1 / (hw - 1) < 4 * S.C_FMT[f]:
                continue
            assert S.bar_used(y, ref, mag, S.A_GAP, S.C_FMT[f]) > 1, (name, f)


# ------------------------------------------------------------------------------------------------ softmax
def _softmax_fp32(x):
    """fp32 softmax in softmax_kernel's order: max, 256 strided partial sums of exp(x - m) then summed, times 1/sum."""
    x = np.asarray(x, np.float32)
    m = x.max(axis=-1, keepdims=True)
    e = np.exp(x - m)
    c = x.shape[-1]
    pad = np.zeros(x.shape[:-1] + ((-c) % 256,), np.float32)
    parts = np.concatenate([e, pad], axis=-1).reshape(x.shape[0], -1, 256).sum(axis=1, dtype=np.float32)
    s = parts.sum(axis=-1, keepdims=True, dtype=np.float32)
    return e * (np.float32(1) / s)


@pytest.mark.parametrize("c", [7, 1000, 4097])
def test_softmax_bar_passes_fp32_and_rejects_wrong_arithmetic(c):
    x = S.softmax_rows(c)
    assert S.softmax_bar_used(_softmax_fp32(x), x) <= 0.5
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.exp(x[2:3])                                                  # no max subtraction, fp32, +-1e4 row
        assert S.softmax_bar_used(e / e.sum(axis=-1, keepdims=True), x[2:3]) > 1
    x64 = x[0].astype(np.float64)                                           # the scale-1 row
    e = np.exp(x64 - x64.max())
    j = e.argsort()[c // 2]                                                 # a term of median size left out of the sum
    assert S.softmax_bar_used(e / (e.sum() - e[j]), x[:1]) > 1
