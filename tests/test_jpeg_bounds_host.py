"""The JPEG kernels never access outside a sample's slot or workspace, whatever its block header holds (no GPU).

csrc/jpeg.cu derives each sample's geometry on the device from its block header (``geom``), clamped into the bound
(H, W), and the workspace layout from the bound alone (``jpeg_ws``).  This restates both in Python, checks the layout
against the library's ``defer_k_jpeg_workspace``, and fuzzes headers (sizes, component count, sampling, restart
interval, entropy offset and length, with negative and huge values) to check that every index the three kernels derive
stays inside the slot, the workspace fields and the ``subs_cap`` / ``mcu_cap`` capacities, and that bit positions fit
in an int.  The kernels are never launched on such headers: the check is of the arithmetic."""
import ctypes as C
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from defer_b200 import _cabi as A  # noqa: E402

SBITS = int(re.search(r"#define DEFER_JPEG_SUBSEQ_BITS (\d+)", (ROOT / "include" / "defer_b200.h").read_text()).group(1))
SUB_FIELDS = 9
INT_MAX = (1 << 31) - 1


def _al(v):
    return (v + 255) // 256 * 256


def jpeg_ws(H, W):
    """jpeg.cu's jpeg_ws: byte offsets of the workspace fields of one sample, and the capacities."""
    hp, wp = (H + 15) // 16 * 16, (W + 15) // 16 * 16
    L = {"slot": H * W * 3}
    L["mcu_cap"] = (hp // 8) * (wp // 8)
    L["blocks_cap"] = 3 * L["mcu_cap"]
    L["subs_cap"] = (L["slot"] * 8 + SBITS - 1) // SBITS + L["mcu_cap"]
    sizes = [("stats", 64), ("coef", L["blocks_cap"] * 128), ("planes", L["blocks_cap"] * 64), ("comp", L["slot"] + 16),
             ("seg_start", (L["mcu_cap"] + 2) * 4), ("seg_total", (L["mcu_cap"] + 1) * 4),
             ("sub_base", (L["mcu_cap"] + 1) * 4), ("sub", L["subs_cap"] * SUB_FIELDS * 4)]
    o = 0
    for name, n in sizes:
        L[name], L[name + "_bytes"] = o, n
        o += _al(n)
    L["stride"] = o
    return L


def geom(blk, H, W, slot):
    """jpeg.cu's geom: the clamped geometry of one block header (int32 values)."""
    g = {"h": min(max(blk[0], 1), H), "w": min(max(blk[1], 1), W), "ncomp": 3 if blk[2] == 3 else 1}
    g["hs"] = min(max(blk[3], 1), 2) if g["ncomp"] == 3 else 1
    g["vs"] = min(max(blk[4], 1), 2) if g["ncomp"] == 3 else 1
    if g["vs"] == 2:
        g["hs"] = 2
    g["ri"] = min(max(blk[5], 0), 65535)
    g["off"] = min(max(blk[6], 0), slot)
    g["len"] = min(max(blk[7], 0), slot - g["off"])
    g["mcux"] = (g["w"] + 8 * g["hs"] - 1) // (8 * g["hs"])
    g["mcuy"] = (g["h"] + 8 * g["vs"] - 1) // (8 * g["vs"])
    g["mcus"] = g["mcux"] * g["mcuy"]
    g["nb0"] = g["hs"] * g["vs"]
    g["bpm"] = g["nb0"] + 2 if g["ncomp"] == 3 else 1
    g["blocks"] = g["mcus"] * g["bpm"]
    g["nseg"] = -(-g["mcus"] // g["ri"]) if g["ri"] else 1
    g["bw"] = [g["mcux"] * (g["hs"] if c == 0 else 1) if c < g["ncomp"] else 0 for c in range(3)]
    g["bh"] = [g["mcuy"] * (g["vs"] if c == 0 else 1) if c < g["ncomp"] else 0 for c in range(3)]
    g["poff"] = list(np.cumsum([0] + [g["bw"][c] * g["bh"][c] * 64 for c in range(3)])[:3])
    return g


def check(blk, H, W):
    """Every index the entropy, IDCT and colour kernels derive from ``blk`` at the bound (H, W), against the slot,
    the workspace fields and the capacities."""
    L = jpeg_ws(H, W)
    g = geom(blk, H, W, L["slot"])
    # entropy kernel: the file bytes it reads, the compacted bytes it writes (at most len), the interval arrays
    assert 0 <= g["off"] and g["off"] + g["len"] <= L["slot"]
    assert g["len"] + 16 <= L["comp_bytes"]
    assert 1 <= g["nseg"] and (g["nseg"] + 1) * 4 <= L["seg_start_bytes"] and g["nseg"] * 4 <= L["seg_total_bytes"]
    assert g["nseg"] * 4 <= L["sub_base_bytes"]
    # subsequences: the most the unstuffed data can need, so the clamp to subs_cap never cuts a real one
    assert -(-g["len"] * 8 // SBITS) + g["nseg"] - 1 <= L["subs_cap"]
    assert L["subs_cap"] * SUB_FIELDS * 4 <= L["sub_bytes"]
    # bit positions, and a subsequence's end, stay ints
    assert g["len"] * 8 + SBITS <= INT_MAX
    # coefficients and planes
    assert g["blocks"] * 128 <= L["coef_bytes"]
    assert g["poff"][2] + g["bw"][2] * g["bh"][2] * 64 <= L["planes_bytes"]
    b = np.arange(g["blocks"])
    m, j = b // g["bpm"], b % g["bpm"]
    c = np.where(j < g["nb0"], 0, j - g["nb0"] + 1)
    mx, my = m % g["mcux"], m // g["mcux"]
    bx = np.where(c == 0, mx * g["hs"] + j % g["hs"], mx)
    by = np.where(c == 0, my * g["vs"] + j // g["hs"], my)
    bw, bh = np.array(g["bw"])[c], np.array(g["bh"])[c]
    assert (bx < bw).all() and (by < bh).all()                    # each IDCT block inside its component's plane
    # colour kernel: the luma sample, the chroma rows / columns upsample() reads, the output pixel
    h, w = g["h"], g["w"]
    assert h <= g["bh"][0] * 8 and w <= g["bw"][0] * 8 and h * w * 3 <= L["slot"]
    if g["ncomp"] == 3:
        rows = h if g["vs"] == 1 else (h + 1) >> 1                  # rows read: y (vs 1), r0 / r1 <= dh - 1 (vs 2)
        cols = w if g["hs"] == 1 else (w + 1) >> 1                  # columns read: x (hs 1), i / in_ <= dw - 1
        assert rows <= g["bh"][1] * 8 and cols <= g["bw"][1] * 8
    return g


BIG = [0, 1, 2, 3, 7, 8, 9, 15, 16, 17, 255, 65535, 65536, (1 << 31) - 1, -1, -(1 << 31), -7]


def _widest(H):
    """The widest bound of height H that the library takes: H * W * 24 + DEFER_JPEG_SUBSEQ_BITS < 2^31."""
    return ((1 << 31) - SBITS - 1) // (24 * H)


def _accepts(H, W):
    return A.load().defer_k_jpeg_workspace(H, W, 1, None, None, None, None) == A.OK


def test_largest_bounds():
    """Beyond the widest bound, the end of the last subsequence (slot * 8 + DEFER_JPEG_SUBSEQ_BITS bits) would not fit
    in an int: such a bound is refused."""
    for H in (8, 9459, 1080):
        assert _accepts(H, _widest(H)) and not _accepts(H, _widest(H) + 1)
    assert not _accepts(8, 11184810)              # H * W * 24 < 2^31, but the last subsequence's end is not


@pytest.mark.parametrize("bound", [(1, 1), (8, 8), (15, 17), (223, 225), (480, 640), (1080, 1920), (8, _widest(8)),
                                   (9459, _widest(9459))])
def test_fuzzed_headers_stay_inside(bound):
    H, W = bound
    assert _accepts(H, W)
    rng = np.random.default_rng(H * 7 + W)
    slot = H * W * 3
    picks = [lambda: int(rng.choice(BIG)), lambda: int(rng.integers(-(1 << 31), 1 << 31)),
             lambda: int(rng.integers(-3, 40)), lambda: int(rng.integers(0, slot + 2))]
    n = 300 if H * W <= 1 << 20 else 30                            # the block walk is per block
    for _ in range(n):
        blk = [picks[int(rng.integers(len(picks)))]() for _ in range(10)]
        if rng.random() < 0.5:
            blk[:5] = [int(rng.integers(H - 2, H + 3)), int(rng.integers(W - 2, W + 3)), 3, 2, int(rng.integers(0, 3))]
        check(blk, H, W)
    for ncomp, hs, vs in ((1, 1, 1), (3, 1, 1), (3, 2, 1), (3, 2, 2), (3, 1, 2)):   # the largest image of each kind
        g = check([H, W, ncomp, hs, vs, 1, 0, slot, 0, 0], H, W)
        assert g["h"] == H and g["w"] == W


def test_layout_matches_library():
    lib = A.load()
    for H, W in ((1, 1), (15, 17), (223, 225), (480, 640), (1080, 1920), (8, _widest(8))):
        total, stride, coef, planes = (C.c_uint64() for _ in range(4))
        A.check(lib.defer_k_jpeg_workspace(H, W, 3, C.byref(total), C.byref(stride), C.byref(coef), C.byref(planes)))
        L = jpeg_ws(H, W)
        assert (stride.value, coef.value, planes.value, total.value) == (L["stride"], L["coef"], L["planes"],
                                                                          3 * L["stride"])
