"""The progressive decode never reads past the block prefix its header declares, nor writes outside the sample's
workspace, whatever the scan table holds (no GPU).

csrc/jpeg.cu clamps each scan entry (``pscan``) and maps scan-order blocks to stream order (``scan_block``).  This
restates both in Python on top of tests/test_jpeg_bounds_host.py's ``geom`` and ``jpeg_ws`` and fuzzes scan entries and
the scan and table counts: every table the kernel loads lies inside the declared prefix, every entropy extent inside
the slot, every scan's intervals inside the interval arrays, and every block it touches inside the coefficients."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import jpeg  # noqa: E402
from test_jpeg_bounds_host import BIG, geom, jpeg_ws  # noqa: E402


def _clamp(v, lo, hi):
    return min(max(v, lo), hi)


def pscan(e, g, ntab, slot):
    """jpeg.cu's pscan: the clamped scan of entry ``e``."""
    p = {"ss": _clamp(e[4], 0, 63)}
    p["se"] = 0 if p["ss"] == 0 else _clamp(e[5], p["ss"], 63)
    inter = e[0] > 1 and g["ncomp"] == 3 and p["ss"] == 0
    p["comp"] = 0 if inter else _clamp(e[1], 0, g["ncomp"] - 1)
    p["ri"] = _clamp(e[8], 0, 65535)
    p["off"] = _clamp(e[9], 0, slot)
    p["len"] = _clamp(e[10], 0, slot - p["off"])
    p["dct"] = [_clamp(e[11 + c], 0, max(ntab - 1, 0)) for c in range(3)]
    p["act"] = _clamp(e[14], 0, max(ntab - 1, 0))
    p["hc"] = g["hs"] if p["comp"] == 0 else 1
    p["vc"] = g["vs"] if p["comp"] == 0 else 1
    if inter or g["ncomp"] == 1:
        p["per"], p["units"], p["cw"] = (g["bpm"] if inter else 1), g["mcus"], g["mcux"]
    else:
        p["per"] = 1
        p["cw"] = (g["w"] * p["hc"] + 8 * g["hs"] - 1) // (8 * g["hs"])
        p["units"] = p["cw"] * ((g["h"] * p["vc"] + 8 * g["vs"] - 1) // (8 * g["vs"]))
    p["nq"] = p["units"] * p["per"]
    p["nseg"] = -(-p["units"] // p["ri"]) if p["ri"] else 1
    return p


def scan_block(g, p, q):
    """jpeg.cu's scan_block, vectorised over q."""
    if p["per"] > 1 or g["ncomp"] == 1:
        return q
    bx, by = q % p["cw"], q // p["cw"]
    if p["comp"] == 0:
        return ((by // p["vc"]) * g["mcux"] + bx // p["hc"]) * g["bpm"] + (by % p["vc"]) * p["hc"] + bx % p["hc"]
    return (by * g["mcux"] + bx) * g["bpm"] + g["nb0"] + p["comp"] - 1


def check(blk, entries, H, W):
    L = jpeg_ws(H, W)
    g = geom(blk, H, W, L["slot"])
    nsc, ntab = _clamp(blk[10], 0, jpeg.MAX_SCANS), _clamp(blk[11], 0, jpeg.MAX_TABLES)
    prefix = jpeg.POOL_OFF + ntab * jpeg.HUFF_INTS
    for e in entries[:nsc]:
        p = pscan(e, g, ntab, L["slot"])
        if p["ss"] > 0 or e[6] == 0:                 # a scan that loads tables: the kernel stops if there are none
            if ntab == 0:
                continue
            for t in p["dct"] + [p["act"]]:
                assert jpeg.POOL_OFF + (t + 1) * jpeg.HUFF_INTS <= prefix
        assert 0 <= p["off"] and p["off"] + p["len"] <= L["slot"] and p["len"] + 16 <= L["comp_bytes"]
        assert p["units"] <= L["mcu_cap"] and (p["nseg"] + 1) * 4 <= L["seg_start_bytes"]
        assert -(-p["len"] * 8 // 8192) + p["nseg"] - 1 <= L["subs_cap"]
        b = scan_block(g, p, np.arange(p["nq"]))
        assert p["nq"] <= g["blocks"] and (b >= 0).all() and (b < g["blocks"]).all()
        assert len(np.unique(b)) == p["nq"]          # a scan touches each block once
    assert jpeg.SCAN_OFF + nsc * jpeg.SCAN_INTS <= prefix


@pytest.mark.parametrize("bound", [(1, 1), (15, 17), (61, 75), (480, 640)])
def test_fuzzed_scans_stay_inside(bound):
    H, W = bound
    rng = np.random.default_rng(H + W)
    slot = H * W * 3
    picks = [lambda: int(rng.choice(BIG)), lambda: int(rng.integers(-(1 << 31), 1 << 31)),
             lambda: int(rng.integers(-3, 70)), lambda: int(rng.integers(0, slot + 2))]
    for _ in range(200):
        blk = [picks[int(rng.integers(len(picks)))]() for _ in range(12)]
        if rng.random() < 0.7:
            blk[:5] = [int(rng.integers(H - 2, H + 3)), int(rng.integers(W - 2, W + 3)), 3, 2, int(rng.integers(0, 3))]
            blk[10], blk[11] = int(rng.integers(0, 40)), int(rng.integers(-2, 40))
        entries = [[picks[int(rng.integers(len(picks)))]() for _ in range(jpeg.SCAN_INTS)] for _ in range(8)]
        check(blk, entries, H, W)


def test_fixture_scans_match_parser():
    """On real files the restated clamps change nothing, and the scan order is jpeg.scan_blocks'."""
    from jpeg_progressive_check import fixture, fixture_names
    for nm in fixture_names():
        info = jpeg.parse(fixture(nm))
        b = jpeg.pack_block(info)
        H, W = max(info.h, 64), max(info.w, 80)          # a bound whose slot holds the file
        g = geom(list(b[:12]), H, W, H * W * 3)
        for s, sc in enumerate(info.scans):
            e = list(b[jpeg.SCAN_OFF + s * jpeg.SCAN_INTS:jpeg.SCAN_OFF + (s + 1) * jpeg.SCAN_INTS])
            p = pscan(e, g, len(info.tables), H * W * 3)
            want, per = jpeg.scan_blocks(info, sc)
            assert p["per"] == per and np.array_equal(scan_block(g, p, np.arange(p["nq"])), want), (nm, s)
            assert (p["ss"], p["se"], p["off"], p["len"]) == (sc.ss, sc.se, sc.offset, sc.length)
