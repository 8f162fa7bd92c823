"""Progressive files at the edges of the device decode, on the host (no GPU).

The crafted valid files of tests/jpeg_progressive_edges.py (EOB runs of 32 767 blocks, past their interval and past
their scan, at subsequence edges; AC refinement edges) decode to the coefficients their writer knows and equal Pillow.
The restatement of the device decode (tests/jpeg_progressive_sync.py) equals the sequential decoder, counters included,
at 8 to 8192-bit subsequences.  The worst cases of the first-scan synchronisation take one round per subsequence of an
interval, as their closed form says; the saturating files' block-offset sums pass 2^31, and without the saturation the
restatement would place blocks outside the scan."""
import io
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import jpeg  # noqa: E402
import jpeg_craft_progressive as P  # noqa: E402
import jpeg_progressive_edges as E  # noqa: E402
import jpeg_progressive_sync as S  # noqa: E402
from jpeg_craft import idct_raw  # noqa: E402

SBITS = int(re.search(r"#define DEFER_JPEG_SUBSEQ_BITS (\d+)", (ROOT / "include" / "defer_b200.h").read_text()).group(1))
VALID = E.eob_cases(SBITS) + E.refine_cases()


@pytest.mark.parametrize("case", VALID, ids=[c[0] for c in VALID])
def test_valid_edges_decode_as_written_and_as_pillow(case):
    name, data, want = case
    st = jpeg.decode_stages(data)
    assert st["progress"]["scans"] == len(st["info"].scans) and st["progress"]["cutoff"] == len(st["coef"])
    assert np.array_equal(st["coef"], want), name
    raw = idct_raw(st["coef"].astype(np.int64), np.ones(64, np.int64))
    if np.abs(raw).max() > 512:      # beyond the IDCT range: against the C path in test_jpeg_idct_range_host.py
        assert name.startswith("al 13")
        return
    Image = pytest.importorskip("PIL.Image")
    assert np.array_equal(st["rgb"], np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))), name


@pytest.mark.parametrize("sbits", [8, 64, 1024, SBITS])
def test_sync_restatement_equals_sequential_on_edges(sbits):
    for name, d, _ in VALID:
        if sbits < 1024 and len(d) > 10000:
            continue
        coef, st = S.sync_progressive(d, sbits)
        want, pr = jpeg.progressive_decode(d)
        assert np.array_equal(coef, want), (name, sbits)
        assert [st[0], st[1], st[4], st[5]] == [pr["T"], pr["R"], pr["cutoff"], pr["scans"]], (name, sbits)


def test_sync_restatement_equals_sequential_on_corrupt_files():
    """One corrupt file per scan kind and damage, at the device's subsequence size."""
    seen = set()
    for name, d, s, kd, dmg, iv, at, q in E.corrupt_cases(SBITS):
        if (kd, dmg) in seen:
            continue
        seen.add((kd, dmg))
        coef, st = S.sync_progressive(d, SBITS)
        want, pr = jpeg.progressive_decode(d)
        assert np.array_equal(coef, want), name
        assert [st[0], st[1], st[4], st[5]] == [pr["T"], pr["R"], pr["cutoff"], pr["scans"]], name


def _first_past_subsequence_1(cases):
    """For each first-scan kind, an invalid code past the first subsequence of its interval, which fails the decode at
    its block."""
    got = {}
    for name, d, s, kd, dmg, iv, at, q in cases:
        if kd in E.FIRST and dmg.startswith("invalid") and at > SBITS and kd not in got:
            pr = jpeg.progressive_decode(d)[1]
            assert (pr["scans"], pr["cutoff"]) == (s, q), name
            got[kd] = name
    return got


def test_corrupt_cases_cover_every_scan_kind_and_damage():
    cases = E.corrupt_cases(SBITS)
    got = {(kd, dmg) for _, _, _, kd, dmg, *_ in cases}
    codes = ["invalid code at the first block", "invalid code at a block straddling a subsequence edge",
             "invalid code at the last block"]
    rst = ["an RST dropped", "an RST duplicated", "RSTs renumbered", "surplus RSTs", "RSTs missing after the first",
           "fill bytes before the markers"]
    for kd in E.KINDS:
        want = ["data cut inside the scan", "empty scan"] + rst + (codes if kd != "dc refine" else [])
        want += ["run past Se", "ZRL past Se"] if kd.startswith("ac") else []
        want += ["size-2 refinement symbol"] if kd == "ac refine" else []
        assert {(kd, w) for w in want} <= got, (kd, set(want) - {d for k, d in got if k == kd})
    assert set(_first_past_subsequence_1(cases)) == set(E.FIRST)
    for name, d, s, kd, dmg, iv, at, q in cases:         # a straddling block starts before an edge and ends after it
        if dmg == "invalid code at a block straddling a subsequence edge":
            assert at % SBITS, name
    ivs = {iv for _, _, _, kd, dmg, iv, *_ in cases if kd == "ac refine" and "RST" not in dmg and iv >= 0}
    assert {0, max(ivs)} <= ivs and any(0 < i < max(ivs) for i in ivs), ivs  # first, middle and last interval


def test_large_corrupt_cases_reach_past_subsequence_1():
    cases = E.corrupt_cases(SBITS, large=True)
    assert jpeg.parse(cases[0][1]).h == 1080
    assert set(_first_past_subsequence_1(cases)) == {"dc first", "ac first"}
    assert {c[3] for c in cases} == {"dc first", "ac first", "ac refine"}


@pytest.mark.parametrize("sbits", [8, 64, 1024, SBITS])
@pytest.mark.parametrize("args", [(64, 64, "gray", "ac", 0), (64, 64, "gray", "ac", 3), (48, 80, "gray", "ac", 7),
                                  (96, 128, "420", "dc", 0), (96, 128, "420", "dc", 5), (64, 200, "gray", "dc", 0)])
def test_worst_case_closed_form_equals_restatement(args, sbits):
    d, want, unit = P.worst_first(*args)
    if sbits == 8 and len(d) > 2000:
        return
    assert np.array_equal(jpeg.decode_stages(d)["coef"], want)
    coef, st = S.sync_progressive(d, sbits)
    assert np.array_equal(coef, want)
    assert np.array_equal(st, P.closed_form_counters(d, sbits, unit)), (st.tolist(), sbits)


def test_saturation_keeps_the_restatement_exact(monkeypatch):
    """A 2048x2048 file whose 80 000 subsequences of 48 bits each own 27 316 blocks: their block-offset sum passes 2^31.
    With the device's saturating sum the restatement equals the sequential decode, and its counters the closed form;
    with an int32 sum that wraps, later subsequences start at negative blocks and write outside the scan."""
    d, want, unit = P.saturating(2048, 2048, 80000, 48, coded=True)
    assert 80000 * 27316 > 2 ** 31
    assert np.array_equal(jpeg.decode_stages(d)["coef"], want)
    coef, st = S.sync_progressive(d, 48)
    assert np.array_equal(coef, want)
    assert np.array_equal(st, P.closed_form_counters(d, 48, unit)), st.tolist()
    monkeypatch.setattr(S, "_sat", lambda v: ((v + 2 ** 31) % 2 ** 32) - 2 ** 31)
    with pytest.raises(IndexError):
        S.sync_progressive(d, 48)


def test_saturating_sum_passes_2_31():
    """Every subsequence of the saturating file's AC scan owns more blocks than the image has (checked on its first,
    a middle and its last subsequence), so the unsaturated block-offset sum is subsequences * blocks > 2^31."""
    h, w, nsubs = E.SAT
    d, want, unit = P.saturating(h, w, nsubs, SBITS)
    info = jpeg.parse(d)
    g = jpeg.geometry(info.h, info.w, 1, 1, 1)
    sc = info.scans[1]
    comp, rst = jpeg.unstuff(d[sc.offset:sc.offset + sc.length])
    assert len(comp) * 8 == nsubs * SBITS and not rst
    r = jpeg.BitReader(comp, 0, len(comp))
    for t in (0, nsubs // 2, nsubs - 1):
        *_, owned = S._run(r, t * SBITS, 0, sc.ss, (t + 1) * SBITS, sc, info.tables, 1, [0], g.blocks)
        assert owned == g.blocks
    assert nsubs * g.blocks > 2 ** 31
    st = P.closed_form_counters(d, SBITS, unit)
    assert st.tolist() == [st[0], 0, -(-g.blocks // SBITS) + nsubs, 2, g.blocks, 2]
    assert len(d) <= h * w * 3
    pr = jpeg.progressive_decode(d, info)[1]
    assert [pr["T"], pr["R"], pr["cutoff"], pr["scans"]] == [st[0], st[1], st[4], st[5]]


def test_split_assemble_round_trip():
    for name, d, _ in VALID[1:4]:
        parts, tail = P.split(d)
        assert P.assemble(parts, tail) == d, name
