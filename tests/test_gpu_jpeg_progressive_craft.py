"""The GPU progressive decode on crafted files: worst-case synchronisation, EOB runs at their limits, AC refinement
edges and corrupt files in every scan kind, at full size.

Each file's coefficients, planes and RGB equal ``jpeg.decode_stages`` (or, for the largest files, what the writer put
in), and all six ``stats`` counters (unstuffed bytes, RST markers, subsequences, rounds, failing block, scans decoded
whole) equal the restatement of tests/jpeg_progressive_sync.py or the closed form the host tests check against it
(``jpeg_craft_progressive.closed_form_counters``).  The files come from tests/jpeg_progressive_edges.py.  No Pillow."""
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
import jpeg_craft as jc  # noqa: E402
import jpeg_craft_progressive as P  # noqa: E402
import jpeg_progressive_edges as E  # noqa: E402
from test_gpu_jpeg import _bits, _decode_dev  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
SBITS = int(re.search(r"#define DEFER_JPEG_SUBSEQ_BITS (\d+)", (ROOT / "include" / "defer_b200.h").read_text()).group(1))
Q1 = [np.ones(64, np.int32)]


def _check(ws, coef_off, plane_off, y, want, stats, name):
    h, w = want["rgb"].shape[:2]
    n = want["coef"].shape[0]
    assert np.array_equal(ws[coef_off:coef_off + n * 128].view(np.int16).reshape(n, 64), want["coef"]), name
    off = plane_off
    for c, p in enumerate(want["planes"]):
        assert np.array_equal(ws[off:off + p.size].reshape(p.shape), p), (name, c)
        off += p.size
    assert np.array_equal(y[:h * w * 3].reshape(h, w, 3), want["rgb"]), name
    got = ws[:24].view(np.int32)
    assert np.array_equal(got, stats), (name, got.tolist(), list(stats))
    return got


def _host(d):
    """decode_stages and the restatement's counters of ``d``."""
    return E.host_expect(d, SBITS)


def _written(d, coef, sub):
    info = jpeg.parse(d)
    return jc.expected(coef, info.h, info.w, sub, Q1)


# ------------------------------------------------------------------------------------------------ worst-case sync
WORST = [(384, 512, "gray", "ac", 0), (384, 512, "gray", "ac", 5), (384, 512, "gray", "ac", 40),
         (256, 384, "420", "dc", 0)]


def test_worst_case_sync():
    """No restart interval, an interval shorter than a subsequence (5 blocks), one of a few subsequences (40 blocks),
    and an interleaved 4:2:0 DC first scan: rounds equal the subsequences of the longest interval."""
    files, wants, stats = [], [], []
    for h, w, sub, kind, ri in WORST:
        d, coef, unit = P.worst_first(h, w, sub, kind, ri)
        files.append(d)
        wants.append(_written(d, coef, sub))
        stats.append(P.closed_form_counters(d, SBITS, unit))
    ws, coef_off, plane_off, y = _decode_dev(files, 480, 640)
    for i, case in enumerate(WORST):
        got = _check(ws[i], coef_off, plane_off, y[i], wants[i], stats[i], case)
        print(f"{case}: {got[3]} rounds for {got[2]} subsequences")
    assert max(int(s[3]) for s in stats) >= 400


def test_worst_case_sync_at_the_largest_slot():
    """The AC first worst case at 1080x1920: 1071-bit blocks, one round per subsequence."""
    H, W = 1080, 1920
    d, coef, unit = P.worst_first(H, W, "gray", "ac")
    stats = P.closed_form_counters(d, SBITS, unit)
    (ws, coef_off, plane_off, y), ms = _decode_dev([d], H, W, timed=True)
    got = _check(ws[0], coef_off, plane_off, y[0], _written(d, coef, "gray"), stats, "1080x1920")
    assert got[3] == got[2] - 4 + 1                          # the DC scan: 4 subsequences, 1 round
    print(f"1080x1920 AC first worst case: {got[3]} rounds for {got[2]} subsequences, {ms:.1f} ms")


# ------------------------------------------------------------------------------------------------ valid edges
def test_eob_and_refinement_edges():
    cases = E.eob_cases(SBITS) + E.refine_cases()
    ws, coef_off, plane_off, y = _decode_dev([d for _, d, _ in cases], 1456, 1456)
    for i, (name, d, coef) in enumerate(cases):
        want, stats = _host(d)
        assert np.array_equal(want["coef"], coef), name
        got = _check(ws[i], coef_off, plane_off, y[i], want, stats, name)
        print(f"{name}: {got.tolist()}")


def test_saturating_block_sum():
    """Every subsequence owns more blocks than the image has; the block-offset sum passes 2^31 (host test) and the
    device's saturating sum keeps the decode exact."""
    h, w, nsubs = E.SAT
    d, coef, unit = P.saturating(h, w, nsubs, SBITS)
    stats = P.closed_form_counters(d, SBITS, unit)
    ws, coef_off, plane_off, y = _decode_dev([d], h, w)
    got = _check(ws[0], coef_off, plane_off, y[0], _written(d, coef, "gray"), stats, "saturating")
    print(f"saturating {h}x{w}: {got.tolist()}")


# ------------------------------------------------------------------------------------------------ corrupt files
def _corrupt(cases, H, W):
    """Decode ``cases`` of ``corrupt_cases`` and check them; returns what their failures reached: (kind, damage),
    (kind, "past subsequence 1") for first scans, and ("refine interval", failing interval)."""
    reach = set()
    wants = E.host_expect_all([c[1] for c in cases], SBITS)
    for lo in range(0, len(cases), 40):
        part = cases[lo:lo + 40]
        ws, coef_off, plane_off, y = _decode_dev([c[1] for c in part], H, W)
        for i, (name, d, s, kd, dmg, iv, at, q) in enumerate(part):
            want, stats = wants[lo + i]
            got = _check(ws[i], coef_off, plane_off, y[i], want, stats, name)
            info = jpeg.parse(d)
            sc = info.scans[s]
            if got[5] == s and got[4] < len(jpeg.scan_blocks(info, sc)[0]):
                reach.add((kd, dmg))
                if kd in E.FIRST and at > SBITS and got[4] == q:
                    reach.add((kd, "past subsequence 1"))
                if kd == "ac refine" and sc.restart:
                    reach.add(("refine interval", int(got[4]) // sc.restart))
    return reach


def test_corrupt_every_scan_kind():
    cases = E.corrupt_cases(SBITS)
    reach = _corrupt(cases, 480, 640)
    print(f"{len(cases)} corrupt files equal to the host; failures reached: {sorted(map(str, reach))}")
    for kd in E.FIRST + ("ac refine",):
        assert any(r[0] == kd for r in reach), kd
    for kd in E.FIRST:
        assert (kd, "past subsequence 1") in reach, kd
    ivs = {r[1] for r in reach if r[0] == "refine interval"}
    assert {0, max(ivs)} <= ivs and any(0 < i < max(ivs) for i in ivs), ivs


def test_corrupt_at_the_largest_slot():
    """A 1080x1920 grayscale file with invalid codes in its DC first, AC first and AC refinement scans."""
    cases = E.corrupt_cases(SBITS, large=True)
    reach = _corrupt(cases, 1080, 1920)
    print(f"{len(cases)} corrupt 1080x1920 files equal to the host; failures reached: {sorted(map(str, reach))}")
    assert {("dc first", "past subsequence 1"), ("ac first", "past subsequence 1")} <= reach
    assert any(r[0] == "ac refine" for r in reach)


# ------------------------------------------------------------------------------------------------ stage level
def test_stage_crafted_and_corrupt_in_reused_slots(monkeypatch):
    """The stage copies only a file's bytes into its slot: files after larger ones must not read their leftovers."""
    from test_gpu_conv_paths import _knobs
    from test_gpu_jpeg_progressive import _stem
    from defer_b200.node import StageRunner
    _knobs(monkeypatch)
    m = _stem(seed=5)
    kw = dict(device=0, dtype="float32", max_batch=4, depth=1, preprocess="caffe", max_image_size=(480, 640),
              interpolation="bilinear")
    r = StageRunner.from_model(m, decode="jpeg", **kw)
    r0 = StageRunner.from_model(m, **kw)
    try:
        base = [b[1] for b in E.bases()]
        corrupt = {c[4]: c[1] for c in E.corrupt_cases(SBITS) if c[3] == "ac first"}
        valid = {n: d for n, d, _ in E.eob_cases(SBITS)[1:] + E.refine_cases()}
        groups = [base[:3] + [base[2]],
                  [valid["eob run past the scan"], corrupt["data cut inside the scan"], valid["zrl ending at se+1"],
                   corrupt["empty scan"]],
                  [corrupt["invalid code at the last block"], valid["eob runs past their interval"],
                   corrupt["ZRL past Se"], valid["refine ZRLs over history"]]]
        for files in groups:
            y = r.predict_jpegs(files)
            y0 = r0.predict_frames([jpeg.decode_jpeg(d)[None] for d in files])
            assert np.array_equal(_bits(y), _bits(y0))
    finally:
        r.close()
        r0.close()
