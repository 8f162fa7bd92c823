"""The JPEG decode beyond the IDCT range, on the host, against libjpeg-turbo's C path (no GPU).

Past +-512 around 128 ``defer_b200.jpeg`` promises the pixels of libjpeg's C code: ``jidctint.c`` wraps each IDCT output
to 10 bits before the clamp, and coefficients are int16 as ``jdhuff.c`` / ``jdphuff.c`` store them.  The reference here
is Pillow's own libjpeg-turbo 3.1 with ``JSIMD_FORCENONE=1`` (tests/libjpeg_c.py), which runs exactly that C code.

- Every file of tests/jpeg_idct_range.py (wrap points in every component and subsampling at odd sizes, one AC
  coefficient per block, all coefficients at their largest, random large coefficients with and without restart
  intervals, a DC predictor past int16, progressive files whose first scans wrap int16 and whose refinements apply on
  top, a 1080x1920 grid) decodes to the coefficients its writer records and to the C path's pixels.
- The corpus does leave the range: the raw IDCT passes +-512 in every file but the controls, the wrap points cover
  every edge of the wrap and the clamp on both signs in every component, and SIMD Pillow, which saturates instead of
  wrapping, decodes most files differently.
- On every committed fixture the C path, SIMD Pillow and ``decode_jpeg`` agree: a Pillow built without SIMD gives the
  same pixels in range.
"""
import io
import sys
from collections import defaultdict
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import jpeg  # noqa: E402
import jpeg_idct_range as R  # noqa: E402
from libjpeg_c import SENTINEL_PIXEL, decode_c, sentinel  # noqa: E402

pytestmark = pytest.mark.timeout(600)
FIXTURES = sorted((ROOT / "tests" / "golden").glob("jpeg*/*.jpg"))


def _simd(data):
    Image = pytest.importorskip("PIL.Image")
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


@pytest.fixture(scope="module")
def corpus():
    return R.corpus(grid=True)


@pytest.fixture(scope="module")
def c_path(corpus):
    return decode_c([c.data for c in corpus])


def test_sentinel_takes_the_c_path():
    """The sentinel (x = 1100) gives idct_range_limit[1100 & 1023] = 204 on the C path; SIMD Pillow saturates."""
    got = decode_c([])                  # checks the sentinel itself, fails if the C path was not taken
    assert got == []
    c = decode_c([sentinel()])[0]
    simd = _simd(sentinel())
    assert (c == SENTINEL_PIXEL).all() and (jpeg.decode_jpeg(sentinel()) == SENTINEL_PIXEL).all()
    print(f"sentinel: C path (JSIMD_FORCENONE=1) {np.unique(c).tolist()}, SIMD Pillow {np.unique(simd).tolist()}")


def test_corpus_decodes_as_written_and_as_libjpeg_c(corpus, c_path):
    bad = []
    for case, ref in zip(corpus, c_path):
        st = jpeg.decode_stages(case.data)
        if st["info"].progressive:
            assert st["progress"]["scans"] == len(st["info"].scans), case.name
        else:
            assert st["decoded"].all(), case.name
        if not np.array_equal(st["coef"], case.coef):
            bad.append((case.name, "coefficients"))
        elif not np.array_equal(st["rgb"], ref):
            bad.append((case.name, f"{int((st['rgb'] != ref).sum())} samples"))
    kinds = sorted({c.kind for c in corpus})
    print(f"{len(corpus)} files ({', '.join(kinds)}) equal the C path; {len(bad)} differ")
    assert not bad, bad


def test_corpus_leaves_the_range(corpus, c_path):
    differ = 0
    for case, ref in zip(corpus, c_path):
        out = any(((r < -512) | (r > 511)).any() for r in R.raw_idct(case))
        simd = _simd(case.data)
        if case.kind == "control":
            assert not out, case.name
            assert np.array_equal(simd, ref) and np.array_equal(jpeg.decode_jpeg(case.data), ref), case.name
        else:
            assert out, case.name
        differ += not np.array_equal(simd, ref)
    n = sum(c.kind != "control" for c in corpus)
    print(f"SIMD Pillow decodes {differ} of the {n} out-of-range files differently from the C path")
    assert differ >= 0.8 * n, (differ, n)


def test_wrap_points_cover_every_edge(corpus):
    """Per subsampling and component, DC-only blocks land on both sides of every edge of the wrap and the clamp, at
    positive and negative x, out to within 0.5 % of the largest and most negative reachable x (255 * 32767 / 8 and
    255 * -32768 / 8)."""
    seen = defaultdict(set)
    reach = defaultdict(lambda: [0, 0])
    for case in corpus:
        if case.kind != "wrap":
            continue
        sub = case.name.split()[1]
        c = case.wrapped[0]
        x = R.raw_idct(case)[c][:, 0, 0]
        for v in x.tolist():
            r = (v + 128) % 1024 - 128
            if r in R.EDGES and not -512 <= v <= 511:
                seen[sub, c].add((r, v > 0))
        reach[sub, c][0] = max(reach[sub, c][0], int(x.max()))
        reach[sub, c][1] = min(reach[sub, c][1], int(x.min()))
    want = {(e, s) for e in R.EDGES for s in (False, True)}
    for sub in R.SUBS:
        for c in range(1 if sub == "gray" else 3):
            assert seen[sub, c] == want, (sub, c, sorted(want - seen[sub, c]))
            assert reach[sub, c][0] >= 0.995 * 255 * 32767 // 8 and reach[sub, c][1] <= 0.995 * 255 * -32768 // 8, \
                (sub, c, reach[sub, c])


def test_corpus_reaches_the_int16_rules(corpus):
    """The cases do what their names say: every zigzag position at +-1023, blocks of every coefficient at its largest,
    DC coefficients stored as the int16 of a predictor past +-32767, and each progressive case."""
    by = defaultdict(list)
    for case in corpus:
        by[case.kind].append(case)
    for case in by["one ac"]:
        zz = case.coef[:, jpeg.ZIGZAG]
        got = {(k, int(v)) for b in zz for k in np.nonzero(b)[0].tolist() for v in [b[k]]}
        assert got == {(k, v) for k in range(1, 64) for v in (-1023, 1023)}, case.name
    full = by["full column"][0].coef
    assert any((b[0] == 32767 and (b[1:] == 1023).all()) for b in full)
    assert any((b[0] == -32768 and (b[1:] == -1023).all()) for b in full)
    for case in by["dc predictor"]:
        info = jpeg.parse(case.data)
        ci = R.comp_index(jpeg.geometry(info.h, info.w, info.ncomp, info.hs, info.vs))
        dc = case.coef[ci == 0, 0].astype(np.int64)
        assert dc.max() > 30000 and dc.min() < -30000 and np.abs(np.diff(dc)).max() > 2047, case.name
    names = [c.name for c in by["progressive"]]
    assert any(n.startswith("al 13 down") for n in names)
    assert {n.split()[3] for n in names if n.startswith("ac first al")} == {"10", "11", "12", "13"}
    assert any(n.startswith("dc first al 13") and n.endswith("refined") for n in names)


@pytest.mark.skipif(not FIXTURES, reason="no committed JPEG fixtures")
def test_fixtures_c_path_equals_simd_and_host():
    """In range the C path, SIMD Pillow and decode_jpeg agree on every committed fixture."""
    files = [p.read_bytes() for p in FIXTURES]
    ref = decode_c(files)
    for p, d, r in zip(FIXTURES, files, ref):
        assert np.array_equal(r, _simd(d)), p.name
        assert np.array_equal(r, jpeg.decode_jpeg(d)), p.name
    print(f"{len(files)} committed fixtures: C path = SIMD Pillow = decode_jpeg")
