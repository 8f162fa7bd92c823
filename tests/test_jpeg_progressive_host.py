"""Progressive JPEG files on the host: ``decode_jpeg`` against Pillow byte for byte, the scan-script refusals, the caps
and the block layout (no GPU).

The matrix: 4:4:4, 4:2:2, 4:2:0 and grayscale; sizes from 1x1 up, including sizes where a component's own block grid is
smaller than its MCU-padded one; quality 5 to 100 and optimised tables; restart markers; the committed fixtures.  The
refusals are made by rewriting the scan headers of a Pillow-written file.  Pillow is only used here."""
import io
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests", ROOT / "tools"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import applications, jpeg  # noqa: E402
from jpeg_progressive_check import corrupt_corpus, fixture, fixture_names  # noqa: E402
from jpeg_progressive_worst_case import refinement_stream  # noqa: E402
from make_jpeg_fixtures import content, encode  # noqa: E402

SUBS = ("444", "422", "420", "gray")


def pillow(data):
    Image = pytest.importorskip("PIL.Image")
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def _check(data):
    assert jpeg.parse(data).progressive
    got = applications.decode_jpeg(data)
    want = pillow(data)
    assert got.dtype == np.uint8 and got.shape == want.shape and got.flags["C_CONTIGUOUS"]
    assert np.array_equal(got, want)


@pytest.mark.parametrize("sub", SUBS)
@pytest.mark.parametrize("size", [(1, 1), (1, 17), (3, 5), (9, 9), (15, 17), (16, 16), (17, 33), (33, 18)])
def test_sizes(size, sub):
    pytest.importorskip("PIL")
    for q in (5, 75, 100):
        _check(encode(content("photo", *size, seed=q), sub, q, progressive=True))


@pytest.mark.parametrize("sub", SUBS)
@pytest.mark.parametrize("opts", [{"quality": 50}, {"quality": 95}, {"quality": 75, "optimize": True},
                                  {"quality": 75, "restart_marker_blocks": 1},
                                  {"quality": 90, "restart_marker_blocks": 5}, {"quality": 50, "restart_marker_rows": 1}])
def test_quality_tables_and_restarts(opts, sub):
    pytest.importorskip("PIL")
    _check(encode(content("photo", 41, 57, seed=3), sub, progressive=True, **opts))


def test_committed_fixtures():
    pytest.importorskip("PIL")
    names = fixture_names()
    assert len(names) >= 30
    for nm in names:
        _check(fixture(nm))


def test_crafted_refinement_stream():
    """tools/jpeg_progressive_worst_case.py's file: an EOB run over every block, then 17-bit refinement symbols."""
    _check(refinement_stream(24, 40))
    _check(refinement_stream(9, 17))


def test_corrupt_corpus_defined():
    """Corrupt files decode to the defined result: a failing scan stops the decode, so the entropy data of the scans
    after it changes nothing."""
    stopped = 0
    for nm, d in corrupt_corpus(seed=0):
        st = jpeg.decode_stages(d)
        pr, scans = st["progress"], st["info"].scans
        assert 0 <= pr["scans"] <= len(scans) and pr["cutoff"] <= len(st["coef"]), nm
        if pr["scans"] + 1 >= len(scans):
            continue
        a = bytearray(d)
        for sc in scans[pr["scans"] + 1:]:                  # zero the later scans' entropy data, markers kept
            a[sc.offset:sc.offset + sc.length] = bytes(sc.length)
        other = jpeg.decode_stages(bytes(a))
        assert np.array_equal(other["coef"], st["coef"]) and other["progress"] == pr, nm
        stopped += 1
    assert stopped >= 5


# ------------------------------------------------------------------------------------------------ refusals
def _base():
    return fixture("photo_61x75_420_q75.jpg")


def _sos(data):
    """Offsets of each SOS segment's payload."""
    info = jpeg.parse(data)
    out = []
    for sc in info.scans:                       # the payload: ns, 2 bytes per component, Ss, Se, Ah << 4 | Al
        out.append(sc.offset - (4 + 2 * len(sc.comps)))
    return out, info


def _with_scan(data, s, ss=None, se=None, ah=None, al=None):
    """``data`` with scan s's Ss, Se, Ah or Al rewritten."""
    offs, info = _sos(data)
    p = offs[s]
    ns = data[p]
    a = bytearray(data)
    q = p + 1 + 2 * ns
    if ss is not None:
        a[q] = ss
    if se is not None:
        a[q + 1] = se
    ah0, al0 = a[q + 2] >> 4, a[q + 2] & 15
    a[q + 2] = ((ah if ah is not None else ah0) << 4) | (al if al is not None else al0)
    return bytes(a)


def test_scan_header_offsets():
    offs, info = _sos(_base())
    for p, sc in zip(offs, info.scans):
        assert _base()[p] == len(sc.comps)


@pytest.mark.parametrize("edit,why", [
    (lambda d: _with_scan(d, 0, se=5), "DC scan with Se = 5"),
    (lambda d: _with_scan(d, 1, ss=6, se=5), "spectral selection 6..5"),
    (lambda d: _with_scan(d, 1, se=64), "spectral selection"),
    (lambda d: _with_scan(d, 0, ah=3, al=1), "Ah = 3, Al = 1"),
    (lambda d: _with_scan(d, 0, al=14), "Al = 14 > 13"),
    (lambda d: _with_scan(d, 1, ah=1, al=0), "bit state"),
])
def test_refused_scan_scripts(edit, why):
    with pytest.raises(ValueError, match="progressive") as e:
        jpeg.parse(edit(_base()))
    assert why in str(e.value)


def test_refuses_ac_before_dc_and_interleaved_ac():
    gray = fixture("photo_61x75_gray_q75.jpg")   # its DC first scan made an AC scan: no DC scan before it
    with pytest.raises(ValueError, match="before its DC scan"):
        jpeg.parse(_with_scan(gray, 0, ss=1, se=5))
    d = _base()                                   # an AC spectral range on the interleaved DC scan
    with pytest.raises(ValueError, match="AC scan of 3 components"):
        jpeg.parse(_with_scan(d, 0, ss=1, se=5))


def test_refuses_block_smoothing():
    """A file whose last scans are missing, its EOI kept: libjpeg would smooth its blocks."""
    d = _base()
    info = jpeg.parse(d)
    last = info.scans[-1]
    start = d.rindex(b"\xff\xda", 0, last.offset)
    with pytest.raises(ValueError, match="block smoothing"):
        jpeg.parse(d[:start] + b"\xff\xd9")


def test_caps(monkeypatch):
    d = _base()
    n = len(jpeg.parse(d).scans)
    monkeypatch.setattr(jpeg, "MAX_SCANS", n - 1)
    with pytest.raises(ValueError, match="DEFER_JPEG_MAX_SCANS"):
        jpeg.parse(d)
    monkeypatch.setattr(jpeg, "MAX_SCANS", n)
    jpeg.parse(d)
    monkeypatch.setattr(jpeg, "MAX_TABLES", 1)
    with pytest.raises(ValueError, match="DEFER_JPEG_MAX_TABLES"):
        jpeg.parse(d)


def test_caps_match_header():
    import re
    h = (ROOT / "include" / "defer_b200.h").read_text()
    for name, v in (("MAX_SCANS", jpeg.MAX_SCANS), ("MAX_TABLES", jpeg.MAX_TABLES), ("SCAN_INTS", jpeg.SCAN_INTS)):
        assert int(re.search(rf"#define DEFER_JPEG_{name} (\d+)", h).group(1)) == v


def test_block_layout():
    d = _base()
    info = jpeg.parse(d)
    b = jpeg.pack_block(info)
    assert b.shape == (jpeg.BLOCK_INTS,) and b[10] == len(info.scans) and b[11] == len(info.tables)
    assert jpeg.block_ints(info) == jpeg.POOL_OFF + len(info.tables) * jpeg.HUFF_INTS
    assert not b[jpeg.block_ints(info):].any() and not b[jpeg.Q_END:jpeg.BASE_INTS].any()
    for s, sc in enumerate(info.scans):
        e = b[jpeg.SCAN_OFF + s * jpeg.SCAN_INTS:jpeg.SCAN_OFF + (s + 1) * jpeg.SCAN_INTS]
        assert e[0] == len(sc.comps) and tuple(e[4:11]) == (sc.ss, sc.se, sc.ah, sc.al, sc.restart, sc.offset, sc.length)
        assert e[9] + e[10] <= len(d)
        if sc.ss == 0 and sc.ah == 0:
            assert all(0 <= t < len(info.tables) for t in e[11:11 + len(sc.comps)])
        if sc.ss > 0:
            assert 0 <= e[14] < len(info.tables)
    bl = jpeg.pack_block(jpeg.parse((ROOT / "tests" / "golden" / "jpeg" / "photo_223x225_420_q75.jpg").read_bytes()))
    assert bl[10] == 0 and bl[11] == 0 and not bl[jpeg.BASE_INTS:].any()
