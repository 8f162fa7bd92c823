"""The test JPEG writer (tests/jpeg_craft.py) against the host decoder and Pillow, and the limits of the decode contract.

- Round trip: ``jpeg.entropy_decode`` of a crafted file returns exactly the coefficients written, for random tables
  (codes up to 16 bits), every subsampling and restart intervals.
- In range, a crafted file decodes as Pillow does: one-symbol tables, 16-bit codes, quantisers from 1 to 255, restart
  intervals of one MCU and of more than one MCU row, and the stream of all-zero bits, whose blocks are 127 bits each.
  The coefficients come from a forward DCT of 8-bit blocks, so any encoder may emit them.
- 0xFF fill bytes before every RSTn marker decode as Pillow does.
- Out of range, ``jpeg.idct_islow`` wraps as jidctint.c's ``idct_range_limit[x & 1023]``: a few hand-computed values
  here; tests/test_jpeg_idct_range_host.py checks the whole out-of-range decode against libjpeg-turbo 3.1's C path.
- The closed form of the rounds of the self-synchronising decode on files whose every bit position decodes (the worst
  case the GPU tests use) equals ``jpeg_check.sync_stats`` at 8, 32 and the device's subsequence size.
"""
import io
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))

from defer_b200 import jpeg  # noqa: E402
import jpeg_craft as jc  # noqa: E402
from jpeg_check import sync_stats  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "jpeg"
SBITS = int(re.search(r"#define DEFER_JPEG_SUBSEQ_BITS (\d+)", (ROOT / "include" / "defer_b200.h").read_text()).group(1))
SUBS = ("gray", "444", "422", "420")


def pillow(data):
    Image = pytest.importorskip("PIL.Image")
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def random_coef(rng, g, dc_span=1000, density=0.2):
    """Coefficients that exercise every symbol: DC differences up to 11 bits, AC values up to 10 bits, zero runs of
    every length (ZRL), blocks ending in a non-zero coefficient 63 (no EOB) and all-zero blocks."""
    coef = np.zeros((g.blocks, 64), np.int32)
    coef[:, 0] = rng.integers(-dc_span, dc_span + 1, g.blocks)
    ac = np.where(rng.random((g.blocks, 63)) < density, rng.integers(-1023, 1024, (g.blocks, 63)), 0)
    ac[rng.random(g.blocks) < 0.1] = 0
    ac[::7, -1] = rng.integers(1, 1024, ac[::7].shape[0])
    ac[::5, :40] = 0
    coef[:, 1:] = ac
    return coef


def _round_trip(data, coef):
    info = jpeg.parse(data)
    raw, decoded = jpeg.entropy_decode(data, info)
    assert decoded.all()
    assert np.array_equal(jpeg.dc_predict(raw, decoded, info), coef)


@pytest.mark.parametrize("sub", SUBS)
@pytest.mark.parametrize("restart", [0, 1, 3, 7])
def test_round_trip(sub, restart):
    rng = np.random.default_rng(len(sub) * 10 + restart)
    h, w = 37, 53
    g = jc.geometry(h, w, sub)
    coef = random_coef(rng, g)
    quant = [rng.integers(1, 256, 64), rng.integers(1, 256, 64)]
    for deep in (0.0, 0.5, 1.0):
        dc, ac = jc.tables_for(coef, g, restart, rng, deep)
        data = jc.craft(h, w, sub, quant, dc, ac, coef=coef, restart=restart)
        _round_trip(data, coef)
        assert jc.assemble(*jc.split(data)) == data
        _round_trip(jc.assemble(*jc.split(data), fill=3), coef)     # fill bytes before RSTn and EOI
        st, want = jpeg.decode_stages(data), jc.expected(coef, h, w, sub, quant)
        assert all(np.array_equal(a, b) for a, b in zip(st["planes"], want["planes"]))
        assert np.array_equal(st["rgb"], want["rgb"])
    assert max(i + 1 for t in ac for i, n in enumerate(t[0]) if n) == 16      # deep = 1 gives 16-bit codes


def test_one_symbol_and_long_codes_decode():
    """A one-symbol table is one 1-bit code; a 16-bit code is read past the 9-bit lookahead."""
    for ln in (1, 9, 10, 16):
        dc, ac = jc.one_symbol(0, ln), jc.one_symbol(0x01, ln)
        bits = "0" * (ln + 63 * (ln + 1))
        data = jc.craft(8, 8, "gray", [np.ones(64, int)], [dc], [ac], bits=[bits])
        coef = np.full((1, 64), -1, np.int32)
        coef[0, 0] = 0
        _round_trip(data, coef)


def _planes(rng, g, h, w):
    """MCU-padded 8-bit planes of a photo-like image (tools/make_jpeg_fixtures.content)."""
    from make_jpeg_fixtures import content
    img = content("photo", g.bh[0] * 8, g.bw[0] * 8, seed=int(rng.integers(1 << 30)))
    return [img[:g.bh[c] * 8, :g.bw[c] * 8, c] for c in range(len(g.bw))]


def _in_range(coef, g, quant):
    comp_of = np.tile(np.array(g.comp_of), g.mcus)
    raw = [jc.idct_raw(coef[comp_of == c], np.asarray(quant[0 if c == 0 else -1])) for c in range(len(g.bw))]
    return all(((r >= -512) & (r <= 511)).all() for r in raw)


QUANTS = {"ones": lambda rng: [np.ones(64, int)] * 2,
          "random": lambda rng: [rng.integers(1, 256, 64), rng.integers(1, 256, 64)],
          "coarse": lambda rng: [np.full(64, 255), np.full(64, 200)],
          "ramp": lambda rng: [np.minimum(1 + 4 * np.arange(64), 255)] * 2}


@pytest.mark.parametrize("sub", SUBS)
@pytest.mark.parametrize("quant", list(QUANTS))
@pytest.mark.parametrize("restart,deep", [(0, 0.0), (1, 1.0), (9, 0.5)])
def test_pillow_in_range(sub, quant, restart, deep):
    """Crafted files of forward-DCT coefficients decode as Pillow does; 9 MCUs is more than one MCU row here."""
    pytest.importorskip("PIL")
    rng = np.random.default_rng(len(sub) + 7 * len(quant) + restart)
    h, w = 29, 43 if sub == "gray" else 61
    g = jc.geometry(h, w, sub)
    assert g.mcux < 9
    q = QUANTS[quant](rng)
    coef = jc.fdct_coef(_planes(rng, g, h, w), g, q)
    assert _in_range(coef, g, q)
    dc, ac = jc.tables_for(coef, g, restart, rng, deep)
    data = jc.craft(h, w, sub, q, dc, ac, coef=coef, restart=restart)
    got = jpeg.decode_stages(data)
    assert np.array_equal(got["coef"], coef)
    assert np.array_equal(got["rgb"], pillow(data))


@pytest.mark.parametrize("sub", ["gray", "420"])
@pytest.mark.parametrize("restart", [0, 5])
def test_pillow_all_zero_stream(sub, restart):
    """One-symbol tables (DC category 0 and AC (0, 1), both code '0') and all-zero bits: every block is 127 bits,
    every AC coefficient -1, and the file decodes as Pillow does."""
    pytest.importorskip("PIL")
    h, w = 64, 128
    data = jc.all_zero_stream(h, w, sub, restart)
    want = jc.expected(jc.all_zero_coef(jc.geometry(h, w, sub)), h, w, sub, [np.ones(64, int)])
    assert np.array_equal(jpeg.decode_stages(data)["coef"], want["coef"])
    assert np.array_equal(jpeg.decode_jpeg(data), want["rgb"])
    assert np.array_equal(want["rgb"], pillow(data))


@pytest.mark.parametrize("name", ["photo_223x225_420_q75_rb1.jpg", "photo_223x225_444_q50_rr1.jpg",
                                  "photo_223x225_gray_q90_rb4.jpg"])
def test_fill_bytes_before_rst(name):
    """0xFF fill bytes before each RSTn stay in the entropy data as bytes past the interval's last block: the decode is
    unchanged, and equals Pillow's."""
    pytest.importorskip("PIL")
    data = (GOLDEN / name).read_bytes()
    head, parts = jc.split(data)
    assert len(parts) > 1
    filled = jc.assemble(head, parts, fill=2)
    assert jpeg.unstuff(filled[len(head):])[1] != jpeg.unstuff(data[len(head):])[1]
    assert np.array_equal(jpeg.decode_jpeg(filled), jpeg.decode_jpeg(data))
    assert np.array_equal(jpeg.decode_jpeg(filled), pillow(filled))


@pytest.mark.parametrize("dc,q,want", [(110, 80, 204), (-60, 80, 255), (100, 64, 0), (63, 64, 255), (-64, 64, 0)])
def test_idct_wraps_out_of_range(dc, q, want):
    """A DC-only block of value x = dc * q / 8 around 128 gives idct_range_limit[x & 1023]: 1100 wraps to 76 (204),
    -600 to 424 (clamped to 255), 800 to -224 (clamped to 0); 504 and -512 are in range and clamp to 255 and 0."""
    coef = np.zeros((1, 64), np.int16)
    coef[0, 0] = dc
    x = dc * q // 8
    assert jc.idct_raw(coef, np.full(64, q)).ravel().tolist() == [x] * 64
    assert (jpeg.idct_islow(coef, np.full(64, q, np.int32)) == want).all()


@pytest.mark.parametrize("sbits", [8, 32, SBITS])
def test_worst_case_rounds_closed_form(sbits):
    """On files whose every bit position decodes, the rounds are the most subsequences in one restart interval (a
    decoder in the wrong phase never meets an invalid code), far more than on encoder-made files.  The other four
    counters follow from the unstuffed length, the markers and the geometry."""
    if sbits <= 32:
        files = [jc.all_zero_stream(16, 64, "gray"), jc.all_zero_stream(16, 48, "420"), jc.all_zero_stream(32, 64, "gray", 3)]
    else:
        files = [jc.all_zero_stream(256, 256, "gray"), jc.all_zero_stream(128, 128, "420"),
                 jc.all_zero_stream(256, 256, "gray", restart=200), jc.all_zero_stream(64, 128, "gray", restart=5),
                 jc.long_code_stream(64, 64)]
    rounds = []
    for data in files:
        want = jc.closed_form_counters(data, sbits)
        got = sync_stats(data, sbits)[2]
        assert np.array_equal(got, want), (got, want)
        rounds.append(int(got[3]))
    assert max(rounds) >= 12, rounds


def test_long_code_stream_coefficients():
    h, w = 64, 64
    data = jc.long_code_stream(h, w)
    assert np.array_equal(jpeg.decode_stages(data)["coef"], jc.long_code_coef(jc.geometry(h, w, "gray")))
