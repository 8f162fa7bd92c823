"""PNG files at ingress on the host: the chunk parser, the per-sample block and ``decode_png`` against Pillow.

``decode_png`` equals ``np.asarray(Image.open(f).convert("RGB"))`` on every committed fixture (tools/make_png_fixtures.py:
every colour type and bit depth, odd sizes, each filter type forced per row, zlib levels 0 / 1 / 9 and strategies
Z_FIXED, Z_HUFFMAN_ONLY and Z_RLE, short palettes, Pillow-written files); every refusal names its reason; the feed path
never inflates; and the compressed slot admits the stored (level 0) encoding of noise at the bound."""
import io
import struct
import sys
import zlib
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import applications, jpeg, png  # noqa: E402
from png_craft import chunk, ihdr, png_file  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "png"


def _fixtures():
    return sorted(GOLDEN.glob("*.png"))


def _pillow(data):
    Image = pytest.importorskip("PIL.Image")
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def test_fixtures_cover_every_mode():
    names = [p.name for p in _fixtures()]
    for ctype, depths in {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}.items():
        for d in depths:
            assert any(f"_c{ctype}_d{d}" in n for n in names), (ctype, d)
    assert len(names) >= 100


@pytest.mark.parametrize("path", _fixtures(), ids=lambda p: p.stem)
def test_decode_png_equals_pillow(path):
    d = path.read_bytes()
    got = applications.decode_png(d)
    assert got.dtype == np.uint8 and got.flags["C_CONTIGUOUS"]
    assert np.array_equal(got, _pillow(d))
    st = png.decode_stages(d)
    assert st["stats"].tolist() == [png.STATUS_OK, st["info"].raw_bytes, 0]


def test_restatement_equals_zlib():
    """The device's inflate, restated, gives zlib's bytes on every fixture's stream."""
    for p in _fixtures():
        d = p.read_bytes()
        info = png.parse(d)
        stream = png.gather(d, info)
        want = zlib.decompressobj().decompress(stream, info.raw_bytes)
        assert png.inflate_restated(stream, info.raw_bytes) == (want, png.STATUS_OK), p.name


def _base():
    return (GOLDEN / "photo_7x9_c2_d8.png").read_bytes()


def _chunks(d):
    out, p = [], 8
    while p < len(d):
        n = int.from_bytes(d[p:p + 4], "big")
        out.append((d[p + 4:p + 8], d[p + 8:p + 8 + n]))
        p += 12 + n
    return out


def _build(chs):
    return png.SIGNATURE + b"".join(chunk(k, b) for k, b in chs)


def _refused(data, match):
    with pytest.raises(ValueError, match=match):
        png.parse(data)


def test_refusals_name_their_reason():
    d = _base()
    chs = _chunks(d)
    idat = [b for k, b in chs if k == b"IDAT"]
    z = b"".join(idat)
    _refused(b"\xff\xd8\xff\xe0", "not a PNG")
    _refused(d[:8] + _build(chs[1:])[8:], "missing IHDR")
    _refused(_build([(b"IHDR", chs[0][1][:12])] + chs[1:]), "malformed IHDR")
    for ctype, depth in ((2, 4), (3, 16), (4, 1), (5, 8), (0, 3)):
        body = struct.pack(">IIBBBBB", 9, 7, depth, ctype, 0, 0, 0)
        _refused(_build([(b"IHDR", body)] + chs[1:]), "malformed IHDR")
    _refused(_build([(b"IHDR", struct.pack(">IIBBBBB", 0, 7, 8, 2, 0, 0, 0))] + chs[1:]), "malformed IHDR")
    _refused(_build([(b"IHDR", struct.pack(">IIBBBBB", 9, 7, 8, 2, 1, 0, 0))] + chs[1:]), "compression method")
    _refused(_build([(b"IHDR", struct.pack(">IIBBBBB", 9, 7, 8, 2, 0, 1, 0))] + chs[1:]), "filter method")
    _refused(_build([(b"IHDR", struct.pack(">IIBBBBB", 9, 7, 8, 2, 0, 0, 1))] + chs[1:]), "Adam7")
    for apng in (b"acTL", b"fcTL", b"fdAT"):
        _refused(_build(chs[:1] + [(apng, b"\0" * 8)] + chs[1:]), "APNG")
    _refused(_build(chs[:1] + chs[-1:]), "missing IDAT")
    _refused(_build(chs[:1] + [(b"IDAT", z[:5]), (b"tEXt", b"a\0b"), (b"IDAT", z[5:])] + chs[-1:]), "not consecutive")
    _refused(_build(chs[:1] + [(b"ABCD", b"")] + chs[1:]), "unknown critical chunk ABCD")
    _refused(_build(chs[:1] + [(b"IDAT", z), (b"ABCD", b"")] + chs[-1:]), "unknown critical chunk")
    bad_crc = png.SIGNATURE + ihdr(9, 7, 8, 2)[:-4] + b"\0\0\0\0" + d[33:]
    _refused(bad_crc, "bad CRC of chunk IHDR")
    _refused(d[:40], "runs past the end")
    for head, why in ((b"\x79\x9c", "compression method"), (b"\x88\x98", "window"), (b"\x78\xbb", "FDICT"),
                      (b"\x78\x9d", "FCHECK")):
        _refused(_build(chs[:1] + [(b"IDAT", head + z[2:])] + chs[-1:]), f"bad zlib header.*{why}")
    _refused(_build(chs[:1] + [(b"IDAT", z[:1])] + chs[-1:]), "bad zlib header")
    for bad in (np.zeros((2, 2), np.uint8), "file.png", np.zeros(4, np.float32)):
        with pytest.raises(ValueError, match="PNG item"):
            png.parse(bad)


def test_palette_refusals_and_rules():
    d = (GOLDEN / "photo_7x9_c3_d8_p256.png").read_bytes()
    chs = _chunks(d)
    no_plte = [c for c in chs if c[0] != b"PLTE"]
    _refused(_build(no_plte), "missing PLTE")
    for bad in (b"", b"\1\2", b"\0" * 771):
        _refused(_build([(k, bad if k == b"PLTE" else b) for k, b in chs]), "malformed PLTE")
    plte = [c for c in chs if c[0] == b"PLTE"]
    _refused(_build(chs[:2] + plte + chs[2:]), "a second PLTE")
    after = [c for c in chs if c[0] != b"PLTE"]
    _refused(_build(after[:-1] + plte + after[-1:]), "after IDAT")
    # a PLTE in an RGB file is a suggestion, ignored; tRNS and other ancillary chunks are skipped
    rgb = _chunks(_base())
    f = _build(rgb[:1] + [(b"PLTE", b"\1\2\3" * 5), (b"tRNS", b"\0\1\0\2\0\3"), (b"gAMA", b"\0\0\xb1\x8f")] + rgb[1:])
    assert np.array_equal(png.decode_png(f), _pillow(f))


def test_crc_rule_is_pillows():
    """A bad CRC before the first IDAT is refused, as Pillow refuses it; IDAT and later CRCs are not checked, as Pillow
    does not check them."""
    d = _base()
    chs = _chunks(d)
    f = png.SIGNATURE + chunk(b"IHDR", chs[0][1]) + chunk(b"tEXt", b"k\0v", crc=1) + b"".join(chunk(k, b) for k, b in chs[1:])
    _refused(f, "bad CRC of chunk tEXt")
    f = png.SIGNATURE + b"".join(chunk(k, b, crc=0 if k in (b"IDAT", b"IEND") else None) for k, b in chs)
    assert np.array_equal(png.decode_png(f), _pillow(f))
    f = png.SIGNATURE + b"".join(chunk(k, b) for k, b in chs[:-1])            # no IEND
    assert np.array_equal(png.decode_png(f), _pillow(f))


def test_idat_cap():
    d = _base()
    chs = _chunks(d)
    z = b"".join(b for k, b in chs if k == b"IDAT")
    ok = _build(chs[:1] + [(b"IDAT", z[i:i + 1]) for i in range(len(z))] + chs[-1:])
    assert np.array_equal(png.decode_png(ok), _pillow(ok))
    many = _build(chs[:1] + [(b"IDAT", z)] + [(b"IDAT", b"")] * png.MAX_IDAT + chs[-1:])
    _refused(many, "DEFER_PNG_MAX_IDAT")


def test_block_layout():
    d = (GOLDEN / "photo_7x9_c3_d4_p7.png").read_bytes()
    info = png.parse(d)
    b = png.pack_block(info)
    assert b.shape == (png.BLOCK_INTS,)
    assert b[:9].tolist() == [7, 9, 3, 4, 5, 1, len(info.idat), info.stream_bytes, 7]
    pal = info.palette.astype(np.int64)
    assert b[png.PAL_OFF:png.PAL_OFF + 7].tolist() == (pal[:, 0] | pal[:, 1] << 8 | pal[:, 2] << 16).tolist()
    assert not b[png.PAL_OFF + 7:png.IDAT_OFF].any()
    assert b[png.IDAT_OFF:png.IDAT_OFF + 2 * len(info.idat)].tolist() == [v for r in info.idat for v in r]
    assert png.block_ints(info) == png.IDAT_OFF + 2 * len(info.idat)
    assert not b[png.block_ints(info):].any()
    header = (ROOT / "include" / "defer_b200.h").read_text()
    assert f"#define DEFER_PNG_MAX_IDAT {png.MAX_IDAT}" in header


def test_feed_path_never_inflates(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("the feed path inflated")
    monkeypatch.setattr(zlib, "decompress", boom)
    monkeypatch.setattr(zlib, "decompressobj", boom)
    for p in _fixtures():
        d, info = png.check_png(p.read_bytes(), (256, 256))
        png.pack_block(info)


def _noise_stored(h, w, ctype, depth, chunk_bytes=8192, seed=0):
    rng = np.random.default_rng(seed)
    bpr = (w * {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype] * depth + 7) // 8
    raw = b"".join(b"\0" + rng.integers(0, 256, bpr, dtype=np.uint8).tobytes() for _ in range(h))
    c = zlib.compressobj(0)
    z = c.compress(raw) + c.flush()
    return png_file(w, h, depth, ctype, z, idat_sizes=[chunk_bytes] * (len(z) // chunk_bytes))


def test_slot_admits_stored_noise_at_the_bound():
    """Level-0 (stored) files of noise at max_image_size fit the slot, in every colour type at its deepest, with libpng's
    8 KiB IDAT chunks, and so does a level-0 file of RGB noise at 1080x1920; a slot of H * W * 3 bytes would not."""
    for ctype, depth in ((6, 16), (2, 16), (4, 16), (0, 16), (2, 8)):
        d = _noise_stored(48, 64, ctype, depth)
        data, info = png.check_png(d, (48, 64))
        assert len(data) <= png.slot_bytes(48, 64)
        assert len(data) > 48 * 64 * 3 or ctype == 0
        assert np.array_equal(png.decode_png(d), _pillow(d))
    d = _noise_stored(1080, 1920, 2, 8, chunk_bytes=8192)
    assert len(png.parse(d).idat) <= png.MAX_IDAT
    png.check_png(d, (1080, 1920))
    assert len(d) > 1080 * 1920 * 3
    with pytest.raises(ValueError, match="larger than the compressed slot"):
        png.check_png(d, (300, 1920))
    with pytest.raises(ValueError, match="outside max_image_size"):
        png.check_png(_base(), (7, 8))
    assert png.slot_bytes(1080, 1920) == 1080 * (1 + 8 * 1920) + 1080 * (1 + 8 * 1920) // 64 + 65536


def test_png_decode_option_checks():
    """decode="png" has decode="jpeg"'s rules in the pipelines: preprocess= and max_image_size= needed, image_size
    refused, batch 1.  jpeg.check_decode alone still takes JPEG only."""
    for dec in ("jpeg", "png"):
        jpeg.check_decode(dec, "caffe", None, (8, 8), png.DECODES)
        for kw in ({"preprocess": "caffe"}, {"max_image_size": (8, 8)},
                   {"preprocess": "caffe", "max_image_size": (8, 8), "image_size": (8, 8)}):
            with pytest.raises(ValueError, match="decode="):
                jpeg.check_decode(dec, kw.get("preprocess"), kw.get("image_size"), kw.get("max_image_size"),
                                  png.DECODES)
    with pytest.raises(ValueError, match="decode="):
        jpeg.check_decode("gif", "caffe", None, (8, 8), png.DECODES)
    with pytest.raises(ValueError, match="decode="):
        jpeg.check_decode("png", "caffe", None, (8, 8))
    with pytest.raises(ValueError, match="each PNG carries its own size"):
        jpeg.check_decode("png", "caffe", (8, 8), (8, 8), png.DECODES)
    from defer_b200.dispatcher import DEFER
    d = DEFER([0], preprocess="caffe", max_image_size=(8, 8), decode="png")
    assert d.decode == "png"
    with pytest.raises(ValueError, match="one PNG file, so batch must be 1"):
        DEFER([0], preprocess="caffe", max_image_size=(8, 8), decode="png", batch=2)
    with pytest.raises(ValueError, match="image_size"):
        DEFER([0], preprocess="caffe", image_size=(8, 8), max_image_size=(8, 8), decode="png")


def test_plans():
    """A decode="png" plan puts PNG_DECODE where a JPEG plan puts JPEG_DECODE, on a PNG input slot; the JPEG plan is
    unchanged by it."""
    from defer_b200 import _cabi as A
    from defer_b200 import keras_like as K
    from defer_b200.planner import plan_stage
    x = K.Input((32, 32, 3))
    y = K.Conv2D(4, 3, name="c")(x)
    m = K.Model(x, y, name="m")
    kw = dict(is_first=True, is_last=True, preprocess="caffe", max_image_size=(40, 60), interpolation="bilinear")
    pj = plan_stage(m, decode="jpeg", **kw)
    pp = plan_stage(m, decode="png", **kw)
    assert [o.kind for o in pp.ops] == [A.OP_PNG_DECODE] + [o.kind for o in pj.ops][1:]
    assert pj.ops[0].kind == A.OP_JPEG_DECODE and pj.bufs[pj.input_buf][3] == A.BUF_JPEG
    assert pp.bufs[pp.input_buf] == (40, 60, 3, A.BUF_PNG) and pp.decode == "png"
    assert pp.bufs[1:] == pj.bufs[1:]
