"""`applications.decode_jpeg` against Pillow, byte for byte, and the refusals of the marker parser (no GPU).

The matrix: 4:4:4, 4:2:2, 4:2:0 and grayscale; quality 5 to 100 and optimised Huffman tables; sizes from 1x1 to 1080x1920;
restart markers every block, every 4 blocks and every MCU row; all-0, all-255 and checkerboard images, which drive the
IDCT's range limit; EXIF, ICC and comment segments.  Pillow is only used here: the product never imports it."""
import io
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from defer_b200 import applications, jpeg  # noqa: E402
from make_jpeg_fixtures import content, encode  # noqa: E402

SUBS = ("444", "422", "420", "gray")


def pillow(data):
    Image = pytest.importorskip("PIL.Image")
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def _check(data):
    got = applications.decode_jpeg(data)
    want = pillow(data)
    assert got.dtype == np.uint8 and got.shape == want.shape and got.flags["C_CONTIGUOUS"]
    assert np.array_equal(got, want)


@pytest.mark.parametrize("sub", SUBS)
@pytest.mark.parametrize("size", [(1, 1), (1, 17), (3, 5), (5, 4), (7, 9), (15, 17), (16, 16), (17, 33), (223, 225)])
def test_sizes(size, sub):
    pytest.importorskip("PIL")
    for q in (5, 75, 100):
        _check(encode(content("photo", *size, seed=q), sub, q))


@pytest.mark.parametrize("sub", SUBS)
@pytest.mark.parametrize("opts", [{"quality": 5}, {"quality": 50}, {"quality": 75}, {"quality": 95}, {"quality": 100},
                                  {"quality": 75, "optimize": True}, {"quality": 75, "restart_marker_blocks": 1},
                                  {"quality": 90, "restart_marker_blocks": 4}, {"quality": 50, "restart_marker_rows": 1}])
def test_quality_tables_and_restarts(opts, sub):
    pytest.importorskip("PIL")
    _check(encode(content("photo", 61, 75, seed=3), sub, **opts))


@pytest.mark.parametrize("kind", ["zero", "full", "checker"])
@pytest.mark.parametrize("sub", SUBS)
def test_range_limit(kind, sub):
    pytest.importorskip("PIL")
    for q in (50, 100):
        _check(encode(content(kind, 33, 47, seed=0), sub, q))


def test_large_frames():
    pytest.importorskip("PIL")
    _check(encode(content("photo", 480, 640, seed=1), "420", 90))
    _check(encode(content("photo", 1080, 1920, seed=2), "420", 50))


def test_metadata_segments():
    pytest.importorskip("PIL")
    exif = b"Exif\0\0MM\0*\0\0\0\x08\0\0" + b"\0" * 40
    _check(encode(content("photo", 40, 60, seed=4), "420", 75, exif=exif, icc_profile=b"\0" * 600, comment=b"x" * 50))


def test_committed_fixtures():
    pytest.importorskip("PIL")
    for p in sorted((ROOT / "tests" / "golden" / "jpeg").glob("*.jpg")):
        if "1080x1920" not in p.name:
            _check(p.read_bytes())


def _segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def _base():
    return (Path(ROOT / "tests" / "golden" / "jpeg" / "photo_223x225_420_q75.jpg")).read_bytes()


def _with_sof(data, payload_fn, marker=None):
    """``data`` with its SOF0 segment's payload rewritten by ``payload_fn`` (and its marker replaced)."""
    i = data.index(b"\xff\xc0")
    n = int.from_bytes(data[i + 2:i + 4], "big")
    payload = payload_fn(bytearray(data[i + 4:i + 2 + n]))
    return data[:i] + _segment(marker if marker is not None else 0xC0, bytes(payload)) + data[i + 2 + n:]


@pytest.mark.parametrize("marker,why", [(0xC2, "progressive"), (0xC3, "lossless"), (0xC9, "arithmetic")])
def test_refuses_other_processes(marker, why):
    with pytest.raises(ValueError, match=why):
        jpeg.parse(_with_sof(_base(), lambda p: p, marker))


def test_refusals():
    d = _base()
    with pytest.raises(ValueError, match="12-bit"):
        jpeg.parse(_with_sof(d, lambda p: bytes([12]) + p[1:]))
    with pytest.raises(ValueError, match="truncated"):
        jpeg.parse(d[:-2])
    with pytest.raises(ValueError, match="more than one scan"):
        jpeg.parse(d[:-2] + b"\xff\xda" + b"\0" * 10 + b"\xff\xd9")

    def sampling(p):                      # 4:4:0: luma 1x2
        p[7] = 0x12
        return p
    with pytest.raises(ValueError, match="sampling"):
        jpeg.parse(_with_sof(d, sampling))

    def rgb_ids(p):
        p[6], p[9], p[12] = 82, 71, 66
        return p
    no_jfif = d[:2] + d[2 + 2 + int.from_bytes(d[4:6], "big"):]
    assert d[2:4] == b"\xff\xe0"
    with pytest.raises(ValueError, match="RGB"):
        jpeg.parse(_with_sof(no_jfif, rgb_ids))
    adobe = no_jfif[:2] + _segment(0xEE, b"Adobe\0\x64\0\0\0\0\0") + no_jfif[2:]
    with pytest.raises(ValueError, match="RGB|Adobe"):
        jpeg.parse(adobe)
    with pytest.raises(ValueError, match="not a JPEG"):
        jpeg.parse(b"\x89PNG....")
    with pytest.raises(ValueError, match="runs past"):
        jpeg.parse(d[:10])
    for bad in (np.zeros((2, 2), np.uint8), "file.jpg", np.zeros(4, np.float32)):
        with pytest.raises(ValueError, match="JPEG item"):
            jpeg.parse(bad)


def test_data_after_eoi_is_ignored():
    """An MPF-style file (a second JPEG after the first one's EOI) and trailing bytes holding FFD9 decode as the first
    image, as Pillow does; the entropy data ends at the first EOI."""
    d = _base()
    second = (ROOT / "tests" / "golden" / "jpeg" / "photo_40x60_420_q75_meta.jpg").read_bytes()
    info = jpeg.parse(d)
    assert d[info.offset + info.length:] == b"\xff\xd9"
    for data in (d + second, d + b"\0\xff\xd9junk\xff\xd9", d[:-2] + b"\xff\xff\xff\xd9"):
        got = jpeg.parse(data)
        assert (got.offset, got.length) == (info.offset, info.length)
        assert np.array_equal(applications.decode_jpeg(data), applications.decode_jpeg(d))
        if pytest.importorskip("PIL"):
            _check(data)
    with pytest.raises(ValueError, match="DNL"):
        jpeg.parse(d[:-2] + b"\xff\xdc\0\x04\0\x10\xff\xd9")      # a DNL marker


def test_refuses_2_and_4_components():
    d = _base()
    with pytest.raises(ValueError, match="components"):
        jpeg.parse(_with_sof(d, lambda p: p[:5] + bytes([4]) + p[6:] + p[-3:]))
    with pytest.raises(ValueError, match="components"):
        jpeg.parse(_with_sof(d, lambda p: p[:5] + bytes([2]) + p[6:12]))


def test_bounds_and_slot():
    d = _base()
    data, info = jpeg.check_jpeg(bytearray(d), (223, 225))
    assert data == d and (info.h, info.w) == (223, 225)
    assert jpeg.check_jpeg(memoryview(d), (300, 300))[1].w == 225
    assert jpeg.check_jpeg(np.frombuffer(d, np.uint8), (300, 300))[1].h == 223
    with pytest.raises(ValueError, match="outside max_image_size"):
        jpeg.check_jpeg(d, (222, 1000))
    with pytest.raises(ValueError, match="larger than the compressed slot"):
        jpeg.check_jpeg(d, (8, 8))


def test_tables_are_memoised():
    d = _base()
    jpeg.dht_tables.cache_clear()
    jpeg.dqt_tables.cache_clear()
    a, b = jpeg.parse(d), jpeg.parse(bytes(d))
    assert a.dc[0] is b.dc[0] and a.quant[0] is b.quant[0]
    assert jpeg.dht_tables.cache_info().hits >= 1 and jpeg.dqt_tables.cache_info().hits >= 1
    blk = jpeg.pack_block(a)
    assert blk.shape == (jpeg.BLOCK_INTS,) and blk[0] == 223 and blk[1] == 225 and blk[6] == a.offset


def test_decode_option_checks():
    for kw in ({"decode": "png", "preprocess": "caffe", "max_image_size": (8, 8)},
               {"decode": "jpeg", "preprocess": "caffe"}, {"decode": "jpeg", "max_image_size": (8, 8)},
               {"decode": "jpeg", "preprocess": "caffe", "max_image_size": (8, 8), "image_size": (8, 8)}):
        with pytest.raises(ValueError, match="decode="):
            jpeg.check_decode(kw.get("decode"), kw.get("preprocess"), kw.get("image_size"), kw.get("max_image_size"))
    from defer_b200.dispatcher import DEFER
    with pytest.raises(ValueError, match="batch must be 1"):
        DEFER([0], preprocess="caffe", max_image_size=(8, 8), decode="jpeg", batch=2)


def test_product_never_imports_pil():
    for p in (ROOT / "defer_b200").rglob("*.py"):
        src = p.read_text()
        assert "import PIL" not in src and "from PIL" not in src, p
