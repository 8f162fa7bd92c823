"""JPEG and PNG files in one pipeline (`decode="image"`) on the host: the sniff and its refusals, the option rules, the
plans, the tagged blocks and the workspace strides.  No GPU needed (the library loads without one).

A file's format is told from its first bytes as Pillow's `Image.open` does: FF D8 FF for a JPEG, the PNG signature for
a PNG.  `jpeg.parse` refuses FF D8 not followed by FF, so a sniff on FF D8 alone would give the same result; the tests
show both.  The `decode="jpeg"`, `decode="png"` and `max_image_size` plans are pinned to what they were before
`decode="image"` existed (tests/golden/image_plan_fingerprints.json, from tests/image_plan_fingerprints.py)."""
import ctypes as C
import json
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import _cabi as A  # noqa: E402
from defer_b200 import applications, image, jpeg, png  # noqa: E402
import png_craft as PC  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
JPEG_FILES = sorted((GOLDEN / "jpeg").glob("*.jpg")) + sorted((GOLDEN / "jpeg_progressive").glob("*.jpg"))
PNG_FILES = sorted((GOLDEN / "png").glob("*.png"))
HEADER = (ROOT / "include" / "defer_b200.h").read_text()


def _define(name):
    return int(re.search(rf"#define {name} (\d+)", HEADER).group(1))


# ------------------------------------------------------------------------------------------------ sniff and refusals
@pytest.mark.parametrize("item,seen", [
    (b"BM" + bytes(60), "first bytes 42 4d 00 00 00 00 00 00"),          # BMP
    (b"GIF89a" + bytes(20), "first bytes 47 49 46 38 39 61 00 00"),      # GIF
    (b"", "an empty item"),
    (b"\xff", "first bytes ff"),
    (b"\xff\xd8\x00" + bytes(40), "first bytes ff d8 00 00 00 00 00 00"),
    (png.SIGNATURE[:7], "first bytes 89 50 4e 47 0d 0a 1a"),             # a PNG signature cut short
])
def test_sniff_refuses_other_items(item, seen):
    for call in (image.sniff, lambda d: image.check_image(d, (64, 64)), image.decode_image):
        with pytest.raises(ValueError, match=re.escape(f"neither a JPEG nor a PNG file ({seen})")):
            call(item)


def test_sniff_on_ff_d8_alone_would_refuse_the_same_files():
    """FF D8 followed by anything but FF is refused by the sniff, and jpeg.parse refuses it as well: the two-byte and
    three-byte SOI tests accept the same files."""
    good = JPEG_FILES[0].read_bytes()
    for b in (0x00, 0x01, 0xD9, 0xFE):
        bad = good[:2] + bytes([b]) + good[3:]
        with pytest.raises(ValueError, match="neither a JPEG nor a PNG file"):
            image.sniff(bad)
        with pytest.raises(ValueError, match="JPEG refused"):
            jpeg.parse(bad)


def test_files_are_routed_by_their_bytes():
    """Every committed fixture goes to its own format's parser and decoder, whatever the caller calls it: a PNG named
    like ImageNet's JPEGs still decodes as a PNG, and each accepted item type gives the same result."""
    for paths, kind in ((JPEG_FILES, "jpeg"), (PNG_FILES, "png")):
        for p in paths[::7]:
            d = p.read_bytes()
            assert image.sniff(d) == kind, p.name
            want = jpeg.decode_jpeg(d) if kind == "jpeg" else png.decode_png(d)
            for item in (d, bytearray(d), memoryview(d), np.frombuffer(d, np.uint8)):
                got_d, got_kind, info = image.check_image(item, (1080, 1920))
                assert got_d == d and got_kind == kind and (info.h, info.w) == want.shape[:2], p.name
            assert np.array_equal(applications.decode_image(d), want), p.name
    with pytest.raises(ValueError, match="an image item is bytes"):
        image.check_image(np.zeros((2, 8), np.uint8), (8, 8))


def test_parser_refusals_pass_through():
    d = PNG_FILES[0].read_bytes()
    info = png.parse(d)
    interlaced = d[:8] + PC.ihdr(info.w, info.h, info.depth, info.ctype, interlace=1) + d[33:]
    with pytest.raises(ValueError, match="Adam7"):
        image.check_image(interlaced, (64, 64))
    with pytest.raises(ValueError, match="no SOI marker"):
        image.check_image(b"\xff\xd8\xff", (64, 64))                    # sniffed as a JPEG, too short for one
    with pytest.raises(ValueError, match="outside max_image_size=\\(30, 30\\)"):
        image.check_image(JPEG_FILES[0].read_bytes(), (30, 30))                  # 31x47
    with pytest.raises(ValueError, match="outside max_image_size=\\(1, 100\\)"):
        image.check_image(d, (1, 100))


def test_jpeg_keeps_its_slot_in_an_image_slot():
    """A JPEG of more than H * W * 3 bytes is refused with check_jpeg's message although the image slot, a PNG slot, would
    hold it; a PNG over that slot is refused with check_png's."""
    d = next(p for p in JPEG_FILES if p.name.startswith("photo_223x225_420")).read_bytes()
    info = jpeg.parse(d)
    H, W = info.h, info.w
    big = d + bytes(H * W * 3 + 1 - len(d))                             # trailing bytes after EOI: the same image
    assert len(big) < png.slot_bytes(H, W)
    assert image.check_image(d, (H, W))[1] == "jpeg"
    with pytest.raises(ValueError, match=re.escape(f"larger than the compressed slot of max_image_size=({H}, {W}) "
                                                   f"({H * W * 3} bytes)")):
        image.check_image(big, (H, W))
    p = PNG_FILES[0].read_bytes()
    pinfo = png.parse(p)
    over = p + bytes(png.slot_bytes(pinfo.h, pinfo.w) + 1 - len(p))
    with pytest.raises(ValueError, match="larger than the compressed slot"):
        image.check_image(over, (pinfo.h, pinfo.w))


# ------------------------------------------------------------------------------------------------ option rules
def test_image_decode_option_checks():
    from defer_b200.dispatcher import DEFER
    jpeg.check_decode("image", "caffe", None, (8, 8), image.DECODES)
    for kw in ({"preprocess": "caffe"}, {"max_image_size": (8, 8)}):
        with pytest.raises(ValueError, match="needs preprocess= and max_image_size="):
            jpeg.check_decode("image", kw.get("preprocess"), None, kw.get("max_image_size"), image.DECODES)
    with pytest.raises(ValueError, match="each image file carries its own size"):
        jpeg.check_decode("image", "caffe", (8, 8), (8, 8), image.DECODES)
    with pytest.raises(ValueError, match="the GPU decodes 'jpeg', 'png' files"):
        jpeg.check_decode("image", "caffe", None, (8, 8), png.DECODES)
    assert jpeg.DECODES == ("jpeg",) and png.DECODES == ("jpeg", "png")
    assert image.DECODES == ("jpeg", "png", "image")
    assert DEFER([0], preprocess="caffe", max_image_size=(8, 8), decode="image").decode == "image"
    with pytest.raises(ValueError, match="one JPEG or PNG file, so batch must be 1"):
        DEFER([0], preprocess="caffe", max_image_size=(8, 8), decode="image", batch=2)
    with pytest.raises(ValueError, match="image_size"):
        DEFER([0], preprocess="caffe", image_size=(8, 8), max_image_size=(8, 8), decode="image")
    with pytest.raises(ValueError, match="needs preprocess="):
        DEFER([0], max_image_size=(8, 8), decode="image")


# ------------------------------------------------------------------------------------------------ plans
@pytest.mark.parametrize("keep,interpolation", [(False, "nearest"), (True, "bicubic")])
def test_image_plan_is_the_jpeg_plan_but_its_decode(keep, interpolation):
    from defer_b200.planner import plan_stage
    m = applications.ResNet50(input_shape=(32, 32, 3))
    kw = dict(is_first=True, is_last=True, preprocess="caffe", max_image_size=(40, 60), interpolation=interpolation,
              keep_aspect_ratio=keep)
    pj = plan_stage(m, decode="jpeg", **kw)
    pi = plan_stage(m, decode="image", **kw)
    assert pi.decode == "image" and pi.ops[0].kind == A.OP_IMAGE_DECODE and pj.ops[0].kind == A.OP_JPEG_DECODE
    assert pi.ops[0].layers == ["load_img(decode image <=40x60)"]
    assert pi.bufs[pi.input_buf] == (40, 60, 3, A.BUF_IMAGE)
    assert [b for i, b in enumerate(pi.bufs) if i != pi.input_buf] == [b for i, b in enumerate(pj.bufs) if i != pj.input_buf]

    def op(o):
        return (o.in0, o.in1, o.out, o.kh, o.kw, o.sh, o.sw, tuple(o.pads), o.flags, o.w_kernel, o.w_scale, o.w_shift,
                o.mode)
    assert [op(o) for o in pi.ops] == [op(o) for o in pj.ops]
    assert [(o.kind, o.layers) for o in pi.ops[1:]] == [(o.kind, o.layers) for o in pj.ops[1:]]
    assert pi.frames == pj.frames and pi.tensor_buf == pj.tensor_buf
    assert pi.input_shape == pj.input_shape and pi.output_shape == pj.output_shape
    assert all(np.array_equal(a, b) for a, b in zip(pi.weights, pj.weights)) and len(pi.weights) == len(pj.weights)


def test_single_format_plans_are_unchanged():
    from image_plan_fingerprints import fingerprints
    want = json.loads((GOLDEN / "image_plan_fingerprints.json").read_text())
    assert fingerprints() == want


# ------------------------------------------------------------------------------------------------ blocks
def test_header_constants():
    assert _define("DEFER_IMAGE_TAG") == image.TAG == 15
    assert (_define("DEFER_IMAGE_JPEG"), _define("DEFER_IMAGE_PNG")) == (image.TAG_JPEG, image.TAG_PNG) == (1, 2)
    assert _define("DEFER_BUF_IMAGE") == A.BUF_IMAGE == 5
    assert re.search(r"DEFER_OP_IMAGE_DECODE = (\d+)", HEADER).group(1) == str(A.OP_IMAGE_DECODE) == "15"
    assert image.BLOCK_INTS == max(jpeg.BLOCK_INTS, png.BLOCK_INTS) == 31196
    assert image.TAG < jpeg.Q_OFF and image.TAG < png.HDR_INTS                   # inside both headers


def test_blocks_carry_the_tag_and_their_format_layout():
    """The tag is in [15], which both single-format layouts leave zero; the rest is the format's own block, and the
    prefix a file uses (what defer_stage_submit_images copies) holds all of it."""
    seen = set()
    for paths, kind, mod in ((JPEG_FILES, "jpeg", jpeg), (PNG_FILES, "png", png)):
        for p in paths:
            d, k, info = image.check_image(p.read_bytes(), (1080, 1920))
            own = mod.pack_block(info)
            assert own[image.TAG] == 0, p.name
            b = image.pack_block(k, info)
            assert b.shape == (image.BLOCK_INTS,) and b[image.TAG] == image.TAGS[kind], p.name
            used = image.block_ints(k, info)
            assert used == mod.block_ints(info), p.name
            want = own.copy()
            want[image.TAG] = image.TAGS[kind]
            assert np.array_equal(b[:len(own)], want) and not b[len(own):].any(), p.name
            assert not want[used:].any(), p.name                              # nothing past the copied prefix
            seen.add((kind, used == jpeg.BASE_INTS if kind == "jpeg" else used == png.IDAT_OFF + 2 * len(info.idat)))
            out = np.zeros(image.BLOCK_INTS, np.int32)
            assert image.pack_block(k, info, out) is out and np.array_equal(out, b)
    assert ("jpeg", True) in seen and ("jpeg", False) in seen and seen >= {("png", True)}   # baseline, progressive, PNG


# ------------------------------------------------------------------------------------------------ workspace
@pytest.mark.parametrize("H,W", [(1, 1), (23, 25), (480, 640), (1080, 1920), (255, 3)])
def test_image_workspace_stride(H, W):
    lib = A.load()
    total, stride, coef, plane, raw = (C.c_uint64() for _ in range(5))
    A.check(lib.defer_k_image_workspace(H, W, 3, *(C.byref(v) for v in (total, stride, coef, plane, raw))))
    js, jc, jp, ps, pr = (C.c_uint64() for _ in range(5))
    A.check(lib.defer_k_jpeg_workspace(H, W, 1, None, C.byref(js), C.byref(jc), C.byref(jp)))
    A.check(lib.defer_k_png_workspace(H, W, 1, None, C.byref(ps), C.byref(pr)))
    s = stride.value
    assert s >= js.value and s >= ps.value and s <= (max(js.value, ps.value) + 255) // 256 * 256
    assert s % 256 == 0 and total.value == 3 * s
    assert (coef.value, plane.value, raw.value) == (jc.value, jp.value, pr.value)


def test_image_entry_points_refuse_bad_arguments():
    lib = A.load()
    assert lib.defer_k_image_workspace(0, 8, 1, None, None, None, None, None) == A.ERR_INVALID
    assert lib.defer_k_image_workspace(20000, 20000, 1, None, None, None, None, None) == A.ERR_INVALID   # jpeg bound
    assert lib.defer_k_image_decode(None, None, 1, 8, 8, None, None, None) == A.ERR_INVALID
    assert lib.defer_stage_submit_images(None, 0, 0, 1, None, None, None, 0) == A.ERR_INVALID
