"""JPEG and PNG files in one pipeline, told apart per file: the sniff, the checks and the per-sample block of
``DEFER(decode="image")``, and ``decode_image``, the host restatement that the GPU decode (``DEFER_OP_IMAGE_DECODE``) is
tested against.

``sniff`` tells a file's format from its first bytes, as ``PIL.Image.open`` does (the ``_accept`` of Pillow's JPEG and
PNG plugins), never from its name: a JPEG starts with FF D8 FF, a PNG with the 8-byte PNG signature.  Anything else is
refused with a ValueError that names its first bytes in hex.  A file that passes is checked by ``jpeg.check_jpeg`` or
``png.check_png`` unchanged, so every refusal of ``decode="jpeg"`` / ``"png"`` applies as it is.  In particular a JPEG
keeps its ``H * W * 3``-byte limit although the image slot, ``png.slot_bytes(H, W)``, is larger: the entropy decode's bit
positions are int32 (``jpeg_bound_ok`` in ``csrc/jpeg.cu``).

``decode_image(data)`` is ``jpeg.decode_jpeg`` or ``png.decode_png`` chosen by the same sniff, and so equals
``np.asarray(PIL.Image.open(io.BytesIO(data)).convert("RGB"))`` byte for byte for the files those accept.
"""
from __future__ import annotations

from typing import Optional, Tuple, Union

import numpy as np

from . import jpeg, png

# ------------------------------------------------------------------------------------------------------ block layout
# One sample's int32 block (include/defer_b200.h, DEFER_OP_IMAGE_DECODE): the file's JPEG or PNG block in that format's
# layout (jpeg.pack_block / png.pack_block), with its tag in [TAG].  Both layouts leave [TAG] zero, and the single-format
# decodes never read it.  Only the prefix a file uses is copied to the GPU (``block_ints``).
TAG = 15                          # DEFER_IMAGE_TAG
TAG_JPEG, TAG_PNG = 1, 2          # DEFER_IMAGE_JPEG, DEFER_IMAGE_PNG
BLOCK_INTS = max(jpeg.BLOCK_INTS, png.BLOCK_INTS)
TAGS = {"jpeg": TAG_JPEG, "png": TAG_PNG}

#: the formats ``DEFER(decode=...)`` / ``plan_stage`` take (``jpeg.check_decode(..., decodes=DECODES)``)
DECODES = png.DECODES + ("image",)

JPEG_MAGIC = b"\xff\xd8\xff"


def _as_bytes(data) -> bytes:
    # a bytearray, memoryview or array is copied: the H2D copy of the item is asynchronous, and the caller may change a
    # mutable buffer after putting it on the queue
    if isinstance(data, (bytes, bytearray, memoryview)):
        return bytes(data)
    if isinstance(data, np.ndarray) and data.dtype == np.uint8 and data.ndim == 1:
        return data.tobytes()
    raise ValueError(f"an image item is bytes, bytearray, memoryview or a 1-D uint8 array holding one JPEG or PNG file, "
                     f"got {type(data).__name__}" + (f" {data.dtype} {data.shape}" if isinstance(data, np.ndarray) else ""))


def sniff(data) -> str:
    """"jpeg" or "png": the format of one file, from its first bytes as Pillow's ``_accept`` functions tell it; or a
    ValueError naming the first bytes."""
    head = _as_bytes(data)[:8]
    if head == png.SIGNATURE:
        return "png"
    if head[:3] == JPEG_MAGIC:
        return "jpeg"
    seen = f"first bytes {head.hex(' ')}" if head else "an empty item"
    raise ValueError(f"image refused: neither a JPEG nor a PNG file ({seen})")


def check_image(data, max_image_size) -> Tuple[bytes, str, Union[jpeg.JpegInfo, png.PngInfo]]:
    """Queue item ``data`` of a ``decode="image"`` pipeline as (file bytes, "jpeg" or "png", parsed header), or a
    ValueError: the file is neither format, or its format's check (``jpeg.check_jpeg`` / ``png.check_png``) refuses it."""
    d = _as_bytes(data)
    kind = sniff(d)
    d, info = (jpeg.check_jpeg if kind == "jpeg" else png.check_png)(d, max_image_size)
    return d, kind, info


def block_ints(kind: str, info) -> int:
    """How much of its block a file uses: its format's prefix (``jpeg.block_ints`` / ``png.block_ints``)."""
    return jpeg.block_ints(info) if kind == "jpeg" else png.block_ints(info)


def pack_block(kind: str, info, out: Optional[np.ndarray] = None) -> np.ndarray:
    """One sample's int32 block (layout above); ``out``: a zeroed int32 [BLOCK_INTS] to write it into."""
    b = np.zeros(BLOCK_INTS, np.int32) if out is None else out
    if kind == "jpeg":
        jpeg.pack_block(info, b[:jpeg.BLOCK_INTS])
    else:
        png.pack_block(info, b[:png.BLOCK_INTS])
    b[TAG] = TAGS[kind]
    return b


def decode_image(data) -> np.ndarray:
    """Keras' ``load_img`` decode of one JPEG or PNG file, told by its first bytes: uint8 (h, w, 3), byte for byte what
    ``np.asarray(PIL.Image.open(io.BytesIO(data)).convert("RGB"))`` gives for the files ``jpeg.parse`` / ``png.parse``
    accept."""
    d = _as_bytes(data)
    return jpeg.decode_jpeg(d) if sniff(d) == "jpeg" else png.decode_png(d)
