"""zlib's C inflate, as an independent reference for ``png.inflate_restated`` on valid and corrupt streams.

``inflate_c(stream, limit)`` runs the system libz (the library Python's ``zlib`` module uses, bound here with ctypes so
that ``msg`` can be read): ``inflateInit_`` and one ``inflate(Z_FINISH)`` with ``avail_out = limit``.  It returns
(bytes produced, status), the status mapped onto the ``png.STATUS_*`` values the restatement reports:
  - ``limit`` bytes produced: OK, whatever zlib says of the stream after them (it decodes the next code before it
    finds no room, and checks the trailer), as the restatement reads nothing past a full image;
  - ``msg`` names the fault: ``MESSAGES``;
  - ``Z_STREAM_END`` or "incorrect data check": the final block ended first, SHORT (the restatement does not read the
    Adler-32 trailer);
  - ``Z_BUF_ERROR`` with no message: zlib waits for input, either inside the deflate data (EXHAUSTED) or for the trailer
    after the final block (SHORT).  ``data_type`` does not tell the two apart, so the stream is inflated again with four
    more bytes, the Adler-32 of the bytes produced: if the final block had ended, zlib reads them as the trailer and
    ends (or, when part of a trailer was there already, finds a bad check) with the same output; four bytes are too few
    to hold both the rest of a block and a trailer, so a stream cut inside the deflate data never does.

Skips the calling test when no libz is found.  Nothing here comes from any other project: it is the system zlib.
"""
from __future__ import annotations

import ctypes as C
import ctypes.util
import zlib
from typing import Tuple

import pytest

from defer_b200 import png

Z_OK, Z_STREAM_END, Z_BUF_ERROR, Z_FINISH = 0, 1, -5, 4

#: zlib's error messages (inflate.c, 1.2.x and 1.3) and the restatement's status for each
MESSAGES = {
    "invalid block type": png.STATUS_BAD_BLOCK,
    "invalid stored block lengths": png.STATUS_BAD_BLOCK,
    "too many length or distance symbols": png.STATUS_BAD_HEADER,
    "invalid code lengths set": png.STATUS_BAD_HEADER,
    "invalid bit length repeat": png.STATUS_BAD_HEADER,
    "invalid literal/lengths set": png.STATUS_BAD_HEADER,
    "invalid distances set": png.STATUS_BAD_HEADER,
    "invalid code -- missing end-of-block": png.STATUS_BAD_HEADER,
    "invalid literal/length code": png.STATUS_BAD_SYMBOL,
    "invalid distance code": png.STATUS_BAD_SYMBOL,
    "invalid distance too far back": png.STATUS_BAD_DISTANCE,
}
DATA_CHECK = "incorrect data check"


class ZStream(C.Structure):
    """``z_stream`` on LP64 (uInt 32 bits, uLong 64 bits)."""
    _fields_ = [("next_in", C.c_void_p), ("avail_in", C.c_uint), ("total_in", C.c_ulong),
                ("next_out", C.c_void_p), ("avail_out", C.c_uint), ("total_out", C.c_ulong),
                ("msg", C.c_char_p), ("state", C.c_void_p),
                ("zalloc", C.c_void_p), ("zfree", C.c_void_p), ("opaque", C.c_void_p),
                ("data_type", C.c_int), ("adler", C.c_ulong), ("reserved", C.c_ulong)]


_LIB = None


def lib():
    """The system libz, or a skip of the calling test."""
    global _LIB
    if _LIB is None:
        name = ctypes.util.find_library("z")
        if name is None:
            pytest.skip("no system libz")
        z = C.CDLL(name)
        z.zlibVersion.restype = C.c_char_p            # the default int return would truncate the pointer
        z.zlibVersion.argtypes = []
        z.inflateInit_.argtypes = [C.POINTER(ZStream), C.c_char_p, C.c_int]
        z.inflate.argtypes = [C.POINTER(ZStream), C.c_int]
        z.inflateEnd.argtypes = [C.POINTER(ZStream)]
        assert C.sizeof(ZStream) == 112
        _LIB = z
    return _LIB


def version() -> str:
    return lib().zlibVersion().decode()


def inflate_raw(stream: bytes, limit: int) -> Tuple[bytes, int, str]:
    """One ``inflate(Z_FINISH)`` of the zlib ``stream`` into ``limit`` bytes: (bytes produced, return code, msg)."""
    z = lib()
    s = ZStream()
    src = C.create_string_buffer(stream, max(1, len(stream)))
    dst = C.create_string_buffer(max(1, limit))
    assert z.inflateInit_(C.byref(s), z.zlibVersion(), C.sizeof(ZStream)) == Z_OK
    try:
        s.next_in, s.avail_in = C.addressof(src), len(stream)
        s.next_out, s.avail_out = C.addressof(dst), limit
        ret = z.inflate(C.byref(s), Z_FINISH)
        msg = s.msg.decode() if s.msg else ""
        return dst.raw[:s.total_out], ret, msg
    finally:
        z.inflateEnd(C.byref(s))


def inflate_c(stream: bytes, limit: int) -> Tuple[bytes, int]:
    """zlib's inflate of ``stream``, at most ``limit`` bytes: (bytes produced, status mapped as the module docstring
    says)."""
    out, ret, msg = inflate_raw(stream, limit)
    if len(out) == limit:
        return out, png.STATUS_OK
    if ret == Z_STREAM_END or msg == DATA_CHECK:
        return out, png.STATUS_SHORT
    if msg:
        if msg not in MESSAGES:
            raise AssertionError(f"zlib message {msg!r} has no status")
        return out, MESSAGES[msg]
    assert ret == Z_BUF_ERROR, (ret, msg)
    again, ret2, msg2 = inflate_raw(stream + zlib.adler32(out).to_bytes(4, "big"), limit)
    if again == out and (ret2 == Z_STREAM_END or msg2 == DATA_CHECK):
        return out, png.STATUS_SHORT
    return out, png.STATUS_EXHAUSTED
