"""Non-interlaced PNG files at ingress: the chunk parser and per-sample block of ``DEFER(decode="png")``, and
``decode_png``, the host restatement that the GPU decode (``DEFER_OP_PNG_DECODE``) is tested against.

``decode_png(data)`` equals ``np.asarray(PIL.Image.open(io.BytesIO(data)).convert("RGB"))`` byte for byte for the files
``parse`` accepts: colour types 0, 2, 3, 4 and 6 at every bit depth the PNG specification allows for them.  The
conversion to RGB is Pillow's, not the specification's:
  - grey at 1 bit opens as mode "1" (0 or 255); at 2 and 4 bits it is scaled by 85 and 17; at 16 bits it opens as "I;16"
    and ``convert("RGB")`` clips the 16-bit value to 255 (it does not take the high byte);
  - RGB, grey+alpha and RGBA at 16 bits keep the high byte of each sample (Pillow's ``;16B`` unpackers);
  - grey+alpha gives R = G = B = grey; alpha (types 4 and 6) and any tRNS chunk are dropped by ``convert("RGB")``;
  - a palette index at or past the PLTE length gives black (0, 0, 0).

The feeder walks chunk headers only and never inflates (``parse``): it reads IHDR and PLTE, the two zlib header bytes
and the position of every IDAT chunk, and the device gathers the zlib stream from those ranges itself.  The zlib
stream is the first run of consecutive IDAT chunks, as Pillow reads it.  CRCs are checked as Pillow checks them: every
chunk before the first IDAT (IHDR, PLTE and ancillary chunks alike) must have a correct CRC; IDAT chunks and everything
after them are not checked, as Pillow does not check them.  Ancillary chunks are skipped.

Refused with a ValueError that names the reason: a missing or wrong signature, a missing, malformed or misplaced IHDR,
a colour type / bit depth pair the specification does not define, compression or filter method other than 0, Adam7
interlace, APNG (acTL, fcTL or fdAT chunks), a palette image without PLTE or with a PLTE that is empty, over 256 entries
or not whole RGB triples, a PLTE after IDAT or a second one, a missing IDAT or IDAT chunks that are not consecutive, an
unknown critical chunk, a chunk that runs past the end of the file, a bad CRC before the first IDAT, a bad zlib header
(CM != 8, a window over 32 KiB, FDICT set, or a header check that fails), more than ``MAX_IDAT`` IDAT chunks, an image
outside ``max_image_size`` and a file larger than the compressed slot (``slot_bytes``).  Pillow decodes some of these
(an unknown critical chunk, a palette image without PLTE); they are refused here because their pixels are not defined
by the specification.

Corrupt compressed data has one defined result here, and the device computes the same (there is no promise to match
zlib or Pillow on it, which raise).  The inflate follows zlib's rules for what is valid; the first of these ends the
stream, and everything the stream produced before it stays:
  - a block type 3, or a stored block whose LEN and NLEN disagree;
  - a dynamic header with more than 286 literal/length or 30 distance codes, a code-length code that is incomplete or
    over-subscribed, a repeat code 16 with no previous length, a repeat past the last length, no code for
    end-of-block, or a literal/length or distance code that is over-subscribed, or incomplete with a longest code
    other than one bit (one-code trees are valid, as in zlib; so is a distance code with no codes, until it is used);
  - a bit pattern that is no code of its table, a literal/length symbol 286 or 287, a distance symbol 30 or 31;
  - a distance past the bytes produced so far;
  - input exhausted before the final block: the bits of the gathered IDAT data run out inside a field or code, which
    is then not applied (bits past the end read as zero while a code is looked up).
The stream also ends, normally, when the output holds ``h * (1 + bytes per row)`` bytes: a match is cut there and
whatever follows is not read, as Pillow stops reading once the image is full.  The Adler-32 trailer is not checked.
Against zlib's ``inflate()`` given the same input and room for the image, this result differs in four cases only
(tests/test_png_zlib_host.py checks that nothing else differs):
  (a) a stored block whose data runs past the end of the input produces none of its bytes here (EXHAUSTED); zlib
      produces the bytes that are there, and so fills the image when they reach its end;
  (b) a dynamic header whose code-length code has no codes at all is refused at once (BAD_HEADER); zlib decodes each
      of the HLIT + HDIST lengths as 0 from one bit and refuses the header for its missing end-of-block code;
  (c) a repeat code 16 as the first code length is refused before its two extra bits are read (BAD_HEADER); zlib reads
      them first;
  (d) a distance code with no codes is refused when used, before any bit of the distance is read (BAD_SYMBOL); zlib
      reads one bit first.
In (b), (c) and (d) the bytes produced are the same and the status differs only when the input ends first, where zlib
still waits for input (EXHAUSTED).
The scanline bytes not produced are zero, and the unfilter and the conversion run over them as over the others.  A
filter type byte above 4 makes its row unfiltered as type 0 (None).

Per sample the device records ``stats``: [0] status (``STATUS_*``), [1] scanline bytes produced, [2] rows with a
filter type above 4.
"""
from __future__ import annotations

import zlib
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np

# ------------------------------------------------------------------------------------------------------ block layout
# One sample's int32 block (include/defer_b200.h, DEFER_OP_PNG_DECODE):
#   [0] h  [1] w  [2] colour type  [3] bit depth  [4] bytes per row (without the filter byte)  [5] filter unit (bytes
#   per complete pixel, at least 1)  [6] IDAT chunks  [7] zlib stream bytes (their total)  [8] PLTE entries  [9..15] 0
#   [PAL_OFF + i]               palette entry i < 256 as r | g << 8 | b << 16, zero past the PLTE length
#   [IDAT_OFF + 2 k, + 1]       IDAT chunk k: payload offset in the file, payload length
# Only the prefix a file uses is copied to the GPU (``block_ints``).
HDR_INTS = 16
PAL_OFF = HDR_INTS
IDAT_OFF = PAL_OFF + 256
MAX_IDAT = 4096                   # DEFER_PNG_MAX_IDAT: IDAT chunks of one file (libpng writes 8 KiB chunks)
BLOCK_INTS = IDAT_OFF + 2 * MAX_IDAT
MAX_BYTES_PER_PIXEL = 8           # RGBA at 16 bits

STATUS_OK = 0                     # the scanlines are complete
STATUS_SHORT = 1                  # the final block ended first: the rest is zero
STATUS_EXHAUSTED = 2              # the input ran out before the final block
STATUS_BAD_BLOCK = 3              # block type 3, or a stored block's LEN != ~NLEN
STATUS_BAD_HEADER = 4             # a dynamic block header zlib refuses
STATUS_BAD_SYMBOL = 5             # no code of its table, or a literal/length symbol 286-287 or distance 30-31
STATUS_BAD_DISTANCE = 6           # a distance past the bytes produced

#: the single-format decodes (``image.DECODES`` adds "image", what ``DEFER(decode=...)`` / ``plan_stage`` take)
DECODES = ("jpeg", "png")

SIGNATURE = b"\x89PNG\r\n\x1a\n"
_DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
_CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def slot_bytes(H: int, W: int) -> int:
    """Bytes of one sample's compressed slot for images up to (H, W) (DEFER_PNG_SLOT_BYTES): the stored-block (level 0)
    encoding of the largest accepted image, ``H * (1 + 8 W)`` scanline bytes, plus 1/64 of that for stored-block and
    IDAT chunk headers (a 5-byte block header per 320 bytes, a 12-byte chunk per 768) and 64 KiB for the signature,
    IHDR, PLTE and ancillary chunks."""
    raw = H * (1 + MAX_BYTES_PER_PIXEL * W)
    return raw + raw // 64 + 65536


@dataclass(frozen=True)
class PngInfo:
    h: int
    w: int
    ctype: int
    depth: int
    idat: Tuple[Tuple[int, int], ...]   # (payload offset, length) of each IDAT chunk of the zlib stream
    palette: Optional[np.ndarray] = None  # uint8 [n, 3] of a palette image

    @property
    def bytes_per_row(self) -> int:
        return (self.w * _CHANNELS[self.ctype] * self.depth + 7) // 8

    @property
    def filter_unit(self) -> int:
        return max(1, _CHANNELS[self.ctype] * self.depth // 8)

    @property
    def raw_bytes(self) -> int:
        return self.h * (1 + self.bytes_per_row)

    @property
    def stream_bytes(self) -> int:
        return sum(n for _, n in self.idat)


def _refuse(why: str):
    raise ValueError(f"PNG refused: {why}")


def _as_bytes(data) -> bytes:
    # a bytearray, memoryview or array is copied: the H2D copy of the item is asynchronous, and the caller may change a
    # mutable buffer after putting it on the queue
    if isinstance(data, (bytes, bytearray, memoryview)):
        return bytes(data)
    if isinstance(data, np.ndarray) and data.dtype == np.uint8 and data.ndim == 1:
        return data.tobytes()
    raise ValueError(f"a PNG item is bytes, bytearray, memoryview or a 1-D uint8 array holding one file, got "
                     f"{type(data).__name__}" + (f" {data.dtype} {data.shape}" if isinstance(data, np.ndarray) else ""))


def parse(data) -> PngInfo:
    """Walk the chunk headers of one PNG file: its geometry, palette and IDAT ranges, or a ValueError naming why the file
    is refused.  Nothing is inflated: of the compressed data only the two zlib header bytes are read."""
    d = _as_bytes(data)
    n = len(d)
    if d[:8] != SIGNATURE:
        _refuse("not a PNG file (no PNG signature)")
    p, ihdr, palette, idat = 8, None, None, []
    idat_done = False                      # the run of IDAT chunks has ended
    while True:
        if p == n and idat:
            break                          # no IEND: Pillow decodes what the IDAT chunks hold
        if p + 8 > n:
            if idat:                       # a torn chunk after the image data is not read, as Pillow does not read it
                break
            _refuse("truncated file (a chunk header runs past the end of the file)")
        ln = int.from_bytes(d[p:p + 4], "big")
        ct = d[p + 4:p + 8]
        if not all(65 <= c <= 90 or 97 <= c <= 122 for c in ct):
            if idat:
                break
            _refuse(f"malformed chunk type {ct!r} at byte {p}")
        name = ct.decode("ascii")
        if ln > 0x7FFFFFFF or p + 12 + ln > n:
            if idat and ct != b"IDAT":
                break
            _refuse(f"chunk {name} of length {ln} runs past the end of the file")
        body = d[p + 8:p + 8 + ln]
        if not idat and ct != b"IDAT" and int.from_bytes(d[p + 8 + ln:p + 12 + ln], "big") != zlib.crc32(ct + body):
            _refuse(f"bad CRC of chunk {name}")
        if ihdr is None and ct != b"IHDR":
            _refuse(f"missing IHDR (the first chunk is {name})")
        if ct == b"IHDR":
            if ihdr is not None:
                _refuse("malformed IHDR (a second IHDR chunk)")
            if ln != 13:
                _refuse(f"malformed IHDR (length {ln}, not 13)")
            w, h = int.from_bytes(body[0:4], "big"), int.from_bytes(body[4:8], "big")
            depth, ctype, comp, filt, inter = body[8:13]
            if w == 0 or h == 0 or w > 0x7FFFFFFF or h > 0x7FFFFFFF:
                _refuse(f"malformed IHDR (image size {w}x{h})")
            if ctype not in _DEPTHS or depth not in _DEPTHS[ctype]:
                _refuse(f"malformed IHDR (colour type {ctype} with bit depth {depth})")
            if comp != 0 or filt != 0:
                _refuse(f"malformed IHDR (compression method {comp}, filter method {filt})")
            if inter == 1:
                _refuse("Adam7 interlace (only non-interlaced PNGs are decoded)")
            if inter != 0:
                _refuse(f"malformed IHDR (interlace method {inter})")
            ihdr = (h, w, ctype, depth)
        elif ct == b"PLTE":
            if idat:
                _refuse("malformed PLTE (after IDAT)")
            if palette is not None:
                _refuse("malformed PLTE (a second PLTE chunk)")
            if ihdr[2] == 3 and (ln == 0 or ln % 3 or ln > 768):
                _refuse(f"malformed PLTE (length {ln}: 1 to 256 RGB entries)")
            palette = np.frombuffer(body, np.uint8)[:ln // 3 * 3].reshape(-1, 3)
        elif ct == b"IDAT":
            if idat_done:
                _refuse("IDAT chunks are not consecutive")
            idat.append((p + 8, ln))
        elif ct in (b"acTL", b"fcTL", b"fdAT"):
            _refuse(f"APNG ({name} chunk; animated PNGs are not decoded)")
        elif ct == b"IEND":
            break
        elif not (ct[0] & 0x20):
            _refuse(f"unknown critical chunk {name}")
        if idat and ct != b"IDAT":
            idat_done = True
        p += 12 + ln
    if ihdr is None:
        _refuse("missing IHDR")
    if not idat:
        _refuse("missing IDAT")
    if len(idat) > MAX_IDAT:
        _refuse(f"{len(idat)} IDAT chunks, more than DEFER_PNG_MAX_IDAT = {MAX_IDAT}")
    h, w, ctype, depth = ihdr
    if ctype == 3 and palette is None:
        _refuse("missing PLTE (a palette image needs one)")
    head = b"".join(d[o:o + k] for o, k in idat[:2])[:2]
    if len(head) < 2:
        head = b"".join(d[o:o + k] for o, k in idat)[:2]
    if len(head) < 2:
        _refuse("bad zlib header (the IDAT data holds fewer than 2 bytes)")
    cmf, flg = head
    if cmf & 15 != 8:
        _refuse(f"bad zlib header (compression method {cmf & 15}, not 8 = deflate)")
    if cmf >> 4 > 7:
        _refuse(f"bad zlib header (window of 2^{(cmf >> 4) + 8} bytes, over 32 KiB)")
    if flg & 0x20:
        _refuse("bad zlib header (FDICT set: a preset dictionary)")
    if ((cmf << 8) | flg) % 31:
        _refuse("bad zlib header (header check FCHECK fails)")
    return PngInfo(h, w, ctype, depth, tuple(idat), palette if ctype == 3 else None)


def block_ints(info: PngInfo) -> int:
    """How much of its block a file uses: the header, the palette and its IDAT ranges."""
    return IDAT_OFF + 2 * len(info.idat)


def pack_block(info: PngInfo, out: Optional[np.ndarray] = None) -> np.ndarray:
    """One sample's int32 block (layout above); ``out``: a zeroed int32 [BLOCK_INTS] to write it into."""
    b = np.zeros(BLOCK_INTS, np.int32) if out is None else out
    npal = 0 if info.palette is None else len(info.palette)
    b[:9] = (info.h, info.w, info.ctype, info.depth, info.bytes_per_row, info.filter_unit, len(info.idat),
             info.stream_bytes, npal)
    if npal:
        pal = info.palette.astype(np.int32)
        b[PAL_OFF:PAL_OFF + npal] = pal[:, 0] | (pal[:, 1] << 8) | (pal[:, 2] << 16)
    if info.idat:
        b[IDAT_OFF:IDAT_OFF + 2 * len(info.idat)] = np.array(info.idat, np.int64).reshape(-1)
    return b


def check_png(data, max_image_size) -> Tuple[bytes, PngInfo]:
    """Queue item ``data`` of a ``decode="png"`` pipeline as (file bytes, parsed header), or a ValueError: the file is
    refused, its image is outside ``max_image_size=(H, W)``, or it is larger than the compressed slot
    (``slot_bytes(H, W)``)."""
    d = _as_bytes(data)
    H, W = max_image_size
    if len(d) > slot_bytes(H, W):
        _refuse(f"a {len(d)}-byte file is larger than the compressed slot of max_image_size=({H}, {W}) "
                f"({slot_bytes(H, W)} bytes)")
    info = parse(d)
    if not (info.h <= H and info.w <= W):
        _refuse(f"a {info.h}x{info.w} image is outside max_image_size=({H}, {W})")
    return d, info


# ------------------------------------------------------------------------------------------------ the host decoder
LBASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258)
LEXT = (0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0)
DBASE = (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
         6145, 8193, 12289, 16385, 24577)
DEXT = (0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13)
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)


class _Stop(Exception):
    def __init__(self, status: int):
        self.status = status


class _Huffman:
    """A canonical code as puff.c decodes it: counts per length and the symbols in canonical order."""

    def __init__(self, lens, codes: bool = False):
        self.count = [0] * 16
        for v in lens:
            self.count[v] += 1
        self.count[0] = 0
        left = 1
        for ln in range(1, 16):
            left = 2 * left - self.count[ln]
            if left < 0:
                raise _Stop(STATUS_BAD_HEADER)                     # over-subscribed
        longest = max([ln for ln in range(1, 16) if self.count[ln]], default=0)
        if codes and longest == 0:
            raise _Stop(STATUS_BAD_HEADER)                         # a code-length code with no codes
        if left > 0 and longest != 0 and (codes or longest != 1):
            raise _Stop(STATUS_BAD_HEADER)                         # incomplete (zlib's inflate_table rule)
        offs = [0] * 16
        for ln in range(1, 15):
            offs[ln + 1] = offs[ln] + self.count[ln]
        self.symbol = [0] * len(lens)
        for s, v in enumerate(lens):
            if v:
                self.symbol[offs[v]] = s
                offs[v] += 1


class _Bits:
    def __init__(self, data: bytes):
        self.data = data
        self.nbits = 8 * len(data)
        self.pos = 16                                              # past the zlib header

    def peek(self, n: int) -> int:                                 # n <= 16; bits past the end read as zero
        q = self.pos >> 3
        return (int.from_bytes(self.data[q:q + 4], "little") >> (self.pos & 7)) & ((1 << n) - 1)

    def take(self, n: int) -> int:
        if self.pos + n > self.nbits:
            raise _Stop(STATUS_EXHAUSTED)
        r = self.peek(n)
        self.pos += n
        return r

    def decode(self, h: _Huffman) -> int:
        v = self.peek(15)
        code = first = index = 0
        for ln in range(1, 16):
            code |= (v >> (ln - 1)) & 1
            count = h.count[ln]
            if code - first < count:
                if self.pos + ln > self.nbits:
                    raise _Stop(STATUS_EXHAUSTED)
                self.pos += ln
                return h.symbol[index + code - first]
            index += count
            first = (first + count) << 1
            code <<= 1
        raise _Stop(STATUS_BAD_SYMBOL)


def _fixed():
    lens = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
    return _Huffman(lens), _Huffman([5] * 32)


def _dynamic(r: _Bits):
    hlit, hdist, hclen = r.take(5) + 257, r.take(5) + 1, r.take(4) + 4
    if hlit > 286 or hdist > 30:
        raise _Stop(STATUS_BAD_HEADER)
    cl = [0] * 19
    for i in range(hclen):
        cl[CL_ORDER[i]] = r.take(3)
    clh = _Huffman(cl, codes=True)
    lens = []
    while len(lens) < hlit + hdist:
        sym = r.decode(clh)
        if sym < 16:
            lens.append(sym)
            continue
        if sym == 16:
            if not lens:
                raise _Stop(STATUS_BAD_HEADER)
            val, rep = lens[-1], 3 + r.take(2)
        elif sym == 17:
            val, rep = 0, 3 + r.take(3)
        else:
            val, rep = 0, 11 + r.take(7)
        if len(lens) + rep > hlit + hdist:
            raise _Stop(STATUS_BAD_HEADER)
        lens += [val] * rep
    if lens[256] == 0:
        raise _Stop(STATUS_BAD_HEADER)
    return _Huffman(lens[:hlit]), _Huffman(lens[hlit:])


def inflate_restated(stream: bytes, limit: int) -> Tuple[bytes, int]:
    """The device's inflate of the gathered zlib ``stream``, at most ``limit`` bytes: (bytes produced, status).  Byte
    for byte zlib's output on valid data; on corrupt data the rule of the module docstring."""
    r = _Bits(stream)
    out = bytearray()
    try:
        while True:
            final = r.take(1)
            btype = r.take(2)
            if btype == 0:
                r.pos = (r.pos + 7) & ~7
                ln, nln = r.take(16), r.take(16)
                if ln != (~nln & 0xFFFF):
                    raise _Stop(STATUS_BAD_BLOCK)
                if r.pos + 8 * ln > r.nbits:
                    raise _Stop(STATUS_EXHAUSTED)
                q = r.pos >> 3
                out += stream[q:q + min(ln, limit - len(out))]
                r.pos += 8 * ln
                if len(out) == limit:
                    return bytes(out), STATUS_OK
            elif btype == 3:
                raise _Stop(STATUS_BAD_BLOCK)
            else:
                lit, dist = _fixed() if btype == 1 else _dynamic(r)
                while True:
                    sym = r.decode(lit)
                    if sym < 256:
                        out.append(sym)
                        if len(out) == limit:
                            return bytes(out), STATUS_OK
                        continue
                    if sym == 256:
                        break
                    sym -= 257
                    if sym >= 29:
                        raise _Stop(STATUS_BAD_SYMBOL)
                    length = LBASE[sym] + r.take(LEXT[sym])
                    ds = r.decode(dist)
                    if ds >= 30:
                        raise _Stop(STATUS_BAD_SYMBOL)
                    d = DBASE[ds] + r.take(DEXT[ds])
                    if d > len(out):
                        raise _Stop(STATUS_BAD_DISTANCE)
                    n = min(length, limit - len(out))
                    start = len(out) - d
                    for i in range(n):
                        out.append(out[start + i % d] if i >= d else out[start + i])
                    if len(out) == limit:
                        return bytes(out), STATUS_OK
            if final:
                return bytes(out), STATUS_SHORT
    except _Stop as e:
        return bytes(out), e.status


def gather(data: bytes, info: PngInfo) -> bytes:
    """The zlib stream: the IDAT payloads, in order."""
    return b"".join(data[o:o + n] for o, n in info.idat)


def inflate(data: bytes, info: PngInfo) -> Tuple[bytes, int]:
    """``inflate_restated`` of the file's stream: (bytes produced, status).  zlib gives the bytes whenever it decodes
    the stream without an error (the restatement equals it there, and is much slower); else the restatement does."""
    stream = gather(data, info)
    limit = info.raw_bytes
    try:
        z = zlib.decompressobj()
        out = z.decompress(stream, limit)
        if len(out) == limit:
            return out, STATUS_OK
        if z.eof:
            return out, STATUS_SHORT
    except zlib.error:
        pass
    return inflate_restated(stream, limit)


def _paeth(a: int, b: int, c: int) -> int:
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def unfilter(raw: bytes, info: PngInfo) -> Tuple[np.ndarray, int]:
    """The scanlines (uint8 [h, bytes per row]) and the number of rows with a filter type above 4 (unfiltered as None),
    of ``raw`` zero-extended to ``h * (1 + bytes per row)`` bytes."""
    bpr, bpp = info.bytes_per_row, info.filter_unit
    buf = np.zeros(info.raw_bytes, np.uint8)
    buf[:len(raw)] = np.frombuffer(raw, np.uint8)
    rows = buf.reshape(info.h, 1 + bpr)
    out = np.zeros((info.h, bpr), np.uint8)
    prev = np.zeros(bpr, np.uint8)
    unknown = 0
    for y in range(info.h):
        ft, cur = int(rows[y, 0]), rows[y, 1:].copy()
        if ft == 1:                                            # bpr is a multiple of bpp
            cur = np.cumsum(cur.reshape(-1, bpp), axis=0, dtype=np.uint8).reshape(-1)
        elif ft == 2:
            cur = (cur.astype(np.uint16) + prev).astype(np.uint8)
        elif ft == 3:
            c, up = bytearray(cur.tobytes()), prev.tobytes()
            for x in range(bpr):
                left = c[x - bpp] if x >= bpp else 0
                c[x] = (c[x] + ((left + up[x]) >> 1)) & 255
            cur = np.frombuffer(bytes(c), np.uint8)
        elif ft == 4:
            c, up = bytearray(cur.tobytes()), prev.tobytes()
            for x in range(bpr):
                a = c[x - bpp] if x >= bpp else 0
                cc = up[x - bpp] if x >= bpp else 0
                c[x] = (c[x] + _paeth(a, up[x], cc)) & 255
            cur = np.frombuffer(bytes(c), np.uint8)
        elif ft > 4:
            unknown += 1
        out[y] = cur
        prev = out[y]
    return out, unknown


def _samples(rows: np.ndarray, info: PngInfo, per_pixel: int) -> np.ndarray:
    """The samples of each row, uint16 [h, w * per_pixel] (sub-byte depths unpacked MSB first, 16 bits big-endian)."""
    d = info.depth
    if d == 16:
        v = rows.astype(np.uint16)
        return (v[:, 0::2] << 8) | v[:, 1::2]
    if d == 8:
        return rows.astype(np.uint16)
    bits = np.unpackbits(rows, axis=1).reshape(info.h, -1, d)
    v = np.zeros(bits.shape[:2], np.uint16)
    for k in range(d):
        v = (v << 1) | bits[:, :, k]
    return v[:, :info.w * per_pixel]


def to_rgb(rows: np.ndarray, info: PngInfo) -> np.ndarray:
    """Pillow's ``convert("RGB")`` of the scanlines in the file's mode and depth (module docstring)."""
    ch = _CHANNELS[info.ctype]
    s = _samples(rows, info, ch).reshape(info.h, info.w, ch)
    d = info.depth
    if info.ctype == 3:
        pal = np.zeros((256, 3), np.uint8)
        pal[:len(info.palette)] = info.palette
        return np.ascontiguousarray(pal[s[:, :, 0]])
    if d == 16:
        if info.ctype == 0:
            g = np.minimum(s[:, :, 0], 255).astype(np.uint8)
            return np.ascontiguousarray(np.repeat(g[:, :, None], 3, axis=2))
        s = s >> 8
    elif d < 8:
        s = s * {1: 255, 2: 85, 4: 17}[d]
    s = s.astype(np.uint8)
    if info.ctype in (0, 4):
        return np.ascontiguousarray(np.repeat(s[:, :, :1], 3, axis=2))
    return np.ascontiguousarray(s[:, :, :3])


def decode_stages(data) -> dict:
    """Every stage of the decode: ``info``, ``raw`` (the scanline bytes the inflate produced), ``rows`` (unfiltered),
    ``rgb``, and ``stats`` (the device's workspace counters, int32 [3])."""
    d = _as_bytes(data)
    info = parse(d)
    raw, status = inflate(d, info)
    rows, unknown = unfilter(raw, info)
    return {"info": info, "raw": raw, "rows": rows, "rgb": to_rgb(rows, info),
            "stats": np.array([status, len(raw), unknown], np.int32)}


def decode_png(data) -> np.ndarray:
    """Keras' ``load_img`` decode of one PNG file: uint8 (h, w, 3), C-contiguous, byte for byte what
    ``np.asarray(PIL.Image.open(io.BytesIO(data)).convert("RGB"))`` gives for the files ``parse`` accepts."""
    d = _as_bytes(data)
    info = parse(d)
    raw, _ = inflate(d, info)
    return to_rgb(unfilter(raw, info)[0], info)
