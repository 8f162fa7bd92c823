"""PNG files no encoder writes: a chunk writer, a small deflate bit writer, and a corpus of crafted streams.

``png_file`` wraps any zlib stream in a PNG of a given size, colour type and depth, split into IDAT chunks where asked.
``BitWriter`` writes deflate blocks bit by bit (stored, fixed Huffman, dynamic Huffman with any code lengths, and raw
header fields), so a test can build what zlib never emits: empty stored blocks, stored blocks that cross IDAT chunk
boundaries, matches at distance 32768 and length 258, an overlapping match, a dynamic header whose repeat codes span the
literal/length and distance lengths, one-code distance trees, and every corruption of the decode's defined result
(defer_b200/png.py)."""
from __future__ import annotations

import struct
import zlib
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from defer_b200 import png

CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def chunk(kind: bytes, body: bytes, crc: Optional[int] = None) -> bytes:
    c = zlib.crc32(kind + body) if crc is None else crc
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", c & 0xFFFFFFFF)


def ihdr(w: int, h: int, depth: int, ctype: int, interlace: int = 0) -> bytes:
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, interlace))


def png_file(w: int, h: int, depth: int, ctype: int, stream: bytes, idat_sizes: Sequence[int] = (),
             palette: Optional[bytes] = None, before: bytes = b"", after: bytes = b"") -> bytes:
    """A PNG of ``stream`` (a zlib stream) split into IDAT chunks of ``idat_sizes`` bytes (the rest in one more chunk);
    ``before`` / ``after``: raw chunks put before the first IDAT / after the last."""
    out = png.SIGNATURE + ihdr(w, h, depth, ctype)
    if palette is not None:
        out += chunk(b"PLTE", palette)
    out += before
    p = 0
    for n in idat_sizes:
        out += chunk(b"IDAT", stream[p:p + n])
        p += n
    if p < len(stream) or not idat_sizes:
        out += chunk(b"IDAT", stream[p:])
    return out + after + chunk(b"IEND", b"")


def bytes_per_row(w: int, depth: int, ctype: int) -> int:
    return (w * CHANNELS[ctype] * depth + 7) // 8


# ------------------------------------------------------------------------------------------------- deflate writer
class BitWriter:
    """Deflate bits, LSB first; ``zlib()`` adds the 2-byte header (and an Adler-32 of ``data`` when given)."""

    def __init__(self):
        self.bits: List[int] = []

    def put(self, v: int, n: int):
        self.bits += [(v >> i) & 1 for i in range(n)]

    def put_code(self, code: int, n: int):        # a Huffman code, MSB first
        self.bits += [(code >> (n - 1 - i)) & 1 for i in range(n)]

    def align(self):
        self.bits += [0] * (-len(self.bits) % 8)

    def tobytes(self) -> bytes:
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(sum(b[i + k] << k for k in range(8)) for i in range(0, len(b), 8))

    def zlib(self, data: Optional[bytes] = None) -> bytes:
        body = self.tobytes()
        return b"\x78\x01" + body + (struct.pack(">I", zlib.adler32(data)) if data is not None else b"")

    # ---- blocks
    def stored(self, data: bytes, final: bool = False, nlen: Optional[int] = None):
        self.put(int(final), 1)
        self.put(0, 2)
        self.align()
        self.put(len(data), 16)
        self.put((~len(data) & 0xFFFF) if nlen is None else nlen, 16)
        for c in data:
            self.put(c, 8)

    def huffman(self, items, final: bool = False, lit_lens: Optional[Sequence[int]] = None,
                dist_lens: Optional[Sequence[int]] = None, header: Optional[List[Tuple[int, int]]] = None):
        """A fixed block (no lengths given) or a dynamic one: ``items`` are literal ints, ('m', length, distance) matches,
        ('sym', s) raw literal/length symbols or ('dsym', s, extra, nbits) raw distance symbols; the block ends with
        end-of-block unless ``items`` ends with 'noeob'.  ``header``: dynamic code-length symbols as (symbol, extra)
        pairs instead of the plain ones written from ``lit_lens`` + ``dist_lens``."""
        dyn = lit_lens is not None
        self.put(int(final), 1)
        self.put(2 if dyn else 1, 2)
        if dyn:
            self._dynamic_header(list(lit_lens), list(dist_lens), header)
            lc, dc = canonical(lit_lens), canonical(dist_lens)
        else:
            lc, dc = canonical(FIXED_LIT), canonical([5] * 32)
        eob = True
        for it in items:
            if it == "noeob":
                eob = False
            elif isinstance(it, int):
                self.put_code(*lc[it])
            elif it[0] == "sym":
                self.put_code(*lc[it[1]])
            elif it[0] == "dsym":
                self.put_code(*dc[it[1]])
                self.put(it[2], it[3])
            else:
                _, length, dist = it
                s = max(i for i, b in enumerate(png.LBASE) if b <= length) if length < 258 else 28
                self.put_code(*lc[257 + s])
                self.put(length - png.LBASE[s], png.LEXT[s])
                d = max(i for i, b in enumerate(png.DBASE) if b <= dist)
                self.put_code(*dc[d])
                self.put(dist - png.DBASE[d], png.DEXT[d])
        if eob:
            self.put_code(*lc[256])

    def _dynamic_header(self, lit: List[int], dist: List[int], header):
        syms = header if header is not None else [(v, 0) for v in lit + dist]
        used = {s for s, _ in syms}
        # lengths of the code-length code: a complete code over the used symbols (at most 7 bits)
        cl_lens = complete_lengths(sorted(used), 7)
        cl = [cl_lens.get(i, 0) for i in range(19)]
        order = png.CL_ORDER
        hclen = max(i for i in range(19) if cl[order[i]]) + 1
        hclen = max(hclen, 4)
        self.put(len(lit) - 257, 5)
        self.put(len(dist) - 1, 5)
        self.put(hclen - 4, 4)
        for i in range(hclen):
            self.put(cl[order[i]], 3)
        cc = canonical(cl)
        for s, extra in syms:
            self.put_code(*cc[s])
            if s == 16:
                self.put(extra, 2)
            elif s == 17:
                self.put(extra, 3)
            elif s == 18:
                self.put(extra, 7)


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8


def canonical(lens: Sequence[int]) -> Dict[int, Tuple[int, int]]:
    """symbol -> (code, length) of the canonical code of ``lens``."""
    count = [0] * 16
    for v in lens:
        count[v] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = {}
    for s, v in enumerate(lens):
        if v:
            out[s] = (nxt[v], v)
            nxt[v] += 1
    return out


def complete_lengths(symbols: Sequence[int], maxlen: int) -> Dict[int, int]:
    """Code lengths of a complete code over ``symbols`` (a one-symbol set gets a 1-bit code plus an unused partner)."""
    n = len(symbols)
    if n == 1:
        return {symbols[0]: 1}
    k = (n - 1).bit_length()                       # 2^(k-1) < n <= 2^k
    short = 2 ** k - n                             # that many get k-1 bits, the rest k bits
    assert k <= maxlen
    return {s: (k - 1 if i < short else k) for i, s in enumerate(symbols)}


def lit_lengths_for(symbols: Sequence[int], n: int = 286) -> List[int]:
    lens = [0] * n
    for s, v in complete_lengths(sorted(set(symbols) | {256}), 15).items():
        lens[s] = v
    return lens


# ------------------------------------------------------------------------------------------------- the corpus
def _scan(w: int, h: int, depth: int, ctype: int, seed: int) -> bytes:
    """Scanlines with random filter types 0..4 and random bytes."""
    rng = np.random.default_rng(seed)
    bpr = bytes_per_row(w, depth, ctype)
    return b"".join(bytes([int(rng.integers(0, 5))]) + rng.integers(0, 256, bpr, dtype=np.uint8).tobytes()
                    for _ in range(h))


def valid_cases() -> Dict[str, bytes]:
    """Crafted files whose streams are valid: each decodes as Pillow decodes it."""
    out = {}
    raw = _scan(40, 20, 8, 2, 1)                                      # 20 rows of 121 bytes
    w = BitWriter()                                                   # empty stored blocks around the data
    w.stored(b"")
    w.stored(raw[:1000])
    w.stored(b"")
    w.stored(raw[1000:], final=True)
    z = w.zlib(raw)
    out["stored_empty_blocks"] = png_file(40, 20, 8, 2, z)
    out["stored_across_idat"] = png_file(40, 20, 8, 2, z, idat_sizes=[1, 3, 7, 500, 2, 900])
    out["idat_one_byte_chunks"] = png_file(40, 20, 8, 2, z, idat_sizes=[1] * 64)
    # a match at distance 32768 and one of length 258 (8-bit grey rows of 1 + 255 bytes, 33280 in all)
    w8, h8 = 255, 130
    rng = np.random.default_rng(2)
    head = rng.integers(0, 256, 32768, dtype=np.uint8)
    head[::256] %= 5                                                  # filter type bytes
    head = head.tobytes()
    data = head + head[:258] + head[258:512]
    items = list(head) + [("m", 258, 32768), ("m", 254, 32768)]
    w = BitWriter()
    w.huffman(items, final=True)
    zz = w.zlib(data)
    assert zlib.decompress(zz) == data
    out["match_32768_258"] = png_file(w8, h8, 8, 0, zz)
    # an overlapping match: distance 1, length 258, repeated (rows of Sub-filtered ones)
    data = bytes([1]) * 777
    w = BitWriter()
    w.huffman([1, ("m", 258, 1), ("m", 258, 1), ("m", 258, 1), 1, 1], final=True)
    out["overlap_1_258"] = png_file(258, 3, 8, 0, w.zlib(data))
    # dynamic: 18 repeats that span the literal/length and distance lengths, and a one-code distance tree
    data = bytes([0]) + bytes([1, 2, 3]) * 40
    lit = lit_lengths_for([0, 1, 2, 3, 257, 258])                      # 286 lengths, 0 from 259 on
    dist = [0] * 3 + [1]                                              # one code: distance symbol 3 (distance 4)
    full = lit + dist
    hdr = []
    i = 0
    while i < len(full):
        if full[i] == 0:
            j = i
            while j < len(full) and full[j] == 0 and j - i < 138:
                j += 1
            if j - i >= 11:
                hdr.append((18, j - i - 11))
                i = j
                continue
            if j - i >= 3:
                hdr.append((17, j - i - 3))
                i = j
                continue
        hdr.append((full[i], 0))
        i += 1
    assert any(s == 18 for s, _ in hdr)
    w = BitWriter()
    w.huffman([0, 1, 2, 3, ("sym", 258), ("dsym", 3, 0, 0)], lit_lens=lit, dist_lens=dist, header=hdr)
    w.huffman([], final=True)
    data = bytes([0, 1, 2, 3, 0, 1, 2, 3])                            # length 4 at distance 4
    assert zlib.decompress(w.zlib(data)) == data
    out["dyn_repeat_spanning_one_dist"] = png_file(7, 1, 8, 0, w.zlib(data))
    # a dynamic block whose distance code has no codes at all (valid while unused), and fixed blocks around it
    w = BitWriter()
    lit = lit_lengths_for([1, 2])
    w.huffman([1, 2, 1], lit_lens=lit, dist_lens=[0])
    w.huffman([2], final=True)
    data = bytes([1, 2, 1, 2])
    assert zlib.decompress(w.zlib(data)) == data
    out["dyn_empty_dist"] = png_file(3, 1, 8, 0, w.zlib(data))
    return out


def corrupt_cases() -> Dict[str, Tuple[bytes, int]]:
    """Crafted files whose streams end early by the defined rule: name -> (file, expected status)."""
    S = png
    out = {}
    good = bytes(range(1, 60))                                         # 8-bit grey, 3 rows of 1 + 19 bytes

    def f(stream, w=19, h=3):
        return png_file(w, h, 8, 0, stream)
    w = BitWriter()
    w.stored(good[:10])
    w.put(1, 1)
    w.put(3, 2)                                                        # block type 3
    out["block_type_3"] = (f(w.zlib()), S.STATUS_BAD_BLOCK)
    w = BitWriter()
    w.stored(good[:10], nlen=0x1234)
    out["stored_nlen"] = (f(w.zlib()), S.STATUS_BAD_BLOCK)
    w = BitWriter()
    w.stored(good[:10])
    w.huffman([1, 2, ("sym", 286)], final=True)
    out["litlen_286"] = (f(w.zlib()), S.STATUS_BAD_SYMBOL)
    w = BitWriter()
    w.huffman([1, 2, ("sym", 287)], final=True)
    out["litlen_287"] = (f(w.zlib()), S.STATUS_BAD_SYMBOL)
    for d in (30, 31):
        w = BitWriter()
        w.huffman([1, 2, 3, ("sym", 257), ("dsym", d, 0, 0)], final=True)
        out[f"dist_{d}"] = (f(w.zlib()), S.STATUS_BAD_SYMBOL)
    w = BitWriter()
    w.huffman([1, 2, 3, ("m", 3, 4)], final=True)                     # distance 4 after 3 bytes
    out["dist_too_far"] = (f(w.zlib()), S.STATUS_BAD_DISTANCE)
    w = BitWriter()
    w.huffman([1, 2, 3], final=False)                                 # input ends before the final block
    out["exhausted"] = (f(w.zlib()), S.STATUS_EXHAUSTED)
    w = BitWriter()
    w.huffman(list(good[:20]) + ["noeob"], final=True)                # input ends inside the block
    out["exhausted_in_block"] = (f(w.zlib()[:-1]), S.STATUS_EXHAUSTED)
    w = BitWriter()
    w.huffman(list(good[:25]), final=True)                            # the final block ends first
    out["short"] = (f(w.zlib()), S.STATUS_SHORT)
    # dynamic headers zlib refuses
    lit = lit_lengths_for([1, 2])
    w = BitWriter()
    w.huffman([1, 2], lit_lens=lit, dist_lens=[1], header=[(16, 0)] + [(v, 0) for v in lit + [1]][3:], final=True)
    out["dyn_16_first"] = (f(w.zlib()), S.STATUS_BAD_HEADER)
    w = BitWriter()
    bad = list(lit)
    bad[1] = bad[2] = 1                                               # over-subscribed: 1, 2 and EOB all of 1 bit
    bad[256] = 1
    w.huffman([], lit_lens=bad, dist_lens=[1], final=True)
    out["dyn_oversubscribed"] = (f(w.zlib()), S.STATUS_BAD_HEADER)
    w = BitWriter()
    inc = [0] * 286
    inc[1], inc[2], inc[256] = 2, 2, 2                                # incomplete with a longest code of 2 bits
    w.huffman([], lit_lens=inc, dist_lens=[1], final=True)
    out["dyn_incomplete"] = (f(w.zlib()), S.STATUS_BAD_HEADER)
    w = BitWriter()
    noeob = [0] * 286
    noeob[1], noeob[2] = 1, 1
    w.huffman([1, "noeob"], lit_lens=noeob, dist_lens=[1], final=True)
    out["dyn_no_eob"] = (f(w.zlib()), S.STATUS_BAD_HEADER)
    w = BitWriter()
    w.put(1, 1)
    w.put(2, 2)
    w.put(30, 5)                                                      # HLIT = 287
    w.put(0, 5)
    w.put(0, 4)
    w.put(0, 32)
    out["dyn_hlit_287"] = (f(w.zlib()), S.STATUS_BAD_HEADER)
    w = BitWriter()
    w.huffman([], lit_lens=lit, dist_lens=[1], header=[(v, 0) for v in lit] + [(18, 100)], final=True)
    out["dyn_repeat_past_end"] = (f(w.zlib()), S.STATUS_BAD_HEADER)
    w = BitWriter()                                                   # a distance code with no codes, used
    w.huffman([1, 2, 3, ("sym", 257), "noeob"], lit_lens=lit_lengths_for([1, 2, 3, 257]), dist_lens=[0], final=True)
    w.put(0, 16)
    out["dyn_empty_dist_used"] = (f(w.zlib()), S.STATUS_BAD_SYMBOL)
    w = BitWriter()                                                   # a one-code distance tree fed the unused code
    w.huffman([1, 2, 3, ("sym", 257), "noeob"], lit_lens=lit_lengths_for([1, 2, 3, 257]), dist_lens=[1], final=True)
    w.put(1, 1)
    w.put(0, 16)
    out["dyn_one_code_dist_unused"] = (f(w.zlib()), S.STATUS_BAD_SYMBOL)
    # scanlines with an unknown filter type: the stream is valid, the row unfilters as None
    raw = b"".join(bytes([ft]) + bytes(range(i, i + 19)) for i, ft in enumerate((7, 1, 200)))
    out["unknown_filter"] = (f(zlib.compress(raw)), S.STATUS_OK)
    return out


def adversarial(nbytes: int, w: int = 1, h: int = 1) -> bytes:
    """About ``nbytes`` of non-final dynamic blocks, each with a maximal header (286 + 30 code lengths written one by one,
    no repeats) and no data, then an empty final block: the worst case of table building per input bit, for a ``w`` x
    ``h`` 8-bit grey image that the stream never fills."""
    lit = [0] * 286
    for s, v in complete_lengths(list(range(286)), 15).items():
        lit[s] = v
    dist = [0] * 30
    for s, v in complete_lengths(list(range(30)), 15).items():
        dist[s] = v
    w1 = BitWriter()
    w1.huffman([], lit_lens=lit, dist_lens=dist)
    unit = BitWriter()
    unit.bits = w1.bits * 8                                           # a whole number of bytes
    unit_bytes = unit.tobytes()
    last = BitWriter()
    last.huffman([], final=True)
    stream = b"\x78\x01" + unit_bytes * max(1, nbytes // len(unit_bytes)) + last.tobytes()
    return png_file(w, h, 8, 0, stream, idat_sizes=[1 << 16] * (len(stream) >> 16))
