"""PNG files no encoder writes: a chunk writer, a small deflate bit writer, and a corpus of crafted streams.

``png_file`` wraps any zlib stream in a PNG of a given size, colour type and depth, split into IDAT chunks where asked.
``BitWriter`` writes deflate blocks bit by bit (stored, fixed Huffman, dynamic Huffman with any code lengths, and raw
header fields), so a test can build what zlib never emits: empty stored blocks, stored blocks that cross IDAT chunk
boundaries, matches at distance 32768 and length 258, an overlapping match, a dynamic header whose repeat codes span the
literal/length and distance lengths, one-code distance trees, codes that use every length from 1 to 15, a one-bit
end-of-block-only code, every corruption of the decode's defined result and each case where that result deviates from
zlib (defer_b200/png.py).  ``filter_rows`` filters image rows forward, so a test can build a file of any size whose
expected scanlines are known without an unfilter."""
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


# ------------------------------------------------------------------------------------------------- forward filters
def filter_rows(x: np.ndarray, bpp: int, types: np.ndarray) -> bytes:
    """The scanlines of image rows ``x`` (uint8 [h, bytes per row]) filtered forward with filter type ``types[r]`` on row
    r, filter unit ``bpp``: each row's type byte and its bytes minus the predictor of the PNG specification.  Every
    neighbour is known on this side, so all four predictors are whole-array operations (no unfilter is run)."""
    h, bpr = x.shape
    xi = x.astype(np.int16)
    a = np.zeros_like(xi)
    a[:, bpp:] = xi[:, :-bpp]
    b = np.zeros_like(xi)
    b[1:] = xi[:-1]
    c = np.zeros_like(xi)
    c[1:, bpp:] = xi[:-1, :-bpp]
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    t = np.asarray(types, np.uint8)
    rows = xi.copy()
    for k, pred in ((1, a), (2, b), (3, (a + b) >> 1), (4, paeth)):
        rows[t == k] -= pred[t == k]
    return np.concatenate([t[:, None], (rows & 255).astype(np.uint8)], axis=1).tobytes()


def encode(x: np.ndarray, w: int, depth: int, ctype: int, types, level: int = 1, chunk_bytes: int = 8192,
           palette: Optional[bytes] = None) -> bytes:
    """A PNG of scanline bytes ``x`` (uint8 [h, bytes per row]): ``filter_rows`` with per-row ``types``, zlib at
    ``level``, IDAT chunks of ``chunk_bytes``."""
    raw = filter_rows(x, max(1, CHANNELS[ctype] * depth // 8), types)
    z = zlib.compress(raw, level)
    return png_file(w, x.shape[0], depth, ctype, z, idat_sizes=[chunk_bytes] * (len(z) // chunk_bytes), palette=palette)


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
    out["dyn_lengths_1_to_15"] = lengths_1_to_15()
    # a literal/length code whose only code is end-of-block, of one bit (incomplete, valid as in zlib), then the data
    w = BitWriter()
    w.huffman([], lit_lens=EOB_ONLY, dist_lens=[0])
    w.huffman([], lit_lens=EOB_ONLY, dist_lens=[1])
    w.stored(raw[:121], final=True)
    assert zlib.decompress(w.zlib(raw[:121])) == raw[:121]
    out["dyn_eob_only"] = png_file(40, 1, 8, 2, w.zlib(raw[:121]))
    return out


EOB_ONLY = [0] * 256 + [1]                                            # HLIT = 257: end-of-block alone, code "0"

# lengths_1_to_15: literal/length and distance codes, each complete and using every code length from 1 to 15 (lengths
# 1..14 once and 15 twice); a literal, a length symbol and two distance symbols have 15-bit codes
_LIT_1_15 = {0: 1, 257: 2, 1: 3, 265: 4, 2: 5, 269: 6, 3: 7, 273: 8, 4: 9, 277: 10, 7: 11, 281: 12, 100: 13, 256: 14,
             255: 15, 285: 15}
_DIST_1_15 = {27: 1, 3: 2, 26: 3, 8: 4, 28: 5, 11: 6, 15: 7, 14: 8, 17: 9, 20: 10, 23: 11, 5: 12, 4: 13, 2: 14,
              0: 15, 29: 15}


def lengths_1_to_15(seed: int = 5) -> bytes:
    """An 8-bit grey 255x130 file of one dynamic block in the codes above, whose data uses every symbol of both codes:
    the 10-bit lookup and the canonical walk of longer codes run in one table.  Filter type bytes (every 256th) are
    0..4: a match that covers one has a distance that is a multiple of 256, so it copies another."""
    assert sum(2.0 ** -v for v in _LIT_1_15.values()) == 1 and sum(2.0 ** -v for v in _DIST_1_15.values()) == 1
    rng = np.random.default_rng(seed)
    lits = [s for s in _LIT_1_15 if s < 256]
    lsyms = [s - 257 for s in _LIT_1_15 if s > 256]
    dsyms = list(_DIST_1_15)
    n, out, items = 256 * 130, bytearray(), []
    todo_l, todo_d = set(lsyms), set(dsyms)
    used_lit = set()
    while len(out) < n:
        p = len(out)
        item = None
        if p % 256 and rng.random() < 0.6:
            ls = int(rng.choice(sorted(todo_l) if todo_l and rng.random() < 0.5 else lsyms))
            near = [d for d in (sorted(todo_d) if todo_d and rng.random() < 0.5 else dsyms) if png.DBASE[d] <= p]
            ds = int(rng.choice(near)) if near else -1
            if ds >= 0:
                length = png.LBASE[ls] + int(rng.integers(0, 1 << png.LEXT[ls]))
                lo, hi = png.DBASE[ds], min(p, png.DBASE[ds] + (1 << png.DEXT[ds]) - 1)
                crosses = (p + length - 1) // 256 > p // 256
                if crosses:                                           # a multiple of 256 in [lo, hi]
                    lo, hi = -(-lo // 256), hi // 256
                step = 256 if crosses else 1
                if lo <= hi and p + length <= n:
                    d = step * int(rng.integers(lo, hi + 1))
                    item = ("m", length, d)
                    todo_l.discard(ls)
                    todo_d.discard(ds)
                    for _ in range(length):
                        out.append(out[-d])
        if item is None:
            v = int(rng.integers(0, 5)) if p % 256 == 0 else int(rng.choice(lits))
            used_lit.add(v)
            item = v
            out.append(v)
        items.append(item)
    assert not todo_l and not todo_d and used_lit == set(lits), (todo_l, todo_d, used_lit)
    lit = [0] * 286
    for s, v in _LIT_1_15.items():
        lit[s] = v
    dist = [0] * 30
    for s, v in _DIST_1_15.items():
        dist[s] = v
    w = BitWriter()
    w.huffman(items, final=True, lit_lens=lit, dist_lens=dist)
    data = bytes(out)
    z = w.zlib(data)
    assert zlib.decompress(z) == data and all(v <= 4 for v in data[::256])
    return png_file(255, 130, 8, 0, z)


def _ends_at_byte(body) -> BitWriter:
    """A writer holding a non-final fixed block of j 9-bit literals (200) and then ``body(writer)``, with j in 0..7
    chosen so that the bits end on a byte boundary: nothing past ``body`` for a decoder to read."""
    for j in range(8):
        w = BitWriter()
        w.huffman([200] * j)
        body(w)
        if len(w.bits) % 8 == 0:
            return w
    raise AssertionError("no prefix aligns the body")


def _empty_cl_header(w: BitWriter, zero_lengths: int):
    """A final dynamic block header whose code-length code has no codes (HLIT 257, HDIST 1, HCLEN 4, all lengths 0),
    then ``zero_lengths`` zero bits (zlib decodes each bit as code length 0)."""
    w.put(1, 1)
    w.put(2, 2)
    w.put(0, 5)
    w.put(0, 5)
    w.put(0, 4)
    w.put(0, 12)
    w.put(0, zero_lengths)


def _sixteen_first(w: BitWriter):
    """A final dynamic block header whose first code length is repeat code 16, its 2 extra bits not written."""
    w.put(1, 1)
    w.put(2, 2)
    w.put(0, 5)
    w.put(0, 5)
    w.put(0, 4)
    for v in (1, 0, 0, 1):                                            # CL_ORDER 16, 17, 18, 0: codes 0 -> "0", 16 -> "1"
        w.put(v, 3)
    w.put_code(1, 1)


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
    w = BitWriter()                                                   # the one-code (end-of-block) tree fed code "1"
    w.huffman([], lit_lens=EOB_ONLY, dist_lens=[0])
    w.huffman(["noeob"], lit_lens=EOB_ONLY, dist_lens=[0], final=True)
    w.put(1, 1)
    w.put(0, 16)
    out["dyn_eob_only_unused"] = (f(w.zlib()), S.STATUS_BAD_SYMBOL)
    # the restatement's deviations from zlib (module docstring of defer_b200/png.py)
    w = BitWriter()                                                   # a code-length code with no codes at all
    w.stored(good[:10])
    _empty_cl_header(w, 400)
    out["dyn_empty_cl_code"] = (f(w.zlib()), S.STATUS_BAD_HEADER)
    w = _ends_at_byte(lambda w: _empty_cl_header(w, 100))             # ... cut before its 258 code lengths
    out["dyn_empty_cl_code_cut"] = (f(w.zlib()), S.STATUS_BAD_HEADER)
    w = _ends_at_byte(_sixteen_first)                                 # repeat code 16 first, cut before its extra bits
    out["dyn_16_first_cut"] = (f(w.zlib()), S.STATUS_BAD_HEADER)
    w = _ends_at_byte(lambda w: w.huffman([1, 2, 3, ("sym", 257), "noeob"], lit_lens=lit_lengths_for([1, 2, 3, 257]),
                                          dist_lens=[0], final=True))
    out["dyn_empty_dist_used_at_end"] = (f(w.zlib()), S.STATUS_BAD_SYMBOL)   # an empty distance code, cut where used
    w = BitWriter()                                                   # a stored block whose data runs past the input
    w.stored(good[:10])
    w.stored(good[10:50], final=True)
    out["stored_truncated"] = (f(w.zlib()[:-15]), S.STATUS_EXHAUSTED)
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
