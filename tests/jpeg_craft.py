"""A baseline-JPEG writer for tests: files whose tables, restart intervals and entropy bits are chosen, not encoded.

``craft`` writes SOI, APP0 (JFIF), DQT, SOF0 (1 or 3 components; 4:4:4, 4:2:2 or 4:2:0), DHT, an optional DRI, SOS, the
entropy-coded data and EOI.  The entropy data is either quantised coefficients, Huffman-coded as DC differences and AC
run/size symbols with EOB and ZRL, or explicit bits per restart interval.  Each interval is padded with 1-bits to a byte,
0xFF bytes are stuffed, RSTn markers go between intervals, and ``fill`` 0xFF fill bytes may go before every marker.

The writer knows the coefficients it wrote, so a test needs no entropy decode to know what a crafted file holds; its
pixels follow from ``jpeg.planes`` and ``jpeg.color_convert``.  ``split`` and ``assemble`` take a file apart into its
header and unstuffed restart intervals and put one together again, which is how the corrupt files of the tests are made.
Pure Python and numpy: no Pillow.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from defer_b200 import jpeg

#: a Huffman table: 16 code-length counts and the symbols in code order
Table = Tuple[Sequence[int], Sequence[int]]
SAMPLING = {"gray": (1, 1, 1), "444": (3, 1, 1), "422": (3, 2, 1), "420": (3, 2, 2)}


def one_symbol(sym: int, length: int = 1) -> Table:
    """A table of one code: ``length`` zero bits for ``sym``."""
    counts = [0] * 16
    counts[length - 1] = 1
    return counts, [sym]


def random_table(rng: np.random.Generator, symbols: Sequence[int], deep: float = 0.3) -> Table:
    """A random canonical table over ``symbols`` (codes of up to 16 bits; the larger ``deep``, the longer the codes).
    One leaf of the code tree stays unused, so no code is all 1-bits."""
    depths = [0]
    while len(depths) < len(symbols) + 1:
        cand = [i for i, d in enumerate(depths) if d < 16]
        i = max(cand, key=lambda i: depths[i]) if rng.random() < deep else cand[int(rng.integers(len(cand)))]
        d = depths.pop(i)
        depths += [d + 1, d + 1]
    depths = sorted(depths)[:len(symbols)]
    syms = [int(s) for s in rng.permutation(np.asarray(symbols))]
    counts = [0] * 16
    for d in depths:
        counts[d - 1] += 1
    return counts, syms


def codes(t: Table) -> Dict[int, Tuple[int, int]]:
    """symbol -> (code, length) of a canonical table."""
    counts, syms = t
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            out[syms[k]] = (code, ln)
            code += 1
            k += 1
        code <<= 1
    return out


def geometry(h: int, w: int, sub: str) -> jpeg.Geometry:
    nc, hs, vs = SAMPLING[sub]
    return jpeg.geometry(h, w, nc, hs, vs)


def _category(v: int) -> int:
    return int(abs(v)).bit_length()


def _bits(v: int, s: int) -> str:
    return format(v if v >= 0 else v + (1 << s) - 1, f"0{s}b") if s else ""


def symbols_of(coef: np.ndarray, g: jpeg.Geometry, restart: int = 0) -> Tuple[List[set], List[set]]:
    """The DC and AC symbols each component of ``coef`` needs (to build tables that cover them)."""
    dc, ac = [set() for _ in range(3)], [set() for _ in range(3)]
    for c, diff, blk in _walk(coef, g, restart):
        dc[c].add(_category(diff))
        ac[c].update(_ac_symbol(run, v) for run, v in _runs(blk))
    return dc, ac


def _walk(coef, g, restart):
    """(component, DC difference, zigzag AC list) of each block in stream order."""
    per = restart * g.bpm if restart else g.blocks
    pred = [0, 0, 0]
    for b in range(g.blocks):
        if b % per == 0:
            pred = [0, 0, 0]
        c = g.comp_of[b % g.bpm]
        dcv = int(coef[b, 0])
        yield c, dcv - pred[c], [int(coef[b, jpeg.ZIGZAG[k]]) for k in range(1, 64)]
        pred[c] = dcv


def _runs(ac: List[int]):
    """(run, value) AC symbols of a block: (15, None) is ZRL, (0, None) is EOB."""
    run = 0
    for v in ac:
        if v == 0:
            run += 1
            continue
        while run > 15:
            yield 15, None
            run -= 16
        yield run, v
        run = 0
    if run:
        yield 0, None


def _ac_symbol(run: int, v: Optional[int]) -> int:
    return (run << 4) | _category(v) if v is not None else 0xF0 if run == 15 else 0


def encode(coef: np.ndarray, g: jpeg.Geometry, dc: Sequence[Table], ac: Sequence[Table], restart: int = 0) -> List[str]:
    """The bits of each restart interval for final quantised coefficients ``coef`` (int [blocks, 64], stream order,
    natural order); ``dc[c]`` / ``ac[c]`` are the tables of component c."""
    dcc, acc = [codes(t) for t in dc], [codes(t) for t in ac]
    per = restart * g.bpm if restart else g.blocks
    out, cur = [], []
    for b, (c, diff, blk) in enumerate(_walk(coef, g, restart)):
        if b and b % per == 0:
            out.append("".join(cur))
            cur = []
        s = _category(diff)
        code, ln = dcc[c][s]
        cur.append(format(code, f"0{ln}b") + _bits(diff, s))
        for run, v in _runs(blk):
            code, ln = acc[c][_ac_symbol(run, v)]
            cur.append(format(code, f"0{ln}b") + (_bits(v, _category(v)) if v is not None else ""))
    out.append("".join(cur))
    return out


def pack(bits) -> bytes:
    """A bit string ('0'/'1' characters) or a 0/1 array, padded with 1-bits to a byte, as bytes (not stuffed)."""
    a = np.frombuffer(bits.encode(), np.uint8) - ord("0") if isinstance(bits, str) else np.asarray(bits, np.uint8)
    pad = -len(a) % 8
    return np.packbits(np.concatenate([a, np.ones(pad, np.uint8)])).tobytes()


def stuff(b: bytes) -> bytes:
    """Insert 0x00 after every 0xFF."""
    a = np.frombuffer(b, np.uint8)
    ff = np.nonzero(a == 0xFF)[0]
    return np.insert(a, ff + 1, 0).tobytes() if len(ff) else bytes(b)


def _seg(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def header(h: int, w: int, sub: str, quant: Sequence[np.ndarray], dc: Sequence[Table], ac: Sequence[Table],
           restart: int = 0) -> bytes:
    """SOI .. SOS.  Component 0 uses quant[0], dc[0], ac[0]; the chroma components use table 1 of each (or 0 if there
    is only one).  ``quant`` tables are in natural order, entries 1..255."""
    nc, hs, vs = SAMPLING[sub]
    out = b"\xff\xd8" + _seg(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")
    for t, q in enumerate(quant):
        q = np.asarray(q).reshape(64)
        assert q.min() >= 1 and q.max() <= 255
        out += _seg(0xDB, bytes([t]) + q[jpeg.ZIGZAG].astype(np.uint8).tobytes())
    tq = [0] + [min(1, len(quant) - 1)] * 2
    comps = b"".join(bytes([i + 1, ((hs << 4) | vs) if i == 0 else 0x11, tq[i]]) for i in range(nc))
    out += _seg(0xC0, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([nc]) + comps)
    for cls, tabs in ((0, dc), (1, ac)):
        for t, (counts, syms) in enumerate(tabs):
            out += _seg(0xC4, bytes([(cls << 4) | t]) + bytes(counts) + bytes(syms))
    if restart:
        out += _seg(0xDD, restart.to_bytes(2, "big"))
    th = [0] + [min(1, len(dc) - 1)] * 2
    sel = b"".join(bytes([i + 1, (th[i] << 4) | th[i]]) for i in range(nc))
    return out + _seg(0xDA, bytes([nc]) + sel + b"\x00\x3f\x00")


def assemble(head: bytes, intervals: Sequence[bytes], fill: int = 0, rst: Optional[Sequence[int]] = None) -> bytes:
    """A file of ``head`` (up to the end of SOS) and the unstuffed bytes of each restart interval: stuffed, with RSTn
    markers between them (``rst`` gives each marker's n, else 0, 1, .., 7, 0, ..), ``fill`` 0xFF bytes before every
    marker, and EOI."""
    out = [head]
    for i, b in enumerate(intervals):
        if i:
            out.append(b"\xff" * fill + bytes([0xFF, 0xD0 + (rst[i - 1] if rst is not None else (i - 1) % 8)]))
        out.append(stuff(b))
    out.append(b"\xff" * fill + b"\xff\xd9")
    return b"".join(out)


def split(data: bytes) -> Tuple[bytes, List[bytes]]:
    """(header up to the end of SOS, unstuffed bytes of each interval between RST markers) of a file ``jpeg.parse``
    accepts; ``assemble(*split(data))`` holds the same entropy data."""
    info = jpeg.parse(data)
    comp, rst = jpeg.unstuff(data[info.offset:info.offset + info.length])
    edges = [0] + rst + [len(comp)]
    return data[:info.offset], [comp[a:b] for a, b in zip(edges[:-1], edges[1:])]


def craft(h: int, w: int, sub: str, quant: Sequence[np.ndarray], dc: Sequence[Table], ac: Sequence[Table], *,
          coef: Optional[np.ndarray] = None, bits: Optional[Sequence] = None, restart: int = 0, fill: int = 0) -> bytes:
    """One baseline file.  The entropy data is ``coef`` (final quantised coefficients, int [blocks, 64] in stream order
    and natural order) Huffman-coded with ``dc`` / ``ac``, or ``bits``: per restart interval, a '0'/'1' string or a 0/1
    array."""
    assert (coef is None) != (bits is None)
    if coef is not None:
        nc = SAMPLING[sub][0]
        per = [0] + [min(1, len(dc) - 1)] * 2
        bits = encode(np.asarray(coef), geometry(h, w, sub), [dc[per[c]] for c in range(nc)],
                      [ac[per[c]] for c in range(nc)], restart)
    return assemble(header(h, w, sub, quant, dc, ac, restart), [pack(b) for b in bits], fill)


def tables_for(coef: np.ndarray, g: jpeg.Geometry, restart: int, rng: np.random.Generator, deep: float = 0.3):
    """Random luma and chroma tables (dc, ac) that cover every symbol ``coef`` needs."""
    dcs, acs = symbols_of(coef, g, restart)
    groups = [[0]] if g.bpm == 1 else [[0], [1, 2]]
    dc = [random_table(rng, sorted(set().union(*(dcs[c] for c in grp)) or {0}), deep) for grp in groups]
    ac = [random_table(rng, sorted(set().union(*(acs[c] for c in grp)) or {0}), deep) for grp in groups]
    return dc, ac


def fdct_coef(img: np.ndarray, g: jpeg.Geometry, quant: Sequence[np.ndarray]) -> np.ndarray:
    """Quantised coefficients (int32 [blocks, 64], stream order) of the MCU-padded uint8 planes ``img[c]`` by a float
    forward DCT, as any encoder may emit: component 0 uses quant[0], the others quant[-1]."""
    k = np.arange(8)
    basis = np.cos((2 * k[None, :] + 1) * k[:, None] * np.pi / 16) * np.where(k == 0, np.sqrt(0.5), 1.0)[:, None] / 2
    comp_of = np.tile(np.array(g.comp_of), g.mcus)
    out = np.zeros((g.blocks, 64), np.int32)
    for c in range(len(g.bw)):
        hc, vc = (g.bw[0] // g.mcux, g.bh[0] // g.mcuy) if c == 0 else (1, 1)
        p = img[c][:g.bh[c] * 8, :g.bw[c] * 8].astype(np.float64) - 128
        b = p.reshape(g.mcuy, vc, 8, g.mcux, hc, 8).transpose(0, 3, 1, 4, 2, 5).reshape(-1, 8, 8)
        f = np.einsum("ux,nxy,vy->nuv", basis, b, basis).reshape(-1, 64)
        q = np.asarray(quant[0] if c == 0 else quant[-1]).reshape(64)
        out[np.nonzero(comp_of == c)[0]] = np.round(f / q).astype(np.int32)
    return out


def idct_raw(coef: np.ndarray, quant: np.ndarray) -> np.ndarray:
    """jidctint.c's ISLOW output of int blocks ``[n, 64]`` before the range limit: int64 ``[n, 8, 8]``, 0 = 128."""
    x = coef.astype(np.int64).reshape(-1, 8, 8) * quant.astype(np.int64).reshape(8, 8)
    ws = np.stack(jpeg._idct_1d([x[:, r, :] for r in range(8)], True), axis=1)
    return np.stack(jpeg._idct_1d([ws[:, :, c] for c in range(8)], False), axis=2)


def info_of(h: int, w: int, sub: str, quant: Sequence[np.ndarray], restart: int = 0) -> jpeg.JpegInfo:
    """A JpegInfo with what ``jpeg.planes`` and ``jpeg.color_convert`` read, for a crafted file's geometry."""
    nc, hs, vs = SAMPLING[sub]
    q = tuple(np.asarray(quant[0 if c == 0 else -1], np.int32).reshape(64) for c in range(nc))
    return jpeg.JpegInfo(h, w, nc, hs, vs, restart, 0, 0, q, (), ())


def expected(coef: np.ndarray, h: int, w: int, sub: str, quant: Sequence[np.ndarray]) -> dict:
    """``coef`` (int16), ``planes`` and ``rgb`` of a crafted file that decodes to final coefficients ``coef``."""
    info = info_of(h, w, sub, quant)
    c16 = np.asarray(coef).astype(np.int16)
    pl = jpeg.planes(c16, info)
    return {"coef": c16, "planes": pl, "rgb": jpeg.color_convert(pl, info)}


def all_zero_coef(g: jpeg.Geometry) -> np.ndarray:
    """What ``all_zero_stream`` holds: DC 0, every AC coefficient -1."""
    coef = np.full((g.blocks, 64), -1, np.int32)
    coef[:, 0] = 0
    return coef


def all_zero_stream(h: int, w: int, sub: str, restart: int = 0) -> bytes:
    """The 127-bit-block stream: all-zero entropy bits under one-symbol tables."""
    g = geometry(h, w, sub)
    per = restart * g.bpm if restart else g.blocks
    n = [min(per, g.blocks - s) * 127 for s in range(0, g.blocks, per)]
    t = 1 if sub == "gray" else 2
    return craft(h, w, sub, [np.ones(64, int)], [one_symbol(0)] * t, [one_symbol(0x01)] * t,
                 bits=[np.zeros(k, np.uint8) for k in n], restart=restart)


def long_code_stream(h: int, w: int) -> bytes:
    """One-symbol 16-bit codes, DC category 11 and AC (0, 7), all-zero bits: 1476-bit blocks, every DC difference
    -2047 and every AC coefficient -127."""
    g = geometry(h, w, "gray")
    return craft(h, w, "gray", [np.ones(64, int)], [one_symbol(11, 16)], [one_symbol(0x07, 16)],
                 bits=[np.zeros(g.blocks * 1476, np.uint8)])


def long_code_coef(g: jpeg.Geometry) -> np.ndarray:
    """What ``long_code_stream`` holds (grayscale, no restart interval)."""
    coef = np.full((g.blocks, 64), -127, np.int64)
    acc = np.cumsum(np.full(g.blocks, -2047, np.int64))
    coef[:, 0] = ((acc + (1 << 15)) % (1 << 16)) - (1 << 15)          # int32 sums, stored as int16
    return coef


def closed_form_counters(data: bytes, sbits: int) -> np.ndarray:
    """The five counters of the device decode (T, R, nsubs, rounds, cutoff) for a file in which every bit position
    starts a valid block and no block ends in an invalid code (one-symbol tables of all-zero codes, all-zero bits):
    a decoder started in the wrong phase never resynchronises, so the true state moves one subsequence per round and
    the rounds are the largest number of subsequences in one restart interval."""
    info = jpeg.parse(data)
    g = jpeg.geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    comp, rst = jpeg.unstuff(data[info.offset:info.offset + info.length])
    nseg = -(-g.mcus // info.restart) if info.restart else 1
    n = [-(-8 * (e - s) // sbits) for s, e in jpeg.segments(len(comp), rst, nseg)]
    return np.array([len(comp), len(rst), sum(n), max([1] + n), g.blocks], np.int32)
