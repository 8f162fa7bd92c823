"""A progressive-JPEG writer for tests: any scan script, over coefficients the writer knows.

``craft`` writes SOI, APP0 (JFIF), DQT, SOF2 (1 or 3 components; 4:4:4, 4:2:2 or 4:2:0), then per scan of the script
the segments asked for before it (COM, a DRI when the restart interval changes, a DQT that redefines a table already
latched), a DHT of fresh random tables covering what the scan needs, SOS and its entropy data, and EOI.  The scans are
encoded as libjpeg's ``jcphuff.c`` encodes them: DC first with its point transform and prediction, DC refinement bits,
AC first with EOB runs (up to 32 767 blocks) and ZRL, AC refinement with its buffered correction bits.  Restart
intervals count MCUs in scans of all components and blocks of the component's own grid in scans of one.

A scan may also be raw: its entropy data given per restart interval, as bits or as symbols under a chosen table, which
is how the tests write what encoders never write.  ``split`` and ``assemble`` take a file apart at its scans and restart
intervals and put it together again with a scan replaced or cut, RST markers dropped, repeated, renumbered, surplus or
missing, and fill bytes.  ``worst_first`` writes the worst case of the device's self-synchronisation for a DC first or
AC first scan, and ``saturating`` a file whose block counts add past 2^31; ``closed_form_counters`` gives the device's
six counters for both.

It returns the file and the final coefficients a decoder must give (int16 ``[blocks, 64]``, stream order, natural
order): each coefficient as the last scan that covered it left it, zero where no scan did.  The block order of a scan is
derived here from the sampling, independently of ``jpeg.scan_blocks``.  Pure Python and numpy: no Pillow.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from defer_b200 import jpeg
from jpeg_craft import SAMPLING, _seg, codes, geometry, one_symbol, pack, random_table, stuff


def scan(comps, ss, se, ah, al, restart=0, com=False, dqt=False, raw=None, table=None, holds=None) -> dict:
    """One entry of a scan script: frame component indices, spectral selection, successive approximation, the restart
    interval in force, and whether a COM segment and a redefining DQT go before it.

    ``raw``: the scan's entropy data as given, not encoded from the coefficients: one entry per restart interval (as many
    as wanted, so RST markers may be missing or surplus), each a '0'/'1' string, a 0/1 array, unstuffed ``bytes``, or a
    list of events ``("s", symbol)`` / ``("b", value, nbits)`` coded under ``table``.  Encoders never write what a raw
    scan can hold: EOB runs past their interval or scan, a ZRL or run past Se, refinement symbols of size 2.  ``holds``
    (int [blocks, 64], stream order, natural order) is what a raw scan leaves in its band; without it the writer does
    not know the final coefficients.  ``table``: the scan's Huffman table (one for all its components), else a random
    one over the symbols it needs."""
    return {"comps": tuple(comps), "ss": ss, "se": se, "ah": ah, "al": al, "restart": restart, "com": com, "dqt": dqt,
            "raw": raw, "table": table, "holds": holds}


def order(h: int, w: int, sub: str, comps: Sequence[int]) -> Tuple[List[int], int]:
    """Stream-order blocks of a scan in scan order, and the blocks per restart-interval unit."""
    nc, hs, vs = SAMPLING[sub]
    g = geometry(h, w, sub)
    if len(comps) > 1 or nc == 1:
        return list(range(g.blocks)), (g.bpm if len(comps) > 1 else 1)
    c = comps[0]
    hc, vc = (hs, vs) if c == 0 else (1, 1)
    cw, ch = -(-w * hc // (hs * 8)), -(-h * vc // (vs * 8))
    out = []
    for by in range(ch):
        for bx in range(cw):
            m = (by // vc) * g.mcux + bx // hc
            j = (by % vc) * hc + bx % hc if c == 0 else hs * vs + c - 1
            out.append(m * g.bpm + j)
    return out, 1


def _cat(v: int) -> int:
    return int(abs(v)).bit_length()


class _Out:
    """Events of one restart interval: ('s', symbol), ('b', value, nbits), and ('m', q): scan-order block q starts."""

    def __init__(self):
        self.ev = []

    def sym(self, s):
        self.ev.append(("s", s))

    def mark(self, q):
        self.ev.append(("m", q))

    def bits(self, v, n):
        if n:
            self.ev.append(("b", v & ((1 << n) - 1), n))


def _dc_first(coef, blks, comp_of, sc, intervals):
    pred, out = {}, None
    for i, b in enumerate(blks):
        if intervals[i] is not out:                   # prediction restarts with each interval
            pred, out = {}, intervals[i]
        out.mark(i)
        c = comp_of[i]
        v = int(coef[b, 0]) >> sc["al"]
        d = v - pred.get(c, 0)
        pred[c] = v
        s = _cat(d)
        out.sym(s)
        out.bits(d if d >= 0 else d - 1, s)


def _ac_first(coef, blks, sc, intervals):
    eob = [0]
    cur = [None]

    def flush():
        if eob[0]:
            r = eob[0].bit_length() - 1
            cur[0].sym(r << 4)
            cur[0].bits(eob[0], r)
            eob[0] = 0
    for i, b in enumerate(blks):
        if intervals[i] is not cur[0]:
            if cur[0] is not None:
                flush()
            cur[0] = intervals[i]
        cur[0].mark(i)
        r = 0
        for k in range(sc["ss"], sc["se"] + 1):
            t = int(coef[b, jpeg.ZIGZAG[k]])
            a = abs(t) >> sc["al"]
            if a == 0:
                r += 1
                continue
            flush()
            while r > 15:
                cur[0].sym(0xF0)
                r -= 16
            n = a.bit_length()
            cur[0].sym((r << 4) | n)
            cur[0].bits(a if t >= 0 else ~a, n)
            r = 0
        if r:
            eob[0] += 1
            if eob[0] == 0x7FFF:
                flush()
    flush()


def _ac_refine(coef, blks, sc, intervals):
    st = {"eob": 0, "be": [], "cur": None}

    def flush():
        if st["eob"]:
            r = st["eob"].bit_length() - 1
            st["cur"].sym(r << 4)
            st["cur"].bits(st["eob"], r)
            st["eob"] = 0
            for x in st["be"]:
                st["cur"].bits(x, 1)
            st["be"] = []
    for i, b in enumerate(blks):
        if intervals[i] is not st["cur"]:
            if st["cur"] is not None:
                flush()
            st["cur"] = intervals[i]
        out = st["cur"]
        out.mark(i)
        ks = range(sc["ss"], sc["se"] + 1)
        absv = {k: abs(int(coef[b, jpeg.ZIGZAG[k]])) >> sc["al"] for k in ks}
        last_new = max([k for k in ks if absv[k] == 1], default=-1)
        r, br = 0, []
        for k in ks:
            t = absv[k]
            if t == 0:
                r += 1
                continue
            while r > 15 and k <= last_new:
                flush()
                out.sym(0xF0)
                r -= 16
                for x in br:
                    out.bits(x, 1)
                br = []
            if t > 1:
                br.append(t & 1)
                continue
            flush()
            out.sym((r << 4) | 1)
            out.bits(0 if int(coef[b, jpeg.ZIGZAG[k]]) < 0 else 1, 1)
            for x in br:
                out.bits(x, 1)
            br, r = [], 0
        if r > 0 or br:
            st["eob"] += 1
            st["be"] += br
            if st["eob"] == 0x7FFF or len(st["be"]) > 1000 - 64 + 1:
                flush()
    flush()


def _encode(events, table) -> str:
    cd = codes(table) if table is not None else {}
    out = []
    for e in events:
        if e[0] == "s":
            c, n = cd[e[1]]
            out.append(format(c, f"0{n}b"))
        elif e[0] == "b":
            out.append(format(e[1], f"0{e[2]}b"))
    return "".join(out)


def block_bits(events, table) -> dict:
    """Scan-order block -> bit offset within its interval where the events of that block begin (the blocks a writer
    marked; a block inside an EOB run has no symbol of its own)."""
    cd = codes(table) if table is not None else {}
    pos, out = 0, {}
    for e in events:
        if e[0] == "m":
            out[e[1]] = pos
        else:
            pos += cd[e[1]][1] if e[0] == "s" else e[2]
    return out


def _interval_bytes(iv, table) -> bytes:
    if isinstance(iv, bytes):
        return iv
    if isinstance(iv, list):
        iv = _encode(iv, table)
    return pack(iv)


def craft(h: int, w: int, sub: str, quant: Sequence[np.ndarray], coef: np.ndarray, script: Sequence[dict],
          seed: int = 0, trace: Optional[list] = None) -> Tuple[bytes, Optional[np.ndarray]]:
    """A progressive file of ``coef`` (int [blocks, 64], stream order, natural order) under ``script`` (``scan``
    entries), and the final coefficients it decodes to (None if a raw scan does not say what it holds).  Component 0
    uses quant[0], the others quant[-1].  ``trace``: a list that gets (events of each interval, table) per scan."""
    rng = np.random.default_rng(seed)
    nc, hs, vs = SAMPLING[sub]
    g = geometry(h, w, sub)
    coef = np.asarray(coef, np.int64)
    want = np.zeros((g.blocks, 64), np.int64)
    out = b"\xff\xd8" + _seg(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")
    for t, q in enumerate(quant):
        out += _seg(0xDB, bytes([t]) + np.asarray(q).reshape(64)[jpeg.ZIGZAG].astype(np.uint8).tobytes())
    tq = [0] + [len(quant) - 1] * 2
    comps = b"".join(bytes([i + 1, ((hs << 4) | vs) if i == 0 else 0x11, tq[i]]) for i in range(nc))
    out += _seg(0xC2, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([nc]) + comps)
    restart, known = 0, True
    for sc in script:
        if sc["com"]:
            out += _seg(0xFE, b"a comment between scans")
        if sc["dqt"]:                                 # a later DQT does not change a latched table
            out += _seg(0xDB, bytes([0]) + bytes(range(100, 164)))
        if sc["restart"] != restart:
            restart = sc["restart"]
            out += _seg(0xDD, restart.to_bytes(2, "big"))
        blks, per = order(h, w, sub, sc["comps"])
        comp_of = [g.comp_of[b % g.bpm] for b in blks]
        units = len(blks) // per
        nseg = -(-units // restart) if restart else 1
        ss, se, ah, al = sc["ss"], sc["se"], sc["ah"], sc["al"]
        band = [0] if ss == 0 else [int(jpeg.ZIGZAG[k]) for k in range(ss, se + 1)]
        if sc.get("raw") is not None:
            evs = [iv for iv in sc["raw"]]
            table = sc.get("table")
            if sc.get("holds") is None:
                known = False
            else:
                want[np.asarray(blks)[:, None], band] = np.asarray(sc["holds"], np.int64)[blks][:, band]
        else:
            ivs = [_Out() for _ in range(nseg)]
            intervals = [ivs[(i // per) // restart if restart else 0] for i in range(len(blks))]
            if ss == 0 and ah == 0:
                _dc_first(coef, blks, comp_of, sc, intervals)
            elif ss == 0:
                for i, b in enumerate(blks):
                    intervals[i].mark(i)
                    intervals[i].bits((int(coef[b, 0]) >> al) & 1, 1)
            elif ah == 0:
                _ac_first(coef, blks, sc, intervals)
            else:
                _ac_refine(coef, blks, sc, intervals)
            c = coef[blks][:, band]                   # what the decode holds after this scan
            want[np.asarray(blks)[:, None], band] = (c >> al) << al if ss == 0 else np.sign(c) * ((np.abs(c) >> al) << al)
            evs = [iv.ev for iv in ivs]
            syms = sorted({e[1] for ev in evs for e in ev if e[0] == "s"})
            table = sc.get("table")
            if table is None and not (ss == 0 and ah > 0):
                table = random_table(rng, syms or [0])
        if trace is not None:
            trace.append((evs, table))
        if table is not None:
            out += _seg(0xC4, bytes([(0 if ss == 0 else 1) << 4]) + bytes(table[0]) + bytes(table[1]))
        sel = b"".join(bytes([c + 1, 0x00]) for c in sc["comps"])
        out += _seg(0xDA, bytes([len(sc["comps"])]) + sel + bytes([ss, se, (ah << 4) | al]))
        for i, iv in enumerate(evs):
            if i:
                out += bytes([0xFF, 0xD0 + (i - 1) % 8])
            out += stuff(_interval_bytes(iv, table))
    return out + b"\xff\xd9", (want.astype(np.int16) if known else None)


def coefficients(h: int, w: int, sub: str, quant, seed: int, zero_from: Optional[int] = None) -> np.ndarray:
    """Quantised coefficients of a seeded photo-like image; ``zero_from``: zigzag coefficients from there on are zero
    (long EOB runs)."""
    from jpeg_craft import fdct_coef
    rng = np.random.default_rng(seed)
    g = geometry(h, w, sub)
    y, x = np.mgrid[0:g.bh[0] * 8, 0:g.bw[0] * 8].astype(np.float64)
    img = []
    for c in range(len(g.bw)):
        p = 128 + 90 * np.sin(x / (5 + 3 * c) + y / (9 + c)) + rng.normal(0, 10, x.shape)
        img.append(np.clip(p, 0, 255).astype(np.uint8))
    coef = fdct_coef(img, g, quant)
    if zero_from is not None:
        coef[:, jpeg.ZIGZAG[zero_from:]] = 0
    return coef


FULL = [(0, 0, 0, 1), (1, 5, 0, 2), (6, 63, 0, 2), (1, 63, 2, 1), (0, 0, 1, 0), (1, 63, 1, 0)]


def corpus() -> List[Tuple[str, bytes, np.ndarray]]:
    """(name, file, final coefficients) of the crafted cases the tests run on the host and on the GPU."""
    q = [np.full(64, 3, np.int32), np.full(64, 5, np.int32)]
    out = []

    def add(name, h, w, sub, script, seed, zero_from=None, quant=q):
        coef = coefficients(h, w, sub, quant, seed, zero_from)
        out.append((name, *craft(h, w, sub, quant, coef, script, seed=seed)))
    comps = {"gray": [(0,)], "444": [(0,), (1,), (2,)], "422": [(0,), (1,), (2,)], "420": [(0,), (1,), (2,)]}
    for sub in ("420", "422", "444", "gray"):
        allc = (0,) if sub == "gray" else (0, 1, 2)
        # separate DC scans per component, DC first with Al = 0, other spectral splits, never-sent 10..63 of chroma
        s = [scan(c, 0, 0, 0, 0) for c in comps[sub]]
        s += [scan(c, 1, 9, 0, 0) for c in comps[sub]]
        s += [scan((0,), 10, 40, 0, 1), scan((0,), 41, 63, 0, 0), scan((0,), 10, 40, 1, 0)]
        add(f"split_{sub}_17x33", 17, 33, sub, s, seed=1)
        # restart intervals in one-component scans, changing between scans, DHT / DRI / COM / DQT between scans
        s = [scan(allc, 0, 0, 0, 2, restart=2)]
        s += [scan(c, 1, 63, 0, 3, restart=3 + i, com=i == 0, dqt=i == 0) for i, c in enumerate(comps[sub])]
        s += [scan(c, 1, 63, 3, 2, restart=5) for c in comps[sub]]
        s += [scan(allc, 0, 0, 2, 1, restart=1), scan(allc, 0, 0, 1, 0, restart=0)]
        s += [scan(c, 1, 63, 2, 1, restart=7, com=True) for c in comps[sub]]
        s += [scan(c, 1, 63, 1, 0) for c in comps[sub]]
        add(f"restart_{sub}_61x75", 61, 75, sub, s, seed=2)
    # refinement from Al = 13 down, one bit per scan
    s = [scan((0,), 0, 0, 0, 13)] + [scan((0,), 0, 0, a + 1, a) for a in range(12, -1, -1)]
    s += [scan((0,), 1, 9, 0, 13)] + [scan((0,), 1, 9, a + 1, a) for a in range(12, 5, -1)]
    s += [scan((0,), 1, 9, 6, 5), scan((0,), 1, 9, 5, 4), scan((0,), 1, 9, 4, 3), scan((0,), 1, 9, 3, 2),
          scan((0,), 1, 9, 2, 1), scan((0,), 1, 9, 1, 0)]
    add("al13_gray_24x40", 24, 40, "gray", s, seed=3, quant=[np.ones(64, np.int32)])
    # long EOB runs: zigzag 20..63 all zero, in one-component scans with and without restart intervals
    s = [scan((0,), *f) for f in FULL]
    add("eob_gray_480x640", 480, 640, "gray", s, seed=4, zero_from=20)
    s = [scan((0, 1, 2), 0, 0, 0, 1)] + [scan((c,), 1, 63, 0, 1, restart=700) for c in range(3)]
    s += [scan((0, 1, 2), 0, 0, 1, 0)] + [scan((c,), 1, 63, 1, 0, restart=300 * (c + 1)) for c in range(3)]
    add("eob_444_223x225", 223, 225, "444", s, seed=5, zero_from=12)
    return out


# ------------------------------------------------------------------------------------------------ taking files apart
def split(data: bytes) -> Tuple[List[Tuple[bytes, List[bytes]]], bytes]:
    """([(the bytes before scan s's entropy data, from the previous scan's end; the unstuffed bytes of each of its restart
    intervals)], the bytes from the last scan's end): fill bytes before a marker are dropped, so
    ``assemble(*split(data))`` holds the same scans."""
    info = jpeg.parse(data)
    parts, p = [], 0
    for sc in info.scans:
        comp, rst = jpeg.unstuff(data[sc.offset:sc.offset + sc.length])
        edges = [0] + rst + [len(comp)]
        parts.append((data[p:sc.offset], [comp[a:b] for a, b in zip(edges[:-1], edges[1:])]))
        p = sc.offset + sc.length
        while data[p + 1] == 0xFF:
            p += 1
    return parts, data[p:]


def assemble(parts, tail: bytes = b"\xff\xd9", fill: int = 0, rst: Optional[dict] = None) -> bytes:
    """A file of ``split``'s parts: each interval stuffed, RSTn markers between the intervals of a scan (``rst[s]``
    gives the n of scan s's markers, else 0, 1, .., 7, 0, ..), and ``fill`` 0xFF bytes before every marker."""
    out = []
    for s, (pre, ivs) in enumerate(parts):
        out.append(b"\xff" * fill + pre if s else pre)
        for i, b in enumerate(ivs):
            if i:
                n = rst[s][i - 1] if rst and s in rst else (i - 1) % 8
                out.append(b"\xff" * fill + bytes([0xFF, 0xD0 + n]))
            out.append(stuff(b))
    return b"".join(out) + b"\xff" * fill + tail


# ------------------------------------------------------------------------------------------------ worst cases
def _dc_walk(h, w, sub, comps, restart, fn):
    """fn(stream-order block, scan-order index, component, index of the block of its component within its interval)
    for each block of a DC first scan."""
    g = geometry(h, w, sub)
    blks, per = order(h, w, sub, comps)
    seen = {}
    for i, b in enumerate(blks):
        u = i // per
        if i % per == 0 and (u == 0 or restart and u % restart == 0):
            seen = {}
        c = g.comp_of[b % g.bpm] if per > 1 else comps[0]
        seen[c] = seen.get(c, 0) + 1
        fn(b, i, c, seen[c])


def worst_first(h: int, w: int, sub: str, kind: str, restart: int = 0) -> Tuple[bytes, np.ndarray, List[int]]:
    """The worst case of the self-synchronisation of a first scan, a valid file: (file, final coefficients, the bits of
    one unit of each scan's stream, 0 for a scan of at most one subsequence per interval).

    ``kind="ac"`` (grayscale): a DC first scan of 1-bit zero differences, then an AC first scan of zigzag 1..63 under a
    one-symbol table whose (run 0, size 1) code is 16 zero bits, over all-zero bits: every coefficient is a 17-bit -1,
    1071 bits per block.  ``kind="dc"``: a DC first scan of every component (interleaved for 4:2:0) whose one code, 16
    zero bits, is category 1: 17-bit blocks of difference -1; then AC first scans of 1..63 that send nothing.  Every bit
    offset starts a valid symbol and never reaches an invalid one, so a decoder started in the wrong phase never
    resynchronises; the true state moves one subsequence per round."""
    nc = SAMPLING[sub][0]
    g = geometry(h, w, sub)
    allc = tuple(range(nc))
    q = [np.ones(64, np.int32)]
    coef = np.zeros((g.blocks, 64), np.int64)
    _, per = order(h, w, sub, allc)
    units = g.blocks // per
    counts = [min(restart, units - u) if restart else units for u in range(0, units, restart or units)]
    if kind == "ac":
        assert sub == "gray"
        coef[:, 1:] = -1
        script = [scan((0,), 0, 0, 0, 0, raw=[np.zeros(g.blocks, np.uint8)], table=one_symbol(0), holds=coef),
                  scan((0,), 1, 63, 0, 0, restart, raw=[np.zeros(n * 63 * 17, np.uint8) for n in counts],
                       table=one_symbol(0x01, 16), holds=coef)]
        return (*craft(h, w, sub, q, coef, script), [1, 63 * 17])

    def dc(b, i, c, n):
        coef[b, 0] = -n
    _dc_walk(h, w, sub, allc, restart, dc)
    script = [scan(allc, 0, 0, 0, 0, restart, raw=[np.zeros(n * per * 17, np.uint8) for n in counts],
                   table=one_symbol(0x01, 16), holds=coef)]
    script += [scan((c,), 1, 63, 0, 0) for c in allc]
    return (*craft(h, w, sub, q, coef, script), [per * 17] + [0] * nc)


def saturating(h: int, w: int, nsubs: int, sbits: int, coded: bool = False) -> Tuple[bytes, np.ndarray, List[int]]:
    """A valid grayscale file whose AC first scan (1..63) is ``nsubs`` subsequences of EOB runs: EOB14 runs of
    2^14 - 1 + 0b10101010101010 = 27305 blocks after their own, each a 2-bit code and its 14 bits.  The first runs end the
    scan's blocks and libjpeg drops the rest, but the blocks the subsequences own add up to nsubs times what one owns.
    ``coded``: 48-bit units of a 1-bit EOB14 and its bits, a block of +1 at zigzag 1 (2-bit code, 1 bit, 3-bit EOB) and
    nine 3-bit EOBs, 27316 blocks, so that later subsequences write coefficients; else 16-bit units of the run alone.
    A unit divides a subsequence, so every subsequence starts in phase."""
    g = geometry(h, w, "gray")
    coef = np.zeros((g.blocks, 64), np.int64)
    unit = 48 if coded else 16
    assert sbits % unit == 0
    if coded:
        table = ([1, 1, 1] + [0] * 13, [0xE0, 0x01, 0x00])           # codes 0, 10, 110
        data = pack("0" + "10101010101010" + "101" + "110" * 10) * (nsubs * sbits // 48)
        coef[27306::27316, 1] = 1
    else:
        table = one_symbol(0xE0, 2)
        data = b"\x2a\xaa" * (nsubs * sbits // 16)
    script = [scan((0,), 0, 0, 0, 0, raw=[np.zeros(g.blocks, np.uint8)], table=one_symbol(0), holds=coef),
              scan((0,), 1, 63, 0, 0, raw=[data], table=table, holds=coef)]
    return (*craft(h, w, "gray", [np.ones(64, np.int32)], coef, script), [1, unit])


def closed_form_counters(data: bytes, sbits: int, unit_bits: Sequence[int]) -> np.ndarray:
    """The six counters of the device decode (unstuffed bytes, RST markers, subsequences, rounds, cutoff, scans decoded
    whole) of a valid file of ``worst_first`` or ``saturating``.  A first scan's subsequences start in the wrong phase
    unless a unit of its stream (``unit_bits``) divides ``sbits``; then the true state reaches the last subsequence of
    an interval after one round per subsequence, else after one round.  A scan of unit 0 has at most one subsequence in
    an interval."""
    info = jpeg.parse(data)
    g = jpeg.geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    T = R = NS = rounds = 0
    for sc, ub in zip(info.scans, unit_bits):
        comp, rst = jpeg.unstuff(data[sc.offset:sc.offset + sc.length])
        T, R = T + len(comp), R + len(rst)
        blks, per = jpeg.scan_blocks(info, sc)
        nseg = -(-(len(blks) // per) // sc.restart) if sc.restart else 1
        n = [-(-8 * (e - s) // sbits) for s, e in jpeg.segments(len(comp), rst, nseg)]
        assert ub or max(n) <= 1
        NS += sum(n)
        rounds += max(n) if ub and sbits % ub else 1
    return np.array([T, R, NS, rounds, g.blocks, len(info.scans)], np.int32)
