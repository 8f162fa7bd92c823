"""Baseline and progressive JPEG files at ingress: the marker parser and per-sample block of ``DEFER(decode="jpeg")``, and ``decode_jpeg``,
the host restatement that the GPU decode (``DEFER_OP_JPEG_DECODE``) is tested against.

``decode_jpeg(data)`` equals ``np.asarray(PIL.Image.open(io.BytesIO(data)).convert("RGB"))`` byte for byte for the files
``parse`` accepts, with Pillow built against libjpeg-turbo 3.1 (its default decode: Huffman, integer ISLOW IDCT, "fancy"
triangular upsampling, fixed-point YCbCr->RGB of ``jdcolor.c``).  Other libjpeg builds, IJG 9 among them, upsample
differently and can give other pixels.

That holds while every output of the IDCT stays within +-512 of 128, as it does for the blocks encoders write from 8-bit
images.  Beyond that range the samples are those of libjpeg's C code: ``jidctint.c`` wraps each output to 10 bits
before the clamp to 0..255 (``idct_range_limit[x & 1023]``), so 128 + 1100 gives 204, not 255, and coefficients are
int16 as ``jdhuff.c`` / ``jdphuff.c`` store them (a DC predictor past 32767, ``v << Al`` of a first scan).  Only
hand-made or corrupt files get there (large coefficients or quantisers).  There the decode equals Pillow whose
libjpeg-turbo 3.1 runs its C path (``JSIMD_FORCENONE=1``, or a build without SIMD), checked against libjpeg-turbo 3.1's
C path on files that cross every edge of the wrap and the clamp (tests/test_jpeg_idct_range_host.py); Pillow's default
on x86, the SIMD IDCT, saturates instead of wrapping and gives other pixels.

The feeder only walks the markers (``parse``) and decodes no Huffman code: past the scan header, byte searches find the
EOI that ends the entropy-coded data.  Tables derived from DQT and DHT segments are memoised on the segment bytes,
as a stream from one encoder repeats them.

The entropy-coded data ends at the first EOI after the scan header (a second SOS or a DNL marker before it is refused);
anything after the EOI, such as the secondary images of an MPF file, is ignored, as libjpeg ignores it.

Accepted: SOF0 / SOF1 with 8-bit samples, one scan holding every component, 1 (grayscale) or 3 (YCbCr) components,
luma sampling 1x1, 2x1 or 2x2 with 1x1 chroma (4:4:4, 4:2:2, 4:2:0), restart intervals, any APPn / COM segments.  Anything
else raises a ``ValueError`` that names the reason.

Progressive files (SOF2) are accepted with the same limits.  Each scan's entropy data ends at the next marker that is not
stuffing, RSTn or fill; DHT, DRI, DQT, COM and APPn segments may come between scans, and each scan uses the Huffman
tables and restart interval in force when it starts, while a component's quantisation table is latched at its first
scan.  The scan script is checked as libjpeg checks it, and what libjpeg only warns about is refused: a DC scan with
Se != 0, an AC scan of several components or of a component before its DC scan, Ss > Se or Se > 63, Ah != 0 with
Al != Ah - 1, Al > 13, a refinement whose Ah is not the coefficients' bit state, and a first scan of coefficients already
sent.  So are DC scans of some but not all of three components, more than ``MAX_SCANS`` scans or ``MAX_TABLES`` distinct
Huffman tables, and files libjpeg-turbo would decode with block smoothing (every component has had a DC scan and some
component's zigzag coefficients 1..9 are not fully refined).  Coefficients 10..63 never sent or only partly refined are
fine: their missing bits are zero.  Bits of a refinement are applied as ``jdphuff.c`` applies them, in int16.

Corrupt entropy data has one defined result here, and the device computes the same (there is no promise to match libjpeg
on it).  The entropy data is unstuffed byte by byte (``unstuff``); restart interval ``k`` is the bytes between the
``k``-th and ``k+1``-th RST marker; bits past an interval's end read as zero; a block is decoded only if it starts before
the interval's end, and at most the interval's own number of blocks is decoded; an invalid Huffman code, or an AC run
past coefficient 63, ends the decode of the whole image: that block and every later block are zero.  DC prediction runs
in int32 per component and restarts with each interval.

A progressive file decodes scan by scan under the same rules for unstuffing, intervals and bits past an interval's end;
the blocks of a scan are walked in its own order (the MCUs of a scan of all components, else the component's own block
grid), and restart intervals count units of that order.  A block that is not inside an EOB run is decoded only if it
starts before its interval's end; the blocks of an EOB run belong to the symbol that starts it, and at most the
interval's own number of blocks is decoded.  An invalid code, a run past Se (a ZRL included), or a refinement symbol of a
size other than 0 or 1 ends the decode: that block and every later block of the scan, in scan order, get nothing from
the scan, no later scan is decoded, and everything the earlier scans and blocks wrote stays.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np

# ------------------------------------------------------------------------------------------------------ block layout
# One sample's int32 block (include/defer_b200.h, DEFER_OP_JPEG_DECODE):
#   [0] h  [1] w  [2] ncomp (1 | 3)  [3] luma h-sampling  [4] luma v-sampling  [5] restart interval (MCUs, 0 = none)
#   [6] entropy-data offset in the file  [7] entropy-data length  [8] MCUs across  [9] MCUs down  [10..15] zero
#   [16 .. 16 + 3*64)                   quantisation table of component c, natural order
#   [Q_END + t * HUFF_INTS ...]         Huffman table t: DC of component 0, 1, 2, then AC of component 0, 1, 2
# A Huffman table is [lookahead[2^LOOKAHEAD] (len << 8 | symbol for codes of <= LOOKAHEAD bits, else 0),
#                     maxcode[17] (largest code of length l, -1 if none), valoff[17] (symbol index - code), vals[256]]
#   [10] scans of a progressive file (0 = baseline)  [11] Huffman tables in its pool
# A progressive file's block goes on past the baseline part (whose six Huffman tables it leaves zero):
#   [SCAN_OFF + s * SCAN_INTS ...]      scan s: components in scan, their frame indices [3], Ss, Se, Ah, Al, restart
#                                       interval (MCUs, or blocks of a one-component scan), entropy offset and length,
#                                       pool index of each component's DC table [3], pool index of the AC table, 0
#   [POOL_OFF + t * HUFF_INTS ...]      Huffman table t of the pool
# Only the prefix a file uses is copied to the GPU: BASE_INTS values for a baseline file (``block_ints``).
HDR_INTS = 16
Q_OFF = HDR_INTS
Q_END = Q_OFF + 3 * 64
LOOKAHEAD = 9
HUFF_INTS = (1 << LOOKAHEAD) + 17 + 17 + 256
BASE_INTS = Q_END + 6 * HUFF_INTS
MAX_SCANS = 32                    # DEFER_JPEG_MAX_SCANS: scans of one progressive file
MAX_TABLES = 32                   # DEFER_JPEG_MAX_TABLES: distinct Huffman tables of one progressive file
SCAN_INTS = 16
SCAN_OFF = BASE_INTS
POOL_OFF = SCAN_OFF + MAX_SCANS * SCAN_INTS
BLOCK_INTS = POOL_OFF + MAX_TABLES * HUFF_INTS

#: zigzag position k -> natural (row-major) index
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int32)

_SOF_NAMES = {0xC3: "lossless", 0xC5: "differential (hierarchical)",
              0xC6: "differential progressive", 0xC7: "differential lossless", 0xC9: "arithmetic-coded",
              0xCA: "arithmetic-coded progressive", 0xCB: "arithmetic-coded lossless",
              0xCD: "arithmetic-coded differential", 0xCE: "arithmetic-coded differential progressive",
              0xCF: "arithmetic-coded differential lossless"}


@dataclass(frozen=True)
class Scan:
    """One scan of a progressive file."""
    comps: Tuple[int, ...]        # frame indices of its components (all of them, in frame order, or one)
    ss: int                       # spectral selection Ss..Se (zigzag), successive approximation Ah, Al
    se: int
    ah: int
    al: int
    restart: int                  # restart interval in force at the scan: MCUs, or blocks of a one-component scan
    offset: int                   # entropy-coded data: data[offset:offset + length]
    length: int
    dc: Tuple[int, ...]           # pool index of each component's DC table (a DC first scan), else -1
    ac: int                       # pool index of the AC table (an AC scan), else -1


@dataclass(frozen=True)
class JpegInfo:
    h: int
    w: int
    ncomp: int
    hs: int                       # luma sampling factors (1 for grayscale)
    vs: int
    restart: int                  # restart interval in MCUs, 0 = none
    offset: int                   # entropy-coded data: data[offset:offset + length] (up to the EOI marker)
    length: int
    quant: Tuple[np.ndarray, ...]  # per component, int32 [64] natural order
    dc: Tuple[np.ndarray, ...]     # per component, int32 [HUFF_INTS] (baseline)
    ac: Tuple[np.ndarray, ...]
    scans: Tuple[Scan, ...] = ()   # progressive: its scans in file order, and the Huffman tables they use
    tables: Tuple[np.ndarray, ...] = ()

    @property
    def progressive(self) -> bool:
        return bool(self.scans)


def _refuse(why: str):
    raise ValueError(f"JPEG refused: {why}")


@functools.lru_cache(maxsize=256)
def dqt_tables(seg: bytes) -> dict:
    """``{Tq: int32 [64] natural order}`` of one DQT segment's payload (memoised on its bytes; read-only arrays)."""
    out, p = {}, 0
    while p < len(seg):
        pq, tq = seg[p] >> 4, seg[p] & 15
        if pq != 0:
            _refuse("16-bit quantisation table (8-bit samples take 8-bit tables)")
        if tq > 3 or p + 65 > len(seg):
            _refuse("malformed DQT segment")
        q = np.zeros(64, np.int32)
        q[ZIGZAG] = np.frombuffer(seg, np.uint8, 64, p + 1)
        q.setflags(write=False)
        out[tq] = q
        p += 65
    return out


def huff_table(counts: bytes, vals: bytes) -> np.ndarray:
    """The device form of one Huffman table (layout above) from its 16 code-length counts and symbols."""
    t = np.zeros(HUFF_INTS, np.int32)
    lut = t[:1 << LOOKAHEAD]
    maxcode = t[1 << LOOKAHEAD:(1 << LOOKAHEAD) + 17]
    valoff = t[(1 << LOOKAHEAD) + 17:(1 << LOOKAHEAD) + 34]
    t[(1 << LOOKAHEAD) + 34:(1 << LOOKAHEAD) + 34 + len(vals)] = np.frombuffer(vals, np.uint8)
    maxcode[:] = -1
    code, k = 0, 0
    for l in range(1, 17):
        n = counts[l - 1]
        if n:
            valoff[l] = k - code
            for _ in range(n):
                if code >= (1 << l):
                    _refuse("malformed Huffman table (over-subscribed code lengths)")
                if l <= LOOKAHEAD:
                    sh = LOOKAHEAD - l
                    lut[code << sh:(code + 1) << sh] = (l << 8) | vals[k]
                code += 1
                k += 1
            maxcode[l] = code - 1
        code <<= 1
    return t


@functools.lru_cache(maxsize=256)
def dht_tables(seg: bytes) -> dict:
    """``{(Tc, Th): int32 [HUFF_INTS]}`` of one DHT segment's payload (memoised on its bytes; read-only arrays)."""
    out, p = {}, 0
    while p < len(seg):
        if p + 17 > len(seg):
            _refuse("malformed DHT segment")
        tc, th = seg[p] >> 4, seg[p] & 15
        counts = seg[p + 1:p + 17]
        n = sum(counts)
        if tc > 1 or th > 3 or n > 256 or p + 17 + n > len(seg):
            _refuse("malformed DHT segment")
        vals = seg[p + 17:p + 17 + n]
        if tc == 0 and any(v > 11 for v in vals):
            _refuse("DC Huffman symbol above 11 (8-bit samples)")
        if tc == 1 and any((v & 15) > 10 for v in vals):
            _refuse("AC Huffman symbol with a size above 10 (8-bit samples)")
        t = huff_table(counts, vals)
        t.setflags(write=False)
        out[(tc, th)] = t
        p += 17 + n
    return out


def _as_bytes(data) -> bytes:
    # a bytearray, memoryview or array is copied: the H2D copy of the item is asynchronous, and the caller may change a
    # mutable buffer after putting it on the queue
    if isinstance(data, (bytes, bytearray, memoryview)):
        return bytes(data)
    if isinstance(data, np.ndarray) and data.dtype == np.uint8 and data.ndim == 1:
        return data.tobytes()
    raise ValueError(f"a JPEG item is bytes, bytearray, memoryview or a 1-D uint8 array holding one file, got "
                     f"{type(data).__name__}" + (f" {data.dtype} {data.shape}" if isinstance(data, np.ndarray) else ""))


def parse(data) -> JpegInfo:
    """Walk the markers of one JPEG file; its geometry, tables and entropy-data extent, or a ValueError naming why the
    file is refused.  Every segment length is checked against the buffer; the entropy data is not read."""
    d = _as_bytes(data)
    n = len(d)
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        _refuse("not a JPEG file (no SOI marker)")
    p = 2
    qt, ht, frame, restart, progressive = {}, {}, None, 0, False
    jfif, adobe = False, None
    while True:
        if p >= n or d[p] != 0xFF:
            _refuse(f"malformed file (no marker at byte {p})")
        while p < n and d[p] == 0xFF:
            p += 1
        if p >= n:
            _refuse("truncated file (no EOI marker)")
        m = d[p]
        p += 1
        if m == 0xD9:
            _refuse("no scan before the EOI marker")
        if m in (0x01,) or 0xD0 <= m <= 0xD8:
            _refuse(f"unexpected marker 0xFF{m:02X} outside the scan")
        if p + 2 > n:
            _refuse("truncated file (no EOI marker)")
        ln = (d[p] << 8) | d[p + 1]
        if ln < 2 or p + ln > n:
            _refuse(f"segment 0xFF{m:02X} of length {ln} runs past the end of the file")
        seg = d[p + 2:p + ln]
        p += ln
        if m == 0xE0 and seg[:5] == b"JFIF\0":
            jfif = True
        elif m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
            adobe = seg[11]
        elif m == 0xDB:
            qt.update(dqt_tables(seg))
        elif m == 0xC4:
            ht.update(dht_tables(seg))
        elif m == 0xDD:
            if len(seg) != 2:
                _refuse("malformed DRI segment")
            restart = (seg[0] << 8) | seg[1]
        elif m in (0xC0, 0xC1, 0xC2):
            progressive = m == 0xC2
            if frame is not None:
                _refuse("more than one frame")
            if len(seg) < 6:
                _refuse("malformed SOF segment")
            prec, h, w, nc = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if prec != 8:
                _refuse(f"{prec}-bit samples (only 8-bit JPEGs are decoded)")
            if nc not in (1, 3):
                _refuse(f"{nc} components (1 or 3 are decoded; 2 or 4, e.g. CMYK, are not)")
            if len(seg) != 6 + 3 * nc:
                _refuse("malformed SOF segment")
            if h == 0 or w == 0:
                _refuse(f"image size {h}x{w} (a height defined by a DNL marker is not supported)")
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nc)]
            frame = (h, w, comps)
        elif m in _SOF_NAMES:
            _refuse(f"{_SOF_NAMES[m]} JPEG (only baseline, extended sequential and progressive Huffman JPEGs are "
                    "decoded)")
        elif m == 0xDA:
            break
        elif 0xE0 <= m <= 0xEF or m == 0xFE:
            pass
        else:
            _refuse(f"unsupported marker 0xFF{m:02X}")
    if frame is None:
        _refuse("no SOF0/SOF1/SOF2 frame before the scan")
    h, w, comps = frame
    nc = len(comps)
    ids = tuple(c[0] for c in comps)
    if nc == 3 and not jfif and ((adobe is not None and adobe == 0) or (adobe is None and ids == (82, 71, 66))):
        _refuse("RGB colour transform (Adobe or 'RGB' component ids; only YCbCr is decoded)")
    if nc == 3 and adobe is not None and adobe not in (0, 1) and not jfif:
        _refuse(f"Adobe colour transform {adobe}")
    if progressive:
        return _parse_progressive(d, p, seg, h, w, comps, qt, ht, restart)
    ns = seg[0] if seg else 0
    if len(seg) != 4 + 2 * ns:
        _refuse("malformed SOS segment")
    if ns != nc:
        _refuse("more than one scan (a scan holds only some of the components)")
    scan = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
    if [c[0] for c in scan] != [c[0] for c in comps]:
        _refuse("scan components out of frame order")
    ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
    if (ss, se, ahal) != (0, 63, 0):
        _refuse("spectral selection or successive approximation in a sequential scan")
    hs, vs = _sampling(comps)
    quant, dc, ac = [], [], []
    for (cid, _, _, tq), (_, td, ta) in zip(comps, scan):
        if tq not in qt:
            _refuse(f"component {cid} uses undefined quantisation table {tq}")
        if (0, td) not in ht or (1, ta) not in ht:
            _refuse(f"component {cid} uses an undefined Huffman table")
        quant.append(qt[tq])
        dc.append(ht[(0, td)])
        ac.append(ht[(1, ta)])
    # Inside the scan an 0xFF is followed by 0x00, RSTn or another 0xFF, so the first EOI after the scan header ends it;
    # what follows (e.g. the secondary images of an MPF file) is not read.  Three byte searches, no Huffman decoding.
    end = d.find(b"\xff\xd9", p)
    if end < 0:
        _refuse("truncated file (no EOI marker)")
    if d.find(b"\xff\xda", p, end) >= 0:
        _refuse("more than one scan")
    if d.find(b"\xff\xdc", p, end) >= 0:
        _refuse("DNL marker after the scan")
    while end > p and d[end - 1] == 0xFF:      # fill bytes before the marker
        end -= 1
    return JpegInfo(h, w, nc, hs, vs, restart, p, end - p, tuple(quant), tuple(dc), tuple(ac))


def _sampling(comps) -> Tuple[int, int]:
    """Luma sampling factors (hs, vs) of the frame's components, or a refusal."""
    if len(comps) == 1:
        return 1, 1
    hs, vs = comps[0][1], comps[0][2]
    if (hs, vs) not in ((1, 1), (2, 1), (2, 2)) or any((c[1], c[2]) != (1, 1) for c in comps[1:]):
        _refuse("sampling factors " + ",".join(f"{c[1]}x{c[2]}" for c in comps)
                + " (4:4:4, 4:2:2 and 4:2:0 are decoded)")
    return hs, vs


def _parse_progressive(d: bytes, p: int, seg: bytes, h: int, w: int, comps, qt: dict, ht: dict, restart: int) -> JpegInfo:
    """The scans of a progressive file, from its first SOS (payload ``seg``, entropy data from ``p``) to the EOI.  The
    scan script is checked as libjpeg's ``start_pass_phuff_decoder`` checks it, and what libjpeg only warns about is
    refused here too; so is a file libjpeg would decode with block smoothing.  Each scan's entropy data ends at the next
    marker that is not stuffing, RSTn or fill: one vectorised byte search per file."""
    nc = len(comps)
    hs, vs = _sampling(comps)
    b = np.frombuffer(d, np.uint8)
    nxt = b[1:]
    ends = np.nonzero((b[:-1] == 0xFF) & (nxt != 0) & ((nxt < 0xD0) | (nxt > 0xD7)) & (nxt != 0xFF))[0]
    ids = [c[0] for c in comps]
    bits = [[-1] * 64 for _ in range(nc)]         # libjpeg's coef_bits: -1 = never sent, else the last scan's Al
    quant: List[Optional[np.ndarray]] = [None] * nc
    scans, pool, pool_ix = [], [], {}

    def table(key, cid):
        if key not in ht:
            _refuse(f"component {cid} uses an undefined Huffman table")
        t = ht[key]
        if id(t) not in pool_ix:
            if len(pool) == MAX_TABLES:
                _refuse(f"more than {MAX_TABLES} distinct Huffman tables in one progressive file (DEFER_JPEG_MAX_TABLES)")
            pool_ix[id(t)] = len(pool)
            pool.append(t)
        return pool_ix[id(t)]

    while True:                                   # at a scan: seg is its SOS payload, p its first entropy byte
        if len(scans) == MAX_SCANS:
            _refuse(f"more than {MAX_SCANS} scans in one progressive file (DEFER_JPEG_MAX_SCANS)")
        ns = seg[0] if seg else 0
        if ns < 1 or len(seg) != 4 + 2 * ns:
            _refuse("malformed SOS segment")
        sel = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
        if any(c[0] not in ids for c in sel):
            _refuse("scan of a component the frame does not have")
        idx = [ids.index(c[0]) for c in sel]
        if idx != sorted(set(idx)):
            _refuse("scan components repeated or out of frame order")
        ss, se, ah, al = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns] >> 4, seg[3 + 2 * ns] & 15
        if ss == 0 and se != 0:
            _refuse(f"bad progressive scan script: a DC scan with Se = {se}")
        if ss != 0 and (ss > se or se > 63):
            _refuse(f"bad progressive scan script: spectral selection {ss}..{se}")
        if ss != 0 and ns != 1:
            _refuse(f"bad progressive scan script: an AC scan of {ns} components")
        if ah != 0 and al != ah - 1:
            _refuse(f"bad progressive scan script: successive approximation Ah = {ah}, Al = {al}")
        if al > 13:
            _refuse(f"bad progressive scan script: Al = {al} > 13")
        if 1 < ns < nc:
            _refuse(f"progressive DC scan of {ns} of {nc} components (interleaved scans of all components or "
                    "scans of one are decoded)")
        for c in idx:
            if ss > 0 and bits[c][0] < 0:
                _refuse(f"bad progressive scan script: an AC scan of component {ids[c]} before its DC scan")
            for k in range(ss, se + 1):
                cur = bits[c][k]
                if ah != max(cur, 0):
                    _refuse(f"bad progressive scan script: component {ids[c]} coefficient {k} refined with Ah = "
                            f"{ah}, its bit state is {cur}")
                if ah == 0 and cur >= 0:
                    _refuse(f"bad progressive scan script: component {ids[c]} coefficient {k} sent twice")
                bits[c][k] = al
            if quant[c] is None:                  # latch_quant_tables: a later DQT does not change it
                tq = comps[c][3]
                if tq not in qt:
                    _refuse(f"component {ids[c]} uses undefined quantisation table {tq}")
                quant[c] = qt[tq]
        dc = tuple(table((0, td), cid) for cid, td, _ in sel) if ss == 0 and ah == 0 else (-1,) * ns
        ac = table((1, sel[0][2]), sel[0][0]) if ss > 0 else -1
        i = int(np.searchsorted(ends, p))
        if i == len(ends):
            _refuse("truncated file (no EOI marker)")
        end = int(ends[i])
        e = end
        while e > p and d[e - 1] == 0xFF:         # fill bytes before the marker
            e -= 1
        scans.append(Scan(tuple(idx), ss, se, ah, al, restart, p, e - p, dc + (-1,) * (3 - ns), ac))
        p = end
        while True:                               # the markers up to the next scan or the EOI
            while p < len(d) and d[p] == 0xFF:
                p += 1
            if p >= len(d):
                _refuse("truncated file (no EOI marker)")
            m = d[p]
            p += 1
            if m == 0xD9:
                break
            if m == 0xDC:
                _refuse("DNL marker after the scan")
            if m in (0x01,) or 0xD0 <= m <= 0xD8 or 0xC0 <= m <= 0xCF and m != 0xC4:
                _refuse(f"unexpected marker 0xFF{m:02X} between scans")
            if p + 2 > len(d):
                _refuse("truncated file (no EOI marker)")
            ln = (d[p] << 8) | d[p + 1]
            if ln < 2 or p + ln > len(d):
                _refuse(f"segment 0xFF{m:02X} of length {ln} runs past the end of the file")
            seg = d[p + 2:p + ln]
            p += ln
            if m == 0xDA:
                break
            if m == 0xDB:
                qt.update(dqt_tables(seg))
            elif m == 0xC4:
                ht.update(dht_tables(seg))
            elif m == 0xDD:
                if len(seg) != 2:
                    _refuse("malformed DRI segment")
                restart = (seg[0] << 8) | seg[1]
            elif not (0xE0 <= m <= 0xEF or m == 0xFE):
                _refuse(f"unsupported marker 0xFF{m:02X} between scans")
        if m == 0xD9:
            break
    # libjpeg-turbo 3.1 smooths blocks (smoothing_ok) when every component has had a DC scan, none of its quantisers of
    # zigzag 0..9 is zero, and some component's coefficients 1..9 are not fully refined
    if (all(bits[c][0] >= 0 for c in range(nc)) and all(int(q[n]) != 0 for q in quant for n in ZIGZAG[:10])
            and any(bits[c][k] != 0 for c in range(nc) for k in range(1, 10))):
        _refuse("incomplete progression: zigzag coefficients 1..9 are not all fully refined, which libjpeg decodes "
                "with block smoothing (not supported)")
    q = tuple(x if x is not None else np.zeros(64, np.int32) for x in quant)
    first = scans[0].offset
    last = max(s.offset + s.length for s in scans)
    return JpegInfo(h, w, nc, hs, vs, 0, first, last - first, q, (), (), tuple(scans), tuple(pool))


@dataclass(frozen=True)
class Geometry:
    mcux: int
    mcuy: int
    bpm: int                         # blocks per MCU
    comp_of: Tuple[int, ...]         # component of each block within the MCU
    bw: Tuple[int, ...]              # blocks across / down per component plane
    bh: Tuple[int, ...]

    @property
    def mcus(self) -> int:
        return self.mcux * self.mcuy

    @property
    def blocks(self) -> int:
        return self.mcus * self.bpm


def geometry(h: int, w: int, ncomp: int, hs: int, vs: int) -> Geometry:
    if ncomp == 1:
        mx, my = -(-w // 8), -(-h // 8)
        return Geometry(mx, my, 1, (0,), (mx,), (my,))
    mx, my = -(-w // (8 * hs)), -(-h // (8 * vs))
    return Geometry(mx, my, hs * vs + 2, (0,) * (hs * vs) + (1, 2), (mx * hs, mx, mx), (my * vs, my, my))


def block_ints(info: JpegInfo) -> int:
    """How much of its block a file uses: the baseline part, or up to the last Huffman table of its pool."""
    return POOL_OFF + len(info.tables) * HUFF_INTS if info.progressive else BASE_INTS


def pack_block(info: JpegInfo, out: Optional[np.ndarray] = None) -> np.ndarray:
    """One sample's int32 block (layout above); ``out``: a zeroed int32 [BLOCK_INTS] to write it into."""
    b = np.zeros(BLOCK_INTS, np.int32) if out is None else out
    g = geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    b[:12] = (info.h, info.w, info.ncomp, info.hs, info.vs, info.restart, info.offset, info.length, g.mcux, g.mcuy,
              len(info.scans), len(info.tables))
    for c in range(info.ncomp):
        b[Q_OFF + 64 * c:Q_OFF + 64 * (c + 1)] = info.quant[c]
        if not info.progressive:
            b[Q_END + c * HUFF_INTS:Q_END + (c + 1) * HUFF_INTS] = info.dc[c]
            b[Q_END + (3 + c) * HUFF_INTS:Q_END + (4 + c) * HUFF_INTS] = info.ac[c]
    for i, sc in enumerate(info.scans):
        comps = sc.comps + (0,) * (3 - len(sc.comps))
        b[SCAN_OFF + i * SCAN_INTS:SCAN_OFF + (i + 1) * SCAN_INTS] = (
            len(sc.comps), *comps, sc.ss, sc.se, sc.ah, sc.al, sc.restart, sc.offset, sc.length, *sc.dc, sc.ac, 0)
    for t, tab in enumerate(info.tables):
        b[POOL_OFF + t * HUFF_INTS:POOL_OFF + (t + 1) * HUFF_INTS] = tab
    return b


DECODES = ("jpeg",)               # the format this module parses; image.DECODES: every format a pipeline decodes


def check_decode(decode, preprocess, image_size, max_image_size, decodes=DECODES) -> None:
    """``decode=`` of ``DEFER`` / ``plan_stage``: None, or one of ``decodes`` together with ``preprocess`` and
    ``max_image_size``.  The pipelines pass ``image.DECODES``, which adds "png" and "image" (either, told per file)."""
    if decode is None:
        return
    if decode not in decodes:
        raise ValueError(f"decode={decode!r}: the GPU decodes {', '.join(map(repr, decodes))} files")
    if image_size is not None:
        what = "image file" if decode == "image" else decode.upper()
        raise ValueError(f"decode={decode!r} and image_size={image_size}: each {what} carries its own size; give "
                         "max_image_size=(H, W), the largest image the pipeline takes")
    if preprocess is None or max_image_size is None:
        raise ValueError(f"decode={decode!r} needs preprocess= and max_image_size=: the decoded images are resized and "
                         "preprocessed on the GPU as Keras' load_img and preprocess_input do")


def check_jpeg(data, max_image_size) -> Tuple[bytes, JpegInfo]:
    """Queue item ``data`` of a ``decode="jpeg"`` pipeline as (file bytes, parsed header), or a ValueError: the file is
    refused, its image is outside ``max_image_size=(H, W)``, or it is larger than the compressed slot (H * W * 3 bytes)."""
    d = _as_bytes(data)
    H, W = max_image_size
    if len(d) > H * W * 3:
        _refuse(f"a {len(d)}-byte file is larger than the compressed slot of max_image_size=({H}, {W}) ({H * W * 3} bytes)")
    info = parse(d)
    if not (info.h <= H and info.w <= W):
        _refuse(f"a {info.h}x{info.w} image is outside max_image_size=({H}, {W})")
    return d, info


# ------------------------------------------------------------------------------------------------ the host decoder
def unstuff(entropy: bytes) -> Tuple[bytes, List[int]]:
    """The entropy data without its stuffing and RST markers, and the compacted offset where each RST marker was.  Byte
    ``i`` is dropped if it follows an 0xFF and is 0x00 or 0xD0..0xD7, or is an 0xFF followed by 0xD0..0xD7."""
    b = np.frombuffer(entropy, np.uint8)
    prev_ff = np.zeros(len(b), bool)
    prev_ff[1:] = b[:-1] == 0xFF
    rst = (b >= 0xD0) & (b <= 0xD7)
    marker = np.zeros(len(b), bool)
    marker[:-1] = (b[:-1] == 0xFF) & rst[1:]
    keep = ~((prev_ff & ((b == 0) | rst)) | marker)
    pos = np.cumsum(keep) - keep
    return b[keep].tobytes(), [int(v) for v in pos[marker]]


def segments(comp_len: int, rst: List[int], nseg: int) -> List[Tuple[int, int]]:
    """Byte range ``[start, end)`` of each of the ``nseg`` restart intervals in the compacted data."""
    starts = [0] + list(rst)
    out = []
    for k in range(nseg):
        s = starts[k] if k < len(starts) else comp_len
        e = starts[k + 1] if k + 1 < len(starts) else comp_len
        out.append((s, e))
    return out


class BitReader:
    """MSB-first bits of ``buf[start:end]`` (bytes); bits past the end read as zero."""

    def __init__(self, buf: bytes, start: int, end: int):
        self.buf = buf[start:end] + b"\0\0\0\0"
        self.nbits = 8 * (end - start)

    def peek16(self, pos: int) -> int:
        if pos >= self.nbits:
            return 0
        i = pos >> 3
        v = (int.from_bytes(self.buf[i:i + 4], "big") >> (16 - (pos & 7))) & 0xFFFF
        left = self.nbits - pos
        if left < 16:
            v &= ~((1 << (16 - left)) - 1) & 0xFFFF
        return v


def decode_symbol(t: np.ndarray, peek: int) -> Tuple[int, int]:
    """(length, symbol) of the code at the top of the 16-bit ``peek``, or (0, 0) for an invalid code."""
    e = int(t[peek >> (16 - LOOKAHEAD)])
    if e:
        return e >> 8, e & 255
    base = 1 << LOOKAHEAD
    for l in range(LOOKAHEAD + 1, 17):
        code = peek >> (16 - l)
        if code <= t[base + l]:
            return l, int(t[base + 34 + min(max(code + int(t[base + 17 + l]), 0), 255)])
    return 0, 0


def extend(v: int, s: int) -> int:
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def step_symbol(r: BitReader, pos: int, k: int, dc_t, ac_t):
    """Decode one symbol (code + extra bits) of a block at coefficient ``k`` (0 = DC).  Returns
    ``(new_pos, new_k, zigzag index written or -1, value)``; ``new_k == 64`` ends the block; None for an invalid code."""
    if k == 0:
        l, s = decode_symbol(dc_t, r.peek16(pos))
        if l == 0:
            return None
        s &= 15
        v = extend(r.peek16(pos + l) >> (16 - s), s) if s else 0
        return pos + l + s, 1, 0, v
    l, sym = decode_symbol(ac_t, r.peek16(pos))
    if l == 0:
        return None
    run, s = sym >> 4, sym & 15
    if s == 0:
        if run != 15:
            return pos + l, 64, -1, 0
        if k + 16 > 64:
            return None
        return pos + l, k + 16, -1, 0
    if k + run > 63:
        return None
    v = extend(r.peek16(pos + l) >> (16 - s), s)
    return pos + l + s, k + run + 1, k + run, v


def entropy_decode(data, info: Optional[JpegInfo] = None) -> Tuple[np.ndarray, np.ndarray]:
    """Sequential Huffman decode: int16 ``[blocks, 64]`` in stream order and natural coefficient order, DC still as the
    difference, and which blocks decoded (the others are zero)."""
    d = _as_bytes(data)
    info = info or parse(d)
    g = geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    comp, rst = unstuff(d[info.offset:info.offset + info.length])
    ri = info.restart
    nseg = -(-g.mcus // ri) if ri else 1
    coef = np.zeros((g.blocks, 64), np.int16)
    decoded = np.zeros(g.blocks, bool)
    for k, (s, e) in enumerate(segments(len(comp), rst, nseg)):
        r = BitReader(comp, s, e)
        first = k * ri * g.bpm if ri else 0
        nblk = (min(ri, g.mcus - k * ri) if ri else g.mcus) * g.bpm
        pos = 0
        for i in range(nblk):
            if pos >= r.nbits:
                break
            c = g.comp_of[i % g.bpm]
            kk, blk = 0, np.zeros(64, np.int16)
            while kk < 64:
                st = step_symbol(r, pos, kk, info.dc[c], info.ac[c])
                if st is None:
                    return coef, decoded
                pos, kk, z, v = st
                if z >= 0:
                    blk[ZIGZAG[z]] = v
            coef[first + i] = blk
            decoded[first + i] = True
    return coef, decoded


def dc_predict(coef: np.ndarray, decoded: np.ndarray, info: JpegInfo) -> np.ndarray:
    """Final quantised coefficients: DC differences summed per component in int32, restarting with each interval; blocks
    that did not decode are zero and add nothing."""
    g = geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    out = coef.copy()
    out[~decoded] = 0
    diffs = out[:, 0].astype(np.int64)
    per = info.restart * g.bpm if info.restart else g.blocks
    comp_of = np.tile(np.array(g.comp_of), g.mcus)
    for c in range(info.ncomp):
        for s in range(0, g.blocks, per):
            idx = np.nonzero(comp_of[s:s + per] == c)[0] + s
            acc = np.cumsum(diffs[idx])
            acc = ((acc + (1 << 31)) % (1 << 32)) - (1 << 31)      # int32 wrap
            out[idx, 0] = (((acc + (1 << 15)) % (1 << 16)) - (1 << 15)).astype(np.int16)
    out[~decoded] = 0
    return out


_F = {"0_298631336": 2446, "0_390180644": 3196, "0_541196100": 4433, "0_765366865": 6270, "0_899976223": 7373,
      "1_175875602": 9633, "1_501321110": 12299, "1_847759065": 15137, "1_961570560": 16069, "2_053119869": 16819,
      "2_562915447": 20995, "3_072711026": 25172}


def _idct_1d(s, pass1: bool):
    """libjpeg-turbo's jidctint.c ISLOW butterflies on int64 arrays s[0..7]; pass 1 descales by CONST_BITS - PASS1_BITS
    to int, pass 2 by CONST_BITS + PASS1_BITS + 3."""
    F = _F
    z2, z3 = s[2], s[6]
    z1 = (z2 + z3) * F["0_541196100"]
    tmp2 = z1 + z3 * -F["1_847759065"]
    tmp3 = z1 + z2 * F["0_765366865"]
    tmp0 = (s[0] + s[4]) << 13
    tmp1 = (s[0] - s[4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = s[7], s[5], s[3], s[1]
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * F["1_175875602"]
    tmp0 = tmp0 * F["0_298631336"]
    tmp1 = tmp1 * F["2_053119869"]
    tmp2 = tmp2 * F["3_072711026"]
    tmp3 = tmp3 * F["1_501321110"]
    z1 = z1 * -F["0_899976223"]
    z2 = z2 * -F["2_562915447"]
    z3 = z3 * -F["1_961570560"] + z5
    z4 = z4 * -F["0_390180644"] + z5
    tmp0 += z1 + z3
    tmp1 += z2 + z4
    tmp2 += z2 + z3
    tmp3 += z1 + z4
    sh = 11 if pass1 else 18
    o = [t10 + tmp3, t11 + tmp2, t12 + tmp1, t13 + tmp0, t13 - tmp0, t12 - tmp1, t11 - tmp2, t10 - tmp3]
    o = [(v + (1 << (sh - 1))) >> sh for v in o]
    if pass1:
        return [((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31) for v in o]    # stored as int
    return o


def idct_islow(coef: np.ndarray, quant: np.ndarray) -> np.ndarray:
    """Dequantise and inverse-DCT int16 blocks ``[n, 64]`` (natural order) with int32 ``quant[64]``: uint8 ``[n, 8, 8]``,
    each output wrapped to 10 bits and range-limited as libjpeg's ``idct_range_limit[x & 1023]``."""
    x = coef.astype(np.int64).reshape(-1, 8, 8) * quant.astype(np.int64).reshape(8, 8)
    ws = np.stack(_idct_1d([x[:, r, :] for r in range(8)], True), axis=1)          # columns: ws[n, row, col]
    out = np.stack(_idct_1d([ws[:, :, c] for c in range(8)], False), axis=2)       # rows
    v = ((out & 1023) ^ 512) - 512
    return np.clip(v + 128, 0, 255).astype(np.uint8)


def planes(coef: np.ndarray, info: JpegInfo) -> List[np.ndarray]:
    """The MCU-padded uint8 plane of each component from the final coefficients (stream order)."""
    g = geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    pix = np.empty((g.blocks, 8, 8), np.uint8)
    comp_of = np.tile(np.array(g.comp_of), g.mcus)
    for c in range(info.ncomp):
        idx = np.nonzero(comp_of == c)[0]
        pix[idx] = idct_islow(coef[idx], info.quant[c])
    out = []
    for c in range(info.ncomp):
        hc, vc = (info.hs, info.vs) if c == 0 and info.ncomp == 3 else (1, 1)
        idx = np.nonzero(comp_of == c)[0]
        b = pix[idx].reshape(g.mcuy, g.mcux, vc, hc, 8, 8)          # MCU row, MCU col, block row, block col
        out.append(np.ascontiguousarray(b.transpose(0, 2, 4, 1, 3, 5).reshape(g.bh[c] * 8, g.bw[c] * 8)))
    return out


def _upsample(p: np.ndarray, h: int, w: int, hs: int, vs: int) -> np.ndarray:
    """libjpeg-turbo's chroma upsampling of one downsampled plane to ``(h, w)``: the fancy (triangular) h2v1 / h2v2
    filters when the downsampled width exceeds 2, else pixel replication."""
    if hs == 1 and vs == 1:
        return p[:h, :w].astype(np.int32)
    dh, dw = -(-h // vs), -(-w // hs)
    x = np.arange(w)
    i = x >> 1
    odd = (x & 1) == 1
    if dw <= 2:
        y = np.arange(h) // vs
        return p[y][:, i].astype(np.int32)
    ip = np.maximum(i - 1, 0)
    inx = np.minimum(i + 1, dw - 1)
    if vs == 1:
        a = p[:h, :dw].astype(np.int32)
        even_v = np.where(i == 0, a[:, i], (3 * a[:, i] + a[:, ip] + 1) >> 2)
        odd_v = np.where(i == dw - 1, a[:, i], (3 * a[:, i] + a[:, inx] + 2) >> 2)
        return np.where(odd, odd_v, even_v)
    y = np.arange(h)
    r0 = y >> 1
    r1 = np.where((y & 1) == 0, np.maximum(r0 - 1, 0), np.minimum(r0 + 1, dh - 1))
    a = p.astype(np.int32)
    cs = 3 * a[r0][:, :dw] + a[r1][:, :dw]            # column sums, per output row
    even_v = np.where(i == 0, (cs[:, i] * 4 + 8) >> 4, (3 * cs[:, i] + cs[:, ip] + 8) >> 4)
    odd_v = np.where(i == dw - 1, (cs[:, i] * 4 + 7) >> 4, (3 * cs[:, i] + cs[:, inx] + 7) >> 4)
    return np.where(odd, odd_v, even_v)


def _fix(x: float) -> int:
    return int(x * (1 << 16) + 0.5)


def color_convert(pl: List[np.ndarray], info: JpegInfo) -> np.ndarray:
    """Upsample and convert to packed uint8 RGB ``(h, w, 3)`` (``jdcolor.c`` ycc_rgb_convert; grayscale gives R = G = B)."""
    h, w = info.h, info.w
    y = pl[0][:h, :w].astype(np.int32)
    if info.ncomp == 1:
        return np.repeat(y[:, :, None].astype(np.uint8), 3, axis=2)
    cb = _upsample(pl[1], h, w, info.hs, info.vs) - 128
    cr = _upsample(pl[2], h, w, info.hs, info.vs) - 128
    half = 1 << 15
    r = y + ((_fix(1.40200) * cr + half) >> 16)
    g = y + ((-_fix(0.34414) * cb + half - _fix(0.71414) * cr) >> 16)
    b = y + ((_fix(1.77200) * cb + half) >> 16)
    return np.ascontiguousarray(np.clip(np.stack([r, g, b], axis=2), 0, 255).astype(np.uint8))


# ----------------------------------------------------------------------------------------- progressive files, sequentially
def _i16(v: int) -> int:
    return ((v + 32768) & 0xFFFF) - 32768


def scan_blocks(info: JpegInfo, scan: Scan) -> Tuple[np.ndarray, int]:
    """The stream-order block of each block of ``scan`` in scan order, and the blocks per unit (restart intervals count
    units).  A scan of all components walks the MCUs, as a baseline scan.  A scan of one component walks that
    component's own grid of ``ceil(w * hc / (hmax * 8)) x ceil(h * vc / (vmax * 8))`` blocks, which can be smaller than
    its MCU-padded grid: the padding blocks only get a DC value, from interleaved DC scans."""
    g = geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    if len(scan.comps) > 1 or info.ncomp == 1:
        return np.arange(g.blocks), g.bpm if len(scan.comps) > 1 else 1
    c = scan.comps[0]
    hc, vc = (info.hs, info.vs) if c == 0 else (1, 1)
    cw, ch = -(-info.w * hc // (info.hs * 8)), -(-info.h * vc // (info.vs * 8))
    by, bx = np.divmod(np.arange(cw * ch), cw)
    j = (by % vc) * hc + bx % hc if c == 0 else info.hs * info.vs + c - 1
    return ((by // vc) * g.mcux + bx // hc) * g.bpm + j, 1


def _bit(r: BitReader, pos: int) -> int:
    return r.peek16(pos) >> 15


def _decode_interval(r: BitReader, sc: Scan, tabs, zz, blks, comp_of) -> Optional[int]:
    """Decode one restart interval of scan ``sc`` into the zigzag-order coefficient lists ``zz``: ``blks`` are its
    stream-order blocks in scan order, ``comp_of`` the scan component of each position in a unit.  Returns the index in
    ``blks`` of the block whose decode failed (it and every later block get nothing from the scan), else None."""
    ss, se, al, pos = sc.ss, sc.se, sc.al, 0
    if ss == 0 and sc.ah == 0:                        # DC first
        pred = [0, 0, 0]
        for i, b in enumerate(blks):
            if pos >= r.nbits:
                break
            c = comp_of[i % len(comp_of)]
            l, s = decode_symbol(tabs[sc.dc[c]], r.peek16(pos))
            if l == 0:
                return i
            s &= 15
            v = extend(r.peek16(pos + l) >> (16 - s), s) if s else 0
            pos += l + s
            pred[c] = ((pred[c] + v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)
            zz[b][0] = _i16(pred[c] << al)
        return None
    if ss == 0:                                       # DC refinement: one raw bit per block
        for i, b in enumerate(blks):
            if pos >= r.nbits:
                break
            if _bit(r, pos):
                zz[b][0] = _i16(zz[b][0] | (1 << al))
            pos += 1
        return None
    t, eob = tabs[sc.ac], 0
    if sc.ah == 0:                                    # AC first
        for i, b in enumerate(blks):
            if eob:
                eob -= 1
                continue
            if pos >= r.nbits:
                break
            k, new = ss, {}
            while k <= se:
                l, sym = decode_symbol(t, r.peek16(pos))
                if l == 0:
                    return i
                pos += l
                run, s = sym >> 4, sym & 15
                if s:
                    k += run
                    if k > se:
                        return i
                    new[k] = _i16(extend(r.peek16(pos) >> (16 - s), s) << al)
                    pos += s
                    k += 1
                elif run == 15:
                    if k + 16 > se + 1:
                        return i
                    k += 16
                else:
                    eob = (1 << run) - 1 + ((r.peek16(pos) >> (16 - run)) if run else 0)
                    pos += run
                    break
            for k, v in new.items():
                zz[b][k] = v
        return None
    p1, m1 = 1 << al, -(1 << al)                      # AC refinement

    def correct(v):
        return _i16(v + (p1 if v >= 0 else m1)) if (v & p1) == 0 else v

    for i, b in enumerate(blks):
        if eob == 0 and pos >= r.nbits:
            break
        new, k = list(zz[b]), ss
        if eob == 0:
            while k <= se:
                l, sym = decode_symbol(t, r.peek16(pos))
                if l == 0:
                    return i
                pos += l
                run, s = sym >> 4, sym & 15
                if s:
                    if s != 1:
                        return i
                    s = p1 if _bit(r, pos) else m1
                    pos += 1
                elif run != 15:
                    eob = (1 << run) + ((r.peek16(pos) >> (16 - run)) if run else 0)
                    pos += run
                    break
                while k <= se:                        # skip `run` zero-history coefficients, correcting the others
                    if new[k]:
                        if _bit(r, pos):
                            new[k] = correct(new[k])
                        pos += 1
                    else:
                        run -= 1
                        if run < 0:
                            break
                    k += 1
                if k > se:
                    return i
                if s:
                    new[k] = _i16(s)
                k += 1
        if eob:
            while k <= se:
                if new[k]:
                    if _bit(r, pos):
                        new[k] = correct(new[k])
                    pos += 1
                k += 1
            eob -= 1
        zz[b] = new
    return None


def progressive_decode(data, info: Optional[JpegInfo] = None) -> Tuple[np.ndarray, dict]:
    """Sequential decode of a progressive file, one scan after another: final int16 coefficients ``[blocks, 64]`` in
    stream order and natural order, and the counters the device writes (``T`` unstuffed bytes and ``R`` RST markers
    summed over the scans decoded, ``scans`` completed, ``cutoff`` the scan-order block where the decode failed, else
    the block count)."""
    d = _as_bytes(data)
    info = info or parse(d)
    g = geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    zz = [[0] * 64 for _ in range(g.blocks)]
    st = {"T": 0, "R": 0, "scans": 0, "cutoff": g.blocks}
    for sc in info.scans:
        comp, rst = unstuff(d[sc.offset:sc.offset + sc.length])
        st["T"] += len(comp)
        st["R"] += len(rst)
        blks, per = scan_blocks(info, sc)
        comp_of = list(g.comp_of) if per > 1 else [0]
        units = len(blks) // per
        ri = sc.restart
        nseg = -(-units // ri) if ri else 1
        bad = None
        for k, (s, e) in enumerate(segments(len(comp), rst, nseg)):
            u0 = k * ri if ri else 0
            part = blks[u0 * per:(u0 + (min(ri, units - u0) if ri else units)) * per]
            bad = _decode_interval(BitReader(comp, s, e), sc, info.tables, zz, part, comp_of)
            if bad is not None:
                bad += u0 * per
                break
        if bad is not None:
            st["cutoff"] = bad
            break
        st["scans"] += 1
    coef = np.zeros((g.blocks, 64), np.int16)
    coef[:, ZIGZAG] = np.array(zz, np.int64).astype(np.int16)
    return coef, st


def decode_stages(data) -> dict:
    """Every stage of ``decode_jpeg``: ``info``, ``coef`` (final, ``[blocks, 64]`` stream order), ``decoded`` (per block;
    all of a progressive file's), ``planes`` and ``rgb``; and for a progressive file ``progress``, the counters of
    ``progressive_decode``."""
    d = _as_bytes(data)
    info = parse(d)
    out = {"info": info}
    if info.progressive:
        coef, out["progress"] = progressive_decode(d, info)
        decoded = np.ones(len(coef), bool)
    else:
        raw, decoded = entropy_decode(d, info)
        coef = dc_predict(raw, decoded, info)
    pl = planes(coef, info)
    out.update(coef=coef, decoded=decoded, planes=pl, rgb=color_convert(pl, info))
    return out


def decode_jpeg(data) -> np.ndarray:
    """Decode one baseline or progressive JPEG file to uint8 RGB ``(h, w, 3)``, byte for byte as Keras' ``load_img`` does through Pillow
    (``np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))``, libjpeg-turbo 3.1).  ``DEFER(decode="jpeg")`` runs the
    same decode on the GPU.  Unsupported files raise a ValueError (see ``parse``)."""
    return decode_stages(data)["rgb"]
