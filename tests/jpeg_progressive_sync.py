"""A restatement of the GPU's progressive decode (``progressive_decode`` in csrc/jpeg.cu), scan by scan, in Python.

DC first and AC first scans decode as the device decodes them: each restart interval is cut into subsequences of
``sbits`` bits; every subsequence decodes from the default state (block 0 of its unit, k = Ss) at its first bit to the
first symbol boundary at or past its end, an invalid code restarting it one bit later; then, round after round, each
subsequence whose predecessor left in another state than it entered re-decodes from there.  The blocks a subsequence
owns count the blocks of its EOB runs, clamped to the block count; a segmented prefix sum, saturating at 2^30, gives
each subsequence's first block within its interval.  The write pass finishes the tail of a block begun in the
predecessor, then decodes the blocks it owns, and a failing block is the scan's cut.  A DC first scan then runs the
segmented DC prediction over the blocks before the cut and within each interval's count; an AC first scan clears its
band from the cut on.  DC refinements and AC refinements are decoded as ``jpeg.progressive_decode`` decodes them (the
device reads one bit per block, or one interval per thread after a dry run that finds the cut, with the same result).

``sync_progressive`` returns the final coefficients, which must equal ``jpeg.progressive_decode``'s, and the six
counters the device writes to ``stats``: unstuffed bytes and RST markers over the scans decoded, subsequences and
rounds over their first scans, the cut (or the block count) and the scans decoded whole.  The rounds are deterministic,
as on the device, so all six must equal the device's exactly."""
from __future__ import annotations

import numpy as np

from defer_b200 import jpeg

CAP = 1 << 30


def _sat(v: int) -> int:
    """The device's segmented block-offset sum saturates (SegSat)."""
    return min(v, CAP)


def _pstep(r, pos, k, j, sc, tabs, per, comp_of):
    """pstep: (pos, k, z, v, eob) after one symbol, or None."""
    p = r.peek16(pos)
    if sc.ss == 0:
        l, s = jpeg.decode_symbol(tabs[sc.dc[comp_of[j] if per > 1 else 0]], p)
        if l == 0:
            return None
        s &= 15
        v = jpeg.extend(r.peek16(pos + l) >> (16 - s), s) if s else 0
        return pos + l + s, 1, 0, v, 0
    l, sym = jpeg.decode_symbol(tabs[sc.ac], p)
    if l == 0:
        return None
    pos += l
    run, s = sym >> 4, sym & 15
    if s == 0:
        if run == 15:
            return None if k + 16 > sc.se + 1 else (pos, k + 16, -1, 0, 0)
        eob = (1 << run) - 1 + (r.peek16(pos) >> (16 - run)) if run else 0
        return pos + run, sc.se + 1, -1, 0, eob
    if k + run > sc.se:
        return None
    v = jpeg.extend(r.peek16(pos) >> (16 - s), s)
    return pos + s, k + run + 1, k + run, v, 0


def _run(r, pos, j, k, end, sc, tabs, per, comp_of, blocks):
    """psync_run: (pos, j, k, blocks owned) at the first boundary at or past ``end``."""
    count = 0
    while pos < end:
        if k == sc.ss:
            count += 1
        st = _pstep(r, pos, k, j, sc, tabs, per, comp_of)
        if st is None:
            pos, j, k = pos + 1, 0, sc.ss
            continue
        pos, k, _, _, eob = st
        count += eob
        if k > sc.se:
            k, j = sc.ss, (j + 1) % per
    return pos, j, k, min(count, blocks)


def _first_scan(comp, rst, sc, info, g, zz, sbits):
    """One DC first or AC first scan; returns (cut, subsequences, rounds)."""
    blks, per = jpeg.scan_blocks(info, sc)
    comp_of = list(g.comp_of) if per > 1 else [0]
    units = len(blks) // per
    nq, ri = len(blks), sc.restart
    nseg = -(-units // ri) if ri else 1
    tabs = info.tables
    subs = []                                                # (interval, reader, start, end)
    for k, (s, e) in enumerate(jpeg.segments(len(comp), rst, nseg)):
        r = jpeg.BitReader(comp, s, e)
        for i in range(-(-r.nbits // sbits)):
            subs.append((k, r, i * sbits, min((i + 1) * sbits, r.nbits)))
    entry = [(a, 0, sc.ss) for _, _, a, _ in subs]
    out = [_run(r, a, 0, sc.ss, b, sc, tabs, per, comp_of, g.blocks) for _, r, a, b in subs]
    rounds = 1
    while True:
        pend = {t: out[t - 1][:3] for t in range(1, len(subs))
                if subs[t - 1][0] == subs[t][0] and out[t - 1][:3] != entry[t]}
        if not pend:
            break
        for t, new in pend.items():
            entry[t] = new
            out[t] = _run(subs[t][1], *new, subs[t][3], sc, tabs, per, comp_of, g.blocks)
        rounds += 1
    exp = [(min(ri, units - k * ri) if ri else units) * per for k in range(nseg)]
    pre, seg_total, acc = [], [0] * nseg, 0
    for t, (k, *_rest) in enumerate(subs):
        if t == 0 or subs[t - 1][0] != k:
            acc = 0
        pre.append(acc)
        acc = _sat(acc + out[t][3])
        seg_total[k] = min(acc, exp[k])
    cut = nq
    for t, (k, r, a, b) in enumerate(subs):
        pos, j, kk = entry[t]
        idx, ok = pre[t], True
        while kk != sc.ss:
            st = _pstep(r, pos, kk, j, sc, tabs, per, comp_of)
            if st is None:
                ok = False
                break
            pos, kk, _, _, eob = st
            idx += eob
            if kk > sc.se:
                kk, j = sc.ss, (j + 1) % per
        if not ok:
            continue
        q0 = k * ri * per if ri else 0
        while pos < b and idx < exp[k]:
            q = q0 + idx
            blk, extra = zz[blks[q]], 0
            while True:
                st = _pstep(r, pos, kk, j, sc, tabs, per, comp_of)
                if st is None:
                    ok = False
                    break
                pos, kk, z, v, eob = st
                extra += eob
                if z == 0 and sc.ss == 0:
                    blk[0] = jpeg._i16(v)
                elif z >= 0:
                    blk[z] = jpeg._i16(v << sc.al)
                if kk > sc.se:
                    break
            if not ok:
                cut = min(cut, q)
                break
            kk, j, idx = sc.ss, (j + 1) % per, idx + 1 + extra
    if sc.ss == 0:                                           # DC prediction, per component, in scan order
        acc = {}
        for q in range(nq):
            u = q // per
            if (ri and u % ri == 0 or u == 0) and q % per == 0:
                acc = {}
            c = comp_of[q % per]
            b = blks[q]
            ks = u // ri if ri else 0
            if q < cut and q - (ks * ri * per if ri else 0) < seg_total[ks]:
                acc[c] = (acc.get(c, 0) + zz[b][0]) & 0xFFFFFFFF
                zz[b][0] = jpeg._i16(acc[c] << sc.al)
            else:
                zz[b][0] = 0
    else:
        for q in range(cut, nq):
            for kk in range(sc.ss, sc.se + 1):
                zz[blks[q]][kk] = 0
    return cut, len(subs), rounds


def sync_progressive(data, sbits: int):
    """(final int16 coefficients [blocks, 64] stream order natural order, int32 stats [6]) as the device computes them."""
    info = jpeg.parse(data)
    g = jpeg.geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    zz = [[0] * 64 for _ in range(g.blocks)]
    T = R = NS = rounds = done = 0
    cutoff = g.blocks
    for sc in info.scans:
        comp, rst = jpeg.unstuff(data[sc.offset:sc.offset + sc.length])
        T, R = T + len(comp), R + len(rst)
        if sc.ah == 0:
            cut, ns, rd = _first_scan(comp, rst, sc, info, g, zz, sbits)
            NS, rounds = NS + ns, rounds + rd
        else:
            blks, per = jpeg.scan_blocks(info, sc)
            units = len(blks) // per
            ri = sc.restart
            nseg = -(-units // ri) if ri else 1
            cut = len(blks)
            comp_of = list(g.comp_of) if per > 1 else [0]
            for k, (s, e) in enumerate(jpeg.segments(len(comp), rst, nseg)):
                u0 = k * ri if ri else 0
                part = blks[u0 * per:(u0 + (min(ri, units - u0) if ri else units)) * per]
                bad = jpeg._decode_interval(jpeg.BitReader(comp, s, e), sc, info.tables, zz, part, comp_of)
                if bad is not None:
                    cut = bad + u0 * per
                    break
        if cut < len(jpeg.scan_blocks(info, sc)[0]):
            cutoff = cut
            break
        done += 1
    coef = np.zeros((g.blocks, 64), np.int16)
    coef[:, jpeg.ZIGZAG] = np.array(zz, np.int64).astype(np.int16)
    return coef, np.array([T, R, NS, rounds, cutoff, done], np.int32)
