"""A restatement of the GPU's Huffman decode by self-synchronisation (jpeg_entropy_kernel in csrc/jpeg.cu), in Python.

Per restart interval, the unstuffed bits are cut into subsequences of ``sbits`` bits.  A state at a symbol boundary is
(bit offset, block within the MCU, coefficient index).  Every subsequence first decodes from the default state at its
first bit up to the first boundary at or past its end, and records where it leaves.  Then, round after round, each
subsequence whose predecessor left in a state other than the one it entered re-decodes from there.  An invalid code
restarts a decoder one bit later at block 0, coefficient 0 (on the true path it is a real error, which the write pass
finds).  Once no entry changes, each subsequence owns the blocks that start in it: a prefix sum gives their
positions, and a last pass writes them (finishing a block past the subsequence's end, skipping the tail of one that
started before it).  The result must equal ``jpeg.entropy_decode``; ``sync_decode`` also returns the rounds it took, and
``sync_stats`` the five counters the device writes to its ``stats``.  The rounds are deterministic (every pending
subsequence of a round re-decodes from its predecessor's exit of the round before, as on the device), so all five
counters must equal the device's exactly."""
from __future__ import annotations

import numpy as np

from defer_b200 import jpeg


def _run(r, g, info, pos, j, k, end):
    """Decode to the first boundary at or past ``end``: (pos, j, k, blocks started)."""
    count = 0
    while pos < end:
        if k == 0:
            count += 1
        c = g.comp_of[j]
        st = jpeg.step_symbol(r, pos, k, info.dc[c], info.ac[c])
        if st is None:
            pos, j, k = pos + 1, 0, 0
            continue
        pos, k = st[0], st[1]
        if k >= 64:
            k, j = 0, (j + 1) % g.bpm
    return pos, j, k, count


def sync_decode(data, sbits: int):
    """(coef [blocks, 64] natural order with DC differences, decoded mask, rounds), as the device computes them."""
    coef, decoded, stats = sync_stats(data, sbits)
    return coef, decoded, int(stats[3])


def sync_stats(data, sbits: int):
    """(coef, decoded mask, stats): ``sync_decode``'s coefficients and mask, and int32 [5] of what the device writes to
    ``stats[0..4]``: the unstuffed byte count T, the RST marker count R, the subsequence count, the rounds and the
    cutoff (the first block whose decode met an invalid code, or the block count)."""
    info = jpeg.parse(data)
    g = jpeg.geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    comp, rst = jpeg.unstuff(data[info.offset:info.offset + info.length])
    ri = info.restart
    nseg = -(-g.mcus // ri) if ri else 1
    subs = []                                              # (segment, reader, start, end)
    for k, (s, e) in enumerate(jpeg.segments(len(comp), rst, nseg)):
        r = jpeg.BitReader(comp, s, e)
        for i in range(-(-r.nbits // sbits)):
            subs.append((k, r, i * sbits, min((i + 1) * sbits, r.nbits)))
    entry = [(s[2], 0, 0) for s in subs]
    out = []
    for t, (k, r, a, b) in enumerate(subs):
        out.append(_run(r, g, info, a, 0, 0, b))
    rounds = 1
    while True:
        pend = {}
        for t in range(1, len(subs)):
            if subs[t - 1][0] != subs[t][0]:
                continue
            p, j, kk, _ = out[t - 1]
            new = (p, j, kk)
            if new != entry[t]:
                pend[t] = new
        if not pend:
            break
        for t, new in pend.items():
            entry[t] = new
            _, r, _, b = subs[t]
            out[t] = _run(r, g, info, *new, b)
        rounds += 1
    coef = np.zeros((g.blocks, 64), np.int16)
    decoded = np.zeros(g.blocks, bool)
    cutoff = g.blocks
    seg_total = np.zeros(nseg, np.int64)
    done = {}
    for t, (k, r, a, b) in enumerate(subs):
        done[t] = seg_total[k]
        seg_total[k] += out[t][3]
    for t, (k, r, a, b) in enumerate(subs):
        pos, j, kk = entry[t]
        exp_k = (min(ri, g.mcus - k * ri) if ri else g.mcus) * g.bpm
        first = k * ri * g.bpm if ri else 0
        ok = True
        while kk != 0:
            c = g.comp_of[j]
            st = jpeg.step_symbol(r, pos, kk, info.dc[c], info.ac[c])
            if st is None:
                ok = False
                break
            pos, kk = st[0], st[1]
            if kk >= 64:
                kk, j = 0, (j + 1) % g.bpm
        idx = done[t]
        while ok and pos < b and idx < exp_k:
            blk, c = np.zeros(64, np.int16), g.comp_of[j]
            while kk < 64:
                st = jpeg.step_symbol(r, pos, kk, info.dc[c], info.ac[c])
                if st is None:
                    cutoff = min(cutoff, first + idx)
                    ok = False
                    break
                pos, kk, z, v = st
                if z >= 0:
                    blk[jpeg.ZIGZAG[z]] = v
            if not ok:
                break
            coef[first + idx] = blk
            decoded[first + idx] = True
            kk, j, idx = 0, (j + 1) % g.bpm, idx + 1
    for k in range(nseg):
        first = k * ri * g.bpm if ri else 0
        n = (min(ri, g.mcus - k * ri) if ri else g.mcus) * g.bpm
        decoded[first + min(seg_total[k], n):first + n] = False
    decoded[cutoff:] = False
    coef[~decoded] = 0
    return coef, decoded, np.array([len(comp), len(rst), len(subs), rounds, cutoff], np.int32)
