"""Crafted progressive files at the edges of the device's progressive decode, shared by the host and GPU tests.

``eob_cases``: EOB runs at their limits (a run of 32 767 blocks and the encoder's flush there, runs past their restart
interval and past their scan, run symbols that start at, end at and straddle a subsequence edge, a refinement EOB run
carrying over 1000 correction bits across an edge).  ``refine_cases``: AC refinement edges (Se = 63, the single
coefficient band 32..32, bands of non-zero history only, a new coefficient at zigzag 63, ZRLs passing non-zero history,
a ZRL ending a block at exactly Se + 1, Al = 13 down with negative values, restart intervals of one block and of more
than a subsequence).  ``corrupt_cases``: 480x640 files, 4:2:0 and grayscale, with and without restart intervals, with interleaved and
one-component DC first scans, whose luma first scans span several subsequences per interval, damaged in the first scan
of each kind: an invalid code at the first block, at a block straddling a subsequence edge and at the last block, a run and a ZRL past Se, a size-2 refinement symbol, data cut inside the
scan, RST markers dropped, duplicated, renumbered, surplus or missing, fill bytes, an empty scan; and a 1080x1920 grayscale file with invalid codes in its DC first, AC first and AC refinement scans.
Seeded; no Pillow."""
from __future__ import annotations

from typing import List

import numpy as np

from defer_b200 import jpeg
import jpeg_craft_progressive as P
from jpeg_craft import _seg, codes, geometry, pack, random_table

#: the saturating file on the GPU: 2048x4096 grayscale, 20 000 subsequences of EOB runs
SAT = (2048, 4096, 20000)

#: 5-bit codes for the AC first symbols the raw scans here use (no code is all 1-bits)
AC_SYMS = [0x00, 0x01, 0x02] + [r << 4 for r in range(1, 15)] + [0xF0, 0xF1]
FIXED = ([0, 0, 0, 0, len(AC_SYMS)] + [0] * 11, AC_SYMS)


def _bits_of(events, table) -> int:
    cd = codes(table)
    return sum(cd[e[1]][1] if e[0] == "s" else e[2] for e in events if e[0] != "m")


def _eob(n):
    r = n.bit_length() - 1
    return [("s", r << 4)] + ([("b", n - (1 << r), r)] if r else [])


def _fill_to(events, target, coded, want_blocks):
    """Append coded blocks (11 bits: +1 at zigzag 1, then EOB) and empty blocks (a 5-bit EOB) until ``events`` hold
    ``target`` bits; returns the blocks added.  ``coded`` collects the scan-order index of each coded block."""
    have = _bits_of(events, FIXED)
    rest = target - have
    assert rest >= 40
    b = next(b for b in range(11) if (rest - 5 * b) % 11 == 0)
    a = (rest - 5 * b) // 11
    for _ in range(a):
        coded.append(want_blocks[0])
        events += [("s", 0x01), ("b", 1, 1), ("s", 0x00)]
        want_blocks[0] += 1
    for _ in range(b):
        events.append(("s", 0x00))
        want_blocks[0] += 1
    return a + b


def eob_cases(sbits: int) -> List[tuple]:
    """[(name, file, final coefficients or None)] of valid files."""
    out = []
    q = [np.ones(64, np.int32)]
    # a run of exactly 32 767 blocks: 1456x1456 has 33 124, so the encoder flushes at 0x7FFF and sends 357 more
    h = w = 1456
    coef = P.coefficients(h, w, "gray", [np.full(64, 16)], seed=11, zero_from=1)
    tr = []
    out.append(("eob 32767 then 357, 1456x1456", *P.craft(h, w, "gray", q, coef,
                [P.scan((0,), 0, 0, 0, 0), P.scan((0,), 1, 63, 0, 0)], seed=11, trace=tr)))
    assert [e for e in tr[1][0][0] if e[0] != "m"] == _eob(32767) + _eob(357)
    # runs past their restart interval (EOB14 of 32 767 in intervals of 10 blocks) and past the scan
    h, w = 64, 96
    g = geometry(h, w, "gray")
    coef = P.coefficients(h, w, "gray", [np.full(64, 16)], seed=12, zero_from=1)
    hold = np.zeros((g.blocks, 64), np.int64)
    ivs = []
    for i in range(0, g.blocks, 10):
        hold[i, 1] = 1
        ivs.append([("s", 0x01), ("b", 1, 1), ("s", 0xE0), ("b", (1 << 14) - 1, 14)])
    out.append(("eob runs past their interval", *P.craft(h, w, "gray", q, coef, [
        P.scan((0,), 0, 0, 0, 0), P.scan((0,), 1, 63, 0, 0, 10, raw=ivs, table=FIXED, holds=hold)])))
    hold = np.zeros((g.blocks, 64), np.int64)
    hold[:5, 1] = -1
    ev = [x for _ in range(5) for x in (("s", 0x01), ("b", 0, 1), ("s", 0x00))] + _eob(32767)
    out.append(("eob run past the scan", *P.craft(h, w, "gray", q, coef, [
        P.scan((0,), 0, 0, 0, 0), P.scan((0,), 1, 63, 0, 0, raw=[ev], table=FIXED, holds=hold)])))
    # run symbols starting at, ending at and straddling a subsequence edge, one per restart interval of 1200 blocks
    h, w = 480, 480
    g = geometry(h, w, "gray")
    coef = P.coefficients(h, w, "gray", [np.full(64, 16)], seed=13, zero_from=1)
    hold = np.zeros((g.blocks, 64), np.int64)
    ivs = []
    for i, (at, run) in enumerate([(sbits, 300), (sbits - 13, 400), (sbits - 3, 257)]):
        coded, ev, n = [], [], [0]
        _fill_to(ev, at, coded, n)
        ev += _eob(run)
        n[0] += run
        assert _bits_of(ev[:-2], FIXED) == at and _bits_of(ev, FIXED) == at + 13      # 5-bit EOB8 code, 8 bits
        while n[0] < 1200:
            coded.append(n[0])
            ev += [("s", 0x01), ("b", 1, 1), ("s", 0x00)]
            n[0] += 1
        hold[np.asarray(coded) + 1200 * i, 1] = 1
        ivs.append(ev)
    out.append(("eob run symbols at a subsequence edge", *P.craft(h, w, "gray", q, coef, [
        P.scan((0,), 0, 0, 0, 0), P.scan((0,), 1, 63, 0, 0, 1200, raw=ivs, table=FIXED, holds=hold)])))
    # a refinement EOB run of 200 blocks whose 12 600 correction bits cross a subsequence edge
    h, w = 80, 160
    g = geometry(h, w, "gray")
    rng = np.random.default_rng(14)
    coef = rng.choice([-3, -2, 2, 3], (g.blocks, 64)).astype(np.int64)
    coef[:, 0] = 0
    ev = _eob(g.blocks) + [("b", int(coef[b, jpeg.ZIGZAG[k]]) & 1, 1) for b in range(g.blocks) for k in range(1, 64)]
    table = random_table(rng, [0x70])
    assert _bits_of(ev, table) > sbits
    out.append(("refinement eob run, 12600 correction bits", *P.craft(h, w, "gray", q, coef, [
        P.scan((0,), 0, 0, 0, 0), P.scan((0,), 1, 63, 0, 1),
        P.scan((0,), 1, 63, 1, 0, raw=[ev], table=table, holds=coef)])))
    # a ZRL that ends a block at exactly Se + 1, in an AC first scan and in a refinement
    h, w = 24, 40
    g = geometry(h, w, "gray")
    coef = np.zeros((g.blocks, 64), np.int64)
    out.append(("zrl ending at se+1", *P.craft(h, w, "gray", q, coef, [
        P.scan((0,), 0, 0, 0, 0), P.scan((0,), 1, 16, 0, 1, raw=[[("s", 0xF0)] * g.blocks], table=FIXED, holds=coef),
        P.scan((0,), 17, 63, 0, 0), P.scan((0,), 1, 16, 1, 0, raw=[[("s", 0xF0)] * g.blocks], table=FIXED,
                                            holds=coef)])))
    return out


def refine_cases() -> List[tuple]:
    """[(name, file, final coefficients)] of writer-encoded AC refinement edges."""
    out = []
    rng = np.random.default_rng(21)
    q = [np.ones(64, np.int32)]

    def add(name, h, w, coef, ac_script, seed):
        out.append((name, *P.craft(h, w, "gray", q, coef, [P.scan((0,), 0, 0, 0, 0)] + ac_script, seed=seed)))
    h, w = 64, 128
    g = geometry(h, w, "gray")
    nb = g.blocks

    def z(k):
        return int(jpeg.ZIGZAG[k])
    c = np.zeros((nb, 64), np.int64)
    c[:, 0] = rng.integers(-50, 50, nb)
    c[:, z(32)] = rng.choice([-3, -2, -1, 0, 1, 2, 3], nb)        # 32..32: nth_bit in the high word
    for k in (30, 31, 33, 34):
        c[:, z(k)] = rng.choice([-2, -1, 0, 1, 2], nb)
    c[:, z(63)] = rng.choice([-1, 0, 1], nb)                      # new coefficients at zigzag 63
    for k in range(1, 6):                                          # 1..5: non-zero history only
        c[:, z(k)] = rng.choice([-3, -2, 2, 3], nb)
    s = [P.scan((0,), 1, 5, 0, 1), P.scan((0,), 6, 29, 0, 0), P.scan((0,), 30, 31, 0, 1), P.scan((0,), 32, 32, 0, 1),
         P.scan((0,), 33, 63, 0, 1), P.scan((0,), 1, 5, 1, 0), P.scan((0,), 32, 32, 1, 0), P.scan((0,), 30, 31, 1, 0),
         P.scan((0,), 33, 63, 1, 0, restart=1)]
    add("refine 32..32, 1..5 history only, zigzag 63, Se 63, DRI 1", h, w, c, s, 22)
    # ZRLs passing non-zero history before a new coefficient
    c = np.zeros((nb, 64), np.int64)
    for k in (3, 9, 14, 20, 27, 33):
        c[:, z(k)] = rng.choice([-3, -2, 2, 3], nb)
    c[:, z(40)] = rng.choice([-1, 1], nb)
    c[::3, z(58)] = 1
    add("refine ZRLs over history", h, w, c, [P.scan((0,), 1, 63, 0, 1), P.scan((0,), 1, 63, 1, 0)], 23)
    # Al = 13 down to 0 with negative values, one bit per scan
    c = np.zeros((nb, 64), np.int64)
    for k in (1, 2, 5, 17, 44, 63):
        c[:, z(k)] = rng.integers(-(1 << 14) + 1, 1 << 14, nb)
    c[::2, z(2)] = -(1 << 13)
    s = [P.scan((0,), 1, 63, 0, 13)] + [P.scan((0,), 1, 63, a + 1, a, restart=3 if a % 2 else 0)
                                        for a in range(12, -1, -1)]
    add("al 13 down, negative values", h, w, c, s, 24)
    # a refinement whose restart intervals are each longer than a subsequence
    h, w = 256, 256
    c = P.coefficients(h, w, "gray", [np.full(64, 2)], seed=25)
    add("refine, DRI longer than a subsequence", h, w, c,
        [P.scan((0,), 1, 63, 0, 1), P.scan((0,), 1, 63, 1, 0, restart=300)], 25)
    return out


# ------------------------------------------------------------------------------------------------ corrupt files
KINDS = ("dc first", "dc first interleaved", "dc refine", "ac first", "ac refine")
FIRST = ("dc first", "dc first interleaved", "ac first")


def kind(sc) -> str:
    if sc["ss"] == 0 and sc["ah"] == 0:
        return "dc first interleaved" if len(sc["comps"]) > 1 else "dc first"
    return ("dc " if sc["ss"] == 0 else "ac ") + ("first" if sc["ah"] == 0 else "refine")


#: (subsampling, restart interval of interleaved scans in MCUs (one-component scans: 6 times as many blocks), one DC
#: first scan per component) of the 480x640 files the corrupt ones come from
VARIANTS = [("420", 0, False), ("420", 0, True), ("420", 200, False), ("420", 200, True), ("gray", 0, False),
            ("gray", 200, False)]


def bases(h=480, w=640, variants=VARIANTS):
    """[(name, file, final coefficients, script, trace)] of photo-like files whose luma first scans span several
    subsequences, in every interval when there are restart intervals: DC first (interleaved, or one scan per component), AC first
    1..5 and 6..63 of luma at Al 1, chroma AC at Al 0, DC and luma AC refinements."""
    out = []
    for sub, ri, split_dc in variants:
        q = [np.full(64, 8, np.int32), np.full(64, 10, np.int32)]
        coef = P.coefficients(h, w, sub, q, seed=31)
        allc = (0,) if sub == "gray" else (0, 1, 2)
        r1 = 6 * ri                                   # one-component scans count blocks, not MCUs
        ra = ri if len(allc) > 1 else r1
        s = [P.scan((c,), 0, 0, 0, 1, r1) for c in allc] if split_dc else [P.scan(allc, 0, 0, 0, 1, ra)]
        s += [P.scan((0,), 1, 5, 0, 1, r1), P.scan((0,), 6, 63, 0, 1, r1)]
        s += [P.scan((c,), 1, 63, 0, 0, r1) for c in allc[1:]]
        s += [P.scan(allc, 0, 0, 1, 0, ra), P.scan((0,), 1, 63, 1, 0, r1)]
        tr = []
        d, want = P.craft(h, w, sub, q, coef, s, seed=31 + ri, trace=tr)
        out.append((f"{sub} {h}x{w} DRI {ri}{' DC per component' if split_dc else ''}", d, want, s, tr))
    return out


def _with_table(pre: bytes, table, cls: int) -> bytes:
    """``pre`` with its (last) DHT segment replaced by one of ``table``."""
    k = pre.rindex(b"\xff\xc4")
    ln = int.from_bytes(pre[k + 2:k + 4], "big")
    return pre[:k] + _seg(0xC4, bytes([cls << 4]) + bytes(table[0]) + bytes(table[1])) + pre[k + 2 + ln:]


def _recode(parts, s, events, rng, cls):
    """parts with scan s's intervals re-encoded from ``events`` under a fresh table covering their symbols."""
    syms = sorted({e[1] for ev in events for e in ev if e[0] == "s"})
    table = random_table(rng, syms)
    parts = list(parts)
    parts[s] = (_with_table(parts[s][0], table, cls), [P._interval_bytes(ev, table) for ev in events])
    return parts


def _symbol_blocks(ev):
    """(event index, scan-order block) of the marks followed by a symbol that is not an EOB run (blocks that start with
    a code of their own)."""
    out = []
    for i, e in enumerate(ev):
        if e[0] == "m" and i + 1 < len(ev) and ev[i + 1][0] == "s" and (ev[i + 1][1] & 15 or ev[i + 1][1] == 0xF0):
            out.append((i, e[1]))
    return out


def corrupt_cases(sbits: int, seed: int = 0, large: bool = False) -> List[tuple]:
    """[(name, file, scan index, kind, damage, interval index, bit offset in the interval or -1, scan-order block of an
    inserted invalid code or -1)] of corrupt files ``jpeg.parse`` accepts, made from ``bases``.  ``large``: from a
    1080x1920 grayscale base instead, only invalid codes."""
    rng = np.random.default_rng(seed)
    out = []
    for bname, d, _, script, tr in (bases(1080, 1920, [("gray", 0, False)]) if large else bases()):
        parts, tail = P.split(d)
        seen = set()
        for s, sc in enumerate(script):
            kd = kind(sc)
            if kd in seen:                            # the first scan of each kind in each file
                continue
            seen.add(kd)
            evs, table = tr[s]
            nm = f"{bname}, scan {s} ({kd})"
            ivn = len(evs)

            def put(damage, f, iv=-1, at=-1, q=-1):
                out.append((f"{nm}: {damage}", f, s, kd, damage, iv, at, q))
            if sc["ss"] > 0 or sc["ah"] == 0:         # a code: an invalid 16 one-bits at a block
                picks = {}
                b0 = _symbol_blocks(evs[0])
                if b0:
                    picks["invalid code at the first block"] = (0, b0[0][0])
                for iv in range(ivn):                 # a block that starts before an edge and ends after it
                    pos = P.block_bits(evs[iv], table)
                    nxt = dict(zip(sorted(pos), sorted(pos)[1:]))
                    hit = [i for i, q in _symbol_blocks(evs[iv])
                           if q in nxt and pos[q] // sbits < pos[nxt[q]] // sbits and pos[nxt[q]] % sbits]
                    if hit:
                        picks["invalid code at a block straddling a subsequence edge"] = (iv, hit[0])
                        break
                bl = _symbol_blocks(evs[-1])
                if bl:
                    picks["invalid code at the last block"] = (ivn - 1, bl[-1][0])
                if large:                             # and at a block past the middle of the scan
                    iv = ivn // 2
                    sb = _symbol_blocks(evs[iv])
                    picks["invalid code at a middle block"] = (iv, sb[len(sb) // 2][0])
                for damage, (iv, ei) in picks.items():
                    ev = list(evs[iv])
                    at = P.block_bits(ev, table)[ev[ei][1]]
                    bits = P._encode(ev, table)
                    ivs = list(parts[s][1])
                    ivs[iv] = pack(bits[:at] + "1" * 16 + bits[at:])
                    pp = list(parts)
                    pp[s] = (parts[s][0], ivs)
                    put(damage, P.assemble(pp, tail), iv, at, ev[ei][1])
            if large:
                continue
            if sc["ss"] > 0:                          # symbols no valid AC scan holds, in the middle interval
                iv = ivn // 2
                sb = _symbol_blocks(evs[iv])
                i = sb[len(sb) // 2][0]
                width = sc["se"] - sc["ss"] + 1
                bad = {"run past Se": [("s", 0xF0)] * (width // 16) + [("s", (width % 16) << 4 | 1), ("b", 1, 1)],
                       "ZRL past Se": [("s", 0xF0)] * (width // 16 + 1)}
                if sc["ah"]:
                    bad["size-2 refinement symbol"] = [("s", 0x02), ("b", 1, 1)]
                for damage, ins in bad.items():
                    ev = list(evs[iv])
                    at = P.block_bits(ev, table)[ev[i][1]]
                    ev[i + 1:i + 1] = ins
                    ivs_ev = list(evs)
                    ivs_ev[iv] = ev
                    put(damage, P.assemble(_recode(parts, s, ivs_ev, rng, 1), tail), iv, at)
            # data cut inside the scan, an empty scan
            ivs = list(parts[s][1])
            k = ivn // 2
            ivs[k] = ivs[k][:len(ivs[k]) // 2]
            pp = list(parts)
            pp[s] = (parts[s][0], ivs[:k + 1])
            put("data cut inside the scan", P.assemble(pp, tail), k)
            pp = list(parts)
            pp[s] = (parts[s][0], [b""])
            put("empty scan", P.assemble(pp, tail))
            if ivn >= 4:                              # RST markers
                ivs = parts[s][1]
                k = ivn // 2

                def with_ivs(new, rst=None, fill=0):
                    pp = list(parts)
                    pp[s] = (parts[s][0], new)
                    return P.assemble(pp, tail, fill=fill, rst={s: rst} if rst is not None else None)
                put("an RST dropped", with_ivs(ivs[:k] + [ivs[k] + ivs[k + 1]] + ivs[k + 2:]), k)
                put("an RST duplicated", with_ivs(ivs[:k] + [b""] + ivs[k:], [i % 8 for i in range(k)] + [(k - 1) % 8]
                                                  + [i % 8 for i in range(k - 1, ivn - 1)]), k)
                put("RSTs renumbered", with_ivs(ivs, [int(x) for x in rng.integers(0, 8, ivn - 1)]))
                put("surplus RSTs", with_ivs(ivs + [rng.bytes(50), b"", rng.bytes(9)]))
                put("RSTs missing after the first", with_ivs([ivs[0], b"".join(ivs[1:])]), 1)
                put("fill bytes before the markers", with_ivs(ivs, fill=3))
    kept = []
    for c in out:
        jpeg.parse(c[1])
        kept.append(c)
    return kept


def host_expect(d: bytes, sbits: int):
    """``jpeg.decode_stages(d)`` and the six counters of the restatement at ``sbits``, whose coefficients it checks."""
    from jpeg_progressive_sync import sync_progressive
    want = jpeg.decode_stages(d)
    coef, stats = sync_progressive(d, sbits)
    assert np.array_equal(coef, want["coef"])
    return want, stats


def host_expect_all(files, sbits: int):
    """``host_expect`` of each file, in worker processes."""
    import multiprocessing as mp
    import os
    from concurrent.futures import ProcessPoolExecutor
    from functools import partial
    with ProcessPoolExecutor(max_workers=max(1, min(16, os.cpu_count() or 1)), mp_context=mp.get_context("spawn")) as ex:
        return list(ex.map(partial(host_expect, sbits=sbits), files))
