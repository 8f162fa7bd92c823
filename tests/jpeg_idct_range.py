"""Valid JPEG files whose IDCT leaves the +-512 range, shared by the host and GPU tests of that range.

Beyond the range ``defer_b200.jpeg`` follows libjpeg-turbo's C code: ``jidctint.c`` wraps each output to 10 bits before
the 0..255 clamp (``idct_range_limit[x & 1023]``), and the coefficients are int16 as ``jdhuff.c`` / ``jdphuff.c``
store them.  ``corpus()`` plans which of those rules each file reaches:

- ``wrap``: DC-only blocks whose value x = dc * q / 8 around 128 steps across the wrap (x = 511 / 512 mod 1024) and the
  clamp's edges (x = -128 / -127 and 126 / 127 mod 1024), positive and negative, with DC quantisers 8 (x = dc, up to
  +-32767) and 255 (x = 255 d for dc = 8 d, out to the largest and most negative reachable values).  One component at a
  time carries them, in grayscale, 4:4:4, 4:2:2 and 4:2:0, at odd sizes: fancy upsampling sees wrapped chroma at the
  right and bottom edges, pixel replication sees it where the downsampled width is at most 2, and colour conversion
  takes wrapped luma against in-range chroma and the reverse.
- ``one ac``: one AC coefficient per block, each zigzag position 1..63 at +-1023 under quantiser 255; ``full column``:
  blocks whose every coefficient is at its largest, DC +-32767 (or -32768) and every AC +-1023 under 255, the largest
  pass-1 values an accepted file can produce, after a ramp of DC-only blocks (libjpeg's zero-AC column shortcut).
- ``random``: random sparse coefficients up to +-1023 under random and coarse quantisers, every subsampling, without
  restart intervals and with intervals of one MCU and of more than one MCU row.
- ``dc predictor``: DC differences of +2047 for more than 16 blocks of one component and back down, so that the int
  predictor passes +-32767 and each stored coefficient is ``(JCOEF)`` of it.  The writer emits these differences as
  given: derived from the stored coefficients they would not fit a DC symbol.
- ``progressive``: Al = 13 down with negative values; a DC first scan at Al = 13 whose shifted sums wrap int16
  (``(JCOEF)LEFT_SHIFT(s, Al)``), refined down to Al = 0 or not refined; AC first scans at Al = 10..13 of |v| = 1023,
  whose ``v << Al`` wraps int16, and AC refinements applied on top of the wrapped values.  Zigzag 1..9 of every
  component are always refined to Al = 0, so no decoder applies block smoothing.
- ``grid``: one 1080x1920 4:2:0 file of random large coefficients.
- ``control``: two files in range, where every decode agrees.

Each case records the int16 coefficients a libjpeg decoder holds after the entropy decode.  For the AC refinements on
top of wrapped values these follow ``jdphuff.c``'s rule (a correction moves the stored int16 away from zero by its own
sign), which is not the writer's int64 view, so they come from ``refined``, a coefficient-level model of successive
approximation checked against the writer wherever nothing wraps.  Seeded; pure Python and numpy; no Pillow.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence

import numpy as np

from defer_b200 import jpeg
import jpeg_craft as jc
import jpeg_craft_progressive as P

SUBS = ("gray", "444", "422", "420")
#: x mod 1024 on each side of the clamp's edges and of the 10-bit wrap: -128 / -127 give 0 / 1, 126 / 127 give
#: 254 / 255, 511 / 512 give 255 / 0
EDGES = (-128, -127, 126, 127, 511, 512)
#: odd sizes (h, w) of the small wrap-point files: 5x4 and 7x3 have a downsampled width of 2 in 4:2:2 and 4:2:0
SMALL = ((17, 33), (31, 47), (1, 17), (5, 4), (7, 3))
#: the size of the files that sweep the whole reachable range: 192 MCUs of 4:2:0
SWEEP = (191, 255)
GRID = (1080, 1920)
DC_MAX = 2047


@dataclass
class Case:
    name: str
    kind: str
    data: bytes
    coef: np.ndarray                  # int16 [blocks, 64], stream order, natural order
    wrapped: tuple = field(default=())  # wrap files: the component whose DC carries the wrap points


# ------------------------------------------------------------------------------------------------ baseline writing
def full_tables(nc: int, rng: np.random.Generator):
    """Random DC and AC tables (luma, chroma) over every symbol a baseline file may use."""
    dcs = list(range(12))
    acs = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]
    n = 1 if nc == 1 else 2
    return [jc.random_table(rng, dcs, 0.3) for _ in range(n)], [jc.random_table(rng, acs, 0.3) for _ in range(n)]


def encode_diffs(coef: np.ndarray, diffs: np.ndarray, g: jpeg.Geometry, dc, ac) -> List[str]:
    """The bits of one interval (no restart) of blocks whose DC differences are ``diffs`` as given and whose AC
    coefficients are ``coef[:, 1:]`` (natural order)."""
    dcc, acc = [jc.codes(t) for t in dc], [jc.codes(t) for t in ac]
    per = [0] + [min(1, len(dc) - 1)] * 2
    out = []
    for b in range(g.blocks):
        c = per[g.comp_of[b % g.bpm]]
        d = int(diffs[b])
        s = jc._category(d)
        assert s <= 11, d
        code, ln = dcc[c][s]
        out.append(format(code, f"0{ln}b") + jc._bits(d, s))
        for run, v in jc._runs([int(coef[b, jpeg.ZIGZAG[k]]) for k in range(1, 64)]):
            code, ln = acc[c][jc._ac_symbol(run, v)]
            out.append(format(code, f"0{ln}b") + (jc._bits(v, jc._category(v)) if v is not None else ""))
    return ["".join(out)]


def _baseline(name, kind, h, w, sub, quant, coef, rng, restart=0, wrapped=()) -> Case:
    coef = np.asarray(coef, np.int64)
    assert np.abs(coef[:, 1:]).max(initial=0) <= 1023
    dc, ac = full_tables(jc.SAMPLING[sub][0], rng)
    data = jc.craft(h, w, sub, quant, dc, ac, coef=coef, restart=restart)
    return Case(name, kind, data, coef.astype(np.int16), wrapped)


def comp_index(g: jpeg.Geometry) -> np.ndarray:
    """The component of each stream-order block."""
    return np.tile(np.array(g.comp_of), g.mcus)


def _path(targets: Sequence[int], n: int) -> List[int]:
    """``n`` DC values that visit ``targets`` in order from a predictor of 0, each within ``DC_MAX`` of the one before:
    where a target is farther, ramp blocks of +-DC_MAX go between.  Targets past the n-th block are dropped."""
    out, cur, i = [], 0, 0
    while len(out) < n:
        if i < len(targets):
            t = targets[i]
            if abs(t - cur) <= DC_MAX:
                cur, i = t, i + 1
            else:
                cur += DC_MAX if t > cur else -DC_MAX
        out.append(cur)
    return out


def wrap_targets(q: int, order: str, start: int = 0) -> List[int]:
    """DC values whose x = dc * q / 8 is exactly an edge of ``EDGES`` plus a multiple of 1024: q = 8 gives x = dc up to
    +-32767, q = 255 gives x = 255 d for dc = 8 d (with the extremes 32767 and -32768 added).  ``order``: "near" takes
    the values within one DC difference of zero, those out of range first, nearest first, rotated by ``start``; "sweep"
    climbs to the largest, then falls to the most negative."""
    if q == 8:
        vals = {b + 1024 * m for b in EDGES for m in (-32, -31, -15, -7, -3, -2, -1, 0, 1, 2, 3, 7, 15, 31)}
    else:
        inv = pow(255, -1, 1024)
        vals = {8 * (d0 + 1024 * j) for b in EDGES for d0 in [(b * inv) % 1024] for j in range(-5, 5)}
        vals |= {32767, -32768}
    vals = sorted(v for v in vals if -32768 <= v <= 32767)
    if order == "near":
        near = sorted((v for v in vals if abs(v) <= DC_MAX), key=abs)
        out = [v for v in near if not -512 <= v * q // 8 <= 511]
        start %= len(out)
        return out[start:] + out[:start] + [v for v in near if -512 <= v * q // 8 <= 511]
    return [v for v in vals if v > 0] + sorted((v for v in vals if v <= 0), reverse=True)


def wrap_file(sub: str, h: int, w: int, comp: int, q: int, order: str, rng: np.random.Generator,
              start: int = 0) -> Case:
    """DC-only blocks: component ``comp`` walks ``wrap_targets``, the others hold random in-range values."""
    g = jc.geometry(h, w, sub)
    nc = jc.SAMPLING[sub][0]
    qa = np.full(64, q)
    other = np.full(64, 8)
    quant = [qa] if nc == 1 else [qa if comp == 0 else other, qa if comp > 0 else other]
    coef = np.zeros((g.blocks, 64), np.int64)
    ci = comp_index(g)
    for c in range(nc):
        idx = np.nonzero(ci == c)[0]
        if c == comp:
            coef[idx, 0] = _path(wrap_targets(q, order, start), len(idx))
        else:
            qc = quant[0 if c == 0 else 1][0]
            lim = 400 * 8 // int(qc)
            coef[idx, 0] = rng.integers(-lim, lim + 1, len(idx))
    return _baseline(f"wrap {sub} {h}x{w} comp {comp} q{q} {order}", "wrap", h, w, sub, quant, coef, rng,
                     wrapped=(comp,))


def one_ac_file(sub: str, rng: np.random.Generator) -> Case:
    """Zigzag positions 1..63 at +1023 and -1023, one per block, cycling per component; DC 0; quantiser 255."""
    h, w = 71, 111
    g = jc.geometry(h, w, sub)
    coef = np.zeros((g.blocks, 64), np.int64)
    ci = comp_index(g)
    for c in range(jc.SAMPLING[sub][0]):
        for i, b in enumerate(np.nonzero(ci == c)[0]):
            k = 1 + (i // 2) % 63
            coef[b, jpeg.ZIGZAG[k]] = 1023 if i % 2 == 0 else -1023
    return _baseline(f"one ac {sub} {h}x{w}", "one ac", h, w, sub, [np.full(64, 255)] * 2, coef, rng)


def _marked_path(targets: Sequence[int]):
    """``_path`` through every target: (DC values, index of the block each target landed on)."""
    out, at, cur = [], [], 0
    for t in targets:
        while abs(t - cur) > DC_MAX:
            cur += DC_MAX if t > cur else -DC_MAX
            out.append(cur)
        cur = t
        at.append(len(out))
        out.append(cur)
    return out, at


def full_column_file(rng: np.random.Generator) -> Case:
    """Grayscale, quantiser 255: DC-only blocks ramp to 32767; blocks of DC 32767 with every AC +1023, and with every AC
    +-1023 in random signs; DC-only blocks ramp down to -32768; blocks of DC -32768 with every AC -1023, and of DC -32767
    in random signs."""
    h, w = 63, 63
    g = jc.geometry(h, w, "gray")
    targets = [32767] * 4 + [-32768] + [-32767] * 3
    dcs, at = _marked_path(targets)
    assert len(dcs) <= g.blocks
    coef = np.zeros((g.blocks, 64), np.int64)
    coef[:len(dcs), 0] = dcs
    coef[len(dcs):, 0] = dcs[-1]
    coef[at[0], 1:] = 1023
    coef[at[4], 1:] = -1023
    for i in at[1:4] + at[5:]:
        coef[i, 1:] = rng.choice([-1023, 1023], 63)
    return _baseline(f"full column gray {h}x{w}", "full column", h, w, "gray", [np.full(64, 255)], coef, rng)


def random_large(g: jpeg.Geometry, rng: np.random.Generator, density: float) -> np.ndarray:
    """Random sparse coefficients: DC within +-1000, AC up to +-1023, some blocks DC-only."""
    coef = np.zeros((g.blocks, 64), np.int64)
    coef[:, 0] = rng.integers(-1000, 1001, g.blocks)
    ac = np.where(rng.random((g.blocks, 63)) < density, rng.integers(-1023, 1024, (g.blocks, 63)), 0)
    ac[rng.random(g.blocks) < 0.1] = 0
    coef[:, 1:] = ac
    return coef


QUANTS = {"random": lambda rng: [rng.integers(1, 256, 64), rng.integers(1, 256, 64)],
          "coarse": lambda rng: [np.full(64, 255), np.full(64, 200)]}


def random_files(rng: np.random.Generator) -> List[Case]:
    out = []
    for sub in SUBS:
        for qn, qf in QUANTS.items():
            h, w = 29, 43
            g = jc.geometry(h, w, sub)
            for restart in (0, 1, g.mcux + 1):
                coef = random_large(g, rng, 0.2)
                out.append(_baseline(f"random {sub} {h}x{w} {qn} dri {restart}", "random", h, w, sub, qf(rng), coef,
                                     rng, restart))
    return out


def dc_predictor_file(sub: str, rng: np.random.Generator) -> Case:
    """Luma (and in 4:2:0 the Cr component too) takes DC differences of +2047 for 20 blocks, -2047 for 40 and +2047 for
    20: the int predictor climbs past 32767 and falls past -32768, and the stored coefficient is its int16.  The other
    blocks get small differences and a few in-range AC coefficients."""
    h, w = (31, 351) if sub == "gray" else (47, 767)
    g = jc.geometry(h, w, sub)
    ci = comp_index(g)
    diffs = rng.integers(-20, 21, g.blocks)
    for c in ((0,) if sub == "gray" else (0, 2)):
        idx = np.nonzero(ci == c)[0]
        steps = [2047] * 20 + [-2047] * 40 + [2047] * 20
        assert len(idx) > len(steps)
        diffs[idx[:len(steps)]] = steps
    coef = np.zeros((g.blocks, 64), np.int64)
    coef[:, 1:10] = np.where(rng.random((g.blocks, 9)) < 0.3, rng.integers(-20, 21, (g.blocks, 9)), 0)
    for c in range(jc.SAMPLING[sub][0]):
        idx = np.nonzero(ci == c)[0]
        acc = np.cumsum(diffs[idx])                       # the int predictor
        if c == 0:
            assert acc.max() > 32767 and acc.min() < -32768
        coef[idx, 0] = ((acc + (1 << 15)) % (1 << 16)) - (1 << 15)
    quant = [np.full(64, 5)] if sub == "gray" else [np.full(64, 5), np.full(64, 3)]
    dc, ac = full_tables(jc.SAMPLING[sub][0], rng)
    head = jc.header(h, w, sub, quant, dc, ac)
    data = jc.assemble(head, [jc.pack(b) for b in encode_diffs(coef, diffs, g, dc, ac)])
    return Case(f"dc predictor {sub} {h}x{w}", "dc predictor", data, coef.astype(np.int16))


# ------------------------------------------------------------------------------------------------ progressive
def refined(coef: np.ndarray, script: Sequence[dict]) -> np.ndarray:
    """What jdphuff.c holds after ``script`` over the writer's coefficients ``coef`` (int64 [blocks, 64], natural
    order), coefficient by coefficient in int16: a first scan stores ``(JCOEF)(v << Al)``; a DC refinement ORs in its
    bit; an AC refinement either corrects a non-zero coefficient, adding p1 = 1 << Al to one that is >= 0 and -p1 to one
    that is < 0 when the bit is set and the coefficient's bit Al is clear, or sets a zero one that becomes 1 at this
    scan to +-p1.  ``script`` entries carry ``blocks``, the stream-order blocks each scan covers."""
    out = np.zeros(coef.shape, np.int64)

    def i16(v):
        return ((v + (1 << 15)) % (1 << 16)) - (1 << 15)
    for sc in script:
        ss, se, ah, al = sc["ss"], sc["se"], sc["ah"], sc["al"]
        cols = [0] if ss == 0 else [int(jpeg.ZIGZAG[k]) for k in range(ss, se + 1)]
        rows = sc["blocks"]
        t = coef[np.ix_(rows, cols)]
        cur = out[np.ix_(rows, cols)]
        if ss == 0 and ah == 0:
            new = i16((t >> al) << al)
        elif ss == 0:
            new = i16(cur | (((t >> al) & 1) << al))
        elif ah == 0:
            new = i16(np.sign(t) * ((np.abs(t) >> al) << al))
        else:
            a = np.abs(t) >> al
            p1 = 1 << al
            assert ((a > 1) == (cur != 0)).all()           # the writer's history is the decoder's
            corr = (cur != 0) & ((a & 1) == 1) & ((cur & p1) == 0)
            new = np.where(corr, i16(cur + np.where(cur >= 0, p1, -p1)), cur)
            new = np.where((cur == 0) & (a == 1), np.where(t > 0, p1, -p1), new)
        out[np.ix_(rows, cols)] = new
    return out.astype(np.int16)


def _prog(name, h, w, sub, quant, coef, script, seed, exact=True) -> Case:
    """A progressive case; ``exact``: nothing wraps under a refinement, so the writer's own record agrees everywhere,
    else wherever the writer's coefficient fits int16."""
    model = [dict(sc, blocks=np.asarray(P.order(h, w, sub, sc["comps"])[0])) for sc in script]
    want = refined(np.asarray(coef, np.int64), model)
    data, written = P.craft(h, w, sub, quant, coef, script, seed=seed)
    plain = np.abs(np.asarray(coef, np.int64)) < (1 << 15) if not exact else np.ones(want.shape, bool)
    assert np.array_equal(want[plain], written[plain]), name         # where nothing wraps, the writer agrees
    return Case(name, "progressive", data, want)


def progressive_files(rng: np.random.Generator) -> List[Case]:
    import jpeg_progressive_edges as E
    out = [Case(n, "progressive", d, c) for n, d, c in E.refine_cases() if n.startswith("al 13")]
    z19 = [int(jpeg.ZIGZAG[k]) for k in range(1, 10)]
    # DC first at Al = 13: the shifted sums k << 13 wrap int16 for |k| >= 4; refined to Al = 0 bit by bit in 4:2:0
    for sub, refine in (("420", True), ("gray", False)):
        h, w = (31, 47) if sub == "420" else (33, 41)
        g = jc.geometry(h, w, sub)
        nc = jc.SAMPLING[sub][0]
        allc = tuple(range(nc))
        coef = np.zeros((g.blocks, 64), np.int64)
        coef[:, 0] = (rng.integers(-20, 21, g.blocks) << 13) | rng.integers(0, 1 << 13, g.blocks)
        coef[:, z19] = np.where(rng.random((g.blocks, 9)) < 0.5, rng.integers(-60, 61, (g.blocks, 9)), 0)
        s = [P.scan(allc, 0, 0, 0, 13)]
        if refine:
            s += [P.scan(allc, 0, 0, a + 1, a) for a in range(12, -1, -1)]
        s += [P.scan((c,), 1, 63, 0, 0) for c in allc]
        out.append(_prog(f"dc first al 13 {sub} {h}x{w}{' refined' if refine else ''}", h, w, sub,
                         [rng.integers(1, 256, 64), rng.integers(1, 256, 64)][:1 if nc == 1 else 2], coef, s,
                         seed=int(rng.integers(1 << 30))))
    # AC first at Al = 10..13 of |v| = 1023: v << Al wraps int16; luma 1..9 refined on top of the wrapped values
    for al, sub in zip((10, 11, 12, 13), SUBS):
        h, w = 37, 53
        g = jc.geometry(h, w, sub)
        nc = jc.SAMPLING[sub][0]
        ci = comp_index(g)
        coef = np.zeros((g.blocks, 64), np.int64)
        coef[:, 0] = rng.integers(-300, 301, g.blocks)
        sign = rng.choice([-1, 1], (g.blocks, 63))
        big = sign * ((1023 << al) | rng.integers(0, 1 << al, (g.blocks, 63)))
        small = rng.integers(-(1 << al) + 1, 1 << al, (g.blocks, 63))
        pick = rng.random((g.blocks, 63))
        ac = np.where(pick < 0.35, big, np.where(pick < 0.6, small, 0))
        for c in range(1, nc):                            # chroma 1..9 are sent at Al = 0: +-1023 at most
            idx = np.nonzero(ci == c)[0]
            ac[np.ix_(idx, range(9))] = np.where(pick[np.ix_(idx, range(9))] < 0.5,
                                                 rng.integers(-1023, 1024, (len(idx), 9)), 0)
        coef[:, jpeg.ZIGZAG[1:]] = ac
        allc = tuple(range(nc))
        s = [P.scan(allc, 0, 0, 0, 0), P.scan((0,), 1, 9, 0, al)]
        s += [P.scan((0,), 1, 9, a + 1, a, restart=2 if a % 3 == 0 else 0) for a in range(al - 1, -1, -1)]
        s += [P.scan((0,), 10, 63, 0, al)]
        for c in allc[1:]:
            s += [P.scan((c,), 1, 9, 0, 0), P.scan((c,), 10, 63, 0, al, restart=3)]
        q = [rng.integers(1, 256, 64), rng.integers(1, 256, 64)][:1 if nc == 1 else 2]
        out.append(_prog(f"ac first al {al} {sub} {h}x{w}, refined over wrapped values", h, w, sub, q, coef, s,
                         seed=int(rng.integers(1 << 30)), exact=False))
    return out


# ------------------------------------------------------------------------------------------------ the corpus
def control_files(rng: np.random.Generator) -> List[Case]:
    """In range: small coefficients under quantiser 1."""
    out = []
    for sub, (h, w) in (("gray", (17, 33)), ("420", (31, 47))):
        g = jc.geometry(h, w, sub)
        coef = np.zeros((g.blocks, 64), np.int64)
        coef[:, 0] = rng.integers(-400, 401, g.blocks)
        coef[:, 1:] = np.where(rng.random((g.blocks, 63)) < 0.2, rng.integers(-8, 9, (g.blocks, 63)), 0)
        out.append(_baseline(f"control {sub} {h}x{w}", "control", h, w, sub, [np.ones(64, int)] * 2, coef, rng))
    return out


def grid_file() -> Case:
    rng = np.random.default_rng(90)
    h, w = GRID
    g = jc.geometry(h, w, "420")
    return _baseline(f"grid 420 {h}x{w}", "grid", h, w, "420", QUANTS["random"](rng), random_large(g, rng, 0.03), rng)


def corpus(grid: bool = False) -> List[Case]:
    """Every case, the 1080x1920 one only if ``grid``."""
    rng = np.random.default_rng(2024)
    out = []
    for sub in SUBS:
        for c in range(jc.SAMPLING[sub][0]):
            for i, (h, w) in enumerate(SMALL):
                out.append(wrap_file(sub, h, w, c, 8, "near", rng, start=7 * i + 3 * c))
            for q in (8, 255):
                out.append(wrap_file(sub, *SWEEP, c, q, "sweep", rng))
    out += [one_ac_file("gray", rng), one_ac_file("420", rng), full_column_file(rng)]
    out += random_files(rng)
    out += [dc_predictor_file("gray", rng), dc_predictor_file("420", rng)]
    out += progressive_files(rng)
    out += control_files(rng)
    if grid:
        out.append(grid_file())
    return out


def raw_idct(case: Case) -> List[np.ndarray]:
    """jidctint.c's output of each component's blocks before the range limit (int64 [n, 8, 8], 0 = 128)."""
    info = jpeg.parse(case.data)
    g = jpeg.geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    ci = comp_index(g)
    return [jc.idct_raw(case.coef[ci == c], info.quant[c]) for c in range(info.ncomp)]
