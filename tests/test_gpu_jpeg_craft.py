"""The GPU JPEG decode on crafted files: the worst case of its self-synchronisation, and corrupt files.

Worst case: under one-symbol tables of all-zero codes and all-zero entropy bits, every bit position starts a valid
block, so a decoder started in the wrong phase never resynchronises and the true state moves one subsequence per
round: the rounds are the most subsequences in one restart interval.  Each file's coefficients, planes and RGB equal
what the writer put in, and the five counters of ``stats`` (unstuffed bytes, RST markers, subsequences, rounds,
cutoff) equal the restatement's (``jpeg_check.sync_stats``), or for the 1080x1920 file the closed form that the host
tests check against it (``jpeg_craft.closed_form_counters``).

Corrupt files: a seeded corpus of bit flips, byte flips, truncations and missing, extra, renumbered and misplaced RST
markers, each a file ``jpeg.parse`` accepts, decodes as ``jpeg.decode_stages`` defines, with the restatement's counters.
No Pillow here."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests"):
    if str(p) not in sys.path:
        sys.path.insert(0, str(p))

from defer_b200 import jpeg  # noqa: E402
import jpeg_craft as jc  # noqa: E402
from jpeg_check import sync_stats  # noqa: E402
from test_gpu_jpeg import _check_sample, _decode_dev, _fixture  # noqa: E402
from test_jpeg_craft_host import SBITS, random_coef  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

BOUND = (480, 640)


def _check(ws, coef_off, plane_off, y, want, stats, name):
    """Sample ``ws`` / ``y`` of a launch against ``want`` (coef, planes, rgb) and the five counters ``stats``."""
    h, w = want["rgb"].shape[:2]
    n = want["coef"].shape[0]
    assert np.array_equal(ws[coef_off:coef_off + n * 128].view(np.int16).reshape(n, 64), want["coef"]), name
    off = plane_off
    for c, p in enumerate(want["planes"]):
        assert np.array_equal(ws[off:off + p.size].reshape(p.shape), p), (name, c)
        off += p.size
    assert np.array_equal(y[:h * w * 3].reshape(h, w, 3), want["rgb"]), name
    got = ws[:20].view(np.int32)
    assert np.array_equal(got, stats), (name, got.tolist(), stats.tolist())
    return got


# ------------------------------------------------------------------------------------------------ worst-case sync
WORST = {"a: 384x512 gray, 48 subsequences": (384, 512, "gray", 0),
         "b: 384x512 gray, DRI 333 (6 subsequences each)": (384, 512, "gray", 333),
         "b: 384x512 gray, DRI 5 (shorter than a subsequence)": (384, 512, "gray", 5),
         "c: 256x384 4:2:0, 36 subsequences": (256, 384, "420", 0)}


def test_worst_case_sync_matches_restatement():
    files, wants, stats = [], [], []
    for name, (h, w, sub, ri) in WORST.items():
        d = jc.all_zero_stream(h, w, sub, ri)
        files.append(d)
        wants.append(jc.expected(jc.all_zero_coef(jc.geometry(h, w, sub)), h, w, sub, [np.ones(64, int)]))
        stats.append(sync_stats(d, SBITS)[2])
        assert np.array_equal(stats[-1], jc.closed_form_counters(d, SBITS)), name
    ws, coef_off, plane_off, y = _decode_dev(files, *BOUND)
    for i, name in enumerate(WORST):
        got = _check(ws[i], coef_off, plane_off, y[i], wants[i], stats[i], name)
        print(f"{name}: {got[3]} rounds for {got[2]} subsequences, equal to the restatement")
    assert max(int(s[3]) for s in stats) >= 48


def test_worst_case_sync_at_the_largest_slot():
    """(d) A 1080x1920 file whose entropy data fills over 90 % of the slot: one-symbol 16-bit codes, 1476-bit blocks."""
    H, W = 1080, 1920
    d = jc.long_code_stream(H, W)
    info = jpeg.parse(d)
    assert info.length >= 0.9 * H * W * 3 and len(d) <= H * W * 3
    g = jc.geometry(H, W, "gray")
    want = jc.expected(jc.long_code_coef(g), H, W, "gray", [np.ones(64, int)])
    stats = jc.closed_form_counters(d, SBITS)
    (ws, coef_off, plane_off, y), ms = _decode_dev([d], H, W, timed=True)
    got = _check(ws[0], coef_off, plane_off, y[0], want, stats, "d")
    print(f"d: 1080x1920, {info.length} entropy bytes: {got[3]} rounds for {got[2]} subsequences, {ms:.1f} ms")


# ------------------------------------------------------------------------------------------------ corrupt files
def _flip_bits(parts, n, rng):
    """``n`` random bits of the unstuffed intervals flipped."""
    sizes = [len(p) for p in parts]
    a = np.frombuffer(b"".join(parts), np.uint8).copy()
    for b in rng.choice(8 * len(a), n, replace=False):
        a[b >> 3] ^= 0x80 >> (b & 7)
    edges = np.cumsum([0] + sizes)
    return [a[s:e].tobytes() for s, e in zip(edges[:-1], edges[1:])]


def _flip_bytes(data, n, rng):
    """``n`` random bytes of the stuffed entropy data replaced by random values (markers may appear); a file that
    ``jpeg.parse`` accepts."""
    info = jpeg.parse(data)
    while True:
        a = np.frombuffer(data, np.uint8).copy()
        pos = info.offset + rng.choice(info.length, n, replace=False)
        a[pos] = rng.integers(0, 256, n)
        try:
            jpeg.parse(a.tobytes())
            return a.tobytes()
        except ValueError:
            pass


def _put(data, at, raw):
    """``raw`` written over the stuffed entropy data at ``at``."""
    info = jpeg.parse(data)
    p = info.offset + at
    return data[:p] + raw + data[p + len(raw):]


def crafted_420(rng):
    """A 120x160 4:2:0 file with random tables and DRI 7, from random coefficients."""
    h, w, ri = 120, 160, 7
    g = jc.geometry(h, w, "420")
    coef = random_coef(rng, g)
    dc, ac = jc.tables_for(coef, g, ri, rng, 0.5)
    return jc.craft(h, w, "420", [rng.integers(1, 256, 64), rng.integers(1, 256, 64)], dc, ac, coef=coef, restart=ri)


def corpus(seed=0):
    """[(name, file)] of corrupt files, each accepted by ``jpeg.parse``."""
    rng = np.random.default_rng(seed)
    a = _fixture("photo_223x225_420_q75.jpg")            # no restart interval
    b = _fixture("photo_223x225_422_q50_rr1.jpg")        # RST every MCU row
    c = _fixture("photo_223x225_444_q75_rb1.jpg")        # RST every MCU
    d = _fixture("photo_223x225_gray_q90_rb4.jpg")
    e = crafted_420(rng)
    out = []
    for nm, f in (("a", a), ("b", b), ("e", e)):
        head, parts = jc.split(f)
        for n in (1, 8, 64):
            out.append((f"{nm}: {n} bit flips", jc.assemble(head, _flip_bits(parts, n, rng))))
    for nm, f in (("a", a), ("c", c), ("e", e)):
        for n in (1, 4, 16):
            out.append((f"{nm}: {n} byte flips", _flip_bytes(f, n, rng)))
    out.append(("a: a stray RST marker", _put(a, 3000, b"\xff\xd5")))
    out.append(("a: 0xFF before a non-marker byte", _put(a, 5000, b"\xff\x12")))
    out.append(("c: an RST marker overwritten by FF C4", _put(c, c.index(b"\xff\xd3", jpeg.parse(c).offset)
                                                             - jpeg.parse(c).offset, b"\xff\xc4")))
    head, (comp,) = jc.split(a)
    for cut in (1500, 2047, 2048, 2049, len(comp) - 5):
        out.append((f"a: cut at {cut} of {len(comp)} bytes", jc.assemble(head, [comp[:cut]])))
    info = jpeg.parse(a)
    cut = 3072
    while a[info.offset + cut - 1] == 0xFF:
        cut -= 1024
    out.append((f"a: {cut} stuffed bytes", a[:info.offset + cut] + b"\xff\xd9"))
    zhead, (zcomp,) = jc.split(jc.all_zero_stream(64, 128, "gray"))
    out.append(("all-zero stream padded to 2048 bytes", jc.assemble(zhead, [zcomp + b"\xff" * (2048 - len(zcomp))])))
    out.append(("a: RSTs without DRI", jc.assemble(head, [comp[:777], comp[777:4000], comp[4000:]])))
    head, parts = jc.split(b)
    k = len(parts) // 2
    out.append(("b: last interval cut", jc.assemble(head, parts[:-1] + [parts[-1][:len(parts[-1]) // 2]])))
    out.append(("b: one RST dropped", jc.assemble(head, parts[:k] + [parts[k] + parts[k + 1]] + parts[k + 2:])))
    out.append(("b: one RST duplicated", jc.assemble(head, parts[:k] + [b""] + parts[k:],
                                                     rst=[i % 8 for i in range(k)] + [(k - 1) % 8] +
                                                     [i % 8 for i in range(k - 1, len(parts) - 1)])))
    out.append(("b: renumbered RSTs", jc.assemble(head, parts, rst=rng.integers(0, 8, len(parts) - 1))))
    out.append(("b: adjacent RSTs", jc.assemble(head, parts[:k] + [b""] * 3 + parts[k:])))
    out.append(("b: more RSTs than intervals", jc.assemble(head, parts + [rng.bytes(50), b"", rng.bytes(9)])))
    out.append(("b: DRI without RSTs", jc.assemble(head, [b"".join(parts)])))
    head, parts = jc.split(d)
    out.append(("d: fill bytes before RSTs", jc.assemble(head, parts, fill=2)))
    out.append(("d: every RST dropped after the first", jc.assemble(head, [parts[0], b"".join(parts[1:])])))
    for name, f in out:
        jpeg.parse(f)
    return out


def test_corrupt_files_match_host():
    items = corpus()
    ws, coef_off, plane_off, y = _decode_dev([f for _, f in items], *BOUND)
    cut = 0
    for i, (name, f) in enumerate(items):
        want = jpeg.decode_stages(f)
        got = _check_sample(ws[i], coef_off, plane_off, y[i], want, name, sync_stats(f, SBITS)[2])
        cut += int(got[4]) < want["coef"].shape[0]
    print(f"{len(items)} corrupt files, {cut} of them cut by an invalid code, equal to the host")
    assert cut >= 5
