"""The PNG inflate restatement against zlib's C inflate, on valid and corrupt streams.

``png.inflate_restated`` is the reference the GPU inflate is tested against bit for bit; here it is checked against the
system libz (tests/zlib_c.py) on every committed fixture, every crafted stream (tests/png_craft.py) and a seeded corpus of
several thousand truncated, bit-flipped, overwritten and spliced streams (tests/png_mutants.py).  Both must give the same
bytes and the same status.  The only exceptions are the deviations the module docstring of defer_b200/png.py names, each
recognised by an exact predicate; each must occur in the corpus, and none may explain a pair that differs otherwise.

The forward filters that tests/test_gpu_png_full.py builds its full-size files with are checked here as well, against
``png.unfilter`` and against Pillow."""
import collections
import functools
import io
import sys
import warnings
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import png  # noqa: E402
import png_craft as PC  # noqa: E402
import png_mutants  # noqa: E402
import zlib_c  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "png"
EXHAUSTED, OK = png.STATUS_EXHAUSTED, png.STATUS_OK


# ------------------------------------------------------------------------------------------------ the deviations
def stored_cut(stream, limit, restated, c) -> bool:
    """(a) a stored block whose data runs past the input: the restatement stops EXHAUSTED before it, zlib also gives the
    part of the block in the input (up to ``limit``; when that fills the image its status is OK)."""
    (rb, rs), (zb, zs) = restated, c
    if rs != EXHAUSTED or len(zb) <= len(rb) or zb[:len(rb)] != rb:
        return False
    extra = zb[len(rb):]
    if zs == EXHAUSTED:                                      # all of the input's part of the block: the stream's tail
        starts = [len(stream) - len(extra)] if stream.endswith(extra) else []
    elif zs == OK and len(zb) == limit:
        starts, i = [], stream.find(extra, 6)
        while i >= 0:
            starts.append(i)
            i = stream.find(extra, i + 1)
    else:
        return False
    for q in starts:                                         # LEN and NLEN before the data; LEN past the input
        ln, nln = int.from_bytes(stream[q - 4:q - 2], "little"), int.from_bytes(stream[q - 2:q], "little")
        if q >= 6 and ln == (~nln & 0xFFFF) and q + ln > len(stream):
            return True
    return False


#: (b), (c), (d): the restatement refuses where zlib still waits for input; given any more input, zlib refuses with the
#: restatement's status and this message
EARLY_REFUSALS = {
    "empty_code_length_code": (png.STATUS_BAD_HEADER, "invalid code -- missing end-of-block"),
    "repeat_16_first": (png.STATUS_BAD_HEADER, "invalid bit length repeat"),
    "empty_distance_code": (png.STATUS_BAD_SYMBOL, "invalid distance code"),
}


def early_refusal(stream, limit, restated, c):
    """The name of the deviation (b), (c) or (d) that explains the pair, or None: the same bytes, zlib waiting for input
    (EXHAUSTED) where the restatement has refused, and zlib refusing the same way whatever bits follow (zeros or ones)."""
    (rb, rs), (zb, zs) = restated, c
    if rb != zb or zs != EXHAUSTED:
        return None
    for name, (status, msg) in EARLY_REFUSALS.items():
        if rs == status and all(zlib_c.inflate_raw(stream + bytes([fill]) * 64, limit)[::2] == (rb, msg)
                                for fill in (0x00, 0xFF)):
            return name
    return None


def explain(stream, limit, restated, c):
    """None when the restatement and zlib agree, else the name of the deviation that explains the difference, else
    'UNEXPLAINED'."""
    if restated == c:
        return None
    if stored_cut(stream, limit, restated, c):
        return "stored_block_cut"
    return early_refusal(stream, limit, restated, c) or "UNEXPLAINED"


# ------------------------------------------------------------------------------------------------ the corpus
def _streams():
    """(name, zlib stream, limit) of every fixture, crafted file and mutant."""
    files = [(p.name, p.read_bytes()) for p in sorted(GOLDEN.glob("*.png"))]
    files += sorted(PC.valid_cases().items())
    files += [(k, d) for k, (d, _) in sorted(PC.corrupt_cases().items())]
    files += png_mutants.mutants()
    out = []
    for name, d in files:
        info = png.parse(d)
        out.append((name, png.gather(d, info), info.raw_bytes))
    return out


@functools.lru_cache(maxsize=None)
def _results():
    zlib_c.lib()
    return [(name, stream, limit, png.inflate_restated(stream, limit), zlib_c.inflate_c(stream, limit))
            for name, stream, limit in _streams()]


def test_restatement_equals_libz():
    by_status, by_deviation, unexplained = collections.Counter(), collections.Counter(), []
    for name, stream, limit, restated, c in _results():
        by_status[restated[1]] += 1
        why = explain(stream, limit, restated, c)
        if why == "UNEXPLAINED":
            unexplained.append((name, restated[1], len(restated[0]), c[1], len(c[0])))
        elif why is not None:
            by_deviation[why] += 1
    n = len(_results())
    print(f"libz {zlib_c.version()}: {n} streams; restated status: {dict(sorted(by_status.items()))}; "
          f"deviations: {dict(sorted(by_deviation.items()))}")
    assert not unexplained, unexplained[:20]
    assert set(by_status) == set(range(png.STATUS_OK, png.STATUS_BAD_DISTANCE + 1)), by_status
    assert set(by_deviation) == {"stored_block_cut"} | set(EARLY_REFUSALS), by_deviation
    assert sum(by_deviation.values()) < n // 10, by_deviation


def test_crafted_deviations_are_the_named_ones():
    """Each crafted deviation is explained by its own predicate; the crafted corruptions that are not deviations
    equal zlib."""
    want = {"stored_truncated": "stored_block_cut", "dyn_empty_cl_code_cut": "empty_code_length_code",
            "dyn_16_first_cut": "repeat_16_first", "dyn_empty_dist_used_at_end": "empty_distance_code"}
    for name, (d, status) in PC.corrupt_cases().items():
        info = png.parse(d)
        stream = png.gather(d, info)
        restated = png.inflate_restated(stream, info.raw_bytes)
        assert restated[1] == status, name
        assert explain(stream, info.raw_bytes, restated, zlib_c.inflate_c(stream, info.raw_bytes)) == want.get(name), name


def test_short_and_exhausted_are_told_apart():
    """zlib waits for input in both: after the final block (for the trailer) and inside a block.  The retry with the
    Adler-32 appended tells them apart, and so does a trailer cut short."""
    corrupt = PC.corrupt_cases()
    for name, status in (("short", png.STATUS_SHORT), ("exhausted_in_block", png.STATUS_EXHAUSTED),
                         ("exhausted", png.STATUS_EXHAUSTED)):
        d = corrupt[name][0]
        info = png.parse(d)
        stream = png.gather(d, info)
        out, ret, msg = zlib_c.inflate_raw(stream, info.raw_bytes)
        assert (ret, msg) == (zlib_c.Z_BUF_ERROR, "")
        assert zlib_c.inflate_c(stream, info.raw_bytes) == (out, status) == png.inflate_restated(stream, info.raw_bytes)
    w = PC.BitWriter()
    w.huffman([1, 2, 3], final=True)
    z = w.zlib(bytes([1, 2, 3]))
    for cut in range(len(z) - 4, len(z) + 1):               # the trailer: none, part, all
        assert zlib_c.inflate_c(z[:cut], 10) == (bytes([1, 2, 3]), png.STATUS_SHORT)
    assert zlib_c.inflate_c(z, 3) == (bytes([1, 2, 3]), png.STATUS_OK)


def test_deviation_predicates_are_exact():
    """Each predicate explains its own crafted case and nothing near it: not another status, not other bytes."""
    corrupt = PC.corrupt_cases()

    def case(name):
        d = corrupt[name][0]
        info = png.parse(d)
        stream = png.gather(d, info)
        return stream, info.raw_bytes, png.inflate_restated(stream, info.raw_bytes), zlib_c.inflate_c(stream,
                                                                                                    info.raw_bytes)
    stream, limit, (rb, rs), (zb, zs) = case("stored_truncated")
    assert stored_cut(stream, limit, (rb, rs), (zb, zs))
    assert not stored_cut(stream, limit, (rb, png.STATUS_BAD_BLOCK), (zb, zs))
    assert not stored_cut(stream, limit, (rb, rs), (zb[:-1] + bytes([zb[-1] ^ 1]), zs))
    assert not stored_cut(stream, limit, (rb, rs), (zb, png.STATUS_SHORT))
    assert not stored_cut(stream, limit, (rb[:-1], rs), (zb, zs))
    for name, dev in (("dyn_empty_cl_code_cut", "empty_code_length_code"), ("dyn_16_first_cut", "repeat_16_first"),
                      ("dyn_empty_dist_used_at_end", "empty_distance_code")):
        stream, limit, (rb, rs), (zb, zs) = case(name)
        assert early_refusal(stream, limit, (rb, rs), (zb, zs)) == dev
        assert early_refusal(stream, limit, (rb, png.STATUS_BAD_DISTANCE), (zb, zs)) is None
        assert early_refusal(stream, limit, (rb, rs), (zb, png.STATUS_SHORT)) is None
        if rb:
            assert early_refusal(stream, limit, (rb[:-1], rs), (zb[:-1], zs)) is None
    # a stream cut where zlib waits and refusing is not yet defined: the restatement claiming a refusal is not explained
    w = PC.BitWriter()
    w.huffman([1, 2, 3], final=False)
    z = w.zlib()
    assert explain(z, 20, (bytes([1, 2, 3]), png.STATUS_BAD_HEADER), zlib_c.inflate_c(z, 20)) == "UNEXPLAINED"


# ------------------------------------------------------------------------------------------------ forward filters
MODES = [(0, 1), (0, 2), (0, 4), (0, 8), (3, 8), (3, 2), (0, 16), (4, 8), (2, 8), (4, 16), (6, 8), (2, 16), (6, 16)]


def _source(h, w, depth, ctype, seed):
    rng = np.random.default_rng(seed)
    bpr = PC.bytes_per_row(w, depth, ctype)
    y, x = np.mgrid[0:h, 0:bpr]
    smooth = (96 + 60 * np.sin(x / 11.0 + y / 7.0)).astype(np.int64)
    return ((smooth + rng.integers(0, 40, (h, bpr))) & 255).astype(np.uint8)


def _types(h, mode, seed):
    return np.full(h, mode, np.uint8) if mode != "random" else np.random.default_rng(seed).integers(0, 5, h).astype(
        np.uint8)


def _palette(depth):
    return bytes(np.random.default_rng(depth).integers(0, 256, 3 * (1 << depth), dtype=np.uint8))


@pytest.mark.parametrize("ctype,depth", MODES)
def test_forward_filters_invert_unfilter(ctype, depth):
    for h, w in ((1, 1), (5, 3), (9, 17), (4, 33)):
        x = _source(h, w, depth, ctype, h * w)
        for mode in (0, 1, 2, 3, 4, "random"):
            d = PC.encode(x, w, depth, ctype, _types(h, mode, w), palette=_palette(depth) if ctype == 3 else None)
            st = png.decode_stages(d)
            assert np.array_equal(st["rows"], x), (h, w, mode)
            assert st["stats"].tolist() == [png.STATUS_OK, st["info"].raw_bytes, 0]


@pytest.mark.parametrize("ctype,depth", MODES)
def test_forward_filters_decode_as_pillow(ctype, depth):
    Image = pytest.importorskip("PIL.Image")
    h, w = 6, 13
    x = _source(h, w, depth, ctype, 3)
    for mode in (0, 1, 2, 3, 4, "random"):
        d = PC.encode(x, w, depth, ctype, _types(h, mode, 1), palette=_palette(depth) if ctype == 3 else None)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = np.asarray(Image.open(io.BytesIO(d)).convert("RGB"))
        info = png.parse(d)
        assert np.array_equal(png.to_rgb(x, info), want), mode
