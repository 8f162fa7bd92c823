"""The GPU PNG decode at full size and on corrupt streams: row bands past 256, rows up to 15 360 bytes, every filter unit
and type, stream-shape edges, and a seeded mutation corpus.

Valid full-size files are built from a source image ``x`` filtered forward with whole-array predictors
(``png_craft.filter_rows``), so the expected scanlines are ``x`` itself, not the output of ``png.unfilter``: Up, Average
and Paeth rows on both sides of each band of 256 rows that ``png_unfilter_kernel`` works in, at widths 1 and 1920 and
heights around 256 and 512 and up to 1080, at a 1080x1920 bound.  Corrupt full-size files (truncated or bit-flipped past
row 256 of Average and Paeth rows) and several thousand mutants of small streams (tests/png_mutants.py) equal
``png.decode_stages``, the host restatement that tests/test_png_zlib_host.py checks against zlib; the mutants decode the
same over a workspace pre-filled with 0x5A and with 0xA5.  A ``decode="png"`` stage fed valid and corrupt files in one
microbatch equals the ``max_image_size`` stage fed their decoded images.  Nothing here reads Pillow."""
import sys
import zlib
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
from test_gpu_png import check_sample, decode_dev  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

GOLDEN = ROOT / "tests" / "golden" / "png"
BOUND = (1080, 1920)
BATCH = 8                        # about 60 MB of slot, workspace and image per sample at the bound
# (colour type, depth) of every filter unit: 1 byte (grey 1, 2, 4, 8 bits, palette 2 and 8 bits), 2 (grey 16, grey+alpha
# 8), 3 (RGB 8), 4 (grey+alpha 16, RGBA 8), 6 (RGB 16), 8 (RGBA 16)
MODES = [(0, 1), (0, 2), (0, 4), (0, 8), (3, 2), (3, 8), (0, 16), (4, 8), (2, 8), (4, 16), (6, 8), (2, 16), (6, 16)]
FILTERS = (0, 1, 2, 3, 4, "random")


def _source(h, bpr, seed):
    """Smooth rows with noise (zlib finds matches; every filter's residual varies)."""
    rng = np.random.default_rng(seed)
    y = np.arange(h)[:, None]
    x = np.arange(bpr)[None, :]
    smooth = (100 + 70 * np.sin(x / 37.0 + y / 23.0)).astype(np.int64)
    return ((smooth + rng.integers(0, 24, (h, bpr))) & 255).astype(np.uint8)


def _types(h, filt, seed):
    if filt == "random":
        return np.random.default_rng(seed).integers(0, 5, h).astype(np.uint8)
    return np.full(h, filt, np.uint8)


def _palette(depth):
    return bytes(np.random.default_rng(depth).integers(0, 256, 3 * (1 << depth), dtype=np.uint8))


def _valid(h, w, ctype, depth, filt, seed, level=1, chunk_bytes=8192):
    """(file, source scanlines x)"""
    x = _source(h, PC.bytes_per_row(w, depth, ctype), seed)
    d = PC.encode(x, w, depth, ctype, _types(h, filt, seed), level=level, chunk_bytes=chunk_bytes,
                  palette=_palette(depth) if ctype == 3 else None)
    return d, x


def _decode_exact(cases):
    """Decode ``cases`` [(name, file, x)] in microbatches of BATCH at the bound, each with a never-written sample; every
    file must give the scanlines x, their RGB and [OK, scanline bytes, 0]."""
    for b0 in range(0, len(cases), BATCH):
        part = cases[b0:b0 + BATCH]
        ws, raw_off, y = decode_dev([d for _, d, _ in part] + [None], *BOUND)
        for i, (name, d, x) in enumerate(part):
            info = png.parse(d)
            rows = ws[i][raw_off:raw_off + info.raw_bytes].reshape(info.h, 1 + info.bytes_per_row)
            assert np.array_equal(rows[:, 1:], x), name
            assert np.array_equal(y[i][:info.h * info.w * 3].reshape(info.h, info.w, 3), png.to_rgb(x, info)), name
            assert ws[i][:12].view(np.int32).tolist() == [png.STATUS_OK, info.raw_bytes, 0], name
        assert ws[-1][:12].view(np.int32).tolist() == [png.STATUS_EXHAUSTED, 0, 0]
        assert (y[-1][:3] == 0).all() and (y[-1][3:] == 7).all()


def _band_cases():
    """Heights on both sides of each band boundary and the bound, widths 1 and 1920, a random filter type per row (Up,
    Average and Paeth rows cross every boundary), the filter units taken in turn."""
    k = 0
    for h in (255, 256, 257, 511, 512, 513, 1080):
        for w in (1, 1920):
            ctype, depth = MODES[k % len(MODES)]
            k += 1
            yield f"band_{h}x{w}_c{ctype}_d{depth}", *_valid(h, w, ctype, depth, "random", k)


def _unit_cases():
    """Every filter unit with each filter type forced on every row, and random per row, at 300 rows (past the first
    band) and a width that cycles through 1920, 1 and 333."""
    k = 0
    for ctype, depth in MODES:
        for filt in FILTERS:
            w = (1920, 1, 333)[k % 3]
            k += 1
            yield f"unit_c{ctype}_d{depth}_f{filt}_w{w}", *_valid(300, w, ctype, depth, filt, 100 + k)


def test_full_size_bands_match_source():
    _decode_exact(list(_band_cases()))


def test_every_filter_unit_and_type_match_source():
    cases = list(_unit_cases())
    assert len(cases) == len(MODES) * len(FILTERS)
    _decode_exact(cases)


# ------------------------------------------------------------------------------------------------ stream shapes
def _match_32768_near_end():
    """A 1080x1920 RGBA16 file (16.6 MB of scanlines, filter None) whose stream ends with a crafted fixed block: a match
    of length 258 at distance 32768 about 1000 bytes before the end, then literals."""
    h, w = 1080, 1920
    bpr = 8 * w
    x = _source(h, bpr, 7)
    rowlen = 1 + bpr
    p = (h - 1) * rowlen + 1 + bpr - 1000 - 258                     # in the last row's data
    src = p - 32768
    assert src % rowlen and (src + 257) // rowlen == src // rowlen     # the source is data of one row too
    raw = bytearray(PC.filter_rows(x, 8, np.zeros(h, np.uint8)))
    raw[p:p + 258] = raw[src:src + 258]
    x = np.frombuffer(bytes(raw), np.uint8).reshape(h, rowlen)[:, 1:].copy()
    c = zlib.compressobj(1)
    head = c.compress(bytes(raw[:p])) + c.flush(zlib.Z_FULL_FLUSH)   # byte-aligned; the window stays the decoder's
    bw = PC.BitWriter()
    bw.huffman([("m", 258, 32768)] + list(raw[p + 258:]), final=True)
    stream = head + bw.tobytes() + zlib.adler32(bytes(raw)).to_bytes(4, "big")
    assert zlib.decompress(stream) == bytes(raw)
    return PC.png_file(w, h, 16, 6, stream, idat_sizes=[8192] * (len(stream) // 8192)), x


def test_stream_shape_edges():
    cases = []
    # level 0 at the bound's deepest mode, libpng's 8 KiB chunks: the claim behind DEFER_PNG_SLOT_BYTES
    d, x = _valid(1080, 1920, 6, 16, "random", 1, level=0)
    assert len(d) <= png.slot_bytes(*BOUND) and len(png.parse(d).idat) <= png.MAX_IDAT
    png.check_png(d, BOUND)
    cases.append(("stored_1080x1920_rgba16", d, x))
    # exactly MAX_IDAT chunks
    x = _source(400, 3 * 600, 2)
    raw = PC.filter_rows(x, 3, _types(400, "random", 2))
    z = zlib.compress(raw, 6)
    k = len(z) // png.MAX_IDAT
    assert k >= 1
    d = PC.png_file(600, 400, 8, 2, z, idat_sizes=[k] * (png.MAX_IDAT - 1))
    assert len(png.parse(d).idat) == png.MAX_IDAT
    cases.append(("max_idat", d, x))
    cases.append(("match_32768_near_end", *_match_32768_near_end()))
    _decode_exact(cases)


# ------------------------------------------------------------------------------------------------ corrupt at full size
def _corrupt_full():
    """1080-row RGB files of Average and Paeth rows, cut or bit-flipped past row 256: the zero tail and the wrong bytes
    are unfiltered across band boundaries."""
    h, w = 1080, 160
    x = _source(h, 3 * w, 11)
    types = np.array([3 + (r % 2) for r in range(h)], np.uint8)
    raw = PC.filter_rows(x, 3, types)
    z6, z0 = zlib.compress(raw, 6), zlib.compress(raw, 0)
    out = [("cut_40pct", z6[:len(z6) * 4 // 10]), ("cut_75pct", z6[:len(z6) * 3 // 4]), ("stored_cut_55pct",
                                                                                        z0[:len(z0) * 55 // 100])]
    for name, s, frac in (("flip_z6_50pct", z6, 0.5), ("flip_z6_90pct", z6, 0.9), ("flip_stored_60pct", z0, 0.6)):
        b = bytearray(s)
        b[int(len(s) * frac)] ^= 0x10
        out.append((name, bytes(b)))
    return [(name, PC.png_file(w, h, 8, 2, s, idat_sizes=[8192] * (len(s) // 8192))) for name, s in out]


def test_corrupt_full_size_match_host():
    cases = _corrupt_full()
    ws, raw_off, y = decode_dev([d for _, d in cases], *BOUND)
    for i, (name, d) in enumerate(cases):
        info = png.parse(d)
        produced = int(ws[i][4:8].view(np.int32)[0])
        assert 257 * (1 + info.bytes_per_row) < produced <= info.raw_bytes, (name, produced)
        check_sample(ws[i], raw_off, y[i], d, name)


# ------------------------------------------------------------------------------------------------ the mutation corpus
MUTANT_BOUND = (20, 258)
MUTANT_BATCH = 1024


def test_mutants_match_host_over_any_stale_workspace():
    cases = png_mutants.mutants()
    assert len(cases) > 5000
    for name, d in cases:
        info = png.parse(d)
        assert info.h <= MUTANT_BOUND[0] and info.w <= MUTANT_BOUND[1], name
    seen = set()
    for b0 in range(0, len(cases), MUTANT_BATCH):
        part = cases[b0:b0 + MUTANT_BATCH]
        files = [d for _, d in part]
        ws, raw_off, y = decode_dev(files, *MUTANT_BOUND, fill=0x5A)
        ws2, _, y2 = decode_dev(files, *MUTANT_BOUND, fill=0xA5)
        for i, (name, d) in enumerate(part):
            check_sample(ws[i], raw_off, y[i], d, name)
            info = png.parse(d)
            n = info.h * info.w * 3
            rows = [w[i][raw_off:raw_off + info.raw_bytes].reshape(info.h, -1)[:, 1:] for w in (ws, ws2)]
            assert np.array_equal(ws[i][:12], ws2[i][:12]), name
            assert np.array_equal(rows[0], rows[1]), name             # (a filter type byte not produced is not written)
            assert np.array_equal(y[i][:n], y2[i][:n]), name
            seen.add(int(ws[i][:4].view(np.int32)[0]))
    assert seen == set(range(png.STATUS_OK, png.STATUS_BAD_DISTANCE + 1)), seen


# ------------------------------------------------------------------------------------------------ stage level
STAGE_BOUND = (240, 320)


def test_stage_mixed_corrupt_and_valid_equals_frames(monkeypatch):
    """Valid and corrupt files in one microbatch: the defined result of each corrupt file flows through resize and
    preprocess, and its neighbours are exact."""
    from test_gpu_conv_paths import _knobs
    from test_gpu_png import _bits, _stem
    from defer_b200.node import StageRunner
    _knobs(monkeypatch)
    photo = (GOLDEN / "photo_223x225_c2_d8_f4.png").read_bytes()
    info = png.parse(photo)
    stream = png.gather(photo, info)
    corrupt = PC.corrupt_cases()
    files = [photo,
             PC.png_file(info.w, info.h, 8, 2, stream[:len(stream) // 2]),               # cut: the lower half is zero
             (GOLDEN / "photo_63x65_c6_d16.png").read_bytes(),
             corrupt["dist_too_far"][0], corrupt["dyn_empty_cl_code_cut"][0],
             PC.png_file(info.w, info.h, 8, 2, stream[:900] + bytes([stream[900] ^ 4]) + stream[901:]),
             (GOLDEN / "pillow_60x80_p.png").read_bytes(), corrupt["stored_truncated"][0]]
    statuses = [int(png.decode_stages(d)["stats"][0]) for d in files]
    assert statuses.count(png.STATUS_OK) == 3 and len(set(statuses)) >= 4, statuses
    m = _stem(seed=5)
    kw = dict(device=0, dtype="float32", max_batch=len(files), depth=1, preprocess="tf", max_image_size=STAGE_BOUND,
              interpolation="bilinear")
    r = StageRunner.from_model(m, decode="png", **kw)
    r0 = StageRunner.from_model(m, **kw)
    try:
        y = r.predict_pngs(files)
        images = [png.decode_png(d) for d in files]
        y0 = r0.predict_frames([im[None] for im in images])
        dec = r.read_buffer(r.plan.ops[0].out)
        for i, im in enumerate(images):
            h, w = im.shape[:2]
            assert np.array_equal(dec[i].reshape(-1)[:h * w * 3].reshape(h, w, 3), im.astype(np.float32)), i
        assert np.array_equal(_bits(y), _bits(y0))
    finally:
        r.close()
        r0.close()
