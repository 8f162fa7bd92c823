"""Progressive JPEG files on the GPU, bit for bit against the host restatement.

``defer_k_jpeg_decode`` gives the coefficients, planes and RGB of ``jpeg.decode_stages`` byte for byte, and all six
counters of the restatement in tests/jpeg_progressive_sync.py (unstuffed bytes, RST markers, subsequences, rounds, the
failing block, the scans decoded whole), on the committed progressive fixtures, on the crafted scan scripts of
tests/jpeg_craft_progressive.py and on a seeded corpus of corrupt files, alone and mixed with baseline files in one
microbatch.  A ``decode="jpeg"`` stage equals the ``max_image_size`` stage fed
``decode_jpeg(item)`` on mixed items, with the same sample slots taking progressive, then baseline, then progressive
files; ``DEFER`` over one and two stages returns the same bits in FIFO order; submit refuses a scan past its file."""
import ctypes as C
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests", ROOT / "tools"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import _cabi as A  # noqa: E402
from defer_b200 import jpeg  # noqa: E402
from jpeg_craft_progressive import corpus  # noqa: E402
from jpeg_progressive_check import corrupt_corpus, fixture, fixture_names  # noqa: E402
from jpeg_progressive_sync import sync_progressive  # noqa: E402
from jpeg_progressive_worst_case import refinement_stream  # noqa: E402
from test_gpu_jpeg import _bits, _decode_dev, _fixture as baseline_fixture, random_entropy  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
SBITS = int(re.search(r"#define DEFER_JPEG_SUBSEQ_BITS (\d+)", (ROOT / "include" / "defer_b200.h").read_text()).group(1))


def _check(ws, coef_off, plane_off, y, d, name):
    want = jpeg.decode_stages(d)
    info = want["info"]
    g = jpeg.geometry(info.h, info.w, info.ncomp, info.hs, info.vs)
    coef = ws[coef_off:coef_off + g.blocks * 128].view(np.int16).reshape(g.blocks, 64)
    assert np.array_equal(coef, want["coef"]), name
    off = plane_off
    for c, p in enumerate(want["planes"]):
        assert np.array_equal(ws[off:off + p.size].reshape(p.shape), p), (name, c)
        off += p.size
    assert np.array_equal(y[:info.h * info.w * 3].reshape(info.h, info.w, 3), want["rgb"]), name
    st = ws[:24].view(np.int32)
    if info.progressive:
        coef_r, stats = sync_progressive(d, SBITS)
        assert np.array_equal(coef_r, want["coef"]), name
        assert np.array_equal(st, stats), (name, st.tolist(), stats.tolist())
    return st


def test_k_jpeg_decode_progressive_fixtures():
    names = fixture_names()
    files = [fixture(nm) for nm in names]
    ws, coef_off, plane_off, y = _decode_dev(files, 480, 640)
    for i, (nm, d) in enumerate(zip(names, files)):
        _check(ws[i], coef_off, plane_off, y[i], d, nm)


def test_k_jpeg_decode_crafted():
    """Scan scripts Pillow cannot write; each file also decodes to the coefficients its writer knows."""
    cases = corpus()
    ws, coef_off, plane_off, y = _decode_dev([d for _, d, _ in cases], 480, 640)
    for i, (nm, d, want) in enumerate(cases):
        _check(ws[i], coef_off, plane_off, y[i], d, nm)
        g = jpeg.geometry(*(lambda f: (f.h, f.w, f.ncomp, f.hs, f.vs))(jpeg.parse(d)))
        assert np.array_equal(ws[i][coef_off:coef_off + g.blocks * 128].view(np.int16).reshape(-1, 64), want), nm


def test_k_jpeg_decode_progressive_corrupt():
    corpus = corrupt_corpus(seed=0)
    assert len(corpus) >= 40
    files = [f for _, f in corpus]
    ws, coef_off, plane_off, y = _decode_dev(files, 223, 225)
    failed = 0
    for i, (nm, d) in enumerate(corpus):
        st = _check(ws[i], coef_off, plane_off, y[i], d, nm)
        failed += int(st[5] < len(jpeg.parse(d).scans))
    assert failed >= 5                                      # the corpus reaches the failure path


def test_mixed_microbatch():
    """Baseline and progressive files, and random baseline entropy, in one microbatch."""
    prog = ["photo_61x75_420_q75_rb1.jpg", "photo_480x640_420_q75.jpg", "photo_7x9_gray_q5.jpg",
            "photo_223x225_420_q100.jpg"]
    base = ["photo_480x640_420_q75.jpg", "photo_223x225_444_q95.jpg", "photo_1x1_420_q95.jpg"]
    files = []
    for i in range(4):
        files.append(fixture(prog[i]))
        if i < len(base):
            files.append(baseline_fixture(base[i]))
    files.append(random_entropy(baseline_fixture("photo_223x225_420_q75.jpg"), seed=3))
    files.append(refinement_stream(480, 640))             # one 17-bit AC refinement symbol per coefficient
    ws, coef_off, plane_off, y = _decode_dev(files, 480, 640)
    for i, d in enumerate(files):
        _check(ws[i], coef_off, plane_off, y[i], d, i)


# ------------------------------------------------------------------------------------------------ stage level
BOUND = (480, 640)


def _stem(seed):
    from test_gpu_conv_paths import STEMS, _stem_model
    b, h, w, cin, cout, k, s, pad = STEMS["resnet_b1"]
    return _stem_model(h, w, cin, cout, k, s, pad, seed=seed)


@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("mode,interpolation", [("caffe", "nearest"), ("tf", "bilinear")])
def test_stage_progressive_equals_frames(mode, interpolation, dtype, path, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch, **({"DEFER_STREAM_MIN_TILES": 1} if path == "fused" else {"DEFER_STEM_FUSED": 0}))
    m = _stem(seed=len(mode + interpolation))
    kw = dict(device=0, dtype=dtype, max_batch=4, depth=1, preprocess=mode, max_image_size=BOUND,
              interpolation=interpolation)
    r = StageRunner.from_model(m, decode="jpeg", **kw)
    r0 = StageRunner.from_model(m, **kw)
    try:
        groups = [[fixture("photo_480x640_420_q75.jpg"), fixture("photo_61x75_444_q75_rb1.jpg"),
                   baseline_fixture("photo_223x225_gray_q75_rb1.jpg"), fixture("photo_24x40_422_q75.jpg")],
                  [baseline_fixture("photo_480x640_420_q75.jpg"), baseline_fixture("photo_1x1_444_q95.jpg")],
                  [fixture("photo_17x33_gray_q75.jpg"), fixture("photo_223x225_420_q100.jpg")]]
        for files in groups:             # the same slots: progressive, then baseline, then progressive files
            y = r.predict_jpegs(files)
            y0 = r0.predict_frames([jpeg.decode_jpeg(d)[None] for d in files])
            assert np.array_equal(_bits(y), _bits(y0))
    finally:
        r.close()
        r0.close()


def test_submit_refuses_scan_past_file(monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    from defer_b200.resize import pack_frame_tables
    _knobs(monkeypatch)
    r = StageRunner.from_model(_stem(seed=3), device=0, max_batch=2, depth=1, preprocess="caffe", max_image_size=(64, 80),
                               decode="jpeg")
    try:
        d = fixture("photo_61x75_420_q75.jpg")
        info = jpeg.parse(d)

        def call(mutate=lambda b: None):
            blocks = np.concatenate([pack_frame_tables([(info.h, info.w)], (224, 224), r.plan.frames["kw"], "nearest"),
                                     jpeg.pack_block(info)[None]], axis=1)
            nr = blocks.shape[1] - jpeg.BLOCK_INTS
            mutate(blocks[0, nr:])
            sizes = np.array([len(d)], np.uint64)
            ptrs = (C.c_void_p * 1)(C.cast(C.c_char_p(d), C.c_void_p).value)
            return r.lib.defer_stage_submit_jpegs(r.handle, 0, 0, 1, ptrs, sizes.ctypes.data, blocks.ctypes.data,
                                                  blocks.nbytes)
        last = jpeg.SCAN_OFF + (len(info.scans) - 1) * jpeg.SCAN_INTS
        assert call(lambda b: b.__setitem__(last + 10, len(d))) == A.ERR_INVALID       # a scan past the file
        assert call(lambda b: b.__setitem__(10, jpeg.MAX_SCANS + 1)) == A.ERR_INVALID   # over the scan cap
        assert call(lambda b: b.__setitem__(11, jpeg.MAX_TABLES + 1)) == A.ERR_INVALID
        r.sync()
        assert not r.read_buffer(r.plan.input_buf).any()                             # nothing was copied
        assert call() == A.OK
        r.sync()
    finally:
        r.close()


@pytest.mark.parametrize("n_stages", [1, 2])
def test_resnet50_defer_progressive(resnet50, n_stages, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from test_gpu_resize import _run_defer
    _knobs(monkeypatch)
    pool = [fixture("photo_480x640_420_q75.jpg"), baseline_fixture("photo_480x640_420_q75.jpg"),
            fixture("photo_61x75_gray_q50_rr1.jpg"), baseline_fixture("photo_223x225_444_q95.jpg"),
            fixture("photo_223x225_420_q100.jpg"), fixture("photo_1x1_444_q95.jpg")]
    items = [pool[i % len(pool)] for i in range(40)]
    y, io, kernels = _run_defer(resnet50, items, n_stages, preprocess="caffe", max_image_size=BOUND,
                                interpolation="bilinear", decode="jpeg")
    decoded = [jpeg.decode_jpeg(x)[None] for x in items]
    y0, io0, _ = _run_defer(resnet50, decoded, n_stages, preprocess="caffe", max_image_size=BOUND,
                            interpolation="bilinear")
    assert kernels[0] == "jpeg_entropy_kernel+jpeg_idct_kernel+jpeg_color_kernel", kernels
    assert np.array_equal(_bits(y), _bits(y0))
    assert io == io0
