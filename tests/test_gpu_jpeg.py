"""JPEG files at ingress (`decode="jpeg"`) on the GPU, bit for bit against the host restatement.

The contract: `defer_k_jpeg_decode` gives the coefficients, planes and RGB of `jpeg.decode_stages` byte for byte, and the
five counters of the restatement in tests/jpeg_check.py (on the committed fixtures, on a file with random entropy data
and on a never-written sample); a `decode="jpeg"` stage equals the
`max_image_size` stage fed `decode_jpeg(item)`, in both preprocessing modes, dtypes and stem paths and after lane re-use;
and `DEFER` over one and two stages returns what the `max_image_size` pipeline returns for the decoded images, in FIFO
order, and surfaces a refused file as a ValueError.  The fixtures come from tools/make_jpeg_fixtures.py; no Pillow here."""
import ctypes as C
import queue
import re
import sys
import threading
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import _cabi as A  # noqa: E402
from defer_b200 import applications  # noqa: E402
from defer_b200 import jpeg  # noqa: E402
from jpeg_check import sync_stats  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

GOLDEN = ROOT / "tests" / "golden" / "jpeg"
SBITS = int(re.search(r"#define DEFER_JPEG_SUBSEQ_BITS (\d+)", (ROOT / "include" / "defer_b200.h").read_text()).group(1))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _fixture(name):
    return (GOLDEN / name).read_bytes()


def _all_fixtures():
    return sorted(p.name for p in GOLDEN.glob("*.jpg"))


def random_entropy(data, seed):
    """A valid header of ``data`` followed by random entropy bytes and EOI (a defined result, see jpeg.py)."""
    info = jpeg.parse(data)
    rng = np.random.default_rng(seed)
    junk = rng.integers(0, 256, info.length, dtype=np.uint8)
    junk[-1] = 0
    ff = np.nonzero(junk[:-1] == 0xFF)[0]            # each 0xFF is stuffed or an RSTn marker, as inside a scan
    junk[ff + 1] = rng.choice(np.array([0x00] + list(range(0xD0, 0xD8)), np.uint8), len(ff))
    return data[:info.offset] + junk.tobytes() + b"\xff\xd9"


def _decode_dev(files, H, W, timed=False):
    """defer_k_jpeg_decode of ``files`` in slots of the bound (H, W): (workspace, coef offset, plane offset, images); a
    None file is a never-written sample (zero slot, zero block).  ``timed``: also the decode's time in ms (CUDA events)."""
    import torch
    lib = A.load()
    n = len(files)
    slot = H * W * 3
    slots = np.zeros((n, slot), np.uint8)
    blocks = np.zeros((n, jpeg.BLOCK_INTS), np.int32)
    for i, d in enumerate(files):
        if d is not None:
            slots[i, :len(d)] = np.frombuffer(d, np.uint8)
            blocks[i] = jpeg.pack_block(jpeg.parse(d))
    total, stride, coef_off, plane_off = (C.c_uint64() for _ in range(4))
    A.check(lib.defer_k_jpeg_workspace(H, W, n, C.byref(total), C.byref(stride), C.byref(coef_off), C.byref(plane_off)))
    ws = torch.full((total.value,), 0x5A, dtype=torch.uint8, device="cuda")        # stale bytes everywhere
    x = torch.from_numpy(slots.reshape(-1)).cuda()
    b = torch.from_numpy(blocks.reshape(-1)).cuda()
    y = torch.full((n * slot,), 7, dtype=torch.uint8, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]      # on the legacy default stream, as the decode
    torch.cuda.synchronize()
    ev[0].record(torch.cuda.default_stream())
    A.check(lib.defer_k_jpeg_decode(x.data_ptr(), b.data_ptr(), n, H, W, ws.data_ptr(), y.data_ptr(), None))
    ev[1].record(torch.cuda.default_stream())
    torch.cuda.synchronize()
    ws = ws.cpu().numpy().reshape(n, stride.value)
    y = y.cpu().numpy().reshape(n, slot)
    out = ws, coef_off.value, plane_off.value, y
    return (out, ev[0].elapsed_time(ev[1])) if timed else out


def _check_sample(ws, coef_off, plane_off, y, want, name, stats=None):
    info, g = want["info"], jpeg.geometry(want["info"].h, want["info"].w, want["info"].ncomp, want["info"].hs,
                                          want["info"].vs)
    coef = ws[coef_off:coef_off + g.blocks * 128].view(np.int16).reshape(g.blocks, 64)
    assert np.array_equal(coef, want["coef"]), name
    off = plane_off
    for c, p in enumerate(want["planes"]):
        got = ws[off:off + p.size].reshape(p.shape)
        assert np.array_equal(got, p), (name, c)
        off += p.size
    assert np.array_equal(y[:info.h * info.w * 3].reshape(info.h, info.w, 3), want["rgb"]), name
    got = ws[:20].view(np.int32)
    assert 0 <= got[4] <= g.blocks and not want["decoded"][got[4]:].any(), name   # nothing after the cutoff
    if stats is not None:
        assert np.array_equal(got, stats), (name, got.tolist(), stats.tolist())
    return got


def test_k_jpeg_decode_matches_host():
    names = _all_fixtures()
    files = [_fixture(nm) for nm in names]
    files += [random_entropy(_fixture(nm), seed=i) for i, nm in enumerate(
        ["photo_223x225_420_q75.jpg", "photo_223x225_444_q75_rb1.jpg", "photo_223x225_gray_q50_rr1.jpg",
         "photo_480x640_422_q90_rr1.jpg"])]
    names += ["random entropy"] * 4
    ws, coef_off, plane_off, y = _decode_dev(files + [None], 1080, 1920)
    for i, (nm, d) in enumerate(zip(names, files)):
        # all five counters (unstuffed bytes, RST markers, subsequences, rounds, cutoff) equal the restatement's
        _check_sample(ws[i], coef_off, plane_off, y[i], jpeg.decode_stages(d), nm, sync_stats(d, SBITS)[2])
    # a never-written sample: a 1x1 image of value 128, nothing else written
    assert np.array_equal(y[-1][:3], [128, 128, 128])
    assert (y[-1][3:] == 7).all()


def test_k_jpeg_decode_refuses_bad_arguments():
    lib = A.load()
    assert lib.defer_k_jpeg_decode(None, None, 1, 8, 8, None, None, None) == A.ERR_INVALID
    assert lib.defer_k_jpeg_workspace(0, 8, 1, None, None, None, None) == A.ERR_INVALID


# ------------------------------------------------------------------------------------------------ stage level
STAGE_FILES = ["photo_480x640_420_q75.jpg", "photo_223x225_444_q95.jpg", "photo_223x225_gray_q75_rb1.jpg",
               "photo_1x1_444_q95.jpg", "photo_223x225_422_q50_rr1.jpg", "checker_31x47_420_q95.jpg"]
BOUND = (480, 640)


def _stem(seed):
    from test_gpu_conv_paths import STEMS, _stem_model
    b, h, w, cin, cout, k, s, pad = STEMS["resnet_b1"]
    return _stem_model(h, w, cin, cout, k, s, pad, seed=seed)


@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("mode,interpolation", [("caffe", "nearest"), ("tf", "bilinear")])
def test_stage_jpeg_equals_frames(mode, interpolation, dtype, path, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch, **({"DEFER_STREAM_MIN_TILES": 1} if path == "fused" else {"DEFER_STEM_FUSED": 0}))
    m = _stem(seed=len(mode + interpolation))
    files = [_fixture(nm) for nm in STAGE_FILES]
    n = len(files)
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode, max_image_size=BOUND,
                               interpolation=interpolation, decode="jpeg")
    r0 = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode, max_image_size=BOUND,
                                interpolation=interpolation)
    try:
        y = r.predict_jpegs(files)
        images = [jpeg.decode_jpeg(d) for d in files]
        y0 = r0.predict_frames([im[None] for im in images])
        kernels = [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))]
        kernels0 = [r0.op_info(i)["kernel"] for i in range(len(r0.plan.ops))]
        assert kernels == ["jpeg_entropy_kernel+jpeg_idct_kernel+jpeg_color_kernel"] + kernels0, r.describe()
        assert r.num_kernels() == r0.num_kernels() + 3
        dec = r.read_buffer(r.plan.ops[0].out)
        for i, im in enumerate(images):
            h, w = im.shape[:2]
            assert np.array_equal(dec[i].reshape(-1)[:h * w * 3].reshape(h, w, 3), im.astype(np.float32)), STAGE_FILES[i]
        assert np.array_equal(r.read_buffer(r.plan.ops[2].out), r0.read_buffer(r0.plan.ops[1].out))
        assert np.array_equal(_bits(y), _bits(y0))
        info = r.op_info(0)
        assert info["alg_bytes"] > 2 * n * 480 * 640 * 3 and r.time_op(0, iters=3) > 0
        assert r.io_bytes()[0] == n * 480 * 640 * 3
    finally:
        r.close()
        r0.close()


def test_lane_reuse_and_never_written_samples(monkeypatch):
    """Depth 1: a small group after a large one runs on the same slots, blocks and workspace; stale bytes are never read.
    A fresh stage's never-written samples are harmless: they give what a fresh max_image_size stage's do."""
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch)
    m = _stem(seed=2)
    kw = dict(device=0, max_batch=4, depth=1, preprocess="caffe", max_image_size=BOUND, interpolation="bilinear")
    r = StageRunner.from_model(m, decode="jpeg", **kw)
    r0 = StageRunner.from_model(m, **kw)
    try:
        one = [_fixture("photo_17x33_420_q5.jpg")]
        y = r.predict_jpegs(one)
        r0.predict_frames([jpeg.decode_jpeg(one[0])[None]])
        assert np.array_equal(_bits(r.result(0)), _bits(r0.result(0)))
        assert y.shape[0] == 1
        big = [_fixture(nm) for nm in ("photo_480x640_420_q75.jpg", "photo_480x640_422_q90_rr1.jpg",
                                       "photo_223x225_444_q100.jpg", "full_31x47_gray_q95.jpg")]
        small = [_fixture(nm) for nm in ("photo_3x5_420_q5.jpg", "zero_31x47_444_q95.jpg")]
        for group in (big, small, big[:3], small[1:]):
            y = r.predict_jpegs(group)
            y0 = r0.predict_frames([jpeg.decode_jpeg(d)[None] for d in group])
            assert np.array_equal(_bits(y), _bits(y0))
    finally:
        r.close()
        r0.close()


def test_submit_jpegs_refusals_copy_nothing(monkeypatch):
    import torch  # noqa: F401
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    from defer_b200.resize import frame_block_ints, pack_frame_tables
    _knobs(monkeypatch)
    r = StageRunner.from_model(_stem(seed=3), device=0, max_batch=2, depth=1, preprocess="caffe", max_image_size=(40, 60),
                               decode="jpeg")
    frames = StageRunner.from_model(_stem(seed=3), device=0, max_batch=2, depth=1, preprocess="caffe",
                                    max_image_size=(40, 60))
    lib = r.lib
    try:
        d = _fixture("photo_40x60_420_q75_meta.jpg")
        info = jpeg.parse(d)

        def call(mutate=lambda b: None, nbytes=len(d), delta=0, stage=r):
            blocks = np.concatenate([pack_frame_tables([(info.h, info.w)], (224, 224), r.plan.frames["kw"], "nearest"),
                                     jpeg.pack_block(info)[None]], axis=1)
            mutate(blocks[0])
            sizes = np.array([nbytes], np.uint64)
            ptrs = (C.c_void_p * 1)(C.cast(C.c_char_p(d), C.c_void_p).value)
            return lib.defer_stage_submit_jpegs(stage.handle, 0, 0, 1, ptrs, sizes.ctypes.data, blocks.ctypes.data,
                                                blocks.nbytes + delta)
        nr = frame_block_ints((224, 224), r.plan.frames["kw"])               # the JPEG block follows the resize block
        assert call(nbytes=40 * 60 * 3 + 1) == A.ERR_INVALID                     # larger than the slot
        assert call(delta=4) == A.ERR_INVALID
        assert call(lambda b: b.__setitem__(nr, 41)) == A.ERR_INVALID             # JPEG block over the bound
        assert call(lambda b: b.__setitem__(0, 39)) == A.ERR_INVALID              # resize and JPEG headers disagree
        assert call(lambda b: b.__setitem__(nr + 7, len(d))) == A.ERR_INVALID     # entropy data past the file
        assert call(stage=frames) == A.ERR_INVALID                                # a stage without the op
        r.sync()
        assert not r.read_buffer(r.plan.input_buf).any()                        # nothing was copied
        with pytest.raises(ValueError, match="submit_jpegs"):
            r.submit_frames(0, 0, [np.zeros((1, 4, 5, 3), np.uint8)])
        with pytest.raises(ValueError, match="max_image_size"):
            r.submit_jpegs(0, 0, [_fixture("photo_223x225_420_q75.jpg")])
        with pytest.raises(ValueError, match="truncated"):
            r.submit_jpegs(0, 0, [d[:-2]])
        assert call() == A.OK
        r.sync()
        assert np.array_equal(r.read_buffer(r.plan.input_buf)[0].reshape(-1)[:len(d)],
                              np.frombuffer(d, np.uint8).astype(np.float32))
    finally:
        r.close()
        frames.close()


# ------------------------------------------------------------------------------------------------ DEFER end to end
MIXED = ["photo_480x640_420_q75.jpg", "photo_223x225_444_q95.jpg", "photo_223x225_gray_q50_rr1.jpg",
         "photo_1080x1920_420_q50.jpg", "photo_223x225_422_q75_rb1.jpg", "photo_1x1_420_q95.jpg",
         "photo_40x60_420_q75_meta.jpg", "photo_480x640_422_q90_rr1.jpg", "checker_31x47_gray_q95.jpg"]


@pytest.mark.parametrize("n_stages", [1, 2])
def test_resnet50_defer_jpegs(resnet50, n_stages, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from test_gpu_resize import _run_defer
    _knobs(monkeypatch)
    items = [_fixture(MIXED[i % len(MIXED)]) for i in range(40)]     # one full group of 32 and a partial one
    items = [x if i % 3 else bytearray(x) for i, x in enumerate(items)]
    y, io, kernels = _run_defer(resnet50, items, n_stages, preprocess="caffe", max_image_size=(1080, 1920),
                                interpolation="bilinear", decode="jpeg")
    decoded = [jpeg.decode_jpeg(x)[None] for x in items]
    y0, io0, _ = _run_defer(resnet50, decoded, n_stages, preprocess="caffe", max_image_size=(1080, 1920),
                            interpolation="bilinear")
    assert kernels[0] == "jpeg_entropy_kernel+jpeg_idct_kernel+jpeg_color_kernel", kernels
    assert y.shape == (40, 1000)
    assert np.array_equal(_bits(y), _bits(y0))                # FIFO order and every bit
    assert io == io0


def test_defer_surfaces_refused_jpeg(resnet50, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.dispatcher import DEFER
    _knobs(monkeypatch)
    d = DEFER([0], depth=2, coalesce=4, linger_us=2000, preprocess="caffe", max_image_size=(480, 640), decode="jpeg")
    in_q, out_q = queue.Queue(), queue.Queue()
    err = []

    def run():
        try:
            d.run_defer(resnet50, [], in_q, out_q)
        except BaseException as e:  # noqa: BLE001
            err.append(e)
    t = threading.Thread(target=run, daemon=True)
    t.start()
    assert d.wait_ready(300)
    in_q.put(_fixture("photo_223x225_420_q75.jpg"))
    assert out_q.get(timeout=120).shape == (1, 1000)
    in_q.put(_fixture("photo_1080x1920_420_q50.jpg"))          # over the bound
    t.join(timeout=120)
    assert not t.is_alive()
    assert err and isinstance(err[0], ValueError) and "max_image_size" in str(err[0]), err
    d.close()
