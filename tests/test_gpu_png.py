"""PNG files at ingress (`decode="png"`) on the GPU, bit for bit against the host restatement.

`defer_k_png_decode` gives the unfiltered scanlines, RGB and status words of `png.decode_stages` byte for byte on every
committed fixture, in one microbatch of mixed sizes, colour types and depths, with a never-written sample; a
`decode="png"` stage equals the `max_image_size` stage fed `decode_png(item)`; and `DEFER` over ResNet50 returns, per
item and in FIFO order, what the `max_image_size` pipeline returns for the decoded images, with `keep_aspect_ratio` and
a non-nearest interpolation as well.  The fixtures come from tools/make_png_fixtures.py; no Pillow here."""
import ctypes as C
import sys
import zlib
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import _cabi as A  # noqa: E402
from defer_b200 import png  # noqa: E402
import png_craft as PC  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

GOLDEN = ROOT / "tests" / "golden" / "png"


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _fixtures():
    return sorted(p.name for p in GOLDEN.glob("*.png"))


def decode_dev(files, H, W, timed=False, fill=0x5A):
    """defer_k_png_decode of ``files`` in slots of the bound (H, W): (workspace [n, stride], raw offset, images [n, H*W*3]);
    a None file is a never-written sample (zero slot, zero block).  ``timed``: also the decode's time in ms; ``fill``: the
    stale byte the workspace holds before the decode."""
    import torch
    lib = A.load()
    n = len(files)
    slot = png.slot_bytes(H, W)
    slots = np.zeros((n, slot), np.uint8)
    blocks = np.zeros((n, png.BLOCK_INTS), np.int32)
    for i, d in enumerate(files):
        if d is not None:
            slots[i, :len(d)] = np.frombuffer(d, np.uint8)
            png.pack_block(png.parse(d), blocks[i])
    total, stride, raw_off = (C.c_uint64() for _ in range(3))
    A.check(lib.defer_k_png_workspace(H, W, n, C.byref(total), C.byref(stride), C.byref(raw_off)))
    ws = torch.full((total.value,), fill, dtype=torch.uint8, device="cuda")        # stale bytes everywhere
    x = torch.from_numpy(slots.reshape(-1)).cuda()
    b = torch.from_numpy(blocks.reshape(-1)).cuda()
    y = torch.full((n * H * W * 3,), 7, dtype=torch.uint8, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]      # on the legacy default stream, as the decode
    torch.cuda.synchronize()
    ev[0].record(torch.cuda.default_stream())
    A.check(lib.defer_k_png_decode(x.data_ptr(), b.data_ptr(), n, H, W, ws.data_ptr(), y.data_ptr(), None))
    ev[1].record(torch.cuda.default_stream())
    torch.cuda.synchronize()
    out = ws.cpu().numpy().reshape(n, stride.value), raw_off.value, y.cpu().numpy().reshape(n, H * W * 3)
    return (out, ev[0].elapsed_time(ev[1])) if timed else out


def check_sample(ws, raw_off, y, d, name):
    want = png.decode_stages(d)
    info = want["info"]
    bpr = info.bytes_per_row
    rows = ws[raw_off:raw_off + info.raw_bytes].reshape(info.h, 1 + bpr)
    assert np.array_equal(rows[:, 1:], want["rows"]), name
    assert np.array_equal(y[:info.h * info.w * 3].reshape(info.h, info.w, 3), want["rgb"]), name
    assert np.array_equal(ws[:12].view(np.int32), want["stats"]), (name, ws[:12].view(np.int32).tolist(),
                                                                   want["stats"].tolist())


def test_k_png_decode_matches_host():
    names = _fixtures()
    files = [(GOLDEN / nm).read_bytes() for nm in names]
    ws, raw_off, y = decode_dev(files + [None], 256, 260)
    for i, (nm, d) in enumerate(zip(names, files)):
        check_sample(ws[i], raw_off, y[i], d, nm)
    # a never-written sample: a 1x1 black image, nothing else written
    assert (y[-1][:3] == 0).all() and (y[-1][3:] == 7).all()
    assert ws[-1][:12].view(np.int32).tolist() == [png.STATUS_EXHAUSTED, 0, 0]


def test_k_png_decode_refuses_bad_arguments():
    lib = A.load()
    assert lib.defer_k_png_decode(None, None, 1, 8, 8, None, None, None) == A.ERR_INVALID
    assert lib.defer_k_png_workspace(0, 8, 1, None, None, None) == A.ERR_INVALID
    assert lib.defer_k_png_workspace(100000, 100000, 1, None, None, None) == A.ERR_INVALID


# ------------------------------------------------------------------------------------------------ stage level
STAGE_FILES = ["photo_223x225_c2_d8_f4.png", "photo_63x65_c3_d8_z6rle_p256.png", "photo_63x65_c6_d16.png",
               "photo_1x1_c0_d1.png", "photo_31x47_c0_d2_f3.png", "pillow_60x80_p.png"]
BOUND = (240, 320)


def _stem(seed):
    from test_gpu_conv_paths import STEMS, _stem_model
    b, h, w, cin, cout, k, s, pad = STEMS["resnet_b1"]
    return _stem_model(h, w, cin, cout, k, s, pad, seed=seed)


@pytest.mark.parametrize("mode,interpolation,dtype", [("caffe", "nearest", "float32"), ("tf", "bilinear", "bfloat16")])
def test_stage_png_equals_frames(mode, interpolation, dtype, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch)
    m = _stem(seed=len(mode + interpolation))
    files = [(GOLDEN / nm).read_bytes() for nm in STAGE_FILES]
    n = len(files)
    kw = dict(device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode, max_image_size=BOUND,
              interpolation=interpolation)
    r = StageRunner.from_model(m, decode="png", **kw)
    r0 = StageRunner.from_model(m, **kw)
    try:
        y = r.predict_pngs(files)
        images = [png.decode_png(d) for d in files]
        y0 = r0.predict_frames([im[None] for im in images])
        kernels = [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))]
        kernels0 = [r0.op_info(i)["kernel"] for i in range(len(r0.plan.ops))]
        assert kernels == ["png_inflate_kernel+png_unfilter_kernel+png_expand_kernel"] + kernels0, r.describe()
        assert r.num_kernels() == r0.num_kernels() + 3
        dec = r.read_buffer(r.plan.ops[0].out)
        for i, im in enumerate(images):
            h, w = im.shape[:2]
            assert np.array_equal(dec[i].reshape(-1)[:h * w * 3].reshape(h, w, 3), im.astype(np.float32)), STAGE_FILES[i]
        assert np.array_equal(_bits(y), _bits(y0))
        assert r.io_bytes()[0] == n * png.slot_bytes(*BOUND)
        assert r.time_op(0, iters=2) > 0
        with pytest.raises(ValueError, match="submit_pngs"):
            r.submit_frames(0, 0, [np.zeros((1, 4, 5, 3), np.uint8)])
        with pytest.raises(ValueError, match="max_image_size"):
            r.submit_pngs(0, 0, [png_photo(300, 200)])
        with pytest.raises(ValueError, match="Adam7"):
            r.submit_pngs(0, 0, [files[0][:8] + PC.ihdr(225, 223, 8, 2, interlace=1) + files[0][33:]])
    finally:
        r.close()
        r0.close()


def test_submit_pngs_refusals_copy_nothing(monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    from defer_b200.resize import frame_block_ints, pack_frame_tables
    _knobs(monkeypatch)
    r = StageRunner.from_model(_stem(seed=3), device=0, max_batch=2, depth=1, preprocess="caffe", max_image_size=(40, 60),
                               decode="png")
    lib = r.lib
    try:
        d = (GOLDEN / "photo_31x47_c6_d16_f2.png").read_bytes()
        info = png.parse(d)

        def call(mutate=lambda b: None, nbytes=len(d), delta=0):
            blocks = np.concatenate([pack_frame_tables([(info.h, info.w)], (224, 224), r.plan.frames["kw"], "nearest"),
                                     png.pack_block(info)[None]], axis=1)
            mutate(blocks[0])
            sizes = np.array([nbytes], np.uint64)
            ptrs = (C.c_void_p * 1)(C.cast(C.c_char_p(d), C.c_void_p).value)
            return lib.defer_stage_submit_pngs(r.handle, 0, 0, 1, ptrs, sizes.ctypes.data, blocks.ctypes.data,
                                               blocks.nbytes + delta)
        nr = frame_block_ints((224, 224), r.plan.frames["kw"])               # the PNG block follows the resize block
        assert call(nbytes=png.slot_bytes(40, 60) + 1) == A.ERR_INVALID       # larger than the slot
        assert call(delta=4) == A.ERR_INVALID
        assert call(lambda b: b.__setitem__(nr, 41)) == A.ERR_INVALID          # PNG block over the bound
        assert call(lambda b: b.__setitem__(0, 30)) == A.ERR_INVALID           # resize and PNG headers disagree
        assert call(lambda b: b.__setitem__(nr + 3, 4)) == A.ERR_INVALID       # depth 4 in an RGBA file
        assert call(lambda b: b.__setitem__(nr + 4, 1)) == A.ERR_INVALID       # bytes per row
        assert call(lambda b: b.__setitem__(nr + 6, png.MAX_IDAT + 1)) == A.ERR_INVALID
        assert call(lambda b: b.__setitem__(nr + png.IDAT_OFF, len(d))) == A.ERR_INVALID   # IDAT past the file
        assert call(lambda b: b.__setitem__(nr + 7, 1)) == A.ERR_INVALID       # IDAT total
        r.sync()
        assert not r.read_buffer(r.plan.input_buf).any()                     # nothing was copied
        assert call() == A.OK
        r.sync()
        assert np.array_equal(r.read_buffer(r.plan.input_buf)[0].reshape(-1)[:40 * 60 * 3],
                              np.frombuffer(d.ljust(40 * 60 * 3, b"\0")[:40 * 60 * 3], np.uint8).astype(np.float32))
    finally:
        r.close()


# ------------------------------------------------------------------------------------------------ DEFER end to end
def png_photo(h, w, seed=0, ctype=2, level=6):
    """A photo-like 8-bit PNG of h x w (Sub-filtered rows), written with zlib."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([128 + 100 * np.sin(x / (9 + c * 5) + y / (13 + c * 3) + c) for c in range(3)], axis=2)
    img = np.clip(img + rng.normal(0, 6, (h, w, 3)), 0, 255).astype(np.uint8)
    if ctype == 0:
        img = img[:, :, :1]
    rows = img.reshape(h, -1).astype(np.int16)
    c = img.shape[2]
    sub = (rows - np.concatenate([np.zeros((h, c), np.int16), rows[:, :-c]], axis=1)) & 255
    raw = np.concatenate([np.ones((h, 1), np.uint8), sub.astype(np.uint8)], axis=1).tobytes()
    return PC.png_file(w, h, 8, ctype, zlib.compress(raw, level), idat_sizes=[8192] * (len(raw) // 8192))


def _items(n):
    pool = [png_photo(480, 640, 1), (GOLDEN / "photo_223x225_c2_d8_f4.png").read_bytes(), png_photo(300, 451, 2, ctype=0),
            (GOLDEN / "photo_63x65_c6_d16.png").read_bytes(), (GOLDEN / "pillow_60x80_p.png").read_bytes(),
            (GOLDEN / "photo_1x17_c3_d2_p4.png").read_bytes(), png_photo(480, 640, 3, level=0)]
    return [pool[i % len(pool)] for i in range(n)]


@pytest.mark.parametrize("interpolation,keep", [("nearest", False), ("bilinear", True)])
def test_resnet50_defer_pngs(resnet50, interpolation, keep, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from test_gpu_resize import _run_defer
    _knobs(monkeypatch)
    items = _items(40)                                                # one full group of 32 and a partial one
    items = [x if i % 3 else bytearray(x) for i, x in enumerate(items)]
    kw = dict(preprocess="caffe", max_image_size=(480, 640), interpolation=interpolation, keep_aspect_ratio=keep)
    y, io, kernels = _run_defer(resnet50, items, 1, decode="png", **kw)
    y0, io0, _ = _run_defer(resnet50, [png.decode_png(x)[None] for x in items], 1, **kw)
    assert kernels[0] == "png_inflate_kernel+png_unfilter_kernel+png_expand_kernel", kernels
    assert y.shape == (40, 1000)
    assert np.array_equal(_bits(y), _bits(y0))                        # FIFO order and every bit
