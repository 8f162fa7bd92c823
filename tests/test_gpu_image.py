"""JPEG and PNG files in one pipeline (`decode="image"`) on the GPU, bit for bit against the host restatement.

`defer_k_image_decode` gives, on one microbatch that interleaves every committed JPEG, progressive JPEG and PNG fixture
with never-written samples, over a workspace of stale bytes, the image of `image.decode_image` for each sample and the
stats words that its format's own `defer_k_*_decode` gives, in both orders; a `decode="image"` stage equals the
`max_image_size` stage fed `decode_image(item)`, with the fused and the unfused stem, and while the same slots alternate
between the formats; a refused `defer_stage_submit_images` copies nothing; and `DEFER` over ResNet50 returns, per item
and in FIFO order, what the `max_image_size` pipeline returns for the decoded images.  No Pillow here."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import _cabi as A  # noqa: E402
from defer_b200 import image, jpeg, png  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

GOLDEN = ROOT / "tests" / "golden"
IMAGE_KERNELS = ("jpeg_entropy_kernel+jpeg_idct_kernel+jpeg_color_kernel+png_inflate_kernel+png_unfilter_kernel+"
                 "png_expand_kernel")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _read(path):
    return (GOLDEN / path).read_bytes()


def _fixtures():
    jpegs = [f"jpeg/{p.name}" for p in sorted((GOLDEN / "jpeg").glob("*.jpg"))]
    jpegs += [f"jpeg_progressive/{p.name}" for p in sorted((GOLDEN / "jpeg_progressive").glob("*.jpg"))]
    pngs = [f"png/{p.name}" for p in sorted((GOLDEN / "png").glob("*.png"))]
    return jpegs, pngs


def _stats_words(kind, blk_progressive):
    # the words each decoder writes: JPEG [0..4] (+ [5], the scans decoded whole, for a progressive file), PNG [0..2]
    return (6 if blk_progressive else 5) if kind == "jpeg" else 3


class Decode:
    """One kernel-level decode entry point over n samples at the bound (H, W), on device buffers it keeps."""

    def __init__(self, kind, n, H, W):
        import torch
        self.torch, self.lib, self.kind, self.n, self.H, self.W = torch, A.load(), kind, n, H, W
        self.slot = {"jpeg": H * W * 3, "png": png.slot_bytes(H, W), "image": png.slot_bytes(H, W)}[kind]
        self.block_ints = {"jpeg": jpeg.BLOCK_INTS, "png": png.BLOCK_INTS, "image": image.BLOCK_INTS}[kind]
        total, stride = C.c_uint64(), C.c_uint64()
        if kind == "jpeg":
            A.check(self.lib.defer_k_jpeg_workspace(H, W, n, C.byref(total), C.byref(stride), None, None))
        elif kind == "png":
            A.check(self.lib.defer_k_png_workspace(H, W, n, C.byref(total), C.byref(stride), None))
        else:
            A.check(self.lib.defer_k_image_workspace(H, W, n, C.byref(total), C.byref(stride), None, None, None))
        self.stride = stride.value
        self.ws = torch.full((total.value,), 0x5A, dtype=torch.uint8, device="cuda")    # stale bytes everywhere
        self.x = torch.zeros(n * self.slot, dtype=torch.uint8, device="cuda")
        self.b = torch.zeros(n * self.block_ints, dtype=torch.int32, device="cuda")
        self.y = torch.full((n * H * W * 3,), 7, dtype=torch.uint8, device="cuda")

    def run(self, files, timed=False):
        """Decode ``files`` (a None file is a never-written sample: zero slot, zero block) over whatever the workspace
        holds; the images and stats stay on the device.  ``timed``: the decode's time in ms (CUDA events)."""
        torch = self.torch
        assert len(files) == self.n
        self.x.zero_()
        blocks = np.zeros((self.n, self.block_ints), np.int32)
        for i, d in enumerate(files):
            if d is None:
                continue
            self.x[i * self.slot:i * self.slot + len(d)] = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
            if self.kind == "image":
                _, kind, info = image.check_image(d, (self.H, self.W))
                image.pack_block(kind, info, blocks[i])
            elif self.kind == "jpeg":
                jpeg.pack_block(jpeg.parse(d), blocks[i])
            else:
                png.pack_block(png.parse(d), blocks[i])
        self.b.copy_(torch.from_numpy(blocks.reshape(-1)))
        fn = getattr(self.lib, f"defer_k_{self.kind}_decode")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]      # on the legacy default stream, as the decode
        torch.cuda.synchronize()
        ev[0].record(torch.cuda.default_stream())
        A.check(fn(self.x.data_ptr(), self.b.data_ptr(), self.n, self.H, self.W, self.ws.data_ptr(), self.y.data_ptr(),
                   None))
        ev[1].record(torch.cuda.default_stream())
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) if timed else None

    def stats(self, i, words=8):
        return self.ws[i * self.stride:i * self.stride + 4 * words].cpu().numpy().view(np.int32)

    def rgb(self, i, h, w):
        o = i * self.H * self.W * 3
        return self.y[o:o + h * w * 3].cpu().numpy().reshape(h, w, 3)


def test_k_image_decode_matches_each_format():
    jpegs, pngs = _fixtures()
    H, W = 1080, 1920                                                    # the largest JPEG fixture
    order = []
    for k in range(max(len(jpegs), len(pngs))):                         # interleaved, a never-written sample every 25
        order += [p for p in (jpegs[k] if k < len(jpegs) else None, pngs[k] if k < len(pngs) else None) if p]
        if k % 25 == 0:
            order.append(None)
    data = {p: _read(p) for p in order if p}
    # each format's own decode of the same files gives the reference stats words
    want_stats = {}
    for kind, paths in (("jpeg", jpegs), ("png", pngs)):
        dec = Decode(kind, len(paths), H, W)
        dec.run([data[p] for p in paths])
        for i, p in enumerate(paths):
            want_stats[p] = dec.stats(i)
        del dec
    dec = Decode("image", len(order), H, W)
    for files in (order, order[::-1]):                                  # reversed: each slot's workspace held the other format
        dec.run([data[p] if p else None for p in files])
        for i, p in enumerate(files):
            if p is None:                                                # decoded as in a PNG stage: 1x1 black, EXHAUSTED
                assert np.array_equal(dec.rgb(i, 1, 1), np.zeros((1, 1, 3), np.uint8)), i
                assert dec.stats(i, 3).tolist() == [png.STATUS_EXHAUSTED, 0, 0], i
                continue
            kind = image.sniff(data[p])
            want = image.decode_image(data[p])
            h, w = want.shape[:2]
            assert np.array_equal(dec.rgb(i, h, w), want), p
            progressive = kind == "jpeg" and jpeg.parse(data[p]).progressive
            k = _stats_words(kind, progressive)
            assert np.array_equal(dec.stats(i, k), want_stats[p][:k]), (p, dec.stats(i, k).tolist(),
                                                                          want_stats[p][:k].tolist())


def test_k_image_decode_refuses_bad_arguments():
    lib = A.load()
    assert lib.defer_k_image_decode(None, None, 1, 8, 8, None, None, None) == A.ERR_INVALID
    assert lib.defer_k_image_workspace(0, 8, 1, None, None, None, None, None) == A.ERR_INVALID


# ------------------------------------------------------------------------------------------------ stage level
STAGE_FILES = ["jpeg/photo_480x640_420_q75.jpg", "png/photo_223x225_c2_d8_f4.png", "jpeg_progressive/photo_480x640_420_q75.jpg",
               "png/photo_63x65_c6_d16.png", "jpeg/photo_223x225_gray_q75_rb1.jpg", "png/pillow_60x80_p.png",
               "jpeg/photo_1x1_444_q95.jpg", "png/photo_1x1_c0_d1.png"]
BOUND = (480, 640)


def _stem(seed):
    from test_gpu_conv_paths import STEMS, _stem_model
    b, h, w, cin, cout, k, s, pad = STEMS["resnet_b1"]
    return _stem_model(h, w, cin, cout, k, s, pad, seed=seed)


@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("mode,interpolation,dtype", [("caffe", "nearest", "float32"), ("tf", "bilinear", "bfloat16")])
def test_stage_image_equals_frames(mode, interpolation, dtype, path, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch, **({"DEFER_STREAM_MIN_TILES": 1} if path == "fused" else {"DEFER_STEM_FUSED": 0}))
    m = _stem(seed=len(mode + interpolation))
    files = [_read(p) for p in STAGE_FILES]
    n = len(files)
    kw = dict(device=0, dtype=dtype, max_batch=n, depth=1, preprocess=mode, max_image_size=BOUND,
              interpolation=interpolation)
    r = StageRunner.from_model(m, decode="image", **kw)
    r0 = StageRunner.from_model(m, **kw)
    try:
        y = r.predict_images(files)
        images = [image.decode_image(d) for d in files]
        y0 = r0.predict_frames([im[None] for im in images])
        kernels = [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))]
        kernels0 = [r0.op_info(i)["kernel"] for i in range(len(r0.plan.ops))]
        assert kernels == [IMAGE_KERNELS] + kernels0, r.describe()
        assert r.num_kernels() == r0.num_kernels() + 6
        dec = r.read_buffer(r.plan.ops[0].out)
        for i, im in enumerate(images):
            h, w = im.shape[:2]
            assert np.array_equal(dec[i].reshape(-1)[:h * w * 3].reshape(h, w, 3), im.astype(np.float32)), STAGE_FILES[i]
        assert np.array_equal(_bits(y), _bits(y0))
        assert r.io_bytes()[0] == n * png.slot_bytes(*BOUND)
        assert r.op_info(0)["alg_bytes"] > 0 and r.time_op(0, iters=2) > 0
        for call in (r.submit_frames, r.submit_jpegs, r.submit_pngs):
            with pytest.raises(ValueError, match="submit_images"):
                call(0, 0, [files[0]])
        with pytest.raises(ValueError, match="neither a JPEG nor a PNG file"):
            r.submit_images(0, 0, [b"GIF89a" + bytes(40)])
        with pytest.raises(ValueError, match="outside max_image_size"):
            r.submit_images(0, 0, [_read("jpeg/photo_1080x1920_420_q50.jpg")])
    finally:
        r.close()
        r0.close()


def test_slots_alternate_formats(monkeypatch):
    """Depth 1: the same slots, blocks and workspace take JPEG, then PNG, then JPEG files, large ones before small ones;
    nothing of a sample's previous file or format leaks into the next."""
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    _knobs(monkeypatch)
    m = _stem(seed=2)
    kw = dict(device=0, max_batch=4, depth=1, preprocess="caffe", max_image_size=BOUND, interpolation="bilinear")
    r = StageRunner.from_model(m, decode="image", **kw)
    r0 = StageRunner.from_model(m, **kw)
    from test_gpu_png import png_photo
    try:
        big_j = [_read(p) for p in ("jpeg/photo_480x640_420_q75.jpg", "jpeg_progressive/photo_480x640_420_q75.jpg",
                                    "jpeg/photo_480x640_422_q90_rr1.jpg", "jpeg/photo_223x225_444_q100.jpg")]
        big_p = [png_photo(480, 640, 1), png_photo(480, 640, 3, level=0), _read("png/photo_223x225_c2_d8_f4.png"),
                 png_photo(300, 451, 2, ctype=0)]
        small_j = [_read(p) for p in ("jpeg/photo_3x5_420_q5.jpg", "jpeg/zero_31x47_444_q95.jpg",
                                      "jpeg_progressive/photo_15x17_420_q5.jpg", "jpeg/photo_1x1_gray_q100.jpg")]
        small_p = [_read(p) for p in ("png/photo_1x1_c0_d1.png", "png/photo_1x17_c3_d2_p4.png", "png/pillow_60x80_p.png",
                                      "png/photo_63x65_c6_d16.png")]
        mixed = [big_p[0], small_j[0], big_j[1], small_p[2]]
        for group in (big_j, small_p, big_j, big_p, small_j, big_p[:2], small_j[1:3], mixed, mixed[::-1], small_p[:1]):
            y = r.predict_images(group)
            y0 = r0.predict_frames([image.decode_image(d)[None] for d in group])
            assert np.array_equal(_bits(y), _bits(y0))
            dec = r.read_buffer(r.plan.ops[0].out)
            for i, d in enumerate(group):
                im = image.decode_image(d)
                h, w = im.shape[:2]
                assert np.array_equal(dec[i].reshape(-1)[:h * w * 3].reshape(h, w, 3), im.astype(np.float32))
    finally:
        r.close()
        r0.close()


def test_submit_images_refusals_copy_nothing(monkeypatch):
    from test_gpu_conv_paths import _knobs
    from defer_b200.node import StageRunner
    from defer_b200.resize import frame_block_ints, pack_frame_tables
    _knobs(monkeypatch)
    H, W = 40, 60
    r = StageRunner.from_model(_stem(seed=3), device=0, max_batch=2, depth=1, preprocess="caffe", max_image_size=(H, W),
                               decode="image")
    lib = r.lib
    try:
        dp = _read("png/photo_31x47_c6_d16_f2.png")
        dj = _read("jpeg/photo_17x33_420_q5.jpg")

        def call(d, mutate=lambda b: None, nbytes=None, delta=0, hdr=None):
            _, kind, info = image.check_image(hdr or d, (H, W))             # the blocks of hdr (default: d)
            blocks = np.concatenate([pack_frame_tables([(info.h, info.w)], (224, 224), r.plan.frames["kw"], "nearest"),
                                     image.pack_block(kind, info)[None]], axis=1)
            mutate(blocks[0])
            sizes = np.array([len(d) if nbytes is None else nbytes], np.uint64)
            ptrs = (C.c_void_p * 1)(C.cast(C.c_char_p(d), C.c_void_p).value)
            return lib.defer_stage_submit_images(r.handle, 0, 0, 1, ptrs, sizes.ctypes.data, blocks.ctypes.data,
                                                 blocks.nbytes + delta)
        nr = frame_block_ints((224, 224), r.plan.frames["kw"])             # the tagged block follows the resize block
        tag = nr + image.TAG
        big_j = dj + bytes(H * W * 3 + 1 - len(dj))                         # over a JPEG's H * W * 3 bytes, in the slot
        assert len(big_j) < png.slot_bytes(H, W)
        assert call(dj, lambda b: b.__setitem__(tag, 0)) == A.ERR_INVALID      # untagged
        assert call(dj, lambda b: b.__setitem__(tag, 3)) == A.ERR_INVALID      # unknown tag
        assert call(big_j, hdr=dj) == A.ERR_INVALID                             # a JPEG over H * W * 3 bytes
        assert b"the slot takes 4..7200" in lib.defer_last_error()
        assert call(dp, nbytes=png.slot_bytes(H, W) + 1) == A.ERR_INVALID      # a PNG over its slot
        assert call(dj, delta=4) == A.ERR_INVALID
        assert call(dj, lambda b: b.__setitem__(nr + 7, len(dj))) == A.ERR_INVALID    # entropy data past the file
        assert call(dp, lambda b: b.__setitem__(nr + png.IDAT_OFF, len(dp))) == A.ERR_INVALID   # IDAT past the file
        assert call(dp, lambda b: b.__setitem__(nr, H + 1)) == A.ERR_INVALID   # over the bound
        r.sync()
        assert not r.read_buffer(r.plan.input_buf).any()                     # nothing was copied
        assert call(dp) == A.OK
        r.sync()
        assert np.array_equal(r.read_buffer(r.plan.input_buf)[0].reshape(-1)[:H * W * 3],
                              np.frombuffer(dp.ljust(H * W * 3, b"\0")[:H * W * 3], np.uint8).astype(np.float32))
    finally:
        r.close()


# ------------------------------------------------------------------------------------------------ DEFER end to end
def _items(n):
    from test_gpu_png import png_photo
    pool = [_read("jpeg/photo_480x640_420_q75.jpg"), png_photo(480, 640, 1), _read("jpeg_progressive/photo_480x640_420_q75.jpg"),
            _read("png/photo_223x225_c2_d8_f4.png"), _read("jpeg/photo_223x225_422_q50_rr1.jpg"), png_photo(300, 451, 2, ctype=0),
            _read("jpeg/photo_40x60_420_q75_meta.jpg"), _read("png/pillow_60x80_p.png"), _read("jpeg/photo_1x17_gray_q5.jpg"),
            _read("png/photo_1x17_c3_d2_p4.png"), _read("jpeg/photo_480x640_422_q90_rr1.jpg")]
    return [pool[i % len(pool)] for i in range(n)]


@pytest.mark.parametrize("interpolation,keep", [("nearest", False), ("bilinear", True)])
def test_resnet50_defer_images(resnet50, interpolation, keep, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from test_gpu_resize import _run_defer
    _knobs(monkeypatch)
    items = _items(40)                                                # one full group of 32 and a partial one
    items = [x if i % 3 else bytearray(x) for i, x in enumerate(items)]
    kw = dict(preprocess="caffe", max_image_size=(480, 640), interpolation=interpolation, keep_aspect_ratio=keep)
    y, io, kernels = _run_defer(resnet50, items, 1, decode="image", **kw)
    y0, io0, _ = _run_defer(resnet50, [image.decode_image(x)[None] for x in items], 1, **kw)
    assert kernels[0] == IMAGE_KERNELS, kernels
    assert io[0] == png.slot_bytes(480, 640) * 32
    assert y.shape == (40, 1000)
    assert np.array_equal(_bits(y), _bits(y0))                        # FIFO order and every bit
