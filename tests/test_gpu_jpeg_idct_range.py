"""The GPU JPEG decode beyond the IDCT range: the files of tests/jpeg_idct_range.py, bit for bit against the host.

The host tests (tests/test_jpeg_idct_range_host.py) pin ``jpeg.decode_stages`` to libjpeg-turbo's C path on these
files; here the device equals ``decode_stages``, so it follows the same rules: int16 coefficients from DC prediction and
progressive first scans, refinements on top of wrapped values, the 10-bit wrap of ``jidctint.c``, and upsampling and
colour conversion of wrapped samples.  All files go in one microbatch with the 1080x1920 grid, so the IDCT kernel meets
out-of-range blocks across a full grid of CTAs.  A ``decode="jpeg"`` stage, fused and unfused stem, equals the
``max_image_size`` stage fed the host decode of wrap-point files, including ones with fewer than 3 chroma columns.  No
Pillow."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import jpeg  # noqa: E402
import jpeg_idct_range as R  # noqa: E402
from test_gpu_jpeg import _bits, _decode_dev  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]


def test_k_jpeg_decode_beyond_the_range():
    cases = R.corpus(grid=True)
    H, W = R.GRID
    ws, coef_off, plane_off, y = _decode_dev([c.data for c in cases], H, W)
    for i, case in enumerate(cases):
        want = jpeg.decode_stages(case.data)
        assert np.array_equal(want["coef"], case.coef), case.name
        n = len(case.coef)
        assert np.array_equal(ws[i][coef_off:coef_off + n * 128].view(np.int16).reshape(n, 64), want["coef"]), case.name
        off = plane_off
        for c, p in enumerate(want["planes"]):
            assert np.array_equal(ws[i][off:off + p.size].reshape(p.shape), p), (case.name, c)
            off += p.size
        h, w = want["rgb"].shape[:2]
        assert np.array_equal(y[i][:h * w * 3].reshape(h, w, 3), want["rgb"]), case.name
    print(f"{len(cases)} files beyond the IDCT range ({', '.join(sorted({c.kind for c in cases}))}): coefficients, "
          f"planes and RGB equal the host")


#: wrap points at the right and bottom edges and in chroma of downsampled width 2 (5x4, 7x3), in luma and chroma
STAGE = ["wrap 420 5x4 comp 1 q8 near", "wrap 422 7x3 comp 2 q8 near", "wrap 420 17x33 comp 0 q8 near",
         "wrap 420 31x47 comp 2 q8 near", "wrap 444 1x17 comp 1 q8 near", "wrap gray 7x3 comp 0 q8 near"]


@pytest.mark.parametrize("path", ["fused", "unfused"])
def test_stage_beyond_the_range_equals_frames(path, monkeypatch):
    from test_gpu_conv_paths import _knobs
    from test_gpu_jpeg import _stem
    from defer_b200.node import StageRunner
    _knobs(monkeypatch, **({"DEFER_STREAM_MIN_TILES": 1} if path == "fused" else {"DEFER_STEM_FUSED": 0}))
    by = {c.name: c.data for c in R.corpus()}
    files = [by[n] for n in STAGE]
    kw = dict(device=0, dtype="float32", max_batch=len(files), depth=1, preprocess="caffe", max_image_size=(480, 640),
              interpolation="bilinear")
    m = _stem(seed=11)
    r = StageRunner.from_model(m, decode="jpeg", **kw)
    r0 = StageRunner.from_model(m, **kw)
    try:
        y = r.predict_jpegs(files)
        images = [jpeg.decode_jpeg(d) for d in files]
        y0 = r0.predict_frames([im[None] for im in images])
        dec = r.read_buffer(r.plan.ops[0].out)
        for i, im in enumerate(images):
            h, w = im.shape[:2]
            assert np.array_equal(dec[i].reshape(-1)[:h * w * 3].reshape(h, w, 3), im.astype(np.float32)), STAGE[i]
        assert np.array_equal(_bits(y), _bits(y0))
    finally:
        r.close()
        r0.close()
