"""PNG streams no encoder writes (tests/png_craft.py) through the GPU decode.

Every crafted file, valid or corrupt, decodes in one microbatch to the scanlines, RGB and status words of
`png.decode_stages`; and the adversarial stream (maximal dynamic headers on empty blocks, filling the slot of a 480x640
bound) decodes in a bounded time with no sticky error: the next decode on the same device is exact."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import png  # noqa: E402
import png_craft as PC  # noqa: E402
from test_gpu_png import check_sample, decode_dev  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


def test_crafted_streams_match_host():
    cases = dict(PC.valid_cases())
    cases.update({k: d for k, (d, _) in PC.corrupt_cases().items()})
    names = sorted(cases)
    ws, raw_off, y = decode_dev([cases[k] for k in names], 130, 260)
    for i, k in enumerate(names):
        check_sample(ws[i], raw_off, y[i], cases[k], k)
    for k, (d, status) in PC.corrupt_cases().items():
        assert ws[names.index(k)][:4].view(np.int32)[0] == status, k


def test_adversarial_stream_is_bounded():
    H, W = 480, 640
    adv = PC.adversarial(png.slot_bytes(H, W) - 70000, W, H)
    assert len(adv) <= png.slot_bytes(H, W)
    good = (ROOT / "tests" / "golden" / "png" / "photo_223x225_c2_d8_f4.png").read_bytes()
    (ws, raw_off, y), ms = decode_dev([adv] * 32, H, W, timed=True)
    print(f"adversarial: 32 files of {len(adv)} bytes in {ms:.1f} ms")
    assert ms < 4000
    for i in range(32):                                               # the 1x1 image is never filled: black
        assert ws[i][:12].view(np.int32).tolist() == [png.STATUS_SHORT, 0, 0] and not y[i][:3].any()
    ws, raw_off, y = decode_dev([good, adv], H, W)                   # no sticky error: the device still decodes
    check_sample(ws[0], raw_off, y[0], good, "after")
