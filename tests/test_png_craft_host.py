"""PNG streams no encoder writes (tests/png_craft.py), on the host.

Valid crafted files decode as Pillow decodes them; each corrupt one ends its stream with the status the module
docstring of defer_b200/png.py defines, keeps what was produced before the fault, and nothing after the fault changes
the result."""
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

VALID = PC.valid_cases()
CORRUPT = PC.corrupt_cases()


@pytest.mark.parametrize("name", sorted(VALID))
def test_valid_crafted_equal_pillow(name):
    Image = pytest.importorskip("PIL.Image")
    d = VALID[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = np.asarray(Image.open(io.BytesIO(d)).convert("RGB"))
    st = png.decode_stages(d)
    assert np.array_equal(st["rgb"], want)
    assert st["stats"].tolist() == [png.STATUS_OK, st["info"].raw_bytes, 0]
    stream = png.gather(d, st["info"])
    assert png.inflate_restated(stream, st["info"].raw_bytes) == (st["raw"], png.STATUS_OK)


@pytest.mark.parametrize("name", sorted(CORRUPT))
def test_corrupt_streams_end_as_documented(name):
    d, status = CORRUPT[name]
    st = png.decode_stages(d)
    info = st["info"]
    assert st["stats"][0] == status and st["stats"][1] == len(st["raw"])
    assert len(st["raw"]) < info.raw_bytes or status == png.STATUS_OK
    # the rest of the scanlines are zero, then unfiltered and converted as any others
    padded = st["raw"] + bytes(info.raw_bytes - len(st["raw"]))
    rows, _ = png.unfilter(padded, info)
    assert np.array_equal(st["rows"], rows) and np.array_equal(st["rgb"], png.to_rgb(rows, info))
    # what follows the fault is never read: junk appended to the stream changes nothing
    if status not in (png.STATUS_OK, png.STATUS_SHORT, png.STATUS_EXHAUSTED):
        stream = png.gather(d, info)
        got = png.inflate_restated(stream + bytes(range(256)) * 4, info.raw_bytes)
        assert got == (st["raw"], status)


def test_unknown_filter_types_unfilter_as_none():
    d, _ = CORRUPT["unknown_filter"]
    st = png.decode_stages(d)
    assert st["stats"].tolist() == [png.STATUS_OK, 60, 2]
    assert st["rows"][0].tolist() == list(range(0, 19))               # type 7: None
    assert st["rows"][2].tolist() == list(range(2, 21))               # type 200: None


def test_adversarial_file_is_accepted_and_produces_nothing():
    d = PC.adversarial(20000)
    info = png.parse(d)
    st = png.decode_stages(d)
    assert (info.h, info.w) == (1, 1) and st["stats"].tolist() == [png.STATUS_SHORT, 0, 0]
