"""Crafted progressive files and the restatement of the device's per-scan decode (no GPU).

tests/jpeg_craft_progressive.py writes files under scan scripts Pillow cannot write: separate DC scans per component,
DC first at Al = 0, other spectral splits, refinement down from Al = 13, EOB runs over thousands of blocks in
one-component scans with and without restart intervals, restart intervals that change between scans, DHT / DRI / COM
and a redefining DQT between scans, and coefficients 10..63 never sent.  Each decodes to the coefficients the writer
knows, and to Pillow's pixels.  tests/jpeg_progressive_sync.py restates the device's decode; it equals the sequential
decoder, counters included, at subsequence sizes from 8 to 8192 bits, and its rounds stay small on encoder-made files."""
import io
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

from defer_b200 import jpeg  # noqa: E402
from jpeg_craft_progressive import corpus  # noqa: E402
from jpeg_progressive_check import corrupt_corpus, fixture, fixture_names  # noqa: E402
from jpeg_progressive_sync import sync_progressive  # noqa: E402

SBITS = int(re.search(r"#define DEFER_JPEG_SUBSEQ_BITS (\d+)", (ROOT / "include" / "defer_b200.h").read_text()).group(1))
CORPUS = corpus()


@pytest.mark.parametrize("case", CORPUS, ids=[c[0] for c in CORPUS])
def test_crafted_decodes_as_written_and_as_pillow(case):
    name, data, want = case
    st = jpeg.decode_stages(data)
    assert st["progress"]["scans"] == len(st["info"].scans)
    assert np.array_equal(st["coef"], want), name
    Image = pytest.importorskip("PIL.Image")
    assert np.array_equal(st["rgb"], np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))), name


def test_crafted_covers_the_script_features():
    info = {name: jpeg.parse(d) for name, d, _ in CORPUS}
    scans = [s for i in info.values() for s in i.scans]
    assert any(s.ss == 0 and s.ah == 0 and s.al == 0 and len(s.comps) == 1 for s in scans)    # DC first alone, Al 0
    assert any(s.ss == 0 and s.ah == 0 and s.al == 13 for s in scans)
    assert any(s.ss > 0 and s.restart for s in scans) and any(len({s.restart for s in i.scans}) > 2 for i in info.values())
    assert any(len(s.comps) == 1 and s.comps[0] > 0 and s.ss == 0 for s in scans)               # a chroma DC scan


@pytest.mark.parametrize("sbits", [8, 64, 1024, SBITS])
def test_sync_restatement_equals_sequential(sbits):
    cases = [(n, d) for n, d, _ in CORPUS] + [(n, fixture(n)) for n in fixture_names()] + corrupt_corpus(seed=0)
    for name, d in cases:
        if sbits < 64 and len(d) > 20000:
            continue
        coef, st = sync_progressive(d, sbits)
        want, pr = jpeg.progressive_decode(d)
        assert np.array_equal(coef, want), (name, sbits)
        assert [st[0], st[1], st[4], st[5]] == [pr["T"], pr["R"], pr["cutoff"], pr["scans"]], (name, sbits)


def test_rounds_stay_small_on_encoder_made_files():
    """At the device's subsequence size, each DC or AC first scan of a Pillow-written file takes at most 3 rounds (the
    counter sums them over the scans): a property of encoder-made files, not of every valid file."""
    for name in fixture_names():
        d = fixture(name)
        first = sum(1 for s in jpeg.parse(d).scans if s.ah == 0)
        assert sync_progressive(d, SBITS)[1][3] <= 3 * first, name
