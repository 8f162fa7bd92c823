"""The self-synchronising Huffman decode (tests/jpeg_check.py, as the GPU runs it) against the sequential decoder of
`jpeg.entropy_decode`, for several subsequence sizes, with and without restart intervals, on random entropy data and on
the corrupt files of the GPU tests; and its rounds at the device's subsequence size on encoder-made files: a few, however
long the file, so no thread decodes a whole file.  That bound holds for what encoders write, not for every valid file:
on a file whose every bit position decodes, the rounds are the most subsequences in one restart interval
(tests/test_jpeg_craft_host.py), and the GPU tests time that case."""
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from defer_b200 import jpeg  # noqa: E402
from jpeg_check import sync_decode  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "jpeg"
#: the device's subsequence size
SBITS = int(re.search(r"#define DEFER_JPEG_SUBSEQ_BITS (\d+)", (ROOT / "include" / "defer_b200.h").read_text()).group(1))
FILES = ["photo_17x33_420_q5.jpg", "photo_15x17_gray_q100.jpg", "photo_223x225_420_q75.jpg",
         "photo_223x225_444_q75_rb1.jpg", "photo_223x225_422_q90_rb4.jpg", "photo_223x225_gray_q50_rr1.jpg",
         "checker_31x47_420_q95.jpg", "photo_40x60_420_q75_meta.jpg"]


def _same(data, sbits):
    want, dec = jpeg.entropy_decode(data)
    got, gdec, rounds = sync_decode(data, sbits)
    assert np.array_equal(gdec, dec)
    assert np.array_equal(got, want)
    return rounds


@pytest.mark.parametrize("sbits", [8, 32, 257, 1024, 4096, 8192])
def test_sync_equals_sequential(sbits):
    rounds = {}
    for name in FILES:
        data = (GOLDEN / name).read_bytes()
        if sbits < 257 and len(data) > 20000:
            continue                      # Python is slow: the small sizes run on the small files
        rounds[name] = _same(data, sbits)
    print(f"sbits {sbits}: sync rounds {rounds}")
    assert all(r >= 1 for r in rounds.values())
    if sbits >= 4096:             # encoder-made files: longer than the distance a decoder needs to find the true path
        assert max(rounds.values()) <= 3, rounds


def _bounded(data, name):
    """An encoder-made file: its decoders resynchronise within a subsequence, so the rounds stay at 3 or fewer."""
    n_subs = -(-jpeg.parse(data).length * 8 // SBITS)
    rounds = _same(data, SBITS)
    print(f"{name}: {rounds} rounds for {n_subs} subsequences of {SBITS} bits")
    assert n_subs >= 8 and rounds <= 3, (name, rounds, n_subs)


@pytest.mark.parametrize("name", ["photo_480x640_420_q75.jpg", "photo_480x640_422_q90_rr1.jpg"])
def test_rounds_bounded_on_large_files(name):
    _bounded((GOLDEN / name).read_bytes(), name)


@pytest.mark.parametrize("seed", [0, 1])
def test_rounds_bounded_on_benchmark_files(seed):
    """The files tools/jpeg_bench.py times end to end (480x640, q90, 4:2:0)."""
    pytest.importorskip("PIL")
    sys.path.insert(0, str(ROOT / "tools"))
    from make_jpeg_fixtures import content, encode
    _bounded(encode(content("photo", 480, 640, seed=seed), "420", 90), f"jpeg_bench file {seed}")


def test_random_entropy_is_defined():
    from test_gpu_jpeg import random_entropy
    for i, name in enumerate(FILES[2:6]):
        data = random_entropy((GOLDEN / name).read_bytes(), seed=i)
        _same(data, 1024)
        st = jpeg.decode_stages(data)
        assert st["rgb"].shape == (st["info"].h, st["info"].w, 3)
        assert not st["coef"][~st["decoded"]].any()


def test_corrupt_corpus_is_defined():
    """The corrupt files of tests/test_gpu_jpeg_craft.py: each is accepted by the parser, and the restatement of the
    device decode equals the sequential decoder on it."""
    from test_gpu_jpeg_craft import corpus
    for name, data in corpus():
        want, dec = jpeg.entropy_decode(data)
        got, gdec, _ = sync_decode(data, SBITS)
        assert np.array_equal(gdec, dec), name
        assert np.array_equal(got, want), name
