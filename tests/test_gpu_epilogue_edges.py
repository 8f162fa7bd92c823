"""Row and column edges of the staged wgmma epilogue.

The epilogue stages a tile through shared memory 64 columns at a time (two passes at BN 128).  Each consumer thread then
stores 8 channels of the rows t / 8 + 32 k (k = 0..3) and skips rows outside the output.  The cases below reach what the
ResNet shapes do not: a last flat tile with 2 valid rows, so three of a thread's four rows and most threads' rows are
invalid in both passes; a single flat tile of 100 rows; and a 4-D tile of two images whose second image is past the
batch.  The last of these also runs cluster split-K at 2 and 8 CTAs per tile, where each CTA stages and stores only the
column groups it reduced: one group per pass at 8."""
import pytest

from conv_check import ConvCase, assert_conv, check_executors
from defer_b200 import _cabi as A

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

KNOBS = ("DEFER_STREAM", "DEFER_STREAM_MIN_TILES", "DEFER_STREAM_BN", "DEFER_PERSIST_MIN_TILES", "DEFER_UMMA_BN",
         "DEFER_UMMA_SPLITK", "DEFER_UMMA_CLUSTER", "DEFER_UMMA_FORCE_SPLITS", "DEFER_UMMA_FORCE_CSPLIT",
         "DEFER_UMMA_STAGES", "DEFER_MEGA", "DEFER_MEGA_STAGES")

EDGES = {
    # n, h, w, cin, cout, kh, kw, sh, sw, pad t, l, b, r
    "flat_last_tile_2_rows": (1, 10, 13, 64, 256, 1, 1, 1, 1, 0, 0, 0, 0),   # M = 130
    "flat_one_tile_100_rows": (1, 10, 10, 64, 128, 1, 1, 1, 1, 0, 0, 0, 0),
    "tile_n_past_batch": (3, 7, 7, 64, 128, 3, 3, 1, 1, 1, 1, 1, 1),         # 2 x 49 rows per tile, 3 images
}


def _knobs(monkeypatch, **env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


@pytest.fixture(scope="module")
def torch_cuda():
    lib = A.load()
    import torch
    assert torch.cuda.is_available()
    return torch, lib


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("name", list(EDGES))
def test_epilogue_row_edges_every_executor(torch_cuda, fmt_name, name, monkeypatch):
    torch, lib = torch_cuda
    geom = EDGES[name]
    i = list(EDGES).index(name)
    _knobs(monkeypatch)
    check_executors(torch, lib, ConvCase(fmt_name, geom, True, True, seed=70 + i), monkeypatch)
    check_executors(torch, lib, ConvCase(fmt_name, geom, False, False, seed=80 + i, shift=False), monkeypatch)


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("csplit", [2, 8])
def test_cluster_splitk_ragged_tile(torch_cuda, fmt_name, csplit, monkeypatch):
    torch, lib = torch_cuda
    case = ConvCase(fmt_name, EDGES["tile_n_past_batch"], True, True, seed=90 + csplit)
    _knobs(monkeypatch, DEFER_UMMA_CLUSTER=1, DEFER_UMMA_FORCE_CSPLIT=csplit)
    assert_conv(case.run(torch, lib, 2), case.ref, fmt_name, ("cluster split-K", csplit))
