"""TMA im2col A tiles of the wgmma convolution on geometries the applications do not run, bit for bit.

The tiles are 128 consecutive output pixels, loaded with one im2col TMA load per tap and 64-channel block
(tests/test_im2col_host.py restates what each row holds).  The geometries of tests/test_im2col_host.py::IM2COL_EDGES
reach what ResNet, VGG and the other wgmma tests do not: tiles that straddle images with a ragged last tile, a tile over
three images, stride 2 over an odd input, an asymmetric ZeroPadding2D (a 1x1 conv among them), a row of 151 outputs over
301 input columns, and a bounding box whose W and H corners differ.  Each runs on exactly summable operands
(tests/exact_conv.py) through the one-tile, split-K, cluster split-K, persistent-grid and streaming executors, in BF16X2
and BF16."""
import pytest

import exact_conv as X
from test_gpu_conv_exact import EXECUTORS, FAMS, _knobs, run_bits, torch_cuda  # noqa: F401
from test_im2col_host import IM2COL_EDGES

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

RUN = ("one_tile", "split_k3", "cluster2_bn64", "cluster8_bn128", "grid", "stream64", "stream128")


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("name", list(IM2COL_EDGES))
def test_im2col_edges_exact(torch_cuda, name, fmt_name, monkeypatch):  # noqa: F811
    torch, lib = torch_cuda
    i = list(IM2COL_EDGES).index(name)
    g = IM2COL_EDGES[name]
    cases = [X.ExactCase(fmt_name, g, FAMS[i % 4], True, True, seed=7000 + i),
             X.ExactCase(fmt_name, g, FAMS[(i + 1) % 4], False, False, seed=7100 + i, shift=i % 2 == 0)]
    for case in cases:
        want = case.expected_bits("wgmma")
        for ex in RUN:
            backend, env = EXECUTORS[ex]
            _knobs(monkeypatch, **env)
            X.assert_bits(run_bits(torch, lib, case, backend), want, case.out_shape, fmt_name,
                          (name, case.family, ex, f"backend {backend}"))
