"""The wgmma convolution paths the product runs, each against the fp64 oracle and bit for bit against each other.

* tile geometry that ResNet50 never produces (asymmetric padding, non-square kernels) through every executor of
  `defer_k_conv` (the square cases are in tests/test_gpu_kernels.py::RESNET_SHAPES);
* the tensor-core RGB stem at stage level: the fused `conv_stem_kernel` (patch rows built in shared memory by the
  producer warpgroup), and `stem_im2col_kernel` feeding the streaming, persistent-grid and one-tile-per-CTA kernels;
* `conv_mega_kernel` walking a conv block + identity block in one cluster launch, against the per-op kernels;
* the configuration bench.py measures (ResNet50, fp32 parity, 32 images per launch), per image against batch 1;
* programmatic dependent launch (DEFER_PDL=1), which is read once per process, in a subprocess.

Executors that share the K order of every output must agree bitwise; each must also pass the oracle check of
tests/conv_check.py (global and per-channel error) on the operands it actually read."""
import os
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from conv_check import ConvCase, _quantise, assert_conv, check_executors, conv_oracle
from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200 import keras_like as K
from defer_b200.node import DTYPE_TO_FMT, StageRunner

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

TESTS = Path(__file__).resolve().parent
ROOT = TESTS.parent

# every knob that selects an executor; each run below starts from none of them set
KNOBS = ("DEFER_STREAM", "DEFER_STREAM_MIN_TILES", "DEFER_STREAM_BN", "DEFER_PERSIST_MIN_TILES", "DEFER_STEM_FUSED",
         "DEFER_TC_STEM", "DEFER_UMMA_BN", "DEFER_UMMA_SPLITK", "DEFER_UMMA_CLUSTER", "DEFER_UMMA_FORCE_SPLITS",
         "DEFER_UMMA_STAGES", "DEFER_MEGA", "DEFER_MEGA_STAGES")


def _knobs(monkeypatch, **env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


@pytest.fixture(scope="module")
def torch_cuda():
    lib = A.load()          # sets CUDA_DEVICE_MAX_CONNECTIONS before torch touches CUDA
    import torch
    assert torch.cuda.is_available()
    return torch, lib


def _fmt_name(dtype):
    return {A.FMT_BF16X2: "bf16x2", A.FMT_BF16: "bf16"}[DTYPE_TO_FMT[dtype]]


# ------------------------------------------------------------------------------------------------ 1. tile geometry
GEOMETRY = [
    # n, h, w, cin, cout, kh, kw, sh, sw, pad t, l, b, r
    (2, 56, 56, 64, 64, 3, 3, 2, 2, 0, 0, 1, 1),        # TF 'same' at stride 2: all padding after
    (1, 17, 17, 128, 128, 1, 7, 1, 1, 0, 3, 0, 3),      # 1x7: tap -> (tap / kw, tap % kw)
    (1, 17, 17, 128, 128, 7, 1, 1, 1, 3, 0, 3, 0),      # 7x1
    (1, 28, 28, 128, 128, 1, 1, 1, 1, 1, 1, 0, 0),      # 1x1 with top-left padding: the flat [M, C] view must not be used
]


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("geom", GEOMETRY, ids=lambda g: "x".join(map(str, g)))
def test_conv_geometry_every_executor(torch_cuda, fmt_name, geom, monkeypatch):
    torch, lib = torch_cuda
    i = GEOMETRY.index(geom)
    _knobs(monkeypatch)
    check_executors(torch, lib, ConvCase(fmt_name, geom, i % 2 == 0, True, seed=40 + i), monkeypatch)
    # no residual, and a null scale (and every other case a null shift): the epilogue's absent operands
    check_executors(torch, lib, ConvCase(fmt_name, geom, i % 2 == 1, False, seed=50 + i, scale=False, shift=i % 2 == 0),
                    monkeypatch)


# ------------------------------------------------------------------------------------------------ 2. the RGB stem
def _stem_model(h, w, cin, cout, k, s, pad, seed):
    """Input -> [ZeroPadding2D] -> Conv2D -> BatchNormalization -> ReLU; `pad` = 'same' or ((t, b), (l, r))."""
    K.clear_session()
    inp = K.Input(shape=(h, w, cin))
    x = inp if pad == "same" else K.ZeroPadding2D(pad, name="pad")(inp)
    x = K.Conv2D(cout, (k, k), strides=(s, s), padding="same" if pad == "same" else "valid", name="conv")(x)
    x = K.BatchNormalization(name="bn")(x)
    x = K.Activation("relu", name="relu")(x)
    m = K.Model(inp, x, name="stem")
    applications.synthetic_weights(m, seed=seed)
    return m


STEMS = {
    # batch, h, w, cin, cout, k, s, padding
    "resnet_b1": (1, 224, 224, 3, 64, 7, 2, ((3, 3), (3, 3))),
    "resnet_b3": (3, 224, 224, 3, 64, 7, 2, ((3, 3), (3, 3))),
    "vgg": (1, 224, 224, 3, 64, 3, 1, "same"),
    "straddle": (3, 61, 47, 3, 64, 7, 2, ((3, 2), (1, 4))),     # 30 x 23 outputs per image: tiles straddle images
    "cin1_5x5": (2, 40, 36, 1, 64, 5, 1, "same"),
    "cin4_k256": (2, 64, 64, 4, 64, 8, 2, "same"),              # K = 8 * 8 * 4 = 256, the limit
    "wide": (1, 16, 600, 3, 64, 7, 2, ((3, 3), (3, 3))),        # im2col stages 7 rows of 1800 floats: > 48 KB
    "cout128": (2, 64, 64, 3, 128, 7, 2, ((3, 3), (3, 3))),     # C_out != 64: never fused
}

# executor -> (kernel of the stem op, knobs)
STEM_PATHS = {
    "fused": ("conv_stem_kernel", {"DEFER_STREAM_MIN_TILES": 1}),
    "im2col_stream": ("stem_im2col+conv_stream_kernel", {"DEFER_STEM_FUSED": 0, "DEFER_STREAM_MIN_TILES": 1}),
    "im2col_grid": ("stem_im2col+conv_mega_kernel(grid)", {"DEFER_STREAM": 0, "DEFER_PERSIST_MIN_TILES": 1}),
    "im2col_per_cta": ("stem_im2col+conv_umma_kernel", {"DEFER_STREAM_MIN_TILES": 10 ** 9, "DEFER_UMMA_BN": 64}),
}


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("name", list(STEMS))
def test_stem_paths(name, dtype, monkeypatch):
    b, h, w, cin, cout, k, s, pad = STEMS[name]
    fmt_name = _fmt_name(dtype)
    m = _stem_model(h, w, cin, cout, k, s, pad, seed=len(name))
    x = applications.synthetic_input(b, (h, w, cin), seed=len(name))
    outs, ref = {}, {}
    for path, (kernel, env) in list(STEM_PATHS.items()) + [("simt", ("conv_simt_kernel", {}))]:
        _knobs(monkeypatch, **env)
        r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=b, depth=1, conv_backend=1 if path == "simt" else 0)
        try:
            if kernel == "conv_stem_kernel" and cout != 64:
                kernel = "stem_im2col+conv_stream_kernel"
            assert r.op_info(0)["kernel"] == kernel, (path, r.describe())
            r.predict(x)
            outs[path] = y = r.read_layer("relu")
            if not ref:
                op, W = r.plan.ops[0], r.plan.weights
                args = (W[op.w_scale], W[op.w_shift], None, (op.sh, op.sw), op.pads, True)
                ref["tc"] = conv_oracle(_quantise(x, DTYPE_TO_FMT[dtype]), _quantise(W[op.w_kernel], DTYPE_TO_FMT[dtype]), *args)
                ref["simt"] = conv_oracle(x, W[op.w_kernel], *args)
            assert_conv(y, ref["simt" if path == "simt" else "tc"], fmt_name, (name, path))
        finally:
            r.close()
    # same A operand bits (in-kernel patch rows or the im2col matrix) and the same K order on every tensor-core path
    for path in STEM_PATHS:
        assert np.array_equal(outs[path], outs["fused"]), (name, dtype, path)


# ------------------------------------------------------------------------------------------------ 3. megakernel chains
CHAINS = {
    # output spatial: (input channels, bottleneck filters, stride of the conv block, layer in front of the first conv)
    56: (64, (64, 64, 256), 1, "bn"),
    28: (256, (128, 128, 512), 2, "relu"),
    14: (512, (256, 256, 1024), 2, "bn"),
    7: (1024, (512, 512, 2048), 2, "relu"),
}


def _chain_model(spatial, seed=5):
    """[BatchNormalization | ReLU] -> conv block (projection shortcut) -> identity block.  The stage input is fp32 and a
    conv reading it runs on SIMT; the standalone op in front makes every conv of the chain read bf16 planes."""
    cin, filters, stride, head = CHAINS[spatial]
    hin = spatial * stride
    K.clear_session()
    inp = K.Input(shape=(hin, hin, cin))
    x = K.BatchNormalization(name="bn_in")(inp) if head == "bn" else K.Activation("relu", name="relu_in")(inp)
    x = applications._conv_block(x, 3, list(filters), 2, "a", strides=(stride, stride))
    x = applications._identity_block(x, 3, list(filters), 2, "b")
    m = K.Model(inp, x, name="chain")
    applications.synthetic_weights(m, seed=seed)
    return m


def _run_all_buffers(m, x, dtype, **kw):
    """Every buffer of a one-stage run (decoded to fp32) and the runner's describe() / plan."""
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=x.shape[0], depth=1, **kw)
    try:
        r.predict(x)
        return [r.read_buffer(i) for i in range(len(r.plan.bufs))], r.describe(), r.plan
    finally:
        r.close()


def _check_convs_against_oracle(plan, bufs, dtype, what):
    """Each conv of the plan against the fp64 oracle, fed exactly the (decoded) buffers the kernel read."""
    fmt = DTYPE_TO_FMT[dtype]
    W = plan.weights
    for op in plan.ops:
        if op.kind != A.OP_CONV or plan.bufs[op.in0][3] != A.BUF_ACT:
            continue
        res = bufs[op.in1] if op.flags & A.FLAG_RESIDUAL else None
        ref = conv_oracle(bufs[op.in0], _quantise(W[op.w_kernel], fmt), W[op.w_scale], W[op.w_shift], res,
                          (op.sh, op.sw), op.pads, bool(op.flags & A.FLAG_RELU))
        assert_conv(bufs[op.out], ref, _fmt_name(dtype), (what, op.layers))


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("spatial", list(CHAINS))
def test_megakernel_chain_matches_per_op_kernels(spatial, batch, dtype, monkeypatch):
    m = _chain_model(spatial)
    cin, _, stride, _ = CHAINS[spatial]
    x = applications.synthetic_input(batch, (spatial * stride, spatial * stride, cin), seed=spatial + batch)
    runs = {}
    for name, env in (("per_op", {"DEFER_MEGA": 0}), ("mega", {"DEFER_MEGA": 1}),
                      ("mega_ring2", {"DEFER_MEGA": 1, "DEFER_MEGA_STAGES": 2})):
        _knobs(monkeypatch, DEFER_UMMA_SPLITK=0, **env)
        bufs, desc, plan = runs[name] = _run_all_buffers(m, x, dtype)
        n_conv = sum(op.kind == A.OP_CONV for op in plan.ops)
        assert n_conv == 7
        assert ("megakernel group: ops" in desc) == (name != "per_op"), desc
        if name != "per_op":
            first, last = map(int, re.search(r"megakernel group: ops (\d+)\.\.(\d+)", desc).groups())
            assert last - first + 1 == n_conv, desc
        _check_convs_against_oracle(plan, bufs, dtype, name)
    for name in ("mega", "mega_ring2"):
        for i, (a, b) in enumerate(zip(runs[name][0], runs["per_op"][0])):
            assert np.array_equal(a, b), (name, "buffer", i, runs["per_op"][2].describe())


# ------------------------------------------------------------------------------------------------ 4. the benchmark
def test_benchmarked_configuration_per_image(resnet50, monkeypatch):
    """bench.py's single-GPU workload: ResNet50, fp32 parity, 32 images per launch.  The plan is the one the bench
    runs; the stem output and the pooled features of an image do not depend on its position in the microbatch (bitwise
    against a batch-1 run: the K order of a conv does not depend on the batch, the pooling reduces per image)."""
    from oracle import keras_ref
    _knobs(monkeypatch, DEFER_UMMA_SPLITK=0)
    x = applications.synthetic_input(32, seed=23)
    r = StageRunner.from_model(resnet50, device=0, dtype="float32", max_batch=32, depth=1)
    try:
        y = r.predict(x)
        kernels = [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))]
        convs = [i for i, op in enumerate(r.plan.ops) if op.kind == A.OP_CONV]
        assert kernels[convs[0]] == "conv_stem_kernel", kernels
        assert all(kernels[i] == "conv_stream_kernel" for i in convs[1:]), kernels
        bns = [int(v) for v in re.findall(r"wgmma tiles: .*\(BN (\d+)\)", r.describe())]
        assert bns == [128 if r.plan.bufs[r.plan.ops[i].out][2] % 128 == 0 else 64 for i in convs], bns
        act32, gap32 = r.read_layer("activation"), r.read_layer("avg_pool")
    finally:
        r.close()
    r1 = StageRunner.from_model(resnet50, device=0, dtype="float32", max_batch=1, depth=1)
    try:
        assert r1.op_info(convs[0])["kernel"] == "conv_stem_kernel"
        for p in (0, 1, 16, 31):
            r1.predict(x[p:p + 1])
            assert np.array_equal(r1.read_layer("activation")[0], act32[p]), p
            assert np.array_equal(r1.read_layer("avg_pool")[0], gap32[p]), p
    finally:
        r1.close()
    ref = keras_ref.predict(resnet50.to_json(), resnet50.get_weights(), x[[0, 31]])
    for j, p in enumerate((0, 31)):
        assert keras_ref.rel_err(y[p], ref[j]) <= 1e-3, p


# ------------------------------------------------------------------------------------------------ 5. DEFER_PDL
def _pdl_model():
    """The RGB stem, the max-pool and the first conv + identity block of ResNet50 (seeded, fresh names)."""
    K.clear_session()
    inp = K.Input(shape=(224, 224, 3))
    x = K.ZeroPadding2D((3, 3), name="conv1_pad")(inp)
    x = K.Conv2D(64, (7, 7), strides=(2, 2), name="conv1")(x)
    x = K.BatchNormalization(name="bn_conv1")(x)
    x = K.Activation("relu")(x)
    x = K.ZeroPadding2D((1, 1), name="pool1_pad")(x)
    x = K.MaxPooling2D((3, 3), strides=(2, 2))(x)
    x = applications._conv_block(x, 3, [64, 64, 256], 2, "a", strides=(1, 1))
    x = applications._identity_block(x, 3, [64, 64, 256], 2, "b")
    m = K.Model(inp, x, name="pdl")
    applications.synthetic_weights(m, seed=9)
    return m


def run_pdl_stages(out_dir):
    """Every buffer of the _pdl_model stage at batch 1 and 8, saved under `out_dir` (also run in a subprocess)."""
    out_dir = Path(out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    m = _pdl_model()
    for b in (1, 8):
        bufs, _, _ = _run_all_buffers(m, applications.synthetic_input(b, seed=b), "float32")
        np.savez(out_dir / f"batch{b}.npz", *bufs)


def test_pdl_launches_match_default(tmp_path, monkeypatch):
    """DEFER_PDL=1 (programmatic dependent launch of the conv kernels) is read once per process: run it in a child
    process and require the same bits as the default launches here."""
    _knobs(monkeypatch)
    monkeypatch.delenv("DEFER_PDL", raising=False)
    code = (f"import sys; sys.path[:0] = [{str(TESTS)!r}, {str(ROOT)!r}]; import test_gpu_conv_paths as T; "
            f"T.run_pdl_stages({str(tmp_path / 'pdl')!r})")
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env["DEFER_PDL"] = "1"
    p = subprocess.run([sys.executable, "-c", code], env=env, cwd=str(ROOT), capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    run_pdl_stages(tmp_path / "default")
    for b in (1, 8):
        got, want = np.load(tmp_path / "pdl" / f"batch{b}.npz"), np.load(tmp_path / "default" / f"batch{b}.npz")
        assert got.files == want.files
        for f in want.files:
            assert np.array_equal(got[f], want[f]), (b, f)
