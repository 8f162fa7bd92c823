"""Every convolution executor bit for bit against exact expected bits (tests/exact_conv.py).

The operands are exactly summable (every fp32 partial sum of every output is exact, asserted on the host before each
run), so the accumulator is known whatever the K order, split or reduction, and the epilogue is replayed in fp32 as
each kernel documents it.  One wrong term, tap, plane, split partial or epilogue operation anywhere changes the bits:

* `defer_k_conv` wgmma backends: 2 one tile per CTA, its default plan, forced split-K 2 / 3, cluster split-K at 2 / 4 / 8
  CTAs x BN 64 / 128; 3 persistent grid; 4 / 5 streaming BN 64 / 128; 6 / 7 the same planned for a peer's slot - on the
  shape lists of the other convolution tests, BF16X2 and BF16, with and without residual / ReLU / scale / shift;
* operand-ring depths DEFER_UMMA_STAGES, DEFER_STREAM_STAGES and DEFER_PERSIST_STAGES from 2 to the clamp;
* `conv_simt_kernel` in F32, BF16X2 and BF16 (vector and scalar A / B loads and epilogue) and `stem7x7s2_kernel`;
* at stage level: the RGB stems on every path, the megakernel chains at DEFER_MEGA 0 / 1 and DEFER_MEGA_CLUSTER 2 / 4
  (read once per process: in a subprocess), and a conv with a folded affine op (DEFER_FOLD_AFFINE=1).

The module (191 tests) takes 195 s on an H100 80GB HBM3 at a 700 W power limit."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import exact_conv as X
from conv_check import FMTS, _alloc_act, _encode, _ptr
from defer_b200 import _cabi as A
from defer_b200 import keras_like as K
from defer_b200.node import DTYPE_TO_FMT, StageRunner
from test_gpu_conv_paths import CHAINS, GEOMETRY, STEM_PATHS, STEMS, _chain_model, _stem_model
from test_gpu_epilogue_edges import EDGES
from test_gpu_fold_affine import _fold_model
from test_gpu_kernels import RESNET_SHAPES, STREAM_SHAPES

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

TESTS = Path(__file__).resolve().parent
ROOT = TESTS.parent
FAMS = list(X.FAMILIES)

KNOBS = ("DEFER_STREAM", "DEFER_STREAM_MIN_TILES", "DEFER_STREAM_BN", "DEFER_STREAM_STAGES", "DEFER_PERSIST_MIN_TILES",
         "DEFER_PERSIST_STAGES", "DEFER_STEM_FUSED", "DEFER_TC_STEM", "DEFER_UMMA_BN", "DEFER_UMMA_SPLITK",
         "DEFER_UMMA_CLUSTER", "DEFER_UMMA_FORCE_SPLITS", "DEFER_UMMA_FORCE_CSPLIT", "DEFER_UMMA_STAGES", "DEFER_MEGA",
         "DEFER_MEGA_STAGES", "DEFER_MEGA_CLUSTER", "DEFER_FOLD_AFFINE")


def _knobs(monkeypatch, **env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


def _geom(s):
    n, h, w, cin, cout, k, st, pad = s
    return (n, h, w, cin, cout, k, k, st, st, pad, pad, pad, pad)


# ------------------------------------------------------------------------------------------------ the case matrix
# every wgmma shape of the suite: name -> geometry (n, h, w, cin, cout, kh, kw, sh, sw, pad t, l, b, r)
WGMMA_SHAPES = {**{f"resnet{i}": _geom(s) for i, s in enumerate(RESNET_SHAPES)},
                **{f"stream{i}": _geom(s) for i, s in enumerate(STREAM_SHAPES)},
                **{f"geometry{i}": g for i, g in enumerate(GEOMETRY)}, **EDGES}

# conv_simt_kernel: GEOMETRY, the shapes test_conv_simt_shapes runs, and the scalar paths (C_in % 4 != 0: per-element A
# loads; C_out % 4 != 0: per-element B loads and epilogue; a C_out tail past the last 64-column block)
SIMT_SHAPES = {**{f"geometry{i}": g for i, g in enumerate(GEOMETRY)},
               **{f"simt{i}": _geom(s) for i, s in enumerate(RESNET_SHAPES[:8] + [(1, 230, 230, 3, 64, 7, 2, 0),
                                                                                (2, 9, 11, 8, 12, 3, 2, 1)])},
               "cin6": (2, 9, 11, 6, 12, 3, 3, 2, 2, 1, 1, 1, 1), "cout13": (1, 10, 10, 8, 13, 3, 3, 1, 1, 1, 1, 1, 1),
               "cin5_cout70": (2, 7, 9, 5, 70, 3, 3, 1, 1, 1, 0, 1, 2)}

# stem7x7s2_kernel (fp32 image, 7x7/2, 3 -> 64): 31 x 31 and 20 x 27 outputs, not multiples of its 8 x 8 tile
STEM_SHAPES = {"stem61": (2, 61, 61, 3, 64, 7, 7, 2, 2, 3, 3, 3, 3), "stem40x53": (1, 40, 53, 3, 64, 7, 7, 2, 2, 3, 2, 2, 3)}

# two shapes whose K loop (36 and 32 k-blocks) is longer than any ring
RING_SHAPES = {"resnet20": _geom(RESNET_SHAPES[20]), "stream8": _geom(STREAM_SHAPES[8])}


def wgmma_cases(name, fmt_name):
    """Two cases per shape: residual with ReLU on every other shape; no residual, no scale and every other shape no
    shift.  The families rotate over the shapes, so each family meets every executor."""
    i = list(WGMMA_SHAPES).index(name)
    g = WGMMA_SHAPES[name]
    return [X.ExactCase(fmt_name, g, FAMS[i % 4], i % 2 == 0, True, seed=1000 + i),
            X.ExactCase(fmt_name, g, FAMS[(i + 1) % 4], i % 2 == 1, False, seed=2000 + i, scale=False, shift=i % 2 == 0)]


def ring_cases(name, fmt_name):
    g = RING_SHAPES[name]
    j = list(RING_SHAPES).index(name)
    return [X.ExactCase(fmt_name, g, FAMS[(2 * j + f) % 4], True, True, seed=3000 + 10 * j + f) for f in (0, 1)]


def simt_cases(name, fmt_name):
    i = list(SIMT_SHAPES).index(name)
    g = SIMT_SHAPES[name]
    return [X.ExactCase(fmt_name, g, FAMS[i % 4], i % 2 == 0, True, seed=4000 + i),
            X.ExactCase(fmt_name, g, FAMS[(i + 2) % 4], i % 2 == 1, False, seed=5000 + i, scale=i % 3 != 0,
                        shift=i % 2 == 0)]


def stem_cases(name, fmt_name):
    i = list(STEM_SHAPES).index(name)
    g = STEM_SHAPES[name]
    return [X.ExactCase(fmt_name, g, FAMS[(i + f) % 4], relu, False, seed=6000 + 10 * i + f, scale=f == 0)
            for f, relu in ((0, True), (1, False))]


# ------------------------------------------------------------------------------------------------ defer_k_conv
@pytest.fixture(scope="module")
def torch_cuda():
    lib = A.load()
    import torch
    assert torch.cuda.is_available()
    return torch, lib


def run_bits(torch, lib, case, backend, x_is_f32=False):
    """The raw output words of one defer_k_conv run of `case` on `backend`."""
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = case.geom
    fmt = FMTS[case.fmt_name]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda() if a is not None else None   # noqa: E731
    xd = dev(case.x) if x_is_f32 else _encode(torch, lib, case.x, fmt)
    rd = _encode(torch, lib, case.res, fmt) if case.res is not None else None
    wd, sd, fd = dev(case.wk), dev(case.scale), dev(case.shift)
    yd = _alloc_act(torch, fmt, n * case.ho * case.wo * cout)
    A.check(lib.defer_k_conv(fmt, backend, _ptr(xd), int(x_is_f32), _ptr(wd), _ptr(sd), _ptr(fd), _ptr(rd), _ptr(yd),
                             n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr, A.FLAG_RELU if case.relu else 0, None))
    torch.cuda.synchronize()
    return X.raw_bits(torch, yd, case.fmt_name)


# executor -> (backend, knobs)
EXECUTORS = {
    "one_tile": (2, {"DEFER_UMMA_SPLITK": 0}),
    "default_plan": (2, {}),
    "split_k2": (2, {"DEFER_UMMA_FORCE_SPLITS": 2}),
    "split_k3": (2, {"DEFER_UMMA_FORCE_SPLITS": 3}),
    **{f"cluster{c}_bn{bn}": (2, {"DEFER_UMMA_CLUSTER": 1, "DEFER_UMMA_FORCE_CSPLIT": c, "DEFER_UMMA_BN": bn})
       for c in (2, 4, 8) for bn in (64, 128)},
    "grid": (3, {}),
    "stream64": (4, {}),
    "stream128": (5, {}),
    "peer64": (6, {}),
    "peer128": (7, {}),
}


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("name", list(WGMMA_SHAPES))
def test_wgmma_executors_exact(torch_cuda, name, fmt_name, monkeypatch):
    torch, lib = torch_cuda
    for case in wgmma_cases(name, fmt_name):
        want = case.expected_bits("wgmma")
        for ex, (backend, env) in EXECUTORS.items():
            _knobs(monkeypatch, **env)
            X.assert_bits(run_bits(torch, lib, case, backend), want, case.out_shape, fmt_name,
                          (name, case.family, ex, f"backend {backend}"))


def _ring_settings(fmt_name):
    """(executor, backend, knobs) of every ring depth from 2 to the clamp of each persistent kernel (BF16X2: 4 stages at
    BN 64, 3 at BN 128; BF16: 8 and 6) and of the one-tile kernel at 2 and 8."""
    clamp = {("bf16x2", 64): 4, ("bf16x2", 128): 3, ("bf16", 64): 8, ("bf16", 128): 6}
    out = [(f"umma_stages{s}", 2, {"DEFER_UMMA_SPLITK": 0, "DEFER_UMMA_STAGES": s}) for s in (2, 8)]
    out += [(f"persist_stages{s}", 3, {"DEFER_PERSIST_STAGES": s}) for s in range(2, clamp[(fmt_name, 64)] + 1)]
    for backend, bn in ((4, 64), (5, 128)):
        out += [(f"stream{bn}_stages{s}", backend, {"DEFER_STREAM_STAGES": s}) for s in range(2, clamp[(fmt_name, bn)] + 1)]
    return out


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("name", list(RING_SHAPES))
def test_ring_depths_exact(torch_cuda, name, fmt_name, monkeypatch):
    torch, lib = torch_cuda
    for case in ring_cases(name, fmt_name):
        want = case.expected_bits("wgmma")
        for ex, backend, env in _ring_settings(fmt_name):
            _knobs(monkeypatch, **env)
            X.assert_bits(run_bits(torch, lib, case, backend), want, case.out_shape, fmt_name, (name, case.family, ex))


@pytest.mark.parametrize("fmt_name", ["f32", "bf16x2", "bf16"])
@pytest.mark.parametrize("name", list(SIMT_SHAPES))
def test_simt_conv_exact(torch_cuda, name, fmt_name):
    torch, lib = torch_cuda
    for case in simt_cases(name, fmt_name):
        X.assert_bits(run_bits(torch, lib, case, 1), case.expected_bits("simt"), case.out_shape, fmt_name,
                      (name, case.family, "conv_simt_kernel"))


@pytest.mark.parametrize("fmt_name", ["f32", "bf16x2", "bf16"])
@pytest.mark.parametrize("name", list(STEM_SHAPES))
def test_stem7x7s2_exact(torch_cuda, name, fmt_name, monkeypatch):
    torch, lib = torch_cuda
    monkeypatch.delenv("DEFER_NO_STEM_KERNEL", raising=False)
    for case in stem_cases(name, fmt_name):
        X.assert_bits(run_bits(torch, lib, case, 1, x_is_f32=True), case.expected_bits("stem"), case.out_shape, fmt_name,
                      (name, case.family, "stem7x7s2_kernel"))


# ------------------------------------------------------------------------------------------------ stage level
def _fmt_name(dtype):
    return {A.FMT_BF16X2: "bf16x2", A.FMT_BF16: "bf16"}[DTYPE_TO_FMT[dtype]]


def exact_weights(model, seed, nnz=None, split_w=False, x_mean=4.0):
    """Weights a stage can chain exactly: conv kernels of small integers (times 2^EXP_W with `split_w`, half of them
    with a lo plane), sparse - `nnz` expected non-zeros per output channel, or the density that puts the expected
    sum|terms| / g at TARGET for inputs of mean |x_mean| - and zero bias; BN with gamma = 2^-1, beta on a 2^-2 grid, mean
    0 and variance 1 - eps, so the folded scale is exactly 2^-1 and the folded shift is beta."""
    rng = np.random.default_rng(seed)
    for layer, _ in model.iter_nodes():
        if isinstance(layer, K.Conv2D):
            kh, kw = layer.kernel_size
            shape = (kh, kw, layer.in_channels, layer.filters)
            k = kh * kw * layer.in_channels
            if nnz is not None:
                wk = X.values(rng, shape, False, min(1.0, nnz / k), 0)
                wk = np.sign(wk)                                    # +-1: the magnitudes do not grow along the chain
            else:
                m = X.MEAN_SPLIT if split_w else X.MEAN_SMALL
                wk = X.values(rng, shape, split_w, min(1.0, X.TARGET / (k * x_mean * m)), X.EXP_W)
            w = [wk.astype(np.float32)]
            if layer.use_bias:
                w.append(np.zeros(layer.filters, np.float32))
            layer.set_weights(w)
        elif isinstance(layer, K.BatchNormalization):
            c = layer.get_weights()[0].shape[0]
            layer.set_weights([np.full(c, 0.5, np.float32), (rng.integers(-4, 5, c) * 0.25).astype(np.float32),
                               np.zeros(c, np.float32), np.full(c, 1.0 - layer.epsilon, np.float32)])


def assert_exact_plan_weights(plan):
    """The folded scale of every conv / affine op is exactly 2^-1 (1 for a conv without a BN), the shift on a 2^-2 grid."""
    W = plan.weights
    for op in plan.ops:
        if op.kind in (A.OP_CONV, A.OP_AFFINE) and op.w_scale >= 0:
            sc = W[op.w_scale]
            assert np.all(sc == np.float32(0.5)) or np.all(sc == np.float32(1)), (op.layers, sc[:8])
        if op.kind in (A.OP_CONV, A.OP_AFFINE) and op.w_shift >= 0:
            assert np.all(W[op.w_shift] * 4 == np.round(W[op.w_shift] * 4)), (op.layers, W[op.w_shift][:8])


def _opt(W, i):
    return W[i] if i >= 0 else None


def expected_conv_out(plan, op, bufs, fmt_name, kind):
    """Expected stored value (float32, as decoded) of conv `op` fed the decoded buffers it read."""
    W = plan.weights
    x = bufs[op.in0]
    wk = W[op.w_kernel]
    kh, kw, cin, cout = wk.shape
    geom = (x.shape[0], x.shape[1], x.shape[2], cin, cout, kh, kw, op.sh, op.sw) + tuple(op.pads)
    pairs = X.product_pairs(x, wk, fmt_name if kind != "stem" else "f32", kind)
    X.assert_exactly_summable(pairs, geom, op.layers)
    res = bufs[op.in1] if op.flags & A.FLAG_RESIDUAL else None
    v = X.replay(X.exact_acc(pairs, geom), _opt(W, op.w_scale), _opt(W, op.w_shift), res, bool(op.flags & A.FLAG_RELU),
                 fmt_name, kind)
    return X.decode(v, fmt_name)


def _assert_equal(got, want, what):
    bad = np.argwhere(got != want)
    assert not bad.size, (what, f"{len(bad)} of {got.size} values differ; first at (n, h, w, c) = {tuple(bad[0])}: "
                                f"got {got[tuple(bad[0])]!r}, want {want[tuple(bad[0])]!r}")


def check_stage_convs(plan, bufs, dtype, what):
    """Each conv (and each affine op folded into one) against its exact expected result on the buffers it read."""
    fmt_name = _fmt_name(dtype)
    exp = {}
    n = 0
    for i, op in enumerate(plan.ops):
        if op.kind != A.OP_CONV or plan.bufs[op.in0][3] != A.BUF_ACT:
            continue
        exp[op.out] = want = expected_conv_out(plan, op, bufs, fmt_name, "wgmma")
        if not isinstance(bufs[op.out], str):
            _assert_equal(bufs[op.out], want, (what, i, op.layers))
        n += 1
    for i, op in enumerate(plan.ops):
        if op.kind == A.OP_AFFINE and op.in0 in exp:
            W = plan.weights
            u = X.replay_affine(exp[op.in0], W[op.w_scale], W[op.w_shift], bool(op.flags & A.FLAG_RELU))
            _assert_equal(bufs[op.out], X.decode(u, fmt_name), (what, i, op.layers, "folded affine"))
    return n


def _run_all_buffers(m, x, dtype):
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=x.shape[0], depth=1)
    try:
        r.predict(x)
        bufs = []
        for i in range(len(r.plan.bufs)):
            try:
                bufs.append(r.read_buffer(i))
            except A.DeferError as e:          # a conv store folded away
                bufs.append(str(e))
        return bufs, r.describe(), r.plan, [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))]
    finally:
        r.close()


def stem_image(b, h, w, cin, seed):
    """Integer-valued fp32 image in [-1023, 1023]: values above 255 have a lo plane (the stem's window split)."""
    return np.random.default_rng(seed).integers(-1023, 1024, (b, h, w, cin)).astype(np.float32)


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("name", list(STEMS))
def test_stem_paths_exact(name, dtype, monkeypatch):
    b, h, w, cin, cout, k, s, pad = STEMS[name]
    fmt_name = _fmt_name(dtype)
    i = list(STEMS).index(name)
    m = _stem_model(h, w, cin, cout, k, s, pad, seed=i)
    exact_weights(m, seed=100 + i, split_w=i % 2 == 1, x_mean=512.0)
    x = stem_image(b, h, w, cin, seed=200 + i)
    for path, (kernel, env) in list(STEM_PATHS.items()) + [("simt", ("conv_simt_kernel", {}))]:
        _knobs(monkeypatch, **env)
        r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=b, depth=1, conv_backend=1 if path == "simt" else 0)
        try:
            got_kernel = r.op_info(0)["kernel"]
            if kernel == "conv_stem_kernel" and cout != 64:
                kernel = "stem_im2col+conv_stream_kernel"
            if path == "simt" and got_kernel == "stem7x7s2_kernel":
                kernel = got_kernel
            assert got_kernel == kernel, (path, r.describe())
            r.predict(x)
            y = r.read_layer("relu")
            op = r.plan.ops[0]
            assert op.kind == A.OP_CONV and op.flags & A.FLAG_RELU
            assert_exact_plan_weights(r.plan)
            want = expected_conv_out(r.plan, op, {op.in0: x}, fmt_name, "stem" if path == "simt" else "wgmma")
            _assert_equal(y, want, (name, dtype, path, kernel))
        finally:
            r.close()


def chain_input(spatial, batch, seed):
    cin, _, stride, _ = CHAINS[spatial]
    hin = spatial * stride
    return np.random.default_rng(seed).integers(-8, 9, (batch, hin, hin, cin)).astype(np.float32)


def run_chain_exact(spatial, dtype, batch=2):
    """The chain at `spatial` with exact weights under the current knobs: every conv exact; returns describe()."""
    m = _chain_model(spatial)
    exact_weights(m, seed=300 + spatial, nnz=4)
    bufs, desc, plan, _ = _run_all_buffers(m, chain_input(spatial, batch, seed=400 + spatial), dtype)
    assert_exact_plan_weights(plan)
    assert check_stage_convs(plan, bufs, dtype, (spatial, dtype, desc)) == 7
    return desc


@pytest.mark.parametrize("mega", [0, 1])
@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("spatial", list(CHAINS))
def test_chain_exact(spatial, dtype, mega, monkeypatch):
    _knobs(monkeypatch, DEFER_MEGA=mega, DEFER_UMMA_SPLITK=0)
    desc = run_chain_exact(spatial, dtype)
    assert ("megakernel group: ops" in desc) == bool(mega), desc


@pytest.mark.parametrize("cluster", [2, 4])
def test_mega_cluster_exact(cluster, monkeypatch):
    """DEFER_MEGA_CLUSTER is read once per process: each size runs in a child process."""
    _knobs(monkeypatch)
    code = (f"import sys; sys.path[:0] = [{str(TESTS)!r}, {str(ROOT)!r}]; import test_gpu_conv_exact as T\n"
            f"for s in {list(CHAINS)!r}:\n"
            f"    for d in ('float32', 'bfloat16'):\n"
            f"        assert 'megakernel group: ops' in T.run_chain_exact(s, d)\n"
            f"print('exact', {cluster})")
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env.update(DEFER_MEGA="1", DEFER_MEGA_CLUSTER=str(cluster), DEFER_UMMA_SPLITK="0")
    p = subprocess.run([sys.executable, "-c", code], env=env, cwd=str(ROOT), capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and f"exact {cluster}" in p.stdout, p.stdout[-2000:] + p.stderr[-4000:]


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
def test_folded_affine_exact(dtype, monkeypatch):
    """conv -> + residual -> BN -> ReLU with the BN+ReLU folded into the conv's epilogue as a second output."""
    m = _fold_model(residual=True, keep_store=False, relu=True)
    exact_weights(m, seed=500, nnz=16)
    x = np.random.default_rng(501).integers(-8, 9, (2, 28, 28, 128)).astype(np.float32)
    _knobs(monkeypatch, DEFER_FOLD_AFFINE=1, DEFER_STREAM_MIN_TILES=10 ** 9, DEFER_UMMA_SPLITK=0)
    bufs, desc, plan, kernels = _run_all_buffers(m, x, dtype)
    ai = next(i for i, op in enumerate(plan.ops) if op.kind == A.OP_AFFINE)
    ci = next(i for i, op in enumerate(plan.ops) if op.out == plan.ops[ai].in0)
    assert kernels[ci] == "conv_umma_aff_kernel" and "fused into" in kernels[ai], kernels
    assert_exact_plan_weights(plan)
    assert check_stage_convs(plan, bufs, dtype, (dtype, desc)) == 2
