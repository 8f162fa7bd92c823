"""Every convolution the applications run, bit for bit on exactly summable operands (tests/exact_conv.py), at the batches
their plans run: 1, bench.py's 32 for ResNet50 / ResNet50V2, 4 for VGG16's large maps (tests/app_convs.py).

a. per kernel: each geometry of tests/app_convs.py::APP_CONVS with each epilogue its plans give it, through the 15 wgmma
   executors of `defer_k_conv` (test_gpu_conv_exact.EXECUTORS), in BF16X2 and BF16, into outputs pre-filled with NaN;
b. at stage level, at default knobs: block chains built with the applications' own builders at their real maps and
   channels - ResNet50's conv4 block a (`res4a_branch1`) and block b, the first and the stride-2 last block of each
   ResNet V2 stack (the max-pool shortcut) with the next pre-activation BN + ReLU, one conv5 block, VGG16's blocks 2 to 5 -
   in float32 and bfloat16, ResNet V2 with DEFER_FOLD_AFFINE 0 and 1.  Every conv and every folded affine output is exact.
   The executor guard builds (without running) the whole application's stage at the same batch, dtype and knobs, and
   requires each chain conv to get the kernel and the describe() tiling of the same layer there;
c. the RGB stems at 224 x 224 on the fused `conv_stem_kernel`: ResNet's 7x7/2 with BN and ReLU, ResNet V2's with a bias
   and no ReLU, VGG16's 3x3/1, at batch 1 and 32, under the same guard.

The module (130 tests) takes about 11.5 minutes on an H100 80GB HBM3 at a 700 W power limit, most of it the host's exact
reference (the RGB stems at batch 32 take up to 19 s each).
"""
import functools
import re

import numpy as np
import pytest

import app_convs as C
import exact_conv as X
from conv_check import FMTS, _encode, _ptr
from defer_b200 import _cabi as A
from defer_b200 import applications
from defer_b200 import keras_like as K
from defer_b200.node import StageRunner
from test_gpu_conv_exact import (EXECUTORS, _fmt_name, _knobs, _run_all_buffers, assert_exact_plan_weights,
                                 check_stage_convs, exact_weights, expected_conv_out, stem_image)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DTYPES = ["float32", "bfloat16"]


@pytest.fixture(scope="module")
def torch_cuda():
    lib = A.load()
    import torch
    assert torch.cuda.is_available()
    return torch, lib


# ------------------------------------------------------------------------------------------------ a. per kernel
def _run(torch, lib, case, backend, dev):
    """One defer_k_conv run of `case` on `backend` over the device operands `dev` into an output filled with NaN words,
    so an output the kernel never writes cannot match an expected zero."""
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = case.geom
    fmt = FMTS[case.fmt_name]
    xd, rd, wd, sd, fd = dev
    planes = 2 if fmt == A.FMT_BF16X2 else 1
    yd = torch.full((planes * n * case.ho * case.wo * cout,), -1, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    A.check(lib.defer_k_conv(fmt, backend, _ptr(xd), 0, _ptr(wd), _ptr(sd), _ptr(fd), _ptr(rd), _ptr(yd),
                             n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr, A.FLAG_RELU if case.relu else 0, None))
    torch.cuda.synchronize()
    return X.raw_bits(torch, yd, case.fmt_name)


@pytest.mark.parametrize("fmt_name", ["bf16x2", "bf16"])
@pytest.mark.parametrize("name", list(C.APP_CONVS))
def test_app_conv_every_executor_exact(torch_cuda, name, fmt_name, monkeypatch):
    torch, lib = torch_cuda
    fmt = FMTS[fmt_name]
    runs = []
    for args in C.kernel_cases(fmt_name):
        if args[0] != name:
            continue
        case = C.exact_case(fmt_name, *args)
        want = case.expected_bits("wgmma")
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda() if a is not None else None   # noqa: E731
        operands = (_encode(torch, lib, case.x, fmt), _encode(torch, lib, case.res, fmt) if case.res is not None else None,
                    dev(case.wk), dev(case.scale), dev(case.shift))
        for ex, (backend, env) in EXECUTORS.items():
            _knobs(monkeypatch, **env)
            X.assert_bits(_run(torch, lib, case, backend, operands), want, case.out_shape, fmt_name,
                          (name, f"batch {case.geom[0]}", f"residual {args[2]}", f"relu {args[3]}", case.family, ex))
        runs.append(f"batch {case.geom[0]} residual={int(args[2])} relu={int(args[3])} {case.family}")
        del operands
    assert runs
    print(f"\n{name} {fmt_name}: {len(runs)} cases x {len(EXECUTORS)} executors ({', '.join(EXECUTORS)}): "
          + "; ".join(runs))


# ------------------------------------------------------------------------------------------------ guard
def _tiles(desc, i):
    """The `wgmma tiles:` line describe() prints under op i, or '' (no tensor-core plan)."""
    lines = desc.splitlines()
    k = next(j for j, l in enumerate(lines) if re.match(rf"\s*\[\s*{i}\]", l))
    nxt = lines[k + 1] if k + 1 < len(lines) else ""
    return nxt.strip() if nxt.strip().startswith("wgmma tiles:") else ""


def _conv_name(model, op):
    return next(n for n in op.layers if isinstance(model.get_layer(n), K.Conv2D))


def _executors(model, plan, desc, kernels):
    """{conv layer: (kernel, tiles line)} of a built stage."""
    return {_conv_name(model, op): (kernels[i], _tiles(desc, i)) for i, op in enumerate(plan.ops) if op.kind == A.OP_CONV}


@functools.lru_cache(maxsize=None)
def _whole_model_executors(app, batch, dtype, fold):
    """The executor of every conv of `app`'s whole-model stage at this batch, dtype and DEFER_FOLD_AFFINE (built, not
    run; the caller has set the knobs)."""
    m = C.build(app)
    r = StageRunner.from_model(m, device=0, dtype=dtype, max_batch=batch, depth=1)
    try:
        return _executors(m, r.plan, r.describe(), [r.op_info(i)["kernel"] for i in range(len(r.plan.ops))])
    finally:
        r.close()


def assert_same_executors(app, model, plan, desc, kernels, batch, dtype, fold):
    """Each conv of the chain runs the kernel and tiling the same layer gets in the whole application; returns them."""
    mine = _executors(model, plan, desc, kernels)
    whole = _whole_model_executors(app, batch, dtype, fold)
    for layer, got in mine.items():
        assert layer in whole, (app, layer)
        assert got == whole[layer], (app, layer, batch, dtype, f"fold {fold}", "chain", got, "application", whole[layer])
    return mine


# ------------------------------------------------------------------------------------------------ b. stage level
def _resnet50_conv4():
    """ResNet50's conv4 block a (projection shortcut res4a_branch1, 1x1/2 512 -> 1024 with the Add and ReLU fused) and
    identity block b, from a ReLU over the 28 x 28 x 512 input: every conv reads bf16 planes."""
    K.clear_session()
    inp = K.Input(shape=(28, 28, 512))
    x = K.Activation("relu", name="relu_in")(inp)
    x = applications._conv_block(x, 3, [256, 256, 1024], 4, "a")
    x = applications._identity_block(x, 3, [256, 256, 1024], 4, "b")
    return K.Model(inp, x, name="resnet50_conv4")


# ResNet V2 stack: (input map, input channels, filters, blocks in ResNet50V2, stride of the last block)
V2_STACKS = {"conv2": (56, 64, 64, 3, 2), "conv3": (28, 256, 128, 4, 2), "conv4": (14, 512, 256, 6, 2),
             "conv5": (7, 1024, 512, 3, 1)}


def _v2_stack(stack):
    """The first block of a ResNet V2 stack (conv shortcut) and its last block (stride 2 and the 1x1/2 max-pool shortcut;
    conv5: stride 1, identity shortcut), then what reads the last `_out` in the application: the next stack's first
    pre-activation BN + ReLU, or post_bn + post_relu.  With DEFER_FOLD_AFFINE=1 both `_out` convs fold an affine op."""
    hw, cin, f, blocks, stride = V2_STACKS[stack]
    K.clear_session()
    inp = K.Input(shape=(hw, hw, cin))
    x = applications._block2(inp, f, conv_shortcut=True, name=f"{stack}_block1")
    x = applications._block2(x, f, stride=stride, name=f"{stack}_block{blocks}")
    nxt = f"conv{int(stack[-1]) + 1}_block1_preact_" if stack != "conv5" else "post_"
    x = K.BatchNormalization(epsilon=1.001e-5, name=nxt + "bn")(x)
    x = K.Activation("relu", name=nxt + "relu")(x)
    return K.Model(inp, x, name=f"v2_{stack}")


def _vgg_blocks():
    """VGG16's blocks 2 to 5 (conv runs and pools) from a ReLU over the 112 x 112 x 64 input."""
    K.clear_session()
    inp = K.Input(shape=(112, 112, 64))
    x = K.Activation("relu", name="relu_in")(inp)
    for bi, (n, f) in enumerate([(2, 128), (3, 256), (3, 512), (3, 512)], start=2):
        for ci in range(1, n + 1):
            x = K.Conv2D(f, (3, 3), activation="relu", padding="same", name=f"block{bi}_conv{ci}")(x)
        x = K.MaxPooling2D((2, 2), strides=(2, 2), name=f"block{bi}_pool")(x)
    return K.Model(inp, x, name="vgg_blocks")


# name -> (application, builder, batches, DEFER_FOLD_AFFINE settings, expected number of convs)
CHAINS = {
    "resnet50_conv4": ("ResNet50", _resnet50_conv4, (1, C.BENCH_BATCH), (0,), 7),
    **{f"v2_{s}": ("ResNet50V2", functools.partial(_v2_stack, s), (1, C.BENCH_BATCH), (0, 1), 7) for s in V2_STACKS},
    "vgg_blocks": ("VGG16", _vgg_blocks, (1, C.VGG_BATCH), (0,), 11),
}


def _vary_preact_scales(model, seed):
    """ResNet V2's pre-activation and post BNs (the affine ops DEFER_FOLD_AFFINE folds) get gamma 2^-1 or 1 per channel:
    with exact_weights' uniform 2^-1, a folded output that read a neighbouring channel's scale would keep its bits."""
    rng = np.random.default_rng(seed)
    for layer, _ in model.iter_nodes():
        if isinstance(layer, K.BatchNormalization) and layer.name.endswith(("_preact_bn", "post_bn")):
            g, b, m, v = layer.get_weights()
            layer.set_weights([rng.choice(np.float32([0.5, 1.0]), g.shape[0]), b, m, v])


def _assert_exact_weights(plan):
    """Every folded scale is 2^-1 or 1 per channel, every shift on a 2^-2 grid."""
    W = plan.weights
    for op in plan.ops:
        if op.kind in (A.OP_CONV, A.OP_AFFINE) and op.w_scale >= 0:
            assert np.all((W[op.w_scale] == np.float32(0.5)) | (W[op.w_scale] == np.float32(1))), op.layers
        if op.kind in (A.OP_CONV, A.OP_AFFINE) and op.w_shift >= 0:
            assert np.all(W[op.w_shift] * 4 == np.round(W[op.w_shift] * 4)), op.layers


def _chain_cases():
    return [(name, b, dtype, fold) for name, (_, _, batches, folds, _) in CHAINS.items()
            for b in batches for dtype in DTYPES for fold in folds]


@pytest.mark.parametrize("name,batch,dtype,fold", _chain_cases(),
                         ids=[f"{n}-b{b}-{d}-fold{f}" for n, b, d, f in _chain_cases()])
def test_app_chain_exact(name, batch, dtype, fold, monkeypatch):
    app, builder, _, _, n_convs = CHAINS[name]
    i = list(CHAINS).index(name)
    m = builder()
    exact_weights(m, seed=800 + i, nnz=4)
    _vary_preact_scales(m, seed=850 + i)
    hw, _, cin = m.input.shape[1:]
    x = np.random.default_rng(900 + 10 * i + batch).integers(-8, 9, (batch, hw, hw, cin)).astype(np.float32)
    _knobs(monkeypatch, **({"DEFER_FOLD_AFFINE": 1} if fold else {}))
    bufs, desc, plan, kernels = _run_all_buffers(m, x, dtype)
    _assert_exact_weights(plan)
    assert check_stage_convs(plan, bufs, dtype, (name, batch, dtype, fold, desc)) == n_convs
    ex = assert_same_executors(app, m, plan, desc, kernels, batch, dtype, fold)
    folded = [k for k in kernels if k.startswith("affine (fused into")]
    if fold:
        assert len(folded) == 2, kernels
    print(f"\n{name} batch {batch} {dtype} fold {fold}: {n_convs} convs and {len(folded)} folded affine outputs exact; "
          f"executors as in {app}: " + "; ".join(f"{l} {k} [{t.split(':', 1)[-1].strip()}]" for l, (k, t) in ex.items()))


# ------------------------------------------------------------------------------------------------ c. the RGB stems
def _resnet_stem(v2):
    """The applications' stem up to pool1: conv1 + bn_conv1 + ReLU (ResNet50), conv1_conv with its bias alone (V2)."""
    K.clear_session()
    inp = K.Input(shape=(224, 224, 3))
    x = K.ZeroPadding2D(padding=((3, 3), (3, 3)), name="conv1_pad")(inp)
    if v2:
        x = K.Conv2D(64, 7, strides=2, name="conv1_conv")(x)
    else:
        x = K.Conv2D(64, (7, 7), strides=(2, 2), padding="valid", name="conv1")(x)
        x = K.BatchNormalization(name="bn_conv1")(x)
        x = K.Activation("relu")(x)
    x = K.ZeroPadding2D(padding=((1, 1), (1, 1)), name="pool1_pad")(x)
    x = K.MaxPooling2D(3, strides=2, name="pool1_pool")(x)
    return K.Model(inp, x, name="stem")


def _vgg_stem():
    K.clear_session()
    inp = K.Input(shape=(224, 224, 3))
    x = K.Conv2D(64, (3, 3), activation="relu", padding="same", name="block1_conv1")(inp)
    return K.Model(inp, x, name="vgg_stem")


# name -> (application, builder, (residual, relu) of the conv)
STEMS = {
    "resnet50": ("ResNet50", functools.partial(_resnet_stem, False), (False, True)),
    "resnet50v2": ("ResNet50V2", functools.partial(_resnet_stem, True), (False, False)),
    "vgg16": ("VGG16", _vgg_stem, (False, True)),
}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("batch", C.STEM_BATCHES)
@pytest.mark.parametrize("name", list(STEMS))
def test_app_stem_exact(name, batch, dtype, monkeypatch):
    app, builder, (res, relu) = STEMS[name]
    i = list(STEMS).index(name)
    m = builder()
    exact_weights(m, seed=950 + i, split_w=i % 2 == 1, x_mean=512.0)
    x = stem_image(batch, 224, 224, 3, seed=960 + i + batch)
    _knobs(monkeypatch)
    bufs, desc, plan, kernels = _run_all_buffers(m, x, dtype)
    ci = next(j for j, op in enumerate(plan.ops) if op.kind == A.OP_CONV)
    op = plan.ops[ci]
    assert kernels[ci] == "conv_stem_kernel", desc
    assert (bool(op.flags & A.FLAG_RESIDUAL), bool(op.flags & A.FLAG_RELU)) == (res, relu), op.layers
    assert_exact_plan_weights(plan)
    want = expected_conv_out(plan, op, {op.in0: x}, _fmt_name(dtype), "wgmma")
    got = bufs[op.out]
    bad = np.argwhere(got != want)
    assert not bad.size, (name, batch, dtype, f"{len(bad)} of {got.size} differ; first at {tuple(bad[0])}: "
                                               f"got {got[tuple(bad[0])]!r}, want {want[tuple(bad[0])]!r}")
    ex = assert_same_executors(app, m, plan, desc, kernels, batch, dtype, 0)
    print(f"\n{name} stem batch {batch} {dtype}: exact; executor as in {app}: {ex}")
