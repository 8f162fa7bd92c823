"""Every convolution the applications run, as the planner plans them (not a test module).

`plan_convs(app)` walks `planner.plan_stage` over one whole application at 224 x 224 and returns each conv op's geometry,
its epilogue flags and whether an AFFINE op reads its output (ResNet V2's `_preact_bn` / `post_bn`, which
DEFER_FOLD_AFFINE=1 folds into that conv's epilogue).  `APP_CONVS` and `STEM_CONVS` below are that walk over the seven
applications, deduplicated by geometry and written out, so that a new geometry or epilogue in a plan fails
tests/test_app_convs_host.py until it is added here - and with it to the exact matrix of
tests/test_gpu_app_convs_exact.py.

A geometry is (h, w, cin, cout, kh, kw, sh, sw, pad t, l, b, r) of the conv's input map; an epilogue is (residual, ReLU,
affine reader).  Each geometry runs at batch 1, at bench.py's microbatch of 32 when ResNet50 or ResNet50V2 plans it, and
VGG16's maps of 56 and larger at batch 4 (the exact reference of a 224 x 224 x 64 3x3 conv at batch 32 would cost the
host minutes).  The RGB stems read the fp32 image and run on the fused stem kernel at stage level, at batch 1 and 32.
"""
APPS = ("ResNet50", "ResNet101", "ResNet152", "ResNet50V2", "ResNet101V2", "ResNet152V2", "VGG16")
BENCH_BATCH = 32                          # bench.py's microbatch
BENCH_APPS = ("ResNet50", "ResNet50V2")   # the applications run at it
VGG_BATCH, VGG_MIN_MAP = 4, 56            # VGG16's large maps: the batch that bounds the host cost of the reference
STEM_BATCHES = (1, BENCH_BATCH)

# name of one occurrence: (geometry, epilogues (residual, relu, affine reader), batches)
APP_CONVS = {
    "VGG16:block1_conv2": ((224, 224, 64, 64, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1, 4)),
    "VGG16:block2_conv1": ((112, 112, 64, 128, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1, 4)),
    "VGG16:block2_conv2": ((112, 112, 128, 128, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1, 4)),
    "ResNet50:res2a_branch2a": ((56, 56, 64, 64, 1, 1, 1, 1, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "ResNet50:res2a_branch2b": ((56, 56, 64, 64, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1, 32)),
    "ResNet50V2:conv2_block3_2_conv": ((56, 56, 64, 64, 3, 3, 2, 2, 1, 1, 1, 1), ((False, True, False),), (1, 32)),
    "ResNet50:res2a_branch2c": ((56, 56, 64, 256, 1, 1, 1, 1, 0, 0, 0, 0),
                                ((False, False, False), (True, False, True), (True, True, False)), (1, 32)),
    "VGG16:block3_conv1": ((56, 56, 128, 256, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1, 4)),
    "ResNet50:res2b_branch2a": ((56, 56, 256, 64, 1, 1, 1, 1, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "ResNet50:res3a_branch2a": ((56, 56, 256, 128, 1, 1, 2, 2, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "VGG16:block3_conv2": ((56, 56, 256, 256, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1, 4)),
    "ResNet50:res3a_branch1": ((56, 56, 256, 512, 1, 1, 2, 2, 0, 0, 0, 0),
                               ((False, False, False), (True, True, False)), (1, 32)),
    "ResNet50V2:conv2_block3_3_conv": ((28, 28, 64, 256, 1, 1, 1, 1, 0, 0, 0, 0), ((True, False, True),), (1, 32)),
    "ResNet50:res3a_branch2b": ((28, 28, 128, 128, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1, 32)),
    "ResNet50V2:conv3_block4_2_conv": ((28, 28, 128, 128, 3, 3, 2, 2, 1, 1, 1, 1), ((False, True, False),), (1, 32)),
    "ResNet50:res3a_branch2c": ((28, 28, 128, 512, 1, 1, 1, 1, 0, 0, 0, 0),
                                ((False, False, False), (True, False, True), (True, True, False)), (1, 32)),
    "ResNet50V2:conv3_block1_1_conv": ((28, 28, 256, 128, 1, 1, 1, 1, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "ResNet50V2:conv3_block1_0_conv": ((28, 28, 256, 512, 1, 1, 1, 1, 0, 0, 0, 0), ((False, False, False),), (1, 32)),
    "VGG16:block4_conv1": ((28, 28, 256, 512, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1,)),
    "ResNet50:res3b_branch2a": ((28, 28, 512, 128, 1, 1, 1, 1, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "ResNet50:res4a_branch2a": ((28, 28, 512, 256, 1, 1, 2, 2, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "VGG16:block4_conv2": ((28, 28, 512, 512, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1,)),
    "ResNet50:res4a_branch1": ((28, 28, 512, 1024, 1, 1, 2, 2, 0, 0, 0, 0),
                               ((False, False, False), (True, True, False)), (1, 32)),
    "ResNet50V2:conv3_block4_3_conv": ((14, 14, 128, 512, 1, 1, 1, 1, 0, 0, 0, 0), ((True, False, True),), (1, 32)),
    "ResNet50:res4a_branch2b": ((14, 14, 256, 256, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1, 32)),
    "ResNet50V2:conv4_block6_2_conv": ((14, 14, 256, 256, 3, 3, 2, 2, 1, 1, 1, 1), ((False, True, False),), (1, 32)),
    "ResNet50:res4a_branch2c": ((14, 14, 256, 1024, 1, 1, 1, 1, 0, 0, 0, 0),
                                ((False, False, False), (True, False, True), (True, True, False)), (1, 32)),
    "ResNet50V2:conv4_block1_1_conv": ((14, 14, 512, 256, 1, 1, 1, 1, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "VGG16:block5_conv1": ((14, 14, 512, 512, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1,)),
    "ResNet50V2:conv4_block1_0_conv": ((14, 14, 512, 1024, 1, 1, 1, 1, 0, 0, 0, 0), ((False, False, False),), (1, 32)),
    "ResNet50:res4b_branch2a": ((14, 14, 1024, 256, 1, 1, 1, 1, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "ResNet50:res5a_branch2a": ((14, 14, 1024, 512, 1, 1, 2, 2, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "ResNet50:res5a_branch1": ((14, 14, 1024, 2048, 1, 1, 2, 2, 0, 0, 0, 0),
                               ((False, False, False), (True, True, False)), (1, 32)),
    "ResNet50V2:conv4_block6_3_conv": ((7, 7, 256, 1024, 1, 1, 1, 1, 0, 0, 0, 0), ((True, False, True),), (1, 32)),
    "ResNet50:res5a_branch2b": ((7, 7, 512, 512, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), (1, 32)),
    "ResNet50:res5a_branch2c": ((7, 7, 512, 2048, 1, 1, 1, 1, 0, 0, 0, 0),
                                ((False, False, False), (True, False, True), (True, True, False)), (1, 32)),
    "ResNet50V2:conv5_block1_1_conv": ((7, 7, 1024, 512, 1, 1, 1, 1, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
    "ResNet50V2:conv5_block1_0_conv": ((7, 7, 1024, 2048, 1, 1, 1, 1, 0, 0, 0, 0), ((False, False, False),), (1, 32)),
    "ResNet50:res5b_branch2a": ((7, 7, 2048, 512, 1, 1, 1, 1, 0, 0, 0, 0), ((False, True, False),), (1, 32)),
}

# the RGB stems (fp32 image in): ResNet's 7x7/2 with BN and ReLU, ResNet V2's with a bias and no ReLU, VGG16's 3x3/1
STEM_CONVS = {
    "VGG16:block1_conv1": ((224, 224, 3, 64, 3, 3, 1, 1, 1, 1, 1, 1), ((False, True, False),), STEM_BATCHES),
    "ResNet50:conv1": ((224, 224, 3, 64, 7, 7, 2, 2, 3, 3, 3, 3), ((False, False, False), (False, True, False)),
                       STEM_BATCHES),
}


def build(app, weights=None):
    from defer_b200 import applications
    return getattr(applications, app)(weights=weights)


def plan_convs(app, model=None):
    """[(geometry, (residual, relu, affine reader), conv layer name, stem)] of every conv op of `app`'s whole-model plan."""
    from defer_b200 import _cabi as A
    from defer_b200 import keras_like as K
    from defer_b200 import planner
    m = model if model is not None else build(app)
    plan = planner.plan_stage(m, True, True)
    read_by_affine = {op.in0 for op in plan.ops if op.kind == A.OP_AFFINE}
    out = []
    for op in plan.ops:
        if op.kind != A.OP_CONV:
            continue
        h, w, cin, elem = plan.bufs[op.in0]
        geom = (h, w, cin, plan.bufs[op.out][2], op.kh, op.kw, op.sh, op.sw) + tuple(op.pads)
        epi = (bool(op.flags & A.FLAG_RESIDUAL), bool(op.flags & A.FLAG_RELU), op.out in read_by_affine)
        conv = next(n for n in op.layers if isinstance(m.get_layer(n), K.Conv2D))
        out.append((geom, epi, conv, elem != A.BUF_ACT))
    return out


def batches_of(apps, geom, stem):
    """The batches a geometry planned by `apps` runs at (the rule of the module docstring)."""
    if stem:
        return STEM_BATCHES
    b = [1]
    if set(apps) & set(BENCH_APPS):
        b.append(BENCH_BATCH)
    if "VGG16" in apps and geom[0] >= VGG_MIN_MAP:
        b.append(VGG_BATCH)
    return tuple(b)


def walk():
    """{geometry: {"names": [app:layer], "epilogues": set, "apps": [app], "stem": bool}} over the seven applications."""
    out = {}
    for app in APPS:
        for geom, epi, conv, stem in plan_convs(app):
            e = out.setdefault(geom, {"names": [], "epilogues": set(), "apps": [], "stem": stem})
            e["names"].append(f"{app}:{conv}")
            e["epilogues"].add(epi)
            if app not in e["apps"]:
                e["apps"].append(app)
    return out


def kernel_epilogues(epilogues):
    """The distinct (residual, relu) pairs: what a defer_k_conv run sees (the affine reader is a stage-level fold)."""
    return sorted({(r, relu) for r, relu, _ in epilogues})


def kernel_cases(fmt_name):
    """[(name, batch, residual, relu, family, seed)] of the per-kernel matrix: every geometry of APP_CONVS at each of its
    batches with each of its epilogues.  The families rotate so that each meets every geometry class and every batch."""
    import exact_conv as X
    fams = list(X.FAMILIES)
    out = []
    for i, (name, (geom, epis, batches)) in enumerate(APP_CONVS.items()):
        for j, (res, relu) in enumerate(kernel_epilogues(epis)):
            for k, b in enumerate(batches):
                out.append((name, b, res, relu, fams[(i + j + k) % 4], 7000 + 100 * i + 10 * j + k))
    return out


def exact_case(fmt_name, name, batch, res, relu, family, seed):
    import exact_conv as X
    geom = APP_CONVS[name][0]
    return X.ExactCase(fmt_name, (batch,) + geom, family, relu, res, seed=seed)


def n_outputs():
    """Output elements of the per-kernel matrix in one format (the size of the host's exact reference)."""
    n = 0
    for name, b, *_ in kernel_cases("bf16"):
        h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = APP_CONVS[name][0]
        n += b * ((h + pt + pb - kh) // sh + 1) * ((w + pl + pr - kw) // sw + 1) * cout
    return n
