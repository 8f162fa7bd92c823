"""The case list of tests/test_gpu_app_convs_exact.py against the applications' plans, without a GPU.

* coverage guard: every conv op of every application's whole-model plan maps to a case of tests/app_convs.py with the
  epilogue the plan gives it, so a geometry a planner or builder change introduces fails here until the exact matrix
  runs it;
* each case's epilogues and batches are exactly those the plans give it, and its name is one of its occurrences;
* every case that the older exact matrix (test_gpu_conv_exact.WGMMA_SHAPES / STEM_SHAPES) lacks is exactly summable in
  each of the four operand families at each of its batches;
* the host time to build the expected bits of the whole per-kernel matrix, and that every case's expected output has
  values on both sides of zero before the store (a case whose outputs were all one value would check little)."""
import time

import numpy as np
import pytest

import app_convs as C
import exact_conv as X
import test_gpu_conv_exact as G


@pytest.fixture(scope="module")
def walked():
    return C.walk()


def _old_geometries():
    return {g[1:] for g in list(G.WGMMA_SHAPES.values()) + list(G.STEM_SHAPES.values())}


def _table():
    return {**C.APP_CONVS, **C.STEM_CONVS}


def test_every_app_conv_has_a_case(walked):
    by_geom = {g: (name, set(epis)) for name, (g, epis, _) in _table().items()}
    n_ops = 0
    missing = []
    for app in C.APPS:
        for geom, epi, conv, _ in C.plan_convs(app):
            n_ops += 1
            if geom not in by_geom or epi not in by_geom[geom][1]:
                missing.append((app, conv, geom, epi))
    assert not missing, ("conv ops of the applications' plans without an exact case in tests/app_convs.py", missing)
    new = [g for g in walked if g not in _old_geometries()]
    print(f"\n{n_ops} conv ops in {len(C.APPS)} applications: {len(walked)} distinct geometries, {len(new)} not in the "
          f"older exact matrix; all {len(walked)} have cases")
    assert len(walked) == len(_table())


def test_cases_carry_the_plans_epilogues_and_batches(walked):
    for name, (geom, epis, batches) in _table().items():
        assert geom in walked, (name, "no application plans this geometry any more")
        w = walked[geom]
        assert w["stem"] == (name in C.STEM_CONVS), name
        assert set(epis) == w["epilogues"], (name, epis, w["epilogues"])
        assert len(set(epis)) == len(epis), name
        assert tuple(batches) == C.batches_of(w["apps"], geom, w["stem"]), (name, batches, w["apps"])
        assert name in w["names"], (name, w["names"][:4])


def test_new_cases_are_exactly_summable_in_every_family():
    """Both formats: the BF16 products are the hi*hi subset of the BF16X2 ones on the same grid, so the BF16X2 bound
    implies the BF16 one; the grids are asserted equal."""
    old = _old_geometries()
    worst = 0.0
    n = 0
    for name, (geom, _, batches) in C.APP_CONVS.items():
        if geom in old:
            continue
        for b in batches:
            for fam in X.FAMILIES:
                case = X.ExactCase("bf16x2", (b,) + geom, fam, False, False, seed=1)
                pairs = case.pairs("wgmma")
                worst = max(worst, X.assert_exactly_summable(pairs, case.geom, (name, b, fam)))
                (xh, wh), = X.product_pairs(case.x, case.wk, "bf16", "wgmma")
                assert X.quantum(xh) * X.quantum(wh) == (X.quantum(*[a for a, _ in pairs])
                                                        * X.quantum(*[w for _, w in pairs])), (name, b, fam)
                n += 1
    print(f"\n{n} new (case, batch, family) operand sets: worst sum|terms| / g = 2^{np.log2(worst):.2f} (bound 2^22)")


def test_host_time_of_the_expected_bits():
    t0 = time.perf_counter()
    n = 0
    for fmt_name in ("bf16x2", "bf16"):
        for args in C.kernel_cases(fmt_name):
            case = C.exact_case(fmt_name, *args)
            v = case.expected_value("wgmma")
            case.expected_bits("wgmma")
            if not args[3]:                                     # no ReLU: both signs are stored
                assert np.any(v > 0) and np.any(v < 0), (fmt_name, args)
            else:
                assert np.any(v > 0) and np.any(v == 0), (fmt_name, args)
            n += 1
    dt = time.perf_counter() - t0
    print(f"\nexpected bits of the per-kernel matrix: {n} cases, {2 * C.n_outputs() / 1e6:.1f} M outputs in BF16X2 and "
          f"BF16, {dt:.1f} s on this host")
