"""Balanced cut selection - the caller side of ``DEFER._partition`` (SURVEY.md 8f, rank 1).

The reference takes the cut list by hand (``test/test.py:15-18``); pipeline throughput is
1 / max(stage time), so a poorly balanced list wastes GPUs (with the reference's own 8-stage list the
first stage - stem + 3 residual blocks - is ~2x the median stage).  ``balanced_cuts`` picks the cut layers
that minimise the slowest stage:

* candidates are *articulation points* of the layer DAG (every input->output path crosses them - what
  ``dag_util.construct_model`` needs) that are also the tail of a fused op of the single-stage plan, so a
  cut never breaks a conv+BN+Add+ReLU fusion (cutting after the post-Add ReLU also spares the consumer the
  standalone ReLU a cut at ``add_k`` costs);
* per-op cost is either measured (``StageRunner.time_op`` on a GPU) or the analytic batch-1 model
  ``launch_us + alg_bytes / HBM``;
* an O(stages x candidates^2) DP minimises the maximum stage cost (ties: smaller sum of squares).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

from . import _cabi as A
from . import keras_like as K
from .planner import Plan, plan_stage

HBM_GBS = 3350.0          # H100 SXM data-sheet HBM3 bandwidth
LAUNCH_US = 2.0           # per-launch cost with several microbatches in flight (device launch rate)


def articulation_layers(model: K.Model) -> List[str]:
    """Layers whose output tensor is the only live tensor right after they execute."""
    nodes = list(model.iter_nodes())
    remaining: Dict[str, int] = {l.name: 0 for l, _ in nodes}
    for _, ins in nodes:
        for p in ins or []:
            remaining[p] += 1
    live: Dict[str, int] = {}
    out = []
    last = nodes[-1][0].name
    for layer, ins in nodes:
        for p in ins or []:
            live[p] -= 1
            if live[p] == 0:
                del live[p]
        if remaining[layer.name] > 0:
            live[layer.name] = remaining[layer.name]
        if list(live.keys()) == [layer.name] and ins is not None and layer.name != last:
            out.append(layer.name)
    return out


def analytic_op_costs(plan: Plan, act_bytes: int = 4, batch: int = 1) -> List[float]:
    costs = []
    for op in plan.ops:
        hi, wi, ci, _ = plan.bufs[op.in0]
        ho, wo, co, _ = plan.bufs[op.out]
        by = batch * (hi * wi * ci + ho * wo * co) * act_bytes
        if op.kind == A.OP_CONV:
            by += op.kh * op.kw * ci * co * act_bytes + (batch * ho * wo * co * act_bytes if op.flags & A.FLAG_RESIDUAL else 0)
        elif op.kind == A.OP_DENSE:
            by += hi * wi * ci * co * 4
        costs.append(LAUNCH_US + by / (HBM_GBS * 1e3))
    return costs


def minimax_partition(costs: Sequence[float], n_parts: int, allowed: Sequence[int]) -> List[int]:
    """Split ``costs`` into ``n_parts`` contiguous parts; a part may end only after an index in ``allowed``.
    Returns the ``n_parts - 1`` chosen end indices minimising the maximum part sum."""
    n = len(costs)
    pre = [0.0]
    for c in costs:
        pre.append(pre[-1] + c)
    ends = sorted(set(i for i in allowed if 0 <= i < n - 1))
    if len(ends) < n_parts - 1:
        raise ValueError(f"only {len(ends)} legal cut points for {n_parts} stages")
    INF = float("inf")
    pts = ends + [n - 1]
    # best[k][j] = (max, sumsq) splitting costs[0..pts[j]] into k parts, last part ending at pts[j]
    best = [[(INF, INF)] * len(pts) for _ in range(n_parts + 1)]
    arg = [[-1] * len(pts) for _ in range(n_parts + 1)]
    for j, e in enumerate(pts):
        s = pre[e + 1]
        best[1][j] = (s, s * s)
    for k in range(2, n_parts + 1):
        for j, e in enumerate(pts):
            for i in range(j):
                pm, ps = best[k - 1][i]
                if pm == INF:
                    continue
                seg = pre[e + 1] - pre[pts[i] + 1]
                cand = (max(pm, seg), ps + seg * seg)
                if cand < best[k][j]:
                    best[k][j] = cand
                    arg[k][j] = i
    j = len(pts) - 1
    if best[n_parts][j][0] == INF:
        raise ValueError("no feasible partition")
    cuts = []
    for k in range(n_parts, 1, -1):
        j = arg[k][j]
        cuts.append(pts[j])
    return sorted(cuts)


def balanced_cuts(model: K.Model, n_stages: int, op_costs: Optional[Sequence[float]] = None,
                  act_bytes: int = 4) -> Tuple[List[str], List[float]]:
    """Cut layer names for ``DEFER.run_defer`` and the predicted per-stage cost (same unit as ``op_costs``).

    ``op_costs[i]`` is the cost of op ``i`` of ``plan_stage(model, True, True)`` (e.g. measured microseconds);
    default: the analytic model."""
    if n_stages <= 1:
        return [], []
    plan = plan_stage(model, True, True)
    costs = list(op_costs) if op_costs is not None else analytic_op_costs(plan, act_bytes)
    if len(costs) != len(plan.ops):
        raise ValueError(f"{len(costs)} costs for {len(plan.ops)} ops")
    arts = set(articulation_layers(model))
    allowed, name_at = [], {}
    for i, op in enumerate(plan.ops):
        tail = op.layers[-1]
        if tail in arts and plan.bufs[op.out][3] == A.BUF_ACT:
            allowed.append(i)
            name_at[i] = tail
    idx = minimax_partition(costs, n_stages, allowed)
    bounds = [-1] + idx + [len(costs) - 1]
    stage_costs = [sum(costs[bounds[k] + 1:bounds[k + 1] + 1]) for k in range(n_stages)]
    return [name_at[i] for i in idx], stage_costs
