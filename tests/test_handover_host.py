"""Host-side checks of the step orders and the checker tests/test_gpu_handover.py relies on (no GPU needed).

Every order steps each (stage, microbatch) once, submits before stage 0 runs, and collects results FIFO with at most `depth`
outstanding.  The checker rejects results shifted by `depth` either way, two swapped lanes and a torn result, each with its
own diagnosis, when every microbatch has its own input.  With inputs that repeat with a period dividing `depth` (every
multi-lane test before these) the same stale slots pass: that is why the GPU tests feed distinct inputs."""
import numpy as np
import pytest

import handover_check as H


def _positions(events):
    return {ev: i for i, ev in enumerate(events)}


@pytest.mark.parametrize("order", H.SCHEDULES)
@pytest.mark.parametrize("depth", [1, 2, 3, 4])
@pytest.mark.parametrize("n_stages", [1, 2, 8])
def test_schedule_steps_everything_once_and_collects_fifo(order, n_stages, depth):
    n = 3 * depth + 2
    ev = H.schedule(order, n_stages, n, depth)
    assert len(ev) == len(set(ev)) == n * (n_stages + 2)
    pos = _positions(ev)
    for seq in range(n):
        assert pos[("submit", seq)] < pos[("step", 0, seq)]
        assert pos[("step", n_stages - 1, seq)] < pos[("result", seq)]
        for st in range(n_stages):
            if seq >= depth:                               # a lane runs its microbatches in order on every stage
                assert pos[("step", st, seq - depth)] < pos[("step", st, seq)]
    results = [e[1] for e in ev if e[0] == "result"]
    assert results == list(range(n))
    outstanding = 0
    for e in ev:
        if e[0] == "step" and e[1] == n_stages - 1:
            outstanding += 1
            assert outstanding <= depth, (order, e)
        elif e[0] == "result":
            outstanding -= 1
    assert outstanding == 0


@pytest.mark.parametrize("depth", [1, 2, 4])
def test_schedules_differ_where_they_should(depth):
    n_stages, n = 4, 3 * depth + 2
    disp = _positions(H.schedule("dispatcher", n_stages, n, depth))
    major = _positions(H.schedule("stage_major", n_stages, n, depth))
    first = _positions(H.schedule("consumer_first", n_stages, n, depth))
    for seq in range(n):
        # dispatcher: the feeder waits for the result before it reuses the lane (DEFER, bench.py)
        if seq + depth < n:
            assert disp[("result", seq)] < disp[("submit", seq + depth)]
        # consumer_first: every consumer is stepped before its producer, so its ready-flag wait spins
        for st in range(1, n_stages):
            assert first[("step", st, seq)] < first[("step", st - 1, seq)]
        # stage_major: stage 0 reuses a lane before the previous microbatch on it has been collected
        if seq + depth < n:
            assert major[("step", 0, seq + depth)] < major[("result", seq)]
        # ... and runs the whole window before stage 1 starts on it
        w0 = seq - seq % depth
        assert all(major[("step", 0, s)] < major[("step", 1, seq)] for s in range(w0, min(w0 + depth, n)))


# ------------------------------------------------------------------------------------------------ the checker
def _refs(n, seed=0):
    """n softmax rows, as the last stage of the test models gives."""
    z = np.random.default_rng(seed).standard_normal((n, 1, 1000)).astype(np.float32) * 2
    e = np.exp(z - z.max(axis=-1, keepdims=True))
    return list(e / e.sum(axis=-1, keepdims=True))


DEPTHS = [1, 2, 3, 4]


@pytest.mark.parametrize("depth", DEPTHS)
def test_correct_results_pass_and_references_are_distinct(depth):
    n = 3 * depth + 2
    refs = _refs(n)
    H.check_results([r.copy() for r in refs], refs, depth)
    assert H.n_distinct(refs) == n


@pytest.mark.parametrize("depth", DEPTHS)
def test_stale_slot_is_diagnosed(depth):
    """Every lane hands back the microbatch before: a ready flag raised before the copy lands."""
    n = 3 * depth + 2
    refs = _refs(n)
    got = [refs[s - depth] if s >= depth else refs[s] for s in range(n)]
    bad = H.diagnose(got, refs, depth)
    assert [(s, k) for s, k, _ in bad] == [(s, "stale") for s in range(depth, n)]
    with pytest.raises(AssertionError, match=f"seq {depth} .*stale slot"):
        H.check_results(got, refs, depth)


@pytest.mark.parametrize("depth", DEPTHS)
def test_overwritten_result_is_diagnosed(depth):
    """result(seq) collected after seq + depth ran on the lane."""
    n = 3 * depth + 2
    refs = _refs(n)
    got = [refs[s + depth] if s + depth < n else refs[s] for s in range(n)]
    bad = H.diagnose(got, refs, depth)
    assert [(s, k) for s, k, _ in bad] == [(s, "overwritten") for s in range(n - depth)]


@pytest.mark.parametrize("depth", [2, 3, 4])
def test_swapped_lanes_are_diagnosed(depth):
    """Lanes 0 and 1 take each other's slot."""
    n = 3 * depth + 2
    refs = _refs(n)
    partner = {0: 1, 1: 0}

    def src(s):
        lane = s % depth
        t = s - lane + partner.get(lane, lane)
        return t if t < n else s
    got = [refs[src(s)] for s in range(n)]
    bad = H.diagnose(got, refs, depth)
    want = [(s, "other_seq") for s in range(n) if src(s) != s]
    assert want and [(s, k) for s, k, _ in bad] == want
    assert all(f"equals the result of seq {src(s)}" in m for s, _, m in bad)


@pytest.mark.parametrize("depth", DEPTHS)
def test_torn_result_is_diagnosed(depth):
    """One result is half its own microbatch and half the one before on its lane."""
    n = 3 * depth + 2
    refs = _refs(n)
    seq = depth + 1
    torn = refs[seq].copy()
    torn[..., 500:] = refs[seq - depth][..., 500:]
    got = [r.copy() for r in refs]
    got[seq] = torn
    assert [(s, k) for s, k, _ in H.diagnose(got, refs, depth)] == [(seq, "torn")]


@pytest.mark.parametrize("period,depth", [(1, 1), (1, 2), (2, 2), (1, 3), (3, 3), (1, 4), (2, 4), (4, 4)])
def test_inputs_repeating_with_a_period_dividing_depth_are_blind(period, depth):
    """Inputs that cycle with a period dividing depth give each lane one input for ever: a stale slot holds the same bits as
    a fresh one and the check passes.  Such a run says nothing about the hand-over."""
    n = 3 * depth + 2
    base = _refs(period)
    refs = [base[s % period] for s in range(n)]
    stale = [refs[s - depth] if s >= depth else refs[s] for s in range(n)]
    H.check_results(stale, refs, depth)
    assert H.n_distinct(refs) == 0


@pytest.mark.parametrize("period,depth", [(3, 2), (2, 3), (3, 4), (5, 4)])
def test_inputs_repeating_with_a_period_not_dividing_depth_see_a_stale_slot(period, depth):
    n = 3 * depth + 2
    base = _refs(period)
    refs = [base[s % period] for s in range(n)]
    stale = [refs[s - depth] if s >= depth else refs[s] for s in range(n)]
    with pytest.raises(AssertionError):
        H.check_results(stale, refs, depth)


def test_n_distinct_needs_a_real_difference():
    refs = _refs(3)
    near = refs[0] * np.float32(1 + 1e-5)                  # bitwise different, relatively the same
    assert H.n_distinct(refs + [near]) == 2
