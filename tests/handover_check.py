"""Same-process chains of stages, the step orders they are driven in, and a bitwise checker of their results.

A microbatch `seq` runs on lane `seq % depth` of every stage: the lane's input slot, its ready / free flags and (on the last
stage) its output buffer are reused by `seq + depth`.  When every microbatch a slot has held is the same data, a broken
hand-over (a ready flag raised before the copy lands, a free flag raised before the last reader, a lane taking another lane's
slot, a partial group keeping stale samples) still gives the right answer, so the chains here take one input per microbatch,
and `check_results` says which microbatch a wrong result belongs to.

Step orders (`schedule`), each a list of ("submit", seq) | ("step", stage, seq) | ("result", seq):
  dispatcher      per seq: submit, step stages 0..n-1 (DEFER's feeder, bench.py)
  stage_major     per window of `depth` seqs: submit all, step stage 0 for the window, then stage 1, ... (producers run ahead
                  and meet the free-flag waits of consumers still working on the previous window)
  consumer_first  per seq: step stages n-1..1, then submit and step stage 0 (every ready-flag wait spins, as when one process
                  per GPU steps a downstream rank first)
At most `depth` results are outstanding.  The dispatcher order collects the oldest one before it submits the microbatch that
reuses its lane, as DEFER and bench.py do; the other orders collect it as late as that bound allows, just before the last
stage steps that microbatch, so producers keep running ahead.  The rest are collected at the end."""
import contextlib
import os

import numpy as np

SCHEDULES = ("dispatcher", "stage_major", "consumer_first")


def _core(name, n_stages, n_items, depth):
    if name == "dispatcher":
        for seq in range(n_items):
            yield ("submit", seq)
            for st in range(n_stages):
                yield ("step", st, seq)
    elif name == "stage_major":
        for w in range(0, n_items, depth):
            window = range(w, min(w + depth, n_items))
            for seq in window:
                yield ("submit", seq)
            for st in range(n_stages):
                for seq in window:
                    yield ("step", st, seq)
    elif name == "consumer_first":
        for seq in range(n_items):
            for st in range(n_stages - 1, 0, -1):
                yield ("step", st, seq)
            yield ("submit", seq)
            yield ("step", 0, seq)
    else:
        raise ValueError(f"unknown schedule {name!r}; one of {SCHEDULES}")


def schedule(name, n_stages, n_items, depth):
    """The events of step order `name` for `n_items` microbatches through `n_stages` stages of `depth` lanes."""
    events, inflight = [], []
    collect_at = "submit" if name == "dispatcher" else "step"
    for ev in _core(name, n_stages, n_items, depth):
        last = ev[0] == "step" and ev[1] == n_stages - 1
        if (ev[0] == "submit" or last) and ev[0] == collect_at and len(inflight) == depth:
            events.append(("result", inflight.pop(0)))  # ev starts the microbatch that reuses the oldest result's lane
        if last:
            inflight.append(ev[2])
        events.append(ev)
    return events + [("result", seq) for seq in inflight]


def stage_names(model, cuts):
    return [model.input._keras_history[0].name] + list(cuts) + [model.output._keras_history[0].name]


@contextlib.contextmanager
def open_chain(model, cuts, dtype="float32", batch=1, depth=2, devices=None, use_graph=True, wait_timeout_ms=20000):
    """Build the stages of `model` cut after `cuts`, link and finalize them; on exit sync, unlink and close every one."""
    from defer_b200 import dag_util
    from defer_b200.node import StageRunner
    names = stage_names(model, cuts)
    n = len(names) - 1
    runners = []
    try:
        for i in range(n):
            p = dag_util.construct_model(model, names[i], names[i + 1], part_name=f"part{i + 1}")
            runners.append(StageRunner.from_wire(p.to_json(), p.get_weights(), device=(devices[i] if devices else 0),
                                                 dtype=dtype, max_batch=batch, depth=depth, is_first=(i == 0),
                                                 is_last=(i == n - 1), finalize=False, use_graph=use_graph,
                                                 wait_timeout_ms=wait_timeout_ms))
        for i in range(n - 1):
            runners[i].link_to(runners[i + 1])
        for r in runners:
            r.finalize()
        yield runners
    finally:
        for r in runners:
            try:
                r.sync()
            except Exception:
                pass
        if len(runners) > 1:
            for r in runners:
                try:
                    r.unlink()
                except Exception:
                    pass
        for r in runners:
            r.close()


def run_chain(model, cuts, inputs, dtype="float32", depth=2, devices=None, use_graph=True, pin=False,
              wait_timeout_ms=20000, order="dispatcher"):
    """Run microbatch `seq` = `inputs[seq]` through the chain in step order `order`.  Returns a dict:
      results  the last stage's output per seq
      status   per stage, "ok" or the error its status() raised
      links    copy hop (DEFER_HOP unset or "copy") only: per link, per lane, (producer output buffer, consumer input slot)
               after the last microbatch; None for the hops that store straight into the consumer's slot
      kernels  the kernel of every op of every stage"""
    from defer_b200 import _cabi as A
    inputs = [np.ascontiguousarray(x, dtype=x.dtype) for x in inputs]
    with open_chain(model, cuts, dtype=dtype, batch=inputs[0].shape[0], depth=depth, devices=devices, use_graph=use_graph,
                    wait_timeout_ms=wait_timeout_ms) as runners:
        if pin:
            for x in inputs:
                runners[0].pin(x)
        results = [None] * len(inputs)
        for ev in schedule(order, len(runners), len(inputs), depth):
            if ev[0] == "submit":
                runners[0].submit(ev[1], inputs[ev[1]])
            elif ev[0] == "step":
                runners[ev[1]].step(ev[2])
            else:
                results[ev[1]] = runners[-1].result(ev[1])
        for r in runners:
            r.sync()
        status = []
        for r in runners:
            try:
                r.status()
                status.append("ok")
            except A.DeferError as e:
                status.append(str(e))
        links = None
        if os.environ.get("DEFER_HOP", "copy") == "copy":
            links = [[(p.read_buffer(p.plan.output_buf, lane), c.read_buffer(c.plan.input_buf, lane)) for lane in range(depth)]
                     for p, c in zip(runners, runners[1:])]
        kernels = [[r.op_info(i)["kernel"] for i in range(len(r.plan.ops))] for r in runners]
    return {"results": results, "status": status, "links": links, "kernels": kernels}


# ------------------------------------------------------------------------------------------------ checking
def _rel(a, b):
    return float(np.max(np.abs(a.astype(np.float64) - b))) / max(float(np.max(np.abs(b.astype(np.float64)))), 1e-30)


def diagnose(results, refs, depth):
    """(seq, kind, message) for every result that is not bitwise its own reference.  kind:
      stale        it is the result of seq - depth: the slot still held the previous microbatch (ready raised too early)
      overwritten  it is the result of seq + depth: the lane ran that one over it
      other_seq    it is the result of a microbatch of another lane: a lane mix-up
      torn         it equals no reference: a partly stale or torn slot"""
    bad = []
    for seq, y in enumerate(results):
        if np.array_equal(y, refs[seq]):
            continue
        same = [j for j in range(len(refs)) if j != seq and np.array_equal(y, refs[j])]
        if seq - depth in same:
            kind, msg = "stale", f"equals the result of seq {seq - depth} (stale slot, or ready flag raised too early)"
        elif seq + depth in same:
            kind, msg = "overwritten", f"equals the result of seq {seq + depth} (overwritten by the lane's next microbatch)"
        elif same:
            kind, msg = "other_seq", f"equals the result of seq {same[0]} (lane mix-up)"
        else:
            kind, msg = "torn", f"equals no reference, rel err {_rel(y, refs[seq]):.3e} (partly stale or torn slot)"
        bad.append((seq, kind, f"seq {seq} (lane {seq % depth}): {msg}"))
    return bad


def check_results(results, refs, depth):
    assert len(results) == len(refs), (len(results), len(refs))
    bad = diagnose(results, refs, depth)
    assert not bad, "\n".join(m for _, _, m in bad)


def n_distinct(refs, rel=1e-3):
    """How many references differ from every other one bitwise and by more than `rel` (max-norm relative)."""
    return sum(all(j == i or (not np.array_equal(a, b) and _rel(a, b) > rel) for j, b in enumerate(refs))
               for i, a in enumerate(refs))
