"""The one-process-per-GPU pipeline (reference: src/node.py:76-79,107-108 -> 89-90): `Node.run` on every rank under
torchrun, CUDA-IPC link tokens, each hop writing into an input slot mapped from another process, the result ring in shared
memory and `DistContext.shutdown`; plus the one-process peer-access variant on distinct devices.

Each case of tests/dist_cases.py is one torchrun launch of tests/dist_hop_worker.py on whatever GPUs are visible: rank r
on visible GPU r % n, so one H100 runs every case (its ranks time-slice the device and map each other's slots through
CUDA IPC), and more GPUs spread the ranks.  After torchrun has exited, this process runs the same DEFER pipeline in one
process (same model, cuts, dtype, depth, coalesce, ingress and knobs, every stage on GPU 0) on the same items and
requires:
  * every rank exited 0 and finished its teardown;
  * each item's output bitwise equal to its reference, in FIFO order (a mismatch says whose result it is);
  * the references pairwise distinct, or a stale slot could pass;
  * float items: three outputs within the parity bar of the fp64 oracle (1e-3 in fp32, 6e-2 in bf16);
  * the run's shared-memory control block gone.
The one-process references of the resizing and JPEG ingress are themselves bitwise the host's resize and decode
(tests/test_gpu_resize.py, test_gpu_resize_frames.py, test_gpu_resize_keep_aspect.py, test_gpu_jpeg_progressive.py)."""
import queue
import threading
from pathlib import Path

import numpy as np
import pytest

import dist_cases as D
import handover_check
from defer_b200 import _cabi as A
from defer_b200 import applications

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
ROOT = Path(__file__).resolve().parents[1]


def _n_gpus():
    try:
        return A.device_count()
    except Exception:
        return 0


def _one_process(case, items, monkeypatch):
    """The case's pipeline in this process, every stage on GPU 0: the output of each item, in order."""
    from defer_b200.dispatcher import DEFER
    from test_gpu_fold_affine import _knobs
    _knobs(monkeypatch, **D.knob_env(case))
    model = D.build_model(case)
    d = DEFER([0] * case["ranks"], **D.defer_kwargs(case))
    in_q, out_q = queue.Queue(), queue.Queue()
    for x in items:                     # queued before the feeder starts, as in the worker: the same groups
        in_q.put(x)
    err = []

    def run():
        try:
            d.run_defer(model, D.cuts(case, model), in_q, out_q)
        except BaseException as e:  # noqa: BLE001
            err.append(e)
    t = threading.Thread(target=run, daemon=True)
    t.start()
    try:
        assert d.wait_ready(600)
        outs = [out_q.get(timeout=300) for _ in items]
    finally:
        d.close()
        t.join(timeout=60)
    assert not err, err
    return model, outs


@pytest.mark.parametrize("case", D.CASES, ids=[c["id"] for c in D.CASES])
def test_one_process_per_gpu(case, tmp_path, monkeypatch):
    n_vis = _n_gpus()
    world = case["ranks"]
    port = D.free_port()
    out_dir = tmp_path / "out"
    out_dir.mkdir()
    code, log, secs = D.run_group(D.torchrun_cmd(world, port), env=D.launch_env(case, out_dir), cwd=str(ROOT),
                                  timeout=1200)
    tail = log[-6000:]
    assert code == 0, f"torchrun exited {code} after {secs:.0f} s\n{tail}"
    assert sorted(p.name for p in out_dir.glob("rank*.done")) == [f"rank{r}.done" for r in range(world)], tail
    assert not list(Path("/dev/shm").glob(f"defer_b200_{port}_*")), "the shared-memory control block outlived the run"
    outs = [np.load(out_dir / f"item_{i:03d}.npy") for i in range(case["items"])]

    items = D.make_items(case)
    model, refs = _one_process(case, items, monkeypatch)
    distinct = handover_check.n_distinct(refs)
    worst = None
    if case["ingress"] == "float":
        from oracle import keras_ref
        worst = 0.0
        for i in (0, len(items) // 2, len(items) - 1):
            worst = max(worst, keras_ref.rel_err(outs[i], keras_ref.predict(model.to_json(), model.get_weights(), items[i])))
    layout = D.rank_layout(world, n_vis)
    print(f"{case['id']}: {world} ranks on devices {[d for d, _ in layout]} ({layout[0][1]}), {case['model']}, "
          f"{case['dtype']}, depth {case['depth']}, coalesce {case['coalesce']}, ring {case['ring']}, hop {case['hop']}, "
          f"{case['ingress']} items: {len(items)}, torchrun {secs:.1f} s, "
          f"worst rel err of 3 vs oracle {'-' if worst is None else f'{worst:.3e}'}")
    assert distinct == len(items), "the references must be pairwise distinct, or a stale slot would pass"
    assert all(y.shape == (1, D.OUT_ELEMS) for y in outs), [y.shape for y in outs]
    handover_check.check_results(outs, refs, case["depth"])
    if worst is not None:
        assert worst <= D.TOL[case["dtype"]], worst


def test_pipeline_on_distinct_devices_bitwise(resnet50):
    """One process, stage i on GPU i (peer access): each of a distinct input per microbatch gets the answer of one stage on
    one GPU, bit for bit."""
    n = _n_gpus()
    if n < 2:
        pytest.skip("needs 2 GPUs")
    import handover_check as H
    from test_gpu_model import _items, _oracle, _rel, _single_stage
    k = min(n, 4)
    cuts = applications.default_cuts(resnet50, k)
    xs = _items(11, 700)
    run = H.run_chain(resnet50, cuts, xs, depth=3, devices=list(range(k)))
    assert run["status"] == ["ok"] * k
    assert _rel(run["results"][0], _oracle(resnet50, xs[0])) <= 1e-3
    H.check_results(run["results"], _single_stage(resnet50, xs), depth=3)
