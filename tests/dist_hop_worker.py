"""Worker of tests/test_gpu_dist.py: one process per GPU under torchrun.  Every rank runs the product's `Node.run`
(CUDA-IPC link tokens, device-flag hop over NVLink); rank 0 is also the dispatcher (`DEFER.run_defer`).  Rank 0
feeds a distinct seeded input per item and checks every result against a single-stage run of the same model on its own
GPU (bitwise: the reference hop is a lossless codec, src/node.py:76-79,89-90,107-108), three of them also against the CPU
oracle (<= 1e-3)."""
import os
import queue
import sys
import threading
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def main():
    from defer_b200 import _cabi
    _cabi.load()
    import torch
    from defer_b200 import applications
    from defer_b200.dispatcher import DEFER
    from defer_b200.dist import DistContext
    from defer_b200.node import Node, StageRunner

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local_rank = int(os.environ["LOCAL_RANK"])
    G = int(os.environ.get("HOP_COALESCE", "1"))
    depth = int(os.environ.get("HOP_DEPTH", "3"))
    n_items = int(os.environ.get("HOP_ITEMS", "14"))
    torch.cuda.set_device(local_rank)
    ctx = DistContext(ring=64, out_elems=1000, batch=G)
    node = Node(dist_ctx=ctx, device=local_rank)
    nt = threading.Thread(target=node.run, daemon=True)
    nt.start()
    ok = True
    if rank == 0:
        model = applications.ResNet50()
        cuts = applications.default_cuts(model, world)
        defer = DEFER(list(range(world)), dtype="float32", depth=depth, coalesce=G, linger_us=2000, dist=ctx,
                      wait_timeout_ms=20000)
        in_q, out_q = queue.Queue(), queue.Queue()
        t = threading.Thread(target=defer.run_defer, args=(model, cuts, in_q, out_q), daemon=True)
        t.start()
        assert defer.wait_ready(600), "pipeline did not come up"
        # one input per item: with inputs that repeat, a lane can hand over a stale slot and still give the right answer
        xs = [applications.synthetic_input(1, seed=100 + i) for i in range(n_items)]
        for x in xs:
            in_q.put(x)
        outs = [out_q.get(timeout=120) for _ in range(n_items)]
        from oracle import keras_ref
        single = StageRunner.from_model(model, device=local_rank, dtype="float32", max_batch=G, depth=1)
        try:
            whole = []
            for g in range(0, n_items, G):               # an item's result does not depend on its position in a group
                group = xs[g:g + G]
                y = single.predict(np.concatenate(group + [group[0]] * (G - len(group)), axis=0))
                whole += [y[i:i + 1].copy() for i in range(len(group))]
        finally:
            single.close()
        worst = 0.0
        for i, y in enumerate(outs):
            if y.shape != (1, 1000) or not np.array_equal(y, whole[i]):
                ok = False
                same = [j for j in range(n_items) if y.shape == (1, 1000) and np.array_equal(y, whole[j])]
                print(f"item {i}: pipeline over {world} GPUs differs from the single-stage result "
                      f"(it equals the result of items {same})", flush=True)
        for i in (0, n_items // 2, n_items - 1):
            e = keras_ref.rel_err(outs[i], keras_ref.predict(model.to_json(), model.get_weights(), xs[i]))
            worst = max(worst, e)
            if e > 1e-3:
                ok = False
                print(f"item {i}: rel err {e:.3e} against the oracle", flush=True)
        print(f"hop parity: {n_items} items over {world} GPUs, coalesce {G}, worst rel err of 3 vs oracle {worst:.3e}", flush=True)
        defer.close()
        t.join(timeout=30)
    ctx.shutdown(nt)
    if rank == 0:
        print("HOP_OK" if ok else "HOP_FAIL", flush=True)
        sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
