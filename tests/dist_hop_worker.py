"""Worker of tests/test_gpu_dist.py: one rank of a torchrun launch of one case of tests/dist_cases.py (JSON in the
DEFER_DIST_CASE environment variable).  Every rank runs the product's `Node.run` on visible GPU `local_rank % n` (CUDA-IPC
link tokens, hops into another process's input slot, the result ring in shared memory); rank 0 is also the dispatcher
(`DEFER.run_defer`), fed the case's items, and writes each item's output to item_<i>.npy in DEFER_DIST_OUT.  Every rank
writes rank<r>.done there once `DistContext.shutdown` has returned.  The worker checks nothing itself: the test process
compares the outputs with the same pipeline run in one process."""
import json
import os
import queue
import sys
import threading
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
for _p in (ROOT, ROOT / "tests"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))

import dist_cases as D  # noqa: E402


def main():
    from defer_b200 import _cabi
    _cabi.load()
    import torch
    from defer_b200.dispatcher import DEFER
    from defer_b200.dist import DistContext
    from defer_b200.node import Node

    case = json.loads(os.environ[D.CASE_ENV])
    out_dir = Path(os.environ[D.OUT_ENV])
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local_rank = int(os.environ["LOCAL_RANK"])
    device, backend = D.rank_layout(world, torch.cuda.device_count())[local_rank]
    ctx = DistContext(backend=backend, device=device, ring=case["ring"], out_elems=D.OUT_ELEMS, batch=case["coalesce"])
    node = Node(dist_ctx=ctx, device=device)
    nt = threading.Thread(target=node.run, daemon=True)
    nt.start()
    if rank == 0:
        model = D.build_model(case)
        items = D.make_items(case)
        defer = DEFER(list(range(world)), dist=ctx, **D.defer_kwargs(case))
        in_q, out_q = queue.Queue(), queue.Queue()
        for x in items:             # queued before the feeder starts: groups of `coalesce` in order, as in the reference
            in_q.put(x)
        err = []

        def run():
            try:
                defer.run_defer(model, D.cuts(case, model), in_q, out_q)
            except BaseException as e:  # noqa: BLE001
                err.append(e)
        t = threading.Thread(target=run, daemon=True)
        t.start()
        assert defer.wait_ready(600), "pipeline did not come up"
        print(f"rank 0: {case['id']}: {world} ranks on devices {[d for d, _ in D.rank_layout(world, torch.cuda.device_count())]}"
              f", backend {backend}", flush=True)
        for i in range(len(items)):
            np.save(out_dir / f"item_{i:03d}.npy", out_q.get(timeout=300))
        defer.close()
        t.join(timeout=30)
        if err:
            raise err[0]
    ctx.shutdown(nt)
    (out_dir / f"rank{rank}.done").write_text("")


if __name__ == "__main__":
    main()
