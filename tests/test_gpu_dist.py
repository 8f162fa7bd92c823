"""The real cross-GPU hop (reference: src/node.py:76-79,107-108 -> 89-90): one process per GPU under torchrun,
`Node.run` + CUDA-IPC link tokens + device flags over NVLink, checked numerically; plus the one-process
peer-access variant on distinct devices.  Needs >= 2 GPUs (skipped otherwise)."""
import os
import socket
import subprocess
import sys
from pathlib import Path

import pytest

from defer_b200 import _cabi as A
from defer_b200 import applications

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
ROOT = Path(__file__).resolve().parents[1]


def _n_gpus():
    try:
        return A.device_count()
    except Exception:
        return 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("coalesce", [1, 4])
def test_cross_process_hop_parity(coalesce):
    if _n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    env = dict(os.environ, HOP_COALESCE=str(coalesce), HOP_ITEMS="14")
    env.pop("CUDA_VISIBLE_DEVICES", None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(ROOT / "tests" / "dist_hop_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=540, env=env, cwd=str(ROOT))
    tail = (r.stdout[-3000:] + "\n--- stderr ---\n" + r.stderr[-3000:])
    assert r.returncode == 0 and "HOP_OK" in r.stdout, tail
    print(r.stdout[-500:])


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
