"""Run one conv shape through defer_k_conv a few times (a driver for profilers and for debugging one shape).
usage: run_one_conv.py fmt backend n h w cin cout k s pad [iters]"""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from defer_b200 import _cabi as A

lib = A.load()
import torch  # noqa: E402
import test_gpu_kernels as T  # noqa: E402

fmt = sys.argv[1]
backend = int(sys.argv[2])
n, h, w, cin, cout, k, s, pad = map(int, sys.argv[3:11])
iters = int(sys.argv[11]) if len(sys.argv) > 11 else 3
for i in range(iters):
    err, _, _ = T._conv_case(torch, lib, fmt, backend, n, h, w, cin, cout, k, s, pad, relu=True, residual=True, seed=i)
    print("err", err)
