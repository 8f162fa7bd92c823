"""Test helper: numpy interpreter of a planner.Plan (host-logic check of fusion / folding on CPU).

Uses the oracle's layer arithmetic as the checker; never used by the product.  `run_op` applies one op to the buffers
it reads, so a GPU test can check a single op on the stage's own input buffers.
"""
import numpy as np

from defer_b200 import _cabi as A
from oracle import keras_ref as R


def run_op(plan, op, bufs, W):
    """Output of `op` (shaped like its output buffer) from `bufs` (buffer id -> NHWC array) and the weights `W`."""
    a = bufs[op.in0]
    t, l, b, r = op.pads
    if op.kind == A.OP_CONV:
        xp = np.pad(a, ((0, 0), (t, b), (l, r), (0, 0)))
        y = R.conv2d(xp, W[op.w_kernel], None, (op.sh, op.sw), "valid")
        if op.w_scale >= 0:
            y = y * W[op.w_scale]
        if op.w_shift >= 0:
            y = y + W[op.w_shift]
        if op.flags & A.FLAG_RESIDUAL:
            y = y + bufs[op.in1]
        if op.flags & A.FLAG_RELU:
            y = np.maximum(y, 0)
    elif op.kind == A.OP_MAXPOOL:
        y = R.maxpool2d(np.pad(a, ((0, 0), (t, b), (l, r), (0, 0))), (op.kh, op.kw), (op.sh, op.sw))
    elif op.kind == A.OP_GAP:
        y = a.mean(axis=(1, 2)).reshape(a.shape[0], 1, 1, -1)
    elif op.kind == A.OP_DENSE:
        y = a.reshape(a.shape[0], -1) @ W[op.w_kernel]
        if op.w_shift >= 0:
            y = y + W[op.w_shift]
        if op.flags & A.FLAG_RELU:
            y = np.maximum(y, 0)
        y = y.reshape(a.shape[0], 1, 1, -1)
    elif op.kind == A.OP_SOFTMAX:
        y = R.softmax(a.reshape(a.shape[0], -1)).reshape(a.shape)
    elif op.kind == A.OP_AFFINE:
        y = a * W[op.w_scale] + W[op.w_shift]
        if op.flags & A.FLAG_RELU:
            y = np.maximum(y, 0)
    elif op.kind == A.OP_RELU:
        y = np.maximum(a, 0)
    elif op.kind == A.OP_ADD:
        y = a + bufs[op.in1]
        if op.flags & A.FLAG_RELU:
            y = np.maximum(y, 0)
    elif op.kind == A.OP_PAD:
        y = np.pad(a, ((0, 0), (t, b), (l, r), (0, 0)))
    elif op.kind == A.OP_COPY:
        y = a
    else:
        raise ValueError(op.kind)
    h, w, c, _ = plan.bufs[op.out]
    return np.asarray(y).reshape(a.shape[0], h, w, c)


def run_plan(plan, x, dtype=np.float64):
    bufs = {plan.input_buf: np.asarray(x, dtype)}
    W = [w.astype(dtype) for w in plan.weights]
    for op in plan.ops:
        bufs[op.out] = np.asarray(run_op(plan, op, bufs, W), dtype)
    return bufs
