"""Numpy restatement of `resize_frames_u8_kernel` (DEFER_OP_RESIZE, modes DEFER_RESIZE_SAMPLE_W / _H), clamps included.

Each sample reads its size and tables from its own int32 block (`resize.pack_frame_tables`).  Like the kernel, the
restatement clamps `h_in` / `w_in` into the slot, `first` into the source and `count` into `[0, min(kcap, in_len - first)]`,
and it asserts that every byte it reads lies inside the sample's image - so it also shows that no block content makes the
kernel read outside its slot."""
import numpy as np

from defer_b200.resize import PRECISION_BITS


def pack_slots(images, H, W):
    """The input slots as `defer_stage_submit_frames` fills them: image i's h*w*3 bytes at the start of slot i."""
    slots = np.zeros((len(images), H, W, 3), np.uint8)
    for s, im in zip(slots, images):
        s.reshape(-1)[:im.size] = im.reshape(-1)
    return slots


def _pass(x, axis, first, count, taps):
    in_len = x.shape[axis]
    shape = list(x.shape)
    shape[axis] = len(first)
    bshape = [1] * x.ndim
    bshape[axis] = len(first)
    acc = np.full(shape, 1 << (PRECISION_BITS - 1), np.int64)
    for k in range(taps.shape[1]):
        on = k < count
        idx = np.where(on, first + k, 0)
        assert (idx >= 0).all() and (idx < in_len).all(), "read outside the image"
        w = np.where(on, taps[:, k], 0).astype(np.int64).reshape(bshape)
        acc += np.take(x, idx, axis=axis).astype(np.int64) * w
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def split_block(block, target, kw):
    """(h_in, w_in, width (first, count), width taps, height (first, count), height taps) views of one block."""
    (h_out, w_out), (kw_w, kw_h) = target, kw
    off = 2
    parts = []
    for out_len, k in ((w_out, kw_w), (h_out, kw_h)):
        parts.append(block[off:off + 2 * out_len].reshape(out_len, 2))
        off += 2 * out_len
        parts.append(block[off:off + out_len * k].reshape(out_len, k))
        off += out_len * k
    assert off == block.size
    return (int(block[0]), int(block[1]), *parts)


def resize_frames_host(slots, blocks, target, kw):
    """What the SAMPLE_W and SAMPLE_H passes compute over input slots `(n, H, W, 3)`: `(mid, out)`, with `mid` the width
    pass `(n, H, W_out, 3)` (rows past a sample's height are not written: zero here) and `out` `(n, H_out, W_out, 3)`."""
    n, H, W, _ = slots.shape
    (h_out, w_out), (kw_w, kw_h) = target, kw
    mid = np.zeros((n, H, w_out, 3), np.uint8)
    out = np.zeros((n, h_out, w_out, 3), np.uint8)
    for s in range(n):
        h, w, bw, tw, bh, th = split_block(np.asarray(blocks[s], np.int64), target, kw)
        h, w = min(max(h, 1), H), min(max(w, 1), W)
        img = slots[s].reshape(-1)[:h * w * 3].reshape(h, w, 3)
        fw = np.clip(bw[:, 0], 0, w - 1)
        cw = np.clip(bw[:, 1], 0, np.minimum(kw_w, w - fw))
        mid[s, :h] = _pass(img, 1, fw, cw, tw)
        fh = np.clip(bh[:, 0], 0, h - 1)
        ch = np.clip(bh[:, 1], 0, np.minimum(kw_h, h - fh))
        out[s] = _pass(mid[s, :h], 0, fh, ch, th)
    return mid, out
