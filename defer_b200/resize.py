"""Keras ``load_img(target_size=..., interpolation=...)`` resize, restated from Pillow's ``Image.resize`` on uint8 images.

This module owns the per-axis table format that both the host restatement (``resize_image``) and the planner's
``DEFER_OP_RESIZE`` use, so the two cannot drift apart.  For one axis of ``in_len`` source pixels resized to ``out_len``,
``resize_tables`` gives int32 arrays

* ``first[out]``        - the first source index output ``i`` reads,
* ``count[out]``        - how many consecutive source indices it reads (``1 <= count <= ksize``, ``first + count <= in_len``),
* ``coef[out, ksize]``  - their weights in fixed point with ``PRECISION_BITS`` fractional bits (zero past ``count``),

and one pass over that axis computes, per channel, ``clamp((2**21 + sum_k src[first + k] * coef[k]) >> 22, 0, 255)``.

The filters are Pillow's 8-bit path (``libImaging/Resample.c``): support scaled by ``max(in/out, 1)``, weights normalised
by their sequential sum in double precision and rounded half away from zero.  Pillow resizes the horizontal axis first,
rounds to uint8, then the vertical axis, and skips an axis whose size does not change; ``resize_image`` does the same.
``nearest`` is Pillow's affine nearest path: the source index is ``int(xo)``, where ``xo`` starts at ``0.5 * in/out`` and
accumulates ``+= in/out`` in double precision (the closed form ``floor((i + 0.5) * in/out)`` differs from it at some
sizes).  It fits the same tables with one tap of weight ``1 << 22``: an exact gather, so a 2-D nearest resize is the
horizontal gather followed by the vertical one.

``keep_aspect_ratio=True`` is Keras' centred crop (``keras_crop_box``) given to Pillow as ``Image.resize(..., box=...)``.
A box ``(start, end)`` on an axis only moves the filter: Pillow's ``precompute_coeffs`` takes ``scale = (end - start) /
out_len`` and ``center = start + (i + 0.5) * scale``, and clamps the taps to the whole axis ``[0, in_len)``, not to the box,
so outputs near the box's edges read pixels just outside it (a box resize is not a crop followed by a resize).  Nearest
starts at ``start + 0.5 * scale``.  Pillow skips an axis only when its size does not change *and* its box is the whole
axis; an axis that keeps its size under a partial box is resampled.  A box may be empty (``start == end``, from extreme
aspect ratios): every output then reads around ``start``, as Pillow does.
"""
from __future__ import annotations

import functools
import math
from typing import Tuple

import numpy as np

#: the ``interpolation=`` names Keras' ``load_img`` accepts (its default is "nearest")
INTERPOLATIONS = ("nearest", "bilinear", "bicubic", "hamming", "box", "lanczos")
#: fractional bits of the fixed-point weights (Pillow: 32 - 8 - 2)
PRECISION_BITS = 22


def _box(x: float) -> float:
    return 1.0 if -0.5 < x <= 0.5 else 0.0


def _bilinear(x: float) -> float:
    x = abs(x)
    return 1.0 - x if x < 1.0 else 0.0


_F32_054 = float(np.float32(0.54))   # Pillow writes 0.54f and 0.46f: single-precision constants in a double expression
_F32_046 = float(np.float32(0.46))


def _hamming(x: float) -> float:
    x = abs(x)
    if x == 0.0:
        return 1.0
    if x >= 1.0:
        return 0.0
    x = x * math.pi
    return math.sin(x) / x * (_F32_054 + _F32_046 * math.cos(x))


def _bicubic(x: float) -> float:
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x: float) -> float:
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


#: name -> (filter, support)
_FILTERS = {"box": (_box, 0.5), "bilinear": (_bilinear, 1.0), "hamming": (_hamming, 1.0),
            "bicubic": (_bicubic, 2.0), "lanczos": (_lanczos, 3.0)}


def check_interpolation(name) -> None:
    if name not in INTERPOLATIONS:
        raise ValueError(f"interpolation={name!r}: Keras' load_img accepts {', '.join(map(repr, INTERPOLATIONS))}")


def check_size(size, what: str = "image_size") -> Tuple[int, int]:
    """``size`` as ``(h, w)`` of positive ints, or a ValueError naming ``what``."""
    try:
        h, w = (int(v) for v in size)
        ok = (h, w) == tuple(size)
    except (TypeError, ValueError):
        ok = False
    if not ok or h < 1 or w < 1:
        raise ValueError(f"{what}={size!r}: expected (height, width), two positive integers")
    return h, w


def keras_crop_box(h: int, w: int, target) -> Tuple[int, int, int, int]:
    """The box Keras' ``load_img(target_size=target, keep_aspect_ratio=True)`` gives Pillow's ``Image.resize`` for an
    ``h`` x ``w`` image: ``(left, upper, right, lower)``, the largest centred box with the target's aspect ratio.

    Restated from Keras (``keras.utils.load_img``; ``tf.keras.utils.load_img`` since TF 2.9), where ``(width, height) =
    img.size`` and ``(target_width, target_height)`` is the target::

        crop_height = min(height, (width * target_height) // target_width)
        crop_width  = min(width,  (height * target_width) // target_height)
        hstart = (height - crop_height) // 2
        wstart = (width - crop_width) // 2
        img = img.resize((target_width, target_height), resample,
                         box=[wstart, hstart, wstart + crop_width, hstart + crop_height])

    Keras resizes only when ``img.size`` differs from the target; at the target this box is the whole image anyway."""
    th, tw = check_size(target, "target_size")
    h, w = check_size((h, w), "image size")
    crop_h = min(h, (w * th) // tw)
    crop_w = min(w, (h * tw) // th)
    hstart = (h - crop_h) // 2
    wstart = (w - crop_w) // 2
    return wstart, hstart, wstart + crop_w, hstart + crop_h


def _check_box(in_len: int, box) -> Tuple[int, int]:
    try:
        start, end = (int(v) for v in box)
        ok = (start, end) == tuple(box)
    except (TypeError, ValueError):
        ok = False
    if not ok or not 0 <= start <= end <= in_len or start >= in_len:
        raise ValueError(f"resize_tables: box={box!r} on an axis of {in_len}: needs integers 0 <= start <= end <= {in_len} "
                         f"and start < {in_len}")
    return start, end


def resize_tables(in_len: int, out_len: int, interpolation: str = "nearest",
                  box=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``(first, count, coef)`` of one axis: int32 ``[out_len]``, ``[out_len]`` and ``[out_len, ksize]`` (module docstring).
    ``box = (start, end)``: Pillow's ``resize(..., box=...)`` on this axis (None: the whole axis).

    Plain Python floats on purpose: every step is the double-precision operation Pillow's C code performs, in its order
    (a vectorised sum or a SIMD ``sin`` could round differently).  Pillow holds the box in single precision; integer
    coordinates are exact there up to 2^24."""
    check_interpolation(interpolation)
    if in_len < 1 or out_len < 1:
        raise ValueError(f"resize_tables: sizes must be positive, got {in_len} -> {out_len}")
    in0, in1 = (0, in_len) if box is None else _check_box(in_len, box)
    scale = (in1 - in0) / out_len
    first = np.empty(out_len, np.int32)
    count = np.empty(out_len, np.int32)
    if interpolation == "nearest":
        xo = in0 + scale * 0.5
        for i in range(out_len):
            # Pillow's affine nearest fills a pixel whose index leaves the image with 0; the accumulated position stays
            # below in_len for any size this engine can hold, and the clamp keeps the table valid regardless
            first[i] = min(int(xo), in_len - 1)
            xo += scale
        count[:] = 1
        return first, count, np.full((out_len, 1), 1 << PRECISION_BITS, np.int32)
    filt, filter_support = _FILTERS[interpolation]
    filterscale = max(scale, 1.0)
    support = filter_support * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    coef = np.zeros((out_len, ksize), np.int32)
    one = float(1 << PRECISION_BITS)
    for i in range(out_len):
        center = in0 + (i + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)
        hi = min(int(center + support + 0.5), in_len)
        w = [filt((k + lo - center + 0.5) * ss) for k in range(hi - lo)]
        ww = 0.0
        for v in w:
            ww += v
        for k, v in enumerate(w):
            if ww != 0.0:
                v /= ww
            coef[i, k] = int(v * one - 0.5) if v < 0 else int(v * one + 0.5)   # int() truncates, as the C cast does
        first[i], count[i] = lo, hi - lo
    return first, count, coef


def resize_axis(x: np.ndarray, axis: int, first: np.ndarray, count: np.ndarray, coef: np.ndarray) -> np.ndarray:
    """One pass of the tables over ``axis`` of the uint8 array ``x`` (what ``DEFER_OP_RESIZE`` computes on the GPU)."""
    x = np.asarray(x)
    if x.dtype != np.uint8:
        raise TypeError(f"resize_axis: expected uint8, got {x.dtype}")
    in_len = x.shape[axis]
    acc = np.full(x.shape[:axis] + (len(first),) + x.shape[axis + 1:], 1 << (PRECISION_BITS - 1), np.int64)
    bshape = [1] * x.ndim
    bshape[axis] = len(first)
    for k in range(coef.shape[1]):
        idx = np.minimum(first + k, in_len - 1)                  # taps past `count` have weight 0
        w = np.where(k < count, coef[:, k], 0).astype(np.int64).reshape(bshape)
        acc += np.take(x, idx, axis=axis).astype(np.int64) * w
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def check_keep_aspect_ratio(keep_aspect_ratio, image_size=None, max_image_size=None, resizes: bool = False) -> bool:
    """``keep_aspect_ratio=`` as a bool, or a ValueError: it must be a bool, and True needs a resizing ingress
    (``image_size=`` or ``max_image_size=``; ``resizes`` for ``resize_image``, which always has a target)."""
    if not isinstance(keep_aspect_ratio, (bool, np.bool_)):
        raise ValueError(f"keep_aspect_ratio={keep_aspect_ratio!r}: expected True or False, as Keras' load_img takes")
    if keep_aspect_ratio and not resizes and image_size is None and max_image_size is None:
        raise ValueError("keep_aspect_ratio=True crops each image as Keras' load_img does while resizing it, so it needs "
                         "image_size= or max_image_size= (items at the model input are not resized)")
    return bool(keep_aspect_ratio)


def crop_boxes(h: int, w: int, target, keep_aspect_ratio: bool):
    """``(width box, height box)`` of an ``h`` x ``w`` image resized to ``target``: ``(start, end)`` of Keras' crop
    (``keras_crop_box``) on each axis it does not cover whole, else None.  Both None without ``keep_aspect_ratio`` and
    at the target, where Keras does not resize."""
    if not keep_aspect_ratio or (h, w) == tuple(target):
        return None, None
    left, upper, right, lower = keras_crop_box(h, w, target)
    return (None if (left, right) == (0, w) else (left, right)), (None if (upper, lower) == (0, h) else (upper, lower))


def resize_image(x: np.ndarray, target_size, interpolation: str = "nearest", keep_aspect_ratio: bool = False) -> np.ndarray:
    """Resize uint8 RGB ``x`` of shape ``(h, w, 3)`` or ``(n, h, w, 3)`` to ``target_size = (height, width)``, bit for bit
    as Keras' ``load_img(path, target_size=..., interpolation=..., keep_aspect_ratio=...)`` does with Pillow's
    ``Image.resize``.

    Horizontal pass first, then vertical; an axis whose size does not change is not touched, and an image already at
    ``target_size`` comes back as a copy.  ``keep_aspect_ratio=True`` resizes Keras' centred crop (``keras_crop_box``)
    instead of the whole image, through Pillow's ``box=``; an axis that keeps its size but is cropped is then resampled.
    ``DEFER(..., image_size=(h, w), interpolation=..., keep_aspect_ratio=...)`` runs the same passes on the GPU."""
    check_interpolation(interpolation)
    th, tw = check_size(target_size, "target_size")
    keep = check_keep_aspect_ratio(keep_aspect_ratio, resizes=True)
    x = np.asarray(x)
    if x.dtype != np.uint8 or x.ndim not in (3, 4) or x.shape[-1] != 3:
        raise ValueError(f"resize_image: expected a uint8 RGB image (h, w, 3) or (n, h, w, 3), got {x.dtype} {x.shape}")
    h_ax, w_ax = x.ndim - 3, x.ndim - 2
    box_w, box_h = crop_boxes(x.shape[h_ax], x.shape[w_ax], (th, tw), keep)
    y = x.copy()
    if x.shape[w_ax] != tw or box_w is not None:
        y = resize_axis(y, w_ax, *resize_tables(x.shape[w_ax], tw, interpolation, box_w))
    if x.shape[h_ax] != th or box_h is not None:
        y = resize_axis(y, h_ax, *resize_tables(x.shape[h_ax], th, interpolation, box_h))
    return y


# ------------------------------------------------------------------------------------------------ frames of mixed sizes
# ``DEFER(..., max_image_size=(H, W))`` takes images of any size up to (H, W).  Each sample of a microbatch then carries
# its own tables in a fixed-size int32 block (``DEFER_RESIZE_SAMPLE_W`` / ``_H`` in include/defer_b200.h):
#
#     [h_in, w_in,
#      width axis:  (first, count) [W_out, 2],  taps [W_out, kw_w],
#      height axis: (first, count) [H_out, 2],  taps [H_out, kw_h]]
#
# with taps zero past ``count``, ``kw_w = kcap(W, W_out)`` and ``kw_h = kcap(H, H_out)``.  An axis whose length already
# equals the target gets the identity table (first = i, count 1, one tap of 2^22): an exact copy, which is what Pillow's
# skipping that axis gives.  With ``keep_aspect_ratio`` an axis keeps the identity table only when its crop box is the
# whole axis as well; a box's scale is at most ``in_len / out_len``, so ``kcap`` still bounds its taps.

def kcap(max_len: int, out_len: int, interpolation: str = "nearest") -> int:
    """Taps per output that ``resize_tables(n, out_len, interpolation)`` needs for every source length ``1 <= n <=
    max_len``.  Its ksize, ``2 * ceil(support * max(n / out_len, 1)) + 1``, does not decrease with ``n``, so this is the
    ksize at ``max_len``, computed with the same double-precision steps."""
    check_interpolation(interpolation)
    if max_len < 1 or out_len < 1:
        raise ValueError(f"kcap: sizes must be positive, got {max_len} -> {out_len}")
    if interpolation == "nearest":
        return 1
    support = _FILTERS[interpolation][1] * max(max_len / out_len, 1.0)
    return int(math.ceil(support)) * 2 + 1


@functools.lru_cache(maxsize=1024)
def axis_tables(in_len: int, out_len: int, interpolation: str = "nearest",
                box=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``(first, count, coef)`` of one axis of a per-sample block, memoised per (axis length, target, interpolation,
    box) - ``resize_tables`` is plain Python and costs milliseconds per new length, and a stream of a few resolutions
    repeats its axis lengths.  ``in_len == out_len`` with no box gives the identity table.  The arrays are read-only."""
    if in_len == out_len and box is None:
        t = (np.arange(out_len, dtype=np.int32), np.ones(out_len, np.int32),
             np.full((out_len, 1), 1 << PRECISION_BITS, np.int32))
    else:
        t = resize_tables(in_len, out_len, interpolation, box)
    for a in t:
        a.setflags(write=False)
    return t


def frame_block_ints(target, kw) -> int:
    """int32 values in one sample's block for a model input ``target = (H_out, W_out)`` and ``kw = (kw_w, kw_h)``."""
    (h_out, w_out), (kw_w, kw_h) = target, kw
    return 2 + w_out * (2 + kw_w) + h_out * (2 + kw_h)


def pack_frame_tables(hws, target, kw, interpolation: str = "nearest", keep_aspect_ratio: bool = False) -> np.ndarray:
    """The blocks of images of sizes ``hws = [(h, w), ...]``: int32 ``[len(hws), frame_block_ints(target, kw)]``.
    ``keep_aspect_ratio``: each image's tables resize its Keras crop (``keras_crop_box``)."""
    (h_out, w_out), (kw_w, kw_h) = target, kw
    blocks = np.zeros((len(hws), frame_block_ints(target, kw)), np.int32)
    for blk, (h, w) in zip(blocks, hws):
        blk[0], blk[1] = h, w
        off = 2
        boxes = crop_boxes(int(h), int(w), (h_out, w_out), keep_aspect_ratio)
        for in_len, out_len, k, box in ((w, w_out, kw_w, boxes[0]), (h, h_out, kw_h, boxes[1])):
            first, count, coef = axis_tables(int(in_len), out_len, interpolation, box)
            if coef.shape[1] > k:
                raise ValueError(f"pack_frame_tables: {in_len} -> {out_len} ({interpolation}) needs {coef.shape[1]} taps, "
                                 f"the block holds {k}")
            b = blk[off:off + 2 * out_len].reshape(out_len, 2)
            b[:, 0], b[:, 1] = first, count
            off += 2 * out_len
            blk[off:off + out_len * k].reshape(out_len, k)[:, :coef.shape[1]] = coef
            off += out_len * k
    return blocks


def check_frame(x, max_image_size) -> np.ndarray:
    """Queue item ``x`` of a ``max_image_size=(H, W)`` pipeline as a C-contiguous uint8 ``(k, h, w, 3)`` array (an
    ``(h, w, 3)`` image counts as ``k = 1``) with ``1 <= h <= H`` and ``1 <= w <= W``, or a ValueError naming the bound."""
    H, W = max_image_size
    bound = f"max_image_size=({H}, {W})"
    if not (isinstance(x, np.ndarray) and x.dtype == np.uint8):
        raise ValueError(f"{bound} takes uint8 RGB images (img_to_array(img).astype(np.uint8)), got "
                         f"{getattr(x, 'dtype', type(x).__name__)}; do not preprocess or resize them on the host")
    if x.ndim == 3:
        x = x[None]
    if x.ndim != 4 or x.shape[0] < 1 or x.shape[-1] != 3:
        raise ValueError(f"image shape {tuple(x.shape)} is not (k, h, w, 3), channels-last RGB ({bound})")
    h, w = x.shape[1:3]
    if not (1 <= h <= H and 1 <= w <= W):
        raise ValueError(f"a {h}x{w} image is outside {bound}: needs 1 <= h <= {H} and 1 <= w <= {W}")
    return np.ascontiguousarray(x)
