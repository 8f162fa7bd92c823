"""Stage planner: a (sub-)model in wire format -> fused-op plan for ``defer_stage_create``.

This is the host half of what ``model_from_json`` + ``_make_predict_function`` do on a reference node
(``src/node.py:31-37``): turn the layer list into something executable.  Here the
executable form is a short list of fused ops (``include/defer_b200.h``):

* ``[ZeroPadding2D] -> Conv2D -> [BatchNormalization] -> [Add(other)] -> [relu]`` becomes ONE
  ``DEFER_OP_CONV`` - bias and the inference-mode BN fold to a per-channel scale/shift
  (``y = acc*scale + shift``; moving statistics, so no reduction), the residual is an epilogue read.
* ``[ZeroPadding2D] -> MaxPooling2D`` becomes one ``DEFER_OP_MAXPOOL``.
* ``Dense(softmax)`` becomes ``DENSE`` (fp32 logits) + ``SOFTMAX``.
* anything that cannot fuse (a cut in the middle of a block) falls back to standalone
  ``AFFINE`` / ``RELU`` / ``ADD`` / ``PAD`` ops, so arbitrary cut points stay legal.

A follower is absorbed only when the tensor between the two layers has exactly one consumer and is
not the stage output - otherwise that tensor must exist in memory.

With ``preprocess="caffe"`` or ``"tf"`` (first stage only) the stage input is a uint8 RGB image and a
``PREPROCESS`` op (Keras' ``preprocess_input`` in that mode) writes the fp32 tensor the rest of the plan reads;
the library folds it into the fused RGB stem when it can.  With ``image_size=(h, w)`` as well, the stage input is a uint8
image of that size and up to two ``RESIZE`` ops (width, then height: Keras' ``load_img(target_size=...)`` through Pillow,
tables from ``resize.resize_tables``) bring it to the model's input size before ``PREPROCESS``.
With ``max_image_size=(H, W)`` instead, the stage input is a uint8 slot of that size per sample and two per-sample
``RESIZE`` ops (``RESIZE_SAMPLE_W``, then ``_H``) read each image's size and tables from a block that comes with it
(``resize.pack_frame_tables``); the plan records what the feeder needs to pack them in ``Plan.frames``.  With
``decode="jpeg"`` as well, the stage input is a byte slot of ``H * W * 3`` per sample holding one JPEG file, and a
``JPEG_DECODE`` op in front of the resize pair decodes it into the uint8 slot (``jpeg.pack_block``); with ``decode="png"``
the slot holds one PNG file (``png.slot_bytes(H, W)`` bytes) and a ``PNG_DECODE`` op takes that place (``png.pack_block``);
with ``decode="image"`` the slot of that size holds one JPEG or PNG file and an ``IMAGE_DECODE`` op decodes each sample
in its own format, told by the tag of its block (``image.pack_block``).
``keep_aspect_ratio=True`` resizes Keras' centred crop of each image instead (``resize.keras_crop_box``): with
``image_size`` the two ``RESIZE`` ops carry box tables, and an axis that keeps its length under a partial box is
resampled by an op whose ``mode`` names its axis (``RESIZE_W`` / ``_H``); with ``max_image_size`` the feeder packs each
image's box tables (``Plan.frames["keep_aspect_ratio"]``).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import _cabi as A
from . import keras_like as K
from .applications import caffe_shift, check_model_preprocess, check_preprocess
from .jpeg import check_decode
from .image import DECODES
from .resize import check_interpolation, check_keep_aspect_ratio, check_size, crop_boxes, kcap, resize_tables


def same_pad(size: int, k: int, s: int) -> Tuple[int, int]:
    """TF 'SAME': total = max((ceil(size/s)-1)*s + k - size, 0), the odd element goes after."""
    out = -(-size // s)
    total = max((out - 1) * s + k - size, 0)
    return total // 2, total - total // 2


@dataclass(eq=False)
class PlanOp:
    kind: int
    in0: int
    out: int
    in1: int = -1
    kh: int = 1
    kw: int = 1
    sh: int = 1
    sw: int = 1
    pads: Tuple[int, int, int, int] = (0, 0, 0, 0)   # t, l, b, r
    flags: int = 0
    w_kernel: int = -1
    w_scale: int = -1
    w_shift: int = -1
    mode: int = 0                                     # PREPROCESS: A.PRE_CAFFE | A.PRE_TF
    layers: List[str] = field(default_factory=list)   # reference layer names fused into this op
    # planner-only state
    scale: Optional[np.ndarray] = None                # float64 while folding
    shift: Optional[np.ndarray] = None


@dataclass
class Plan:
    bufs: List[Tuple[int, int, int, int]]             # (h, w, c, elem)
    ops: List[PlanOp]
    weights: List[np.ndarray]
    input_buf: int
    output_buf: int
    input_shape: Tuple[int, ...]
    output_shape: Tuple[int, ...]
    tensor_buf: Dict[str, int]                        # layer name -> buffer id holding its output (if materialised)
    # max_image_size=: {"max_image_size": (H, W), "target": (H_out, W_out), "kw": (kw_w, kw_h), "interpolation": name},
    # plus "keep_aspect_ratio": True when that is on, what the stage's feeder needs to pack each image's table block
    # (resize.pack_frame_tables); None otherwise
    frames: Optional[dict] = None
    # decode="jpeg" / "png": the stage takes JPEG / PNG files (each with its jpeg.pack_block / png.pack_block block after its
    # table block); None otherwise
    decode: Optional[str] = None

    def describe(self) -> str:
        lines = []
        for i, op in enumerate(self.ops):
            lines.append(f"[{i:2d}] {A.KIND_NAMES[op.kind]:8s} b{op.in0}" + (f"+b{op.in1}" if op.in1 >= 0 else "") +
                         f" -> b{op.out} {self.bufs[op.out][:3]} flags={op.flags} <- {','.join(op.layers)}")
        return "\n".join(lines)


def _hwc(shape) -> Tuple[int, int, int]:
    s = tuple(shape[1:])
    if len(s) == 3:
        return int(s[0]), int(s[1]), int(s[2])
    if len(s) == 1:
        return 1, 1, int(s[0])
    raise ValueError(f"unsupported tensor rank {shape}")


def plan_stage(model: K.Model, is_first: bool, is_last: bool, preprocess: Optional[str] = None,
               image_size: Optional[Tuple[int, int]] = None, interpolation: str = "nearest",
               max_image_size: Optional[Tuple[int, int]] = None, decode: Optional[str] = None,
               keep_aspect_ratio: bool = False) -> Plan:
    check_decode(decode, preprocess, image_size, max_image_size, DECODES)
    if preprocess is not None:
        check_preprocess(preprocess)
        if not is_first:
            raise ValueError(f"preprocess={preprocess!r}: only the first stage takes images")
        check_model_preprocess(model, preprocess)
    check_interpolation(interpolation)
    if image_size is not None:
        image_size = check_size(image_size)
        if preprocess is None:
            raise ValueError(f"image_size={image_size}: resizing takes uint8 images and needs preprocess= (float items "
                             "are already preprocessed, and Keras resizes before preprocessing)")
    if max_image_size is not None:
        max_image_size = check_size(max_image_size, "max_image_size")
        if preprocess is None:
            raise ValueError(f"max_image_size={max_image_size}: resizing takes uint8 images and needs preprocess= (float "
                             "items are already preprocessed, and Keras resizes before preprocessing)")
        if image_size is not None:
            raise ValueError(f"max_image_size={max_image_size} and image_size={image_size}: give one (image_size: every "
                             "image has that size; max_image_size: each image has its own size up to that bound)")
    keep = check_keep_aspect_ratio(keep_aspect_ratio, image_size, max_image_size)
    nodes = list(model.iter_nodes())
    # names as recorded at map time (tensor histories may be re-tagged later by Input(tensor=...))
    order = [l.name for l, _ in nodes]
    inputs_of: Dict[str, List[str]] = {l.name: (ins or []) for l, ins in nodes}
    layer_of: Dict[str, K.Layer] = {l.name: l for l, _ in nodes}
    in_name = next(l.name for l, ins in nodes if ins is None)
    out_name = order[-1]
    consumers: Dict[str, int] = {n: 0 for n in order}
    for n in order:
        for p in inputs_of[n]:
            consumers[p] += 1

    # static shape inference over this sub-graph (layer.output may belong to another call site)
    shapes: Dict[str, Tuple] = {}
    for l, ins in nodes:
        if ins is None:
            shapes[l.name] = tuple(model.input.shape)
        else:
            shapes[l.name] = tuple(l.compute_output_shape([shapes[p] for p in ins]))

    bufs: List[Tuple[int, int, int, int]] = []
    ops: List[PlanOp] = []
    weights: List[np.ndarray] = []
    tensor_buf: Dict[str, int] = {}          # tensor (layer name) -> buffer id
    producer: Dict[str, Optional[PlanOp]] = {}   # tensor -> op whose tail it is (None: stage input / alias)
    pending_pad: Dict[str, Tuple[str, Tuple[int, int, int, int]]] = {}  # pad tensor -> (source tensor, pads)

    def new_buf(shape, elem=A.BUF_ACT) -> int:
        h, w, c = _hwc(shape)
        bufs.append((h, w, c, elem))
        return len(bufs) - 1

    def add_weight(a: np.ndarray) -> int:
        weights.append(np.ascontiguousarray(a, dtype=np.float32))
        return len(weights) - 1

    def add_table(a: np.ndarray) -> int:       # RESIZE tables stay int32
        weights.append(np.ascontiguousarray(a, dtype=np.int32))
        return len(weights) - 1

    def emit(op: PlanOp) -> PlanOp:
        ops.append(op)
        return op

    def pos(op: PlanOp) -> int:
        return next(i for i, o in enumerate(ops) if o is op)

    def absorbable(t: str) -> bool:
        return consumers[t] == 1 and t != out_name

    def materialise(t: str) -> int:
        """Buffer id of tensor ``t`` (emits a standalone PAD if it is a deferred ZeroPadding2D)."""
        if t in pending_pad:
            src, pads = pending_pad.pop(t)
            sb = materialise(src)
            if bufs[sb][3] != A.BUF_ACT:
                sb = cast(src, sb, A.BUF_ACT)
            ob = new_buf(shapes[t])
            op = emit(PlanOp(A.OP_PAD, sb, ob, pads=pads, layers=[t]))
            tensor_buf[t] = ob
            producer[t] = op
        return tensor_buf[t]

    def cast(t: str, b: int, elem: int) -> int:
        h, w, c, _ = bufs[b]
        bufs.append((h, w, c, elem))
        nb = len(bufs) - 1
        emit(PlanOp(A.OP_COPY, b, nb, layers=[f"cast({t})"]))
        return nb

    def act_buf(t: str) -> int:
        b = materialise(t)
        if bufs[b][3] != A.BUF_ACT:
            b = cast(t, b, A.BUF_ACT)
            tensor_buf[t] = b
            producer[t] = None
        return b

    def source_with_pad(t: str, allow_pad: bool):
        """(buffer id, pads) for a conv/pool reading tensor ``t``; fuses a deferred ZeroPadding2D."""
        if allow_pad and t in pending_pad and consumers[t] == 1:
            src, pads = pending_pad.pop(t)
            return materialise(src), pads, [t]
        return materialise(t), (0, 0, 0, 0), []

    # stage input
    input_shape = tuple(shapes[in_name][1:])
    frames = None
    if preprocess is None:
        tensor_buf[in_name] = new_buf(shapes[in_name], A.BUF_F32 if is_first else A.BUF_ACT)
        input_buf = tensor_buf[in_name]
    else:
        if _hwc(shapes[in_name])[2] != 3 or len(shapes[in_name]) != 4:
            raise ValueError(f"preprocess={preprocess!r}: the input must be an RGB image (h, w, 3), got {shapes[in_name][1:]}")
        H, W, _ = _hwc(shapes[in_name])
        h, w = image_size or max_image_size or (H, W)
        input_shape = (h, w, 3)
        files, op_decode = {None: (A.BUF_U8, None), "jpeg": (A.BUF_JPEG, A.OP_JPEG_DECODE),
                            "png": (A.BUF_PNG, A.OP_PNG_DECODE), "image": (A.BUF_IMAGE, A.OP_IMAGE_DECODE)}[decode]
        input_buf = img = new_buf((None,) + input_shape, files)
        if decode is not None:
            # the files decode into the image slot the per-sample resize reads (jpeg / png / image.pack_block per file)
            img = emit(PlanOp(op_decode, img, new_buf((None,) + input_shape, A.BUF_U8),
                              layers=[f"load_img(decode {decode} <={h}x{w})"])).out
        if max_image_size is not None:
            # images of mixed sizes up to (h, w): both passes always, the tables come with each image
            # a crop box's scale is at most the axis' own, so kcap bounds the taps with keep_aspect_ratio as well
            kw = (kcap(w, W, interpolation), kcap(h, H, interpolation))
            how = interpolation + (", keep_aspect_ratio" if keep else "")
            op_w = emit(PlanOp(A.OP_RESIZE, img, new_buf((None, h, W, 3), A.BUF_U8), kw=kw[0], mode=A.RESIZE_SAMPLE_W,
                               layers=[f"load_img(width <={w}->{W}, {how})"]))
            img = emit(PlanOp(A.OP_RESIZE, op_w.out, new_buf((None, H, W, 3), A.BUF_U8), kw=kw[1], mode=A.RESIZE_SAMPLE_H,
                              layers=[f"load_img(height <={h}->{H}, {how})"])).out
            frames = {"max_image_size": (h, w), "target": (H, W), "kw": kw, "interpolation": interpolation}
            if keep:
                frames["keep_aspect_ratio"] = True
        # Pillow resizes the width first and skips an axis whose size does not change and whose box is the whole axis
        # (so does Keras: no resize at all when the image is already at target_size).  An axis that keeps its size under
        # a partial box is resampled; its op names the axis in `mode`, as its shapes cannot.
        box_w, box_h = crop_boxes(h, w, (H, W), keep)
        for axis, n_in, n_out, shape, box in (("width", w, W, (h, W, 3), box_w), ("height", h, H, (H, W, 3), box_h)):
            if (n_in == n_out and box is None) or frames is not None:
                continue
            first, count, coef = resize_tables(n_in, n_out, interpolation, box)
            crop = "" if box is None else f" box {box[0]}..{box[1]}"
            mode = 0 if n_in != n_out else (A.RESIZE_W if axis == "width" else A.RESIZE_H)
            op = emit(PlanOp(A.OP_RESIZE, img, new_buf((None,) + shape, A.BUF_U8), kw=coef.shape[1], mode=mode,
                             layers=[f"load_img({axis} {n_in}->{n_out}{crop}, {interpolation})"]))
            op.w_scale = add_table(np.stack([first, count], axis=1))
            op.w_kernel = add_table(coef)
            img = op.out
        op = emit(PlanOp(A.OP_PREPROCESS, img, new_buf(shapes[in_name], A.BUF_F32),
                         mode=A.PRE_MODES[preprocess], layers=[f"preprocess_input({preprocess})"]))
        if preprocess == "caffe":                     # tf: Keras hard-codes 127.5 and 1, no weights
            op.w_shift = add_weight(caffe_shift())
        tensor_buf[in_name] = op.out
    producer[in_name] = None

    for name in order:
        if name == in_name:
            continue
        layer = layer_of[name]
        ins = inputs_of[name]
        cn = layer.class_name
        if cn == "ZeroPadding2D":
            (t, b), (l, r) = layer.padding
            pending_pad[name] = (ins[0], (t, l, b, r))
            continue
        if cn == "Conv2D":
            kh, kw = layer.kernel_size
            sh, sw = layer.strides
            src, pads, fused = source_with_pad(ins[0], allow_pad=(layer.padding == "valid"))
            if layer.padding == "same":
                h, w, _ = _hwc(shapes[ins[0]])
                (pt, pb), (pl, pr) = same_pad(h, kh, sh), same_pad(w, kw, sw)
                pads = (pt, pl, pb, pr)
            if layer.activation not in (None, "relu"):
                raise ValueError(f"{name}: conv activation {layer.activation!r} unsupported")
            ws = layer.get_weights()
            cout = layer.filters
            op = PlanOp(A.OP_CONV, src, new_buf(shapes[name]), kh=kh, kw=kw, sh=sh, sw=sw, pads=pads,
                        flags=A.FLAG_RELU if layer.activation == "relu" else 0, layers=fused + [name])
            op.w_kernel = add_weight(ws[0])
            op.scale = np.ones(cout, np.float64)
            op.shift = ws[1].astype(np.float64) if layer.use_bias else np.zeros(cout, np.float64)
            emit(op)
            tensor_buf[name] = op.out
            producer[name] = op
            continue
        if cn == "BatchNormalization":
            g, b, m, v = (a.astype(np.float64) for a in layer.get_weights())
            inv = g / np.sqrt(v + layer.epsilon)
            p = producer.get(ins[0])
            if (p is not None and p.kind == A.OP_CONV and p.flags == 0 and absorbable(ins[0])):
                p.shift = (p.shift - m) * inv + b
                p.scale = p.scale * inv
                p.layers.append(name)
                tensor_buf[name] = p.out
                producer[name] = p
            else:
                src = act_buf(ins[0])
                op = emit(PlanOp(A.OP_AFFINE, src, new_buf(shapes[name]), layers=[name]))
                op.scale, op.shift = inv, b - m * inv
                tensor_buf[name] = op.out
                producer[name] = op
            continue
        if cn == "Activation":
            act = layer.activation
            if act == "linear":
                tensor_buf[name] = materialise(ins[0])
                producer[name] = None
                continue
            if act == "relu":
                p = producer.get(ins[0])
                if (p is not None and p.kind in (A.OP_CONV, A.OP_AFFINE, A.OP_ADD, A.OP_DENSE)
                        and not (p.flags & A.FLAG_RELU) and absorbable(ins[0])
                        and bufs[p.out][3] == A.BUF_ACT):
                    p.flags |= A.FLAG_RELU
                    p.layers.append(name)
                    tensor_buf[name] = p.out
                    producer[name] = p
                else:
                    src = act_buf(ins[0])
                    op = emit(PlanOp(A.OP_RELU, src, new_buf(shapes[name]), layers=[name]))
                    tensor_buf[name] = op.out
                    producer[name] = op
                continue
            if act == "softmax":
                src = materialise(ins[0])
                if bufs[src][3] != A.BUF_F32:
                    src = cast(ins[0], src, A.BUF_F32)
                op = emit(PlanOp(A.OP_SOFTMAX, src, new_buf(shapes[name], A.BUF_F32), layers=[name]))
                tensor_buf[name] = op.out
                producer[name] = op
                continue
            raise ValueError(f"{name}: activation {act!r}")
        if cn == "Add":
            terms = list(ins)
            # try to fold into the conv that was emitted last among the addends
            cand = [(pos(producer[t]), t) for t in terms
                    if producer.get(t) is not None and producer[t].kind == A.OP_CONV and producer[t].flags == 0
                    and absorbable(t)]
            fused_into = None
            if len(terms) == 2 and cand:
                cpos, t = max(cand)
                other = terms[1] if terms[0] == t else terms[0]
                ob = materialise(other)
                other_pos = -1 if producer.get(other) is None else pos(producer[other])
                # the residual must be ACT format, complete before the conv runs, and not the conv's own output
                if bufs[ob][3] == A.BUF_ACT and other_pos < cpos and ob != producer[t].out:
                    p = producer[t]
                    p.in1 = ob
                    p.flags |= A.FLAG_RESIDUAL
                    p.layers.append(name)
                    fused_into = p
            if fused_into is not None:
                tensor_buf[name] = fused_into.out
                producer[name] = fused_into
            else:
                acc = act_buf(terms[0])
                op = None
                for t in terms[1:]:
                    op = emit(PlanOp(A.OP_ADD, acc, new_buf(shapes[name]), in1=act_buf(t), layers=[name]))
                    acc = op.out
                tensor_buf[name] = acc
                producer[name] = op
            continue
        if cn == "MaxPooling2D":
            src, pads, fused = source_with_pad(ins[0], allow_pad=True)
            if bufs[src][3] != A.BUF_ACT:
                src = cast(ins[0], src, A.BUF_ACT)
            ph, pw = layer.pool_size
            sh, sw = layer.strides
            op = emit(PlanOp(A.OP_MAXPOOL, src, new_buf(shapes[name]), kh=ph, kw=pw, sh=sh, sw=sw, pads=pads,
                             layers=fused + [name]))
            tensor_buf[name] = op.out
            producer[name] = op
            continue
        if cn == "GlobalAveragePooling2D":
            op = emit(PlanOp(A.OP_GAP, act_buf(ins[0]), new_buf(shapes[name]), layers=[name]))
            tensor_buf[name] = op.out
            producer[name] = op
            continue
        if cn == "Flatten":
            # NHWC is already (H, W, C) row-major: Flatten is a re-interpretation of the same bytes
            # (the dense kernel takes F = h*w*c of its input buffer), so it aliases the buffer.
            tensor_buf[name] = act_buf(ins[0])
            producer[name] = None
            continue
        if cn == "Dense":
            src = act_buf(ins[0])
            ws = layer.get_weights()
            softmax = layer.activation == "softmax"
            if layer.activation not in (None, "relu", "softmax"):
                raise ValueError(f"{name}: dense activation {layer.activation!r}")
            ob = new_buf(shapes[name], A.BUF_F32 if softmax else A.BUF_ACT)
            op = emit(PlanOp(A.OP_DENSE, src, ob, flags=A.FLAG_RELU if layer.activation == "relu" else 0, layers=[name]))
            op.w_kernel = add_weight(ws[0])
            if layer.use_bias:
                op.w_shift = add_weight(ws[1])
            if softmax:
                op2 = emit(PlanOp(A.OP_SOFTMAX, ob, new_buf(shapes[name], A.BUF_F32), layers=[name + ":softmax"]))
                tensor_buf[name] = op2.out
                producer[name] = op2
            else:
                tensor_buf[name] = ob
                producer[name] = op
            continue
        raise ValueError(f"planner: unsupported layer class {cn} ({name})")

    out_buf = materialise(out_name)
    want = A.BUF_F32 if is_last else A.BUF_ACT
    if bufs[out_buf][3] != want:
        out_buf = cast(out_name, out_buf, want)
    if out_buf == input_buf:
        raise ValueError("stage computes nothing (output is its input)")

    # finalise folded scale/shift arrays
    for op in ops:
        if op.scale is not None:
            op.w_scale = add_weight(op.scale.astype(np.float32))
        if op.shift is not None:
            op.w_shift = add_weight(op.shift.astype(np.float32))
    return Plan(bufs=bufs, ops=ops, weights=weights, input_buf=input_buf, output_buf=out_buf,
                input_shape=input_shape, output_shape=tuple(shapes[out_name][1:]),
                tensor_buf=dict(tensor_buf), frames=frames, decode=decode)
