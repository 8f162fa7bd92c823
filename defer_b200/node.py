"""Stage runtime: the per-GPU counterpart of the reference compute node
(``src/node.py:19-127``).

``StageRunner`` owns one stage handle of ``libdefer_b200.so``: it is what a reference node holds after
``model_from_json`` + ``set_weights`` + ``_make_predict_function`` (``src/node.py:31-38``), and its
``step`` is the body of the hot loop ``_data_client`` (``src/node.py:103-108``) - except that the
whole recv -> predict -> send of one microbatch is a single asynchronous CUDA-graph launch:
wait-input-flag -> fused sm_90a kernels -> copy-engine hop into the next GPU's input slot -> release flags.

``Node`` keeps the reference's class name and thread roles for the one-process-per-GPU deployment
(``torchrun``): it receives its stage from the dispatcher (``_model_socket`` / ``_weights_socket``
analogue over ``torch.distributed``), wires the NVLink hop with CUDA-IPC link tokens and then runs
the data loop until the dispatcher says stop.
"""
from __future__ import annotations

import ctypes as C
import time
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _cabi as A
from . import keras_like as K
from .node_state import NodeState
from .planner import Plan, plan_stage
from . import image, png
from .jpeg import BLOCK_INTS, check_jpeg, pack_block
from .resize import check_frame, pack_frame_tables

DTYPE_TO_FMT = {
    "float32": A.FMT_BF16X2,        # fp32 parity path on the tensor cores (bf16x3 split, fp32 accumulate)
    "fp32": A.FMT_BF16X2,
    "float32_simt": A.FMT_F32,      # exact fp32 FFMA everywhere (cross-check path)
    "bfloat16": A.FMT_BF16,
    "bf16": A.FMT_BF16,
}


def parse_device(d: Union[int, str]) -> int:
    """``computeNodes[i]`` of the reference is an IP (``src/dispatcher.py:45-55``); here a GPU ordinal
    or a ``"cuda:i"`` string."""
    if isinstance(d, (int, np.integer)):
        return int(d)
    s = str(d).strip()
    if s.startswith("cuda:"):
        return int(s[5:])
    if s.isdigit():
        return int(s)
    raise ValueError(f"compute node {d!r}: expected a GPU ordinal or 'cuda:<i>'")


_STREAMS_PER_DEVICE: Dict[int, int] = {}
MAX_STREAMS_PER_DEVICE = 28   # of CUDA_DEVICE_MAX_CONNECTIONS=32 (see _cabi.load)


class StageRunner:
    """One pipeline stage resident on one GPU."""

    def __init__(self, plan: Plan, device: int = 0, fmt: int = A.FMT_BF16X2, batch: int = 1, depth: int = 2,
                 is_first: bool = True, is_last: bool = True, conv_backend: int = 0, use_graph: bool = True,
                 wait_timeout_ms: int = 0, name: str = "stage"):
        self.lib = A.load()
        self.plan = plan
        self.name = name
        self.device, self.fmt, self.batch, self.depth = int(device), int(fmt), int(batch), int(depth)
        self.is_first, self.is_last = bool(is_first), bool(is_last)
        self.handle = C.c_void_p()
        self._pinned: Dict[int, tuple] = {}
        self._marks: Dict[int, int] = {}
        self._ptr_arrays: Dict[int, object] = {}
        self._streams = 0
        if not (is_first and is_last):
            used = _STREAMS_PER_DEVICE.get(self.device, 0)
            if used + self.depth > MAX_STREAMS_PER_DEVICE:
                raise RuntimeError(
                    f"device {self.device}: {used} lane streams already live, {self.depth} more would exceed "
                    f"{MAX_STREAMS_PER_DEVICE} hardware work queues - flag-waiting lanes could block their own "
                    "producer.  Use fewer stages per GPU or a smaller depth.")
        # a stage planned with preprocess= takes uint8 images (Keras preprocessing in that mode runs on the GPU)
        self.in_dtype = np.uint8 if plan.bufs[plan.input_buf][3] == A.BUF_U8 else np.float32
        # the Keras mode of the stage's PREPROCESS op, for messages (None: no preprocessing; the library refuses a bad mode)
        pre_modes = [o.mode for o in plan.ops if o.kind == A.OP_PREPROCESS]
        self.preprocess = {v: k for k, v in A.PRE_MODES.items()}.get(pre_modes[0]) if pre_modes else None
        # planned with image_size=: the stage resizes its images to the model input first (for messages)
        self.resizes = any(o.kind == A.OP_RESIZE for o in plan.ops)
        # planned with max_image_size=: images of mixed sizes, fed by submit_frames with their table blocks
        self.frames = plan.frames
        # "jpeg" / "png" / "image": fed by submit_jpegs / submit_pngs / submit_images, files with their blocks
        self.decode = plan.decode
        self._tables: Dict[int, tuple] = {}          # per lane: blocks, sizes and images of its latest microbatch (kept alive)
        self.in_shape = (self.batch,) + tuple(plan.input_shape)
        self.out_shape = (self.batch,) + tuple(plan.output_shape)
        self.out_elems = int(np.prod(self.out_shape))

        cfg = A.StageConfig(abi_version=A.ABI_VERSION, device=self.device, fmt=self.fmt, batch=self.batch,
                            depth=self.depth, input_buf=plan.input_buf, output_buf=plan.output_buf,
                            is_first=int(is_first), is_last=int(is_last), conv_backend=int(conv_backend),
                            use_graph=int(use_graph), wait_timeout_ms=int(wait_timeout_ms))
        bufs = (A.BufDesc * len(plan.bufs))(*[A.BufDesc(*b) for b in plan.bufs])
        ops = (A.OpDesc * len(plan.ops))()
        for i, o in enumerate(plan.ops):
            t, l, b, r = o.pads
            ops[i] = A.OpDesc(kind=o.kind, in0=o.in0, in1=o.in1, out=o.out, kh=o.kh, kw=o.kw, sh=o.sh, sw=o.sw,
                              pad_t=t, pad_l=l, pad_b=b, pad_r=r, flags=o.flags, w_kernel=o.w_kernel,
                              w_scale=o.w_scale, w_shift=o.w_shift, mode=o.mode)
        n_w = len(plan.weights)
        wptrs = (C.c_void_p * max(n_w, 1))(*[w.ctypes.data for w in plan.weights])
        wbytes = (C.c_uint64 * max(n_w, 1))(*[w.nbytes for w in plan.weights])
        A.check(self.lib.defer_stage_create(C.byref(cfg), bufs, len(plan.bufs), ops, len(plan.ops), wptrs, wbytes,
                                            n_w, C.byref(self.handle)))
        self._streams = self.depth
        _STREAMS_PER_DEVICE[self.device] = _STREAMS_PER_DEVICE.get(self.device, 0) + self.depth
        self.finalized = False

    # ---- construction helpers
    @classmethod
    def from_model(cls, model: K.Model, device=0, dtype: str = "float32", max_batch: int = 1, depth: int = 1,
                   is_first: bool = True, is_last: bool = True, finalize: bool = True, preprocess: Optional[str] = None,
                   image_size: Optional[Tuple[int, int]] = None, interpolation: str = "nearest",
                   max_image_size: Optional[Tuple[int, int]] = None, decode: Optional[str] = None,
                   keep_aspect_ratio: bool = False, **kw) -> "StageRunner":
        """``preprocess="caffe"`` or ``"tf"`` (first stage only): inputs are uint8 RGB images ``(batch, h, w, 3)`` and the
        stage applies Keras' ``preprocess_input`` in that mode on the GPU (``"tf"`` for the ResNet V2 family).
        ``image_size=(h, w)`` (with ``preprocess``): inputs are uint8 RGB images of that size, resized on the GPU to the
        model's input as Keras' ``load_img(target_size=..., interpolation=...)`` does (``resize.resize_image``).
        ``max_image_size=(H, W)`` (with ``preprocess``, instead of ``image_size``): the same for images of any size up to
        ``(H, W)``, each resized from its own size; feed them with ``submit_frames`` / ``predict_frames``.
        ``decode="jpeg"`` (with ``preprocess`` and ``max_image_size``): inputs are baseline JPEG files of images up to
        ``(H, W)``, decoded on the GPU as Keras' ``load_img`` does (``jpeg.decode_jpeg``); feed them with
        ``submit_jpegs`` / ``predict_jpegs``.  ``decode="png"``: the same for non-interlaced PNG files (``png.decode_png``),
        fed with ``submit_pngs`` / ``predict_pngs``.  ``decode="image"``: either format, told apart per file by its first
        bytes as Pillow does (``image.decode_image``), in one microbatch; fed with ``submit_images`` / ``predict_images``.
        ``keep_aspect_ratio=True`` (with ``image_size`` or ``max_image_size``): each image's centred crop with the model
        input's aspect ratio is resized, as ``load_img(..., keep_aspect_ratio=True)`` does (``resize.keras_crop_box``)."""
        plan = plan_stage(model, is_first=is_first, is_last=is_last, preprocess=preprocess, image_size=image_size,
                          interpolation=interpolation, max_image_size=max_image_size, decode=decode,
                          keep_aspect_ratio=keep_aspect_ratio)
        fmt = dtype if isinstance(dtype, int) else DTYPE_TO_FMT[dtype]
        r = cls(plan, device=parse_device(device), fmt=fmt, batch=max_batch, depth=depth, is_first=is_first,
                is_last=is_last, name=model.name, **kw)
        if finalize and is_first and is_last:
            r.finalize()
        return r

    @classmethod
    def from_wire(cls, model_json, weights: Sequence[np.ndarray], **kw) -> "StageRunner":
        """What a reference node does with what it received (``src/node.py:31,34``)."""
        part = K.model_from_json(model_json)
        part.set_weights(weights)
        return cls.from_model(part, **kw)

    # ---- wiring
    def link_to(self, consumer: "StageRunner") -> None:
        A.check(self.lib.defer_stage_link(self.handle, consumer.handle))

    def export_link(self, role: int) -> bytes:
        buf = C.create_string_buffer(A.LINK_TOKEN_BYTES)
        A.check(self.lib.defer_stage_export_link(self.handle, role, buf))
        return buf.raw

    def import_link(self, role: int, token: bytes) -> None:
        buf = C.create_string_buffer(bytes(token), A.LINK_TOKEN_BYTES)
        A.check(self.lib.defer_stage_import_link(self.handle, role, buf))

    def finalize(self) -> None:
        A.check(self.lib.defer_stage_finalize(self.handle))
        self.finalized = True

    def unlink(self) -> None:
        A.check(self.lib.defer_stage_unlink(self.handle))

    # ---- steady state
    def _host_input(self, x) -> np.ndarray:
        """``x`` as the C-contiguous array the stage copies from.  A stage without preprocessing converts to float32.
        A preprocessing stage takes uint8 only: a float array may be ``img_to_array`` output or already preprocessed,
        and neither can be told apart from the other."""
        if self.frames is not None:
            raise ValueError(f"{self.name}: this stage takes images of mixed sizes up to max_image_size="
                             f"{self.frames['max_image_size']}; feed them with submit_frames / predict_frames")
        if self.in_dtype == np.uint8:
            if getattr(x, "dtype", None) != np.uint8:
                raise TypeError(f"{self.name}: this stage preprocesses uint8 RGB images on the GPU "
                                f"(preprocess={self.preprocess!r}) "
                                f"and got dtype {getattr(x, 'dtype', type(x).__name__)}; pass the image as "
                                "img_to_array(img).astype(np.uint8), not preprocessed or float data")
            if x.ndim != 4 or tuple(x.shape[1:]) != self.in_shape[1:]:   # e.g. channels-first: same bytes, wrong image
                raise ValueError(f"{self.name}: image shape {tuple(x.shape)} is not (k,) + {self.in_shape[1:]} "
                                 "(channels-last RGB" + (f", image_size={self.in_shape[1:3]}" if self.resizes else "") + ")")
            if not x.flags["C_CONTIGUOUS"]:
                x = np.ascontiguousarray(x)
                self._keep = x
            return x
        if not (isinstance(x, np.ndarray) and x.dtype == np.float32 and x.flags["C_CONTIGUOUS"]):
            x = np.ascontiguousarray(x, dtype=np.float32)
            self._keep = x
        return x

    def submit(self, seq: int, x: np.ndarray) -> None:
        """Enqueue the H2D copy of microbatch ``seq``.  ``x`` must stay alive and unmodified until the
        step has consumed it; arrays registered with ``pin`` (or from ``pinned_empty``) copy asynchronously."""
        x = self._host_input(x)
        if tuple(x.shape) != self.in_shape:
            raise ValueError(f"{self.name}: input shape {tuple(x.shape)} != stage input {self.in_shape}")
        A.check(self.lib.defer_stage_submit(self.handle, seq, x.ctypes.data, x.nbytes))

    def submit_part(self, seq: int, index: int, x: np.ndarray) -> None:
        """Coalesced ingress: copy the queue item ``x`` (``k`` samples, usually 1 - ``test/test.py:22``) into samples
        ``[index, index + k)`` of microbatch ``seq``.  Same lifetime rule as ``submit``."""
        x = self._host_input(x)
        if tuple(x.shape[1:]) != self.in_shape[1:]:
            raise ValueError(f"{self.name}: item shape {tuple(x.shape)} does not match stage input {self.in_shape}")
        A.check(self.lib.defer_stage_submit_part(self.handle, seq, index, x.shape[0], x.ctypes.data, x.nbytes))

    def submit_items(self, seq: int, items) -> None:
        """Coalesced ingress, one C call per group: ``items`` are C-contiguous arrays of the stage's input dtype (float32,
        or uint8 on a preprocessing stage) and identical shape ``(k,) + input_shape[1:]``; item i lands in samples
        ``[i*k, (i+1)*k)`` of microbatch ``seq``."""
        if self.in_dtype == np.uint8:
            for x in items:
                if self._host_input(x) is not x:
                    raise ValueError(f"{self.name}: submit_items needs C-contiguous items")
        n = len(items)
        ptrs = self._ptr_arrays.get(n)
        if ptrs is None:
            ptrs = self._ptr_arrays[n] = (C.c_void_p * n)()
        for i, x in enumerate(items):
            ptrs[i] = x.__array_interface__["data"][0]
        x0 = items[0]
        A.check(self.lib.defer_stage_submit_parts(self.handle, seq, 0, n, x0.shape[0], ptrs, x0.nbytes))

    def submit_frames(self, seq: int, index: int, frames) -> None:
        """Ingress of a ``max_image_size=(H, W)`` stage: ``frames`` is a list of uint8 RGB items ``(k, h, w, 3)`` (or
        ``(h, w, 3)``), each of its own size with ``1 <= h <= H`` and ``1 <= w <= W``; their samples go to samples
        ``[index, index + total k)`` of microbatch ``seq``, each with its table block.  One C call copies each image's own
        bytes and then the blocks.  Same lifetime rule as ``submit``."""
        if self.frames is None:
            raise ValueError(f"{self.name}: submit_frames needs a stage planned with max_image_size=")
        if self.decode is not None:
            what = "JPEG and PNG" if self.decode == "image" else self.decode.upper()
            raise ValueError(f"{self.name}: this stage takes {what} files; feed them with "
                             f"submit_{self.decode}s / predict_{self.decode}s")
        bound = self.frames["max_image_size"]
        images = []
        for x in frames:
            x = check_frame(x, bound)
            images.extend(x[j] for j in range(x.shape[0]))
        n = len(images)
        if not 0 <= index <= self.batch - n:
            raise ValueError(f"{self.name}: {n} images from sample {index} do not fit the microbatch of {self.batch}")
        hw = np.array([im.shape[:2] for im in images], np.int32).reshape(n, 2)
        tables = pack_frame_tables(hw, self.frames["target"], self.frames["kw"], self.frames["interpolation"],
                                   self.frames.get("keep_aspect_ratio", False))
        self._tables[seq % self.depth] = (tables, hw, images)
        ptrs = (C.c_void_p * n)(*[im.__array_interface__["data"][0] for im in images])
        A.check(self.lib.defer_stage_submit_frames(self.handle, seq, index, n, ptrs, hw.ctypes.data, tables.ctypes.data,
                                                   tables.nbytes))

    def predict_frames(self, frames) -> np.ndarray:
        """Single-stage ``model.predict`` of a ``max_image_size`` stage: the outputs of the samples of ``frames`` (see
        ``submit_frames``), in order."""
        self.submit_frames(0, 0, frames)
        self.step(0)
        n = sum(1 if np.ndim(x) == 3 else len(x) for x in frames)
        return self.result(0)[:n]

    def submit_jpegs(self, seq: int, index: int, items, infos=None) -> None:
        """Ingress of a ``decode="jpeg"`` stage: ``items`` is a list of JPEG files (``bytes``, ``bytearray``,
        ``memoryview`` or 1-D uint8 arrays), one image each, of sizes up to ``max_image_size``; they go to samples
        ``[index, index + len(items))`` of microbatch ``seq``, each with its resize and JPEG blocks.  The files' markers are
        parsed here (``jpeg.check_jpeg``: a refused file raises a ValueError and nothing is copied); one C call copies each
        file's own bytes and then the blocks.  ``infos``: the items' ``jpeg.check_jpeg`` headers when the caller has
        already checked them (the items are then ``bytes``).  Same lifetime rule as ``submit``."""
        self._refuse_images("submit_jpegs")
        if self.decode != "jpeg":
            raise ValueError(f"{self.name}: submit_jpegs needs a stage planned with decode='jpeg'")
        bound = self.frames["max_image_size"]
        if infos is None:
            items, infos = zip(*[check_jpeg(x, bound) for x in items]) if items else ((), ())
        files = items
        n = len(files)
        if not 1 <= n <= self.batch - index or index < 0:
            raise ValueError(f"{self.name}: {n} files from sample {index} do not fit the microbatch of {self.batch}")
        hw = np.array([(i.h, i.w) for i in infos], np.int32).reshape(n, 2)
        tables = pack_frame_tables(hw, self.frames["target"], self.frames["kw"], self.frames["interpolation"],
                                   self.frames.get("keep_aspect_ratio", False))
        nr = tables.shape[1]
        blocks = np.zeros((n, nr + BLOCK_INTS), np.int32)      # only the prefix each file uses is written and copied
        blocks[:, :nr] = tables
        for k, i in enumerate(infos):
            pack_block(i, blocks[k, nr:])
        sizes = np.array([len(f) for f in files], np.uint64)
        self._tables[seq % self.depth] = (blocks, sizes, files)
        ptrs = (C.c_void_p * n)(*[C.cast(C.c_char_p(f), C.c_void_p).value for f in files])
        A.check(self.lib.defer_stage_submit_jpegs(self.handle, seq, index, n, ptrs, sizes.ctypes.data, blocks.ctypes.data,
                                                  blocks.nbytes))

    def predict_jpegs(self, items) -> np.ndarray:
        """Single-stage ``model.predict`` of a ``decode="jpeg"`` stage: the outputs of the JPEG files ``items``, in order."""
        self.submit_jpegs(0, 0, items)
        self.step(0)
        return self.result(0)[:len(items)]

    def submit_pngs(self, seq: int, index: int, items, infos=None) -> None:
        """Ingress of a ``decode="png"`` stage, as ``submit_jpegs``: ``items`` are PNG files, their chunks are walked here
        (``png.check_png``: a refused file raises a ValueError and nothing is copied), and one C call copies each file's
        own bytes and then its resize block and the part of its PNG block it uses."""
        self._refuse_images("submit_pngs")
        if self.decode != "png":
            raise ValueError(f"{self.name}: submit_pngs needs a stage planned with decode='png'")
        bound = self.frames["max_image_size"]
        if infos is None:
            items, infos = zip(*[png.check_png(x, bound) for x in items]) if items else ((), ())
        files = items
        n = len(files)
        if not 1 <= n <= self.batch - index or index < 0:
            raise ValueError(f"{self.name}: {n} files from sample {index} do not fit the microbatch of {self.batch}")
        hw = np.array([(i.h, i.w) for i in infos], np.int32).reshape(n, 2)
        tables = pack_frame_tables(hw, self.frames["target"], self.frames["kw"], self.frames["interpolation"],
                                   self.frames.get("keep_aspect_ratio", False))
        nr = tables.shape[1]
        blocks = np.zeros((n, nr + png.BLOCK_INTS), np.int32)  # only the prefix each file uses is written and copied
        blocks[:, :nr] = tables
        for k, i in enumerate(infos):
            png.pack_block(i, blocks[k, nr:])
        sizes = np.array([len(f) for f in files], np.uint64)
        self._tables[seq % self.depth] = (blocks, sizes, files)
        ptrs = (C.c_void_p * n)(*[C.cast(C.c_char_p(f), C.c_void_p).value for f in files])
        A.check(self.lib.defer_stage_submit_pngs(self.handle, seq, index, n, ptrs, sizes.ctypes.data, blocks.ctypes.data,
                                                 blocks.nbytes))

    def predict_pngs(self, items) -> np.ndarray:
        """Single-stage ``model.predict`` of a ``decode="png"`` stage: the outputs of the PNG files ``items``, in order."""
        self.submit_pngs(0, 0, items)
        self.step(0)
        return self.result(0)[:len(items)]

    def _refuse_images(self, call: str) -> None:
        if self.decode == "image":
            raise ValueError(f"{self.name}: {call} needs a single-format stage; this stage takes JPEG and PNG files told "
                             "apart per file: feed them with submit_images / predict_images")

    def submit_images(self, seq: int, index: int, items, checked=None) -> None:
        """Ingress of a ``decode="image"`` stage, as ``submit_jpegs``: each of ``items`` is a JPEG or a PNG file, told
        apart by its first bytes and checked here (``image.check_image``: a refused file raises a ValueError and nothing
        is copied).  One C call copies each file's own bytes and then its resize block and the part of its tagged block
        that it uses.  ``checked``: the items' ``image.check_image`` results when the caller has already checked them
        ((bytes, kind, header) each).  Same lifetime rule as ``submit``."""
        if self.decode != "image":
            raise ValueError(f"{self.name}: submit_images needs a stage planned with decode='image'")
        bound = self.frames["max_image_size"]
        if checked is None:
            checked = [image.check_image(x, bound) for x in items]
        n = len(checked)
        if not 1 <= n <= self.batch - index or index < 0:
            raise ValueError(f"{self.name}: {n} files from sample {index} do not fit the microbatch of {self.batch}")
        files = [d for d, _, _ in checked]
        hw = np.array([(i.h, i.w) for _, _, i in checked], np.int32).reshape(n, 2)
        tables = pack_frame_tables(hw, self.frames["target"], self.frames["kw"], self.frames["interpolation"],
                                   self.frames.get("keep_aspect_ratio", False))
        nr = tables.shape[1]
        blocks = np.zeros((n, nr + image.BLOCK_INTS), np.int32)  # only the prefix each file uses is written and copied
        blocks[:, :nr] = tables
        for k, (_, kind, i) in enumerate(checked):
            image.pack_block(kind, i, blocks[k, nr:])
        sizes = np.array([len(f) for f in files], np.uint64)
        self._tables[seq % self.depth] = (blocks, sizes, files)
        ptrs = (C.c_void_p * n)(*[C.cast(C.c_char_p(f), C.c_void_p).value for f in files])
        A.check(self.lib.defer_stage_submit_images(self.handle, seq, index, n, ptrs, sizes.ctypes.data,
                                                   blocks.ctypes.data, blocks.nbytes))

    def predict_images(self, items) -> np.ndarray:
        """Single-stage ``model.predict`` of a ``decode="image"`` stage: the outputs of the JPEG or PNG files ``items``, in
        order."""
        self.submit_images(0, 0, items)
        self.step(0)
        return self.result(0)[:len(items)]

    def step(self, seq: int) -> None:
        A.check(self.lib.defer_stage_step(self.handle, seq))
        if self._marks:
            slot = self._marks.pop(seq, None)
            if slot is not None:
                A.check(self.lib.defer_stage_mark(self.handle, seq, slot))

    def mark_after(self, seq: int, slot: int) -> None:
        """Steady-state timing: record timing event ``slot`` (0 | 1) right behind microbatch ``seq`` when it is stepped."""
        self._marks[int(seq)] = int(slot)

    def mark_elapsed_ms(self) -> float:
        ms = C.c_float(0)
        A.check(self.lib.defer_stage_mark_elapsed(self.handle, C.byref(ms)))
        return ms.value

    def result(self, seq: int, out: Optional[np.ndarray] = None) -> np.ndarray:
        if out is None:
            out = np.empty(self.out_shape, np.float32)
        A.check(self.lib.defer_stage_result(self.handle, seq, out.ctypes.data, out.nbytes))
        return out

    def predict(self, x: np.ndarray) -> np.ndarray:
        """Single-stage ``model.predict`` (reference ``test/local_infer.py:21``)."""
        x = self._host_input(x)
        out = np.empty(self.out_shape, np.float32)
        A.check(self.lib.defer_stage_predict(self.handle, x.ctypes.data, x.nbytes, out.ctypes.data, out.nbytes))
        return out

    def sync(self) -> None:
        A.check(self.lib.defer_stage_sync(self.handle))

    def status(self) -> None:
        A.check(self.lib.defer_stage_status(self.handle))

    # ---- host memory
    def pin(self, x: np.ndarray) -> np.ndarray:
        """Page-lock ``x`` in place so ``submit`` is a true async DMA (kept registered until close)."""
        key = x.ctypes.data
        if key not in self._pinned:
            A.check(self.lib.defer_host_register(x.ctypes.data, x.nbytes))
            self._pinned[key] = (x, x.nbytes)
        return x

    # ---- introspection
    def describe(self) -> str:
        buf = C.create_string_buffer(1 << 16)
        A.check(self.lib.defer_stage_describe(self.handle, buf, len(buf)))
        return buf.value.decode()

    def io_bytes(self):
        a, b = C.c_uint64(0), C.c_uint64(0)
        A.check(self.lib.defer_stage_io_bytes(self.handle, C.byref(a), C.byref(b)))
        return a.value, b.value

    def num_kernels(self) -> int:
        n = C.c_int(0)
        A.check(self.lib.defer_stage_num_kernels(self.handle, C.byref(n)))
        return n.value

    def read_buffer(self, buf_id: int, lane: int = 0) -> np.ndarray:
        h, w, c, _ = self.plan.bufs[buf_id]
        out = np.empty((self.batch, h, w, c), np.float32)
        A.check(self.lib.defer_stage_read_buffer(self.handle, lane, buf_id, out.ctypes.data, out.size))
        return out

    def read_layer(self, layer_name: str, lane: int = 0) -> np.ndarray:
        return self.read_buffer(self.plan.tensor_buf[layer_name], lane)

    def time_op(self, op_index: int, iters: int = 20, flush_l2: bool = True) -> float:
        us = C.c_float(0)
        A.check(self.lib.defer_stage_time_op(self.handle, op_index, iters, int(flush_l2), C.byref(us)))
        return us.value

    def op_info(self, op_index: int) -> dict:
        b, f = C.c_double(0), C.c_double(0)
        name = C.create_string_buffer(128)
        A.check(self.lib.defer_stage_op_info(self.handle, op_index, C.byref(b), C.byref(f), name, 128))
        return {"alg_bytes": b.value, "alg_flops": f.value, "kernel": name.value.decode(),
                "layers": list(self.plan.ops[op_index].layers)}

    def timer_start(self) -> None:
        A.check(self.lib.defer_stage_timer_start(self.handle))

    def timer_stop(self) -> float:
        """Device time (ms) from timer_start to the completion of everything enqueued on all lanes."""
        ms = C.c_float(0)
        A.check(self.lib.defer_stage_timer_stop(self.handle, C.byref(ms)))
        return ms.value

    def arm_timing(self, lane: int = 0) -> None:
        us = C.c_float(0)
        A.check(self.lib.defer_stage_last_step_us(self.handle, lane, C.byref(us)))

    def last_step_us(self, lane: int = 0) -> float:
        us = C.c_float(0)
        A.check(self.lib.defer_stage_last_step_us(self.handle, lane, C.byref(us)))
        return us.value

    def close(self) -> None:
        if self.handle:
            self.lib.defer_stage_sync(self.handle)
            for key in list(self._pinned):
                self.lib.defer_host_unregister(C.c_void_p(key))
            self._pinned.clear()
            self.lib.defer_stage_destroy(self.handle)
            self.handle = C.c_void_p()
            _STREAMS_PER_DEVICE[self.device] = max(0, _STREAMS_PER_DEVICE.get(self.device, 0) - self._streams)
            self._streams = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def pinned_empty(shape, dtype=np.float32) -> np.ndarray:
    """numpy array backed by CUDA pinned host memory (freed when the array is garbage-collected)."""
    lib = A.load()
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = C.c_void_p()
    A.check(lib.defer_host_alloc(C.byref(p), nbytes))
    buf = (C.c_char * nbytes).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dtype).reshape(shape)

    class _Owner:
        def __init__(self, ptr):
            self.ptr = ptr

        def __del__(self):
            try:
                lib.defer_host_free(C.c_void_p(self.ptr))
            except Exception:
                pass
    owner = _Owner(p.value)
    _PINNED_OWNERS[arr.ctypes.data] = owner
    return arr


_PINNED_OWNERS: Dict[int, object] = {}


# ------------------------------------------------------------------------------------------------------
# Node: one process per GPU (torchrun).  Thread roles of reference src/node.py:110-124:
#   _weights_socket + _model_socket -> _receive_stage (torch.distributed object from the dispatcher)
#   _data_server                    -> the device-side ready-flag wait inside the lane graph
#   _data_client                    -> _data_loop (enqueue one graph launch per microbatch)
# ------------------------------------------------------------------------------------------------------

class Node:
    def __init__(self, dist_ctx=None, device: Optional[int] = None, poll_s: float = 20e-6):
        self.ctx = dist_ctx
        self.device = device
        self.poll_s = poll_s
        self.runner: Optional[StageRunner] = None
        self.state: Optional[NodeState] = None

    # -- set-up: receive (architecture JSON, weights, next hop) and build the stage
    def _receive_stage(self, ns: NodeState) -> dict:
        msg = self.ctx.recv_stage()                    # blocks until the dispatcher ships our part
        ns.weights = msg["weights"]                    # src/node.py:54  (after _recv_weights)
        ns.next_node = msg["next_node"]                # src/node.py:40
        return msg

    def run(self):
        """Boot the stage and serve microbatches until the dispatcher stops the pipeline
        (reference ``Node.run`` never returns, ``src/node.py:110-124``)."""
        if self.ctx is None:
            raise RuntimeError("Node.run() needs a DistContext (launch one process per GPU with torchrun); "
                               "single-process pipelines are driven by DEFER.run_defer directly")
        ctx = self.ctx
        ns = self.state = NodeState(chunk_size=512 * 1000)  # src/node.py:111 (kept for interface parity)
        msg = self._receive_stage(ns)
        dev = self.device if self.device is not None else ctx.device
        rank, world = ctx.rank, ctx.world
        runner = StageRunner.from_wire(msg["json"], ns.weights, device=dev, dtype=msg["fmt"], max_batch=msg["batch"],
                                       depth=msg["depth"], is_first=(rank == 0), is_last=(rank == world - 1),
                                       finalize=False, conv_backend=msg.get("conv_backend", 0),
                                       wait_timeout_ms=msg.get("wait_timeout_ms", 0),
                                       preprocess=msg.get("preprocess") if rank == 0 else None,
                                       image_size=msg.get("image_size") if rank == 0 else None,
                                       interpolation=msg.get("interpolation", "nearest"),
                                       max_image_size=msg.get("max_image_size") if rank == 0 else None,
                                       decode=msg.get("decode") if rank == 0 else None,
                                       keep_aspect_ratio=msg.get("keep_aspect_ratio", False) if rank == 0 else False)
        ns.model = runner                               # src/node.py:38
        self.runner = runner
        # wire the hop: my consumer gives me its input-side token, I give it my output-side token
        ctx.exchange_links(runner)
        runner.finalize()
        ctx.ack_ready()                                 # src/node.py:41-42 (the 0x06 acknowledgement)
        self._data_loop(runner)
        # teardown is the launcher's job (DistContext.shutdown): unlink on every rank, barrier, destroy -
        # no collective is issued from this thread once the pipeline is up.

    def _data_loop(self, runner: StageRunner):
        """``_data_client`` (src/node.py:103-108): one graph launch per microbatch.  The wait for the
        input is on the device (ready flag); the host only needs to know how many microbatches exist."""
        ctx = self.ctx
        is_first, is_last = ctx.rank == 0, ctx.rank == ctx.world - 1
        enq = retired = 0
        out = np.empty(runner.out_shape, np.float32) if is_last else None
        while True:
            stop = ctx.stop_requested()
            submitted = ctx.submitted()
            progressed = False
            if is_first:
                enq = submitted            # stage 0 is stepped by the dispatcher's feeder (same process)
            else:
                while enq < submitted and (not is_last or enq - retired < runner.depth):
                    runner.step(enq)
                    enq += 1
                    progressed = True
            if is_last and not is_first and retired < enq:
                runner.result(retired, out)
                ctx.publish_result(retired, out)
                retired += 1
                progressed = True
            if stop and enq >= ctx.submitted() and (is_first or not is_last or retired >= enq):
                break
            if not progressed:
                time.sleep(self.poll_s)
        runner.sync()
