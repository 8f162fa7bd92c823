"""Dispatcher with the reference's API (``src/dispatcher.py:20-115``).

``DEFER(computeNodes).run_defer(model, partition_layers, input_stream, output_stream)`` - same names,
same arguments, same blocking behaviour (callers run it in a daemon thread, ``test/test.py:42``).
What changed underneath:

* ``computeNodes[i]`` is a GPU ordinal (or ``"cuda:i"``) of one 8xH100 box instead of an IP;
* ``_dispatchModels`` still ships ``to_json()`` + ``get_weights()`` per stage (``dispatcher.py:49,57``)
  but "shipping" is an upload into that GPU's HBM through ``defer_stage_create`` (same process) or a
  ``torch.distributed`` object send to the rank that owns the GPU (one process per GPU);
* ``_startDistEdgeInference`` / ``_result_server`` (``dispatcher.py:85-105``) keep their roles - feed
  the first stage from ``input_stream``, drain the last into ``output_stream`` in FIFO order - over
  pinned-memory DMA instead of ZFP+LZ4+TCP.

Non-reference additions: ``close()`` / context manager (the reference can only be killed), keyword-only
``dtype``, ``depth`` (in-flight microbatches per stage), ``batch`` (samples per queue item; reference: 1),
``coalesce``, ``preprocess``, ``image_size``, ``max_image_size``, ``interpolation``, ``keep_aspect_ratio`` and ``decode``.

Preprocessing: the reference's driver runs Keras' ``preprocess_input`` on the host before every ``input_q.put``
(``test/test.py:19-23``).  With ``preprocess="caffe"`` queue items are the uint8 images themselves
(``img_to_array(img).astype(np.uint8)``, shape ``(batch, h, w, 3)``) and the first stage applies the transform on its
GPU, bit for bit what ``applications.preprocess_input`` gives on the host; an image crosses PCIe at 1 B per value
instead of 4.  ``preprocess="tf"`` does the same with the ResNet V2 family's transform
(``applications.resnet_v2_preprocess_input``), and is refused for a model whose Keras preprocessing is caffe mode.
Other item dtypes are refused.

Resizing: the same driver loads every image with ``load_img(path, target_size=(224, 224))``, a Pillow resize on the host.
With ``image_size=(h, w)`` (and ``preprocess``) queue items are uint8 images of that size, e.g. camera frames, and the
first stage resizes them to the model input on its GPU before preprocessing, bit for bit what
``applications.resize_image(item, (H, W), interpolation)`` gives; ``interpolation`` takes the names ``load_img`` accepts
(default ``"nearest"``, as in Keras).  An ``image_size`` equal to the model input changes nothing, as Keras does not
resize then.  Photos and frames from several cameras come in many sizes: with ``max_image_size=(H, W)`` instead, each
queue item is a uint8 image ``(batch, h, w, 3)`` of its own size with ``h <= H`` and ``w <= W``, items of different sizes
share a microbatch, and each gives exactly what ``image_size=(h, w)`` would.  Only the image's own bytes cross PCIe.
With ``decode="jpeg"`` as well, each queue item is a baseline JPEG file (``open(path, "rb").read()``); the first GPU
decodes it exactly as ``load_img`` does with Pillow (``jpeg.decode_jpeg``), so only the compressed file crosses PCIe
and the host only parses its markers.  ``decode="png"`` does the same for non-interlaced PNG files (``png.decode_png``);
the host only walks their chunk headers.  ``decode="image"`` takes both in one pipeline: each item's format is told
from its first bytes, as ``PIL.Image.open`` does, never from a file name, and JPEG and PNG files share a microbatch
(``image.decode_image``).  ``keep_aspect_ratio=True`` (with ``image_size`` or ``max_image_size``, and with
``decode="jpeg"``) resizes each image's centred crop with the model input's aspect ratio instead of squashing the whole
image, as ``load_img(..., keep_aspect_ratio=True)`` does: ``applications.resize_image(item, (H, W), interpolation,
keep_aspect_ratio=True)``.

Coalescing: the reference's queue items are single images and every node runs them one at a time
(``src/node.py:103-108``), re-reading its weights per image.  Here up to ``coalesce`` in-flight queue items are
gathered into ONE engine microbatch (one kernel chain launch per stage, weights streamed once per group); results
are split back into per-item arrays and delivered in FIFO order, so the API contract (item in, ``(batch, 1000)``
out, same order) is unchanged.  A group is launched as soon as ``coalesce`` items are there or the input queue has
been empty for ``linger_us``; unused sample slots of a partial group are computed and dropped.
"""
from __future__ import annotations

import queue
import threading
import time
from typing import List, Optional, Tuple

import numpy as np

from . import keras_like as K
from .applications import check_model_preprocess, check_preprocess
from .jpeg import check_decode, check_jpeg
from .image import DECODES, check_image
from .png import check_png
from .resize import check_frame, check_interpolation, check_keep_aspect_ratio, check_size
from .dag_util import construct_model
from .node import DTYPE_TO_FMT, StageRunner, parse_device


class DEFER:
    def __init__(self, computeNodes, *, dtype: str = "float32", depth: int = 4, batch: Optional[int] = None,
                 coalesce: int = 1, linger_us: float = 200.0, conv_backend: int = 0, dist=None,
                 wait_timeout_ms: int = 0, max_inflight: int = 0, preprocess: Optional[str] = None,
                 image_size: Optional[Tuple[int, int]] = None, interpolation: str = "nearest",
                 max_image_size: Optional[Tuple[int, int]] = None, decode: Optional[str] = None,
                 keep_aspect_ratio: bool = False) -> None:
        check_decode(decode, preprocess, image_size, max_image_size, DECODES)
        if decode is not None and batch not in (None, 1):
            what = "JPEG or PNG" if decode == "image" else decode.upper()
            raise ValueError(f"decode={decode!r}: a queue item is one {what} file, so batch must be 1, got {batch}")
        if preprocess is not None:
            check_preprocess(preprocess)
        check_interpolation(interpolation)
        if image_size is not None:
            image_size = check_size(image_size)
            if preprocess is None:
                raise ValueError(f"image_size={image_size}: resizing takes uint8 images and needs preprocess= (float items "
                                 "are already preprocessed, and Keras resizes before preprocessing)")
        if max_image_size is not None:
            max_image_size = check_size(max_image_size, "max_image_size")
            if preprocess is None:
                raise ValueError(f"max_image_size={max_image_size}: resizing takes uint8 images and needs preprocess= "
                                 "(float items are already preprocessed, and Keras resizes before preprocessing)")
            if image_size is not None:
                raise ValueError(f"max_image_size={max_image_size} and image_size={image_size}: give one (image_size: "
                                 "every image has that size; max_image_size: each image has its own size up to that bound)")
        keep_aspect_ratio = check_keep_aspect_ratio(keep_aspect_ratio, image_size, max_image_size)
        self.computeNodes = list(computeNodes)
        self.preprocess = preprocess        # None | "caffe" | "tf": uint8 queue items, preprocessed on stage 0's GPU
        self.image_size = image_size        # None | (h, w) of the uint8 queue items, resized on stage 0's GPU
        self.interpolation = interpolation
        self.keep_aspect_ratio = keep_aspect_ratio  # resize Keras' centred crop of each image (load_img keep_aspect_ratio)
        self.max_image_size = max_image_size  # None | (H, W): uint8 queue items of any size up to it, resized on stage 0
        self.decode = decode                # None | "jpeg" | "png" | "image": JPEG / PNG / either files, decoded on stage 0
        self.dispatchIP = "localhost"       # reference: socket.gethostbyname(...) (dispatcher.py:23); no sockets here
        self.chunk_size = 512 * 1000        # kept for interface parity (dispatcher.py:24)
        self.dtype = dtype
        self.depth = int(depth)
        self.batch = batch                  # samples per queue item
        self.coalesce = max(1, int(coalesce))
        self.linger_s = max(0.0, float(linger_us)) * 1e-6
        self.conv_backend = conv_backend
        self.dist = dist                    # DistContext when launched one-process-per-GPU
        self.wait_timeout_ms = wait_timeout_ms
        # microbatches between ingress and egress.  One process drives all stages => bounded by the lanes of
        # the last stage (depth).  One process per GPU => every stage has its own `depth` lanes and the chain
        # back-pressures itself through the device flags, so depth x stages may be in flight.
        self.max_inflight = int(max_inflight)
        self.stages: List[StageRunner] = []
        self._stop = threading.Event()
        self._ready = threading.Event()
        self._inflight: Optional[threading.Semaphore] = None
        self._submitted = 0                 # engine microbatches (groups of <= coalesce items) stepped so far
        self._group_n: List[int] = []       # items in microbatch seq (ring indexed by seq)
        self._threads: List[threading.Thread] = []
        self._error: Optional[BaseException] = None
        self.results_delivered = 0          # queue items delivered
        self.items_submitted = 0

    @property
    def engine_batch(self) -> int:
        return (self.batch or 1) * self.coalesce

    # ------------------------------------------------------------------ partition (dispatcher.py:27-42)
    def _partition(self, model: K.Model, layer_parts: List[str]) -> List[K.Model]:
        models = []
        for p in range(len(layer_parts) + 1):
            if p == 0:
                start = model.input._keras_history[0].name
            else:
                start = layer_parts[p - 1]
            if p == len(layer_parts):
                end = model.output._keras_history[0].name
            else:
                end = layer_parts[p]
            part = construct_model(model, start, end, part_name=f"part{p+1}")
            models.append(part)
        return models

    # ------------------------------------------------------------------ placement (dispatcher.py:44-65)
    def _dispatchModels(self, models: list, nodeIPs: List) -> None:
        if len(nodeIPs) < len(models):
            raise ValueError(f"{len(models)} stages but only {len(nodeIPs)} compute nodes")
        n = len(models)
        batch = self.engine_batch           # samples per engine microbatch = item batch x coalesced items
        if self.dist is not None:
            # one process per GPU: ship (json, weights, next hop) to each rank; ranks build + link themselves
            for i in range(n):
                next_node = nodeIPs[i + 1] if i != n - 1 else self.dispatchIP
                self.dist.send_stage(i, {"json": models[i].to_json(), "weights": models[i].get_weights(),
                                         "next_node": str(next_node), "fmt": self.dtype, "batch": batch,
                                         "depth": self.depth, "conv_backend": self.conv_backend,
                                         "wait_timeout_ms": self.wait_timeout_ms,
                                         "preprocess": self.preprocess if i == 0 else None,
                                         "image_size": self.image_size if i == 0 else None,
                                         "interpolation": self.interpolation,
                                         "max_image_size": self.max_image_size if i == 0 else None,
                                         "decode": self.decode if i == 0 else None,
                                         "keep_aspect_ratio": self.keep_aspect_ratio and i == 0})
            self.dist.wait_all_ready()      # the 1-byte ACK of dispatcher.py:64-65
            return
        runners = []
        for i in range(n):
            model_json = models[i].to_json()
            weights = models[i].get_weights()
            r = StageRunner.from_wire(model_json, weights, device=parse_device(nodeIPs[i]), dtype=self.dtype,
                                      max_batch=batch, depth=self.depth, is_first=(i == 0), is_last=(i == n - 1),
                                      finalize=False, conv_backend=self.conv_backend,
                                      wait_timeout_ms=self.wait_timeout_ms,
                                      preprocess=self.preprocess if i == 0 else None,
                                      image_size=self.image_size if i == 0 else None,
                                      interpolation=self.interpolation,
                                      max_image_size=self.max_image_size if i == 0 else None,
                                      decode=self.decode if i == 0 else None,
                                      keep_aspect_ratio=self.keep_aspect_ratio and i == 0)
            r.name = f"part{i+1}"
            runners.append(r)
        for i in range(n - 1):              # next hop = nodeIPs[i+1] (dispatcher.py:51-55)
            runners[i].link_to(runners[i + 1])
        for r in runners:
            r.finalize()
        self.stages = runners

    # ------------------------------------------------------------------ ingress (dispatcher.py:85-93)
    def _startDistEdgeInference(self, input: queue.Queue):
        first = self.stages[0] if self.stages else self.dist.local_runner()
        G, B = self.coalesce, self.batch or 1
        u8 = self.preprocess is not None
        bound = self.max_image_size
        hold, nh = self._hold, len(self._hold)
        get_nowait = input.get_nowait
        submit_items = first.submit_items if hasattr(first, "submit_items") else None
        if submit_items is None:             # duck-typed stages (tests): fall back to one call per item
            def submit_items(seq, group):
                for i, x in enumerate(group):
                    first.submit_part(seq, i * B, x)
        if bound is not None:                # each image with its own size and tables, one C call per group
            def submit_items(seq, group):
                first.submit_frames(seq, 0, group)
        files = self.decode is not None      # JPEG or PNG files
        check_file = {"jpeg": check_jpeg, "png": check_png, "image": check_image}.get(self.decode)
        if files and self.decode == "image":  # each file sniffed and parsed here, either format in one group
            def submit_items(seq, group):
                first.submit_images(seq, 0, [d for d, _, _ in group], group)
        elif files:                          # the files, parsed here, decoded on the GPU
            submit_files = first.submit_pngs if self.decode == "png" else first.submit_jpegs

            def submit_items(seq, group):
                submit_files(seq, 0, [d for d, _ in group], [i for _, i in group])
        try:
            while not self._stop.is_set():
                try:
                    model_input = input.get(timeout=0.05)
                except queue.Empty:
                    continue
                while not self._inflight.acquire(timeout=0.05):
                    if self._stop.is_set():
                        return
                seq = self._submitted
                n = 0
                deadline = None
                group = []
                in_shape = None
                while True:
                    x = model_input
                    if files:                        # (file bytes[, kind], header): refused files raise here, as bad items do
                        x = check_file(x, bound)
                    elif bound is not None:          # any size up to the bound: no same-shape rule within a group
                        x = check_frame(x, bound)
                    elif u8:
                        if not (isinstance(x, np.ndarray) and x.dtype == np.uint8):
                            raise TypeError(f"DEFER(preprocess={self.preprocess!r}) takes uint8 RGB images "
                                            "(img_to_array(img).astype(np.uint8)), got "
                                            f"{getattr(x, 'dtype', type(x).__name__)}; do not preprocess them on the host")
                        x = np.ascontiguousarray(x)
                    elif not (isinstance(x, np.ndarray) and x.dtype == np.float32 and x.flags["C_CONTIGUOUS"]):
                        x = np.ascontiguousarray(x, dtype=np.float32)
                    if not files and x.shape[0] != B:
                        raise ValueError(f"queue item has batch {x.shape[0]}, DEFER was built for batch {B}")
                    if files or bound is not None:
                        pass
                    elif in_shape is None:
                        in_shape = x.shape
                    elif x.shape != in_shape:
                        raise ValueError(f"queue items of one group differ in shape: {x.shape} vs {in_shape}")
                    hold[self.items_submitted % nh] = x      # keep alive until the DMA has certainly happened
                    self.items_submitted += 1
                    group.append(x)
                    n += 1
                    if n == G:
                        break
                    try:                                     # coalesce whatever is already waiting ...
                        model_input = get_nowait()
                    except queue.Empty:                      # ... or arrives within the linger window
                        now = time.perf_counter()
                        if deadline is None:
                            deadline = now + self.linger_s
                        if now >= deadline or self._stop.is_set():
                            break
                        try:
                            model_input = input.get(timeout=deadline - now)
                        except queue.Empty:
                            break
                submit_items(seq, group)                     # one C call: a cudaMemcpyAsync per item on the lane's stream
                self._group_n[seq % len(self._group_n)] = n
                if self.dist is not None:
                    first.step(seq)
                    self.dist.mark_submitted(seq + 1)
                else:
                    for r in self.stages:
                        r.step(seq)
                self._submitted = seq + 1
        except BaseException as e:  # surface in close()/run_defer instead of dying silently
            self._error = e
            self._stop.set()

    # ------------------------------------------------------------------ egress (dispatcher.py:95-105)
    def _result_server(self, output: queue.Queue):
        try:
            self._ready.wait()
            seq = 0
            B = self.batch or 1
            local_last = bool(self.stages) or (self.dist is not None and self.dist.world == 1)
            last = (self.stages[-1] if self.stages else self.dist.local_runner()) if local_last else None
            while not self._stop.is_set():
                if seq >= self._submitted:
                    time.sleep(20e-6)
                    continue
                if last is not None:
                    pred = last.result(seq)
                else:
                    pred = self.dist.wait_result(seq, self._stop)
                    if pred is None:
                        return
                    pred = pred.reshape(self.engine_batch, -1)
                n = self._group_n[seq % len(self._group_n)]
                self._inflight.release()
                seq += 1
                for i in range(n):                           # split the group back into queue items, FIFO
                    item = pred[i * B:(i + 1) * B]
                    while not self._stop.is_set():
                        try:
                            output.put(item, timeout=0.05)
                            break
                        except queue.Full:
                            continue
                    self.results_delivered += 1
        except BaseException as e:
            self._error = e
            self._stop.set()

    # ------------------------------------------------------------------ orchestration (dispatcher.py:107-115)
    def run_defer(self, model: K.Model, partition_layers, input_stream: queue.Queue, output_stream: queue.Queue):
        if self.batch is None:
            self.batch = 1
        check_model_preprocess(model, self.preprocess)   # the partitions no longer know which model they came from
        models_to_dispatch = self._partition(model, partition_layers)
        # the last stage has `depth` result buffers (one process) / the result ring and every stage's lanes bound the
        # chain (one process per GPU): more microbatches in flight than that would overwrite a result before it is read
        cap = self.depth * (self.dist.world if self.dist is not None else 1)
        if self.dist is not None:
            cap = min(cap, self.dist.ring)
        if self.max_inflight <= 0:
            self.max_inflight = cap
        elif self.max_inflight > cap:
            raise ValueError(f"max_inflight {self.max_inflight} exceeds what the pipeline can hold ({cap} = depth "
                             f"{self.depth} x {'ranks' if self.dist is not None else '1'}, result ring included)")
        self._inflight = threading.Semaphore(self.max_inflight)
        self._hold = [None] * ((2 * self.max_inflight + 2) * self.coalesce)
        self._group_n = [0] * (2 * self.max_inflight + 2)
        a = threading.Thread(target=self._result_server, args=(output_stream,), name="defer-result")
        a.start()
        try:
            self._dispatchModels(models_to_dispatch, self.computeNodes)
        except BaseException as e:
            self._error = e
            self._stop.set()
            self._ready.set()
            a.join()
            raise
        self._ready.set()
        b = threading.Thread(target=self._startDistEdgeInference, args=(input_stream,), daemon=True, name="defer-feed")
        b.start()
        self._threads = [a, b]
        a.join()                            # blocks until close(), like the reference blocks forever
        b.join()
        if self._error is not None:
            raise self._error

    # ------------------------------------------------------------------ non-reference: clean shutdown
    def wait_ready(self, timeout: Optional[float] = None) -> bool:
        return self._ready.wait(timeout)

    def close(self):
        self._stop.set()
        for t in self._threads:
            if t is not threading.current_thread():
                t.join(timeout=10)
        if self.dist is not None:
            self.dist.request_stop()
        # Stages write into each other's arenas (outputs + ready flags downstream, free flags upstream): first let
        # EVERY stage finish what is enqueued, then drop every cross-stage mapping, and only then free memory.
        for r in self.stages:
            try:
                r.sync()
            except Exception:
                pass
        for r in self.stages:
            try:
                r.unlink()
            except Exception:
                pass
        for r in self.stages:
            r.close()
        self.stages = []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False
