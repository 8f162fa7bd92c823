"""One-process-per-GPU plumbing (``torchrun``): the control plane that replaces the reference's TCP
ports 5001/5002 and its per-node polling (``src/dispatcher.py:44-65``,
``src/node.py:20-75``).

* stage shipment (architecture JSON + weights + next hop) : ``torch.distributed`` object scatter (gloo);
* hop wiring : each rank exports CUDA-IPC link tokens of its stage arena, all-gathered, neighbours import;
* steady state: NO per-microbatch message.  A small POSIX shared-memory block carries three counters
  (``submitted``, ``done``, ``stop``) and the result ring; ranks poll it from their data loop.  The
  activation hop itself never touches the host (device flags over NVLink, see ``csrc/stage.cu``).

The data path uses no collective: the pipeline is a chain of point-to-point hops (SURVEY.md 8e).
"""
from __future__ import annotations

import os
import time
from multiprocessing import shared_memory
from typing import List, Optional

import numpy as np

_HDR_WORDS = 16     # uint64 header: [0] submitted, [1] stop, [2] done (published), [6] consumed by the dispatcher


class DistContext:
    """``device``: the GPU this rank's stage runs on (default: its local rank).  Ranks that share a GPU (CUDA IPC works
    between processes on one device) need ``backend="gloo"``: NCCL refuses two ranks on one device."""

    def __init__(self, backend: Optional[str] = None, ring: int = 64, out_elems: int = 1000, batch: int = 1,
                 device: Optional[int] = None):
        import torch
        import torch.distributed as dist
        self.torch, self.dist = torch, dist
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", str(self.rank)))
        self.device = self.local_rank if device is None else int(device)
        self.ring = int(ring)
        self.out_elems = int(out_elems) * int(batch)
        self._runner = None
        self._owns_group = False
        # a gloo-only world may have more ranks than the host has GPUs: those ranks stay on the CPU
        self.cuda = torch.cuda.is_available() and self.device < torch.cuda.device_count()
        if not dist.is_initialized():
            use_cuda = self.cuda
            if backend is None:
                backend = "cpu:gloo,cuda:nccl" if use_cuda else "gloo"
            if use_cuda:
                torch.cuda.set_device(self.device)
            dist.init_process_group(backend=backend, rank=self.rank, world_size=self.world)
            self._owns_group = True
        else:
            backend = str(dist.get_backend())
        # collectives run on the GPU only where NCCL carries them; under gloo they stay on the host
        self.nccl = self.cuda and "nccl" in str(backend)
        # control block in POSIX shared memory (single node by construction: NVLink domain of one box)
        port = os.environ.get("MASTER_PORT", "0")
        self.shm_name = f"defer_b200_{port}_{os.environ.get('TORCHELASTIC_RUN_ID', 'x')}"[:60]
        nbytes = _HDR_WORDS * 8 + self.ring * self.out_elems * 4
        if self.rank == 0:
            try:
                old = shared_memory.SharedMemory(name=self.shm_name)
                old.close()
                old.unlink()
            except FileNotFoundError:
                pass
            self.shm = shared_memory.SharedMemory(name=self.shm_name, create=True, size=nbytes)
            self.shm.buf[:nbytes] = b"\0" * nbytes
        self.barrier()
        if self.rank != 0:
            self.shm = shared_memory.SharedMemory(name=self.shm_name)
        self.hdr = np.ndarray((_HDR_WORDS,), dtype=np.uint64, buffer=self.shm.buf, offset=0)
        self.results = np.ndarray((self.ring, self.out_elems), dtype=np.float32, buffer=self.shm.buf,
                                  offset=_HDR_WORDS * 8)
        self.barrier()

    # ------------------------------------------------------------------ collectives (control plane only)
    def barrier(self):
        if self.world > 1:
            if self.nccl:
                self.dist.barrier(device_ids=[self.device])
            else:
                self.dist.barrier()

    def max_over_ranks(self, value: float) -> float:
        if self.world == 1:
            return float(value)
        dev = f"cuda:{self.device}" if self.nccl else "cpu"
        t = self.torch.tensor([float(value)], dtype=self.torch.float64, device=dev)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return float(t.item())

    def sum_over_ranks(self, value: float) -> float:
        if self.world == 1:
            return float(value)
        dev = f"cuda:{self.device}" if self.nccl else "cpu"
        t = self.torch.tensor([float(value)], dtype=self.torch.float64, device=dev)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM)
        return float(t.item())

    # ------------------------------------------------------------------ stage shipment (dispatcher -> nodes)
    def send_stage(self, stage_index: int, msg: dict):
        """Dispatcher side of ``_dispatchModels`` - queued, delivered by ``flush_stages``."""
        if not hasattr(self, "_outbox"):
            self._outbox = [None] * self.world
        self._outbox[stage_index] = msg

    def wait_all_ready(self):
        """Deliver the queued stages (one object scatter) and wait for every node's ACK."""
        self._scatter(self._outbox)
        self._outbox = [None] * self.world
        while not getattr(self, "_all_ready", False):   # set by the local node thread after the ACK barrier
            time.sleep(0.001)

    def _scatter(self, objs):
        recv = [None]
        self.dist.scatter_object_list(recv, objs if self.rank == 0 else None, src=0)
        self._inbox = recv[0]
        return recv[0]

    def recv_stage(self) -> dict:
        """Node side: block until the dispatcher's scatter arrives (``_model_socket``/``_weights_socket``)."""
        if self.rank == 0:
            # rank 0 is dispatcher AND node 0: the dispatcher thread performs the scatter
            while getattr(self, "_inbox", None) is None:
                time.sleep(0.001)
            return self._inbox
        return self._scatter(None)

    def exchange_links(self, runner) -> None:
        """Wire the NVLink hops: all-gather (input-side, output-side) tokens, import the neighbours'."""
        self._runner = runner
        mine = (runner.export_link(0) if self.rank > 0 else b"",
                runner.export_link(1) if self.rank < self.world - 1 else b"")
        allt: List = [None] * self.world
        self.dist.all_gather_object(allt, mine)
        if self.rank < self.world - 1:
            runner.import_link(0, allt[self.rank + 1][0])   # my consumer's input side
        if self.rank > 0:
            runner.import_link(1, allt[self.rank - 1][1])   # my producer's output side

    def ack_ready(self):
        self.barrier()
        self._all_ready = True

    def local_runner(self):
        """The stage this rank serves, once the whole pipeline is wired and acknowledged."""
        while not getattr(self, "_all_ready", False):
            time.sleep(0.001)
        return self._runner

    def shutdown(self, node_thread=None):
        """Orderly teardown: stop -> node loops drain -> unlink everywhere -> barrier -> destroy."""
        if self.rank == 0:
            self.request_stop()
        if node_thread is not None:
            node_thread.join(timeout=120)
        if self._runner is not None:
            self._runner.sync()
            self._runner.unlink()
        self.barrier()
        if self._runner is not None:
            self._runner.close()
            self._runner = None
        self.close()

    # ------------------------------------------------------------------ steady-state counters (shared memory)
    def mark_submitted(self, n: int):
        self.hdr[0] = n

    def submitted(self) -> int:
        return int(self.hdr[0])

    def request_stop(self):
        self.hdr[1] = 1

    def stop_requested(self) -> bool:
        return bool(self.hdr[1])

    def publish_result(self, seq: int, out: np.ndarray):
        # never run more than `ring` rows ahead of the dispatcher's result thread (it would overwrite unread rows)
        while seq - int(self.hdr[6]) >= self.ring:
            if self.stop_requested():
                return
            time.sleep(20e-6)
        self.results[seq % self.ring, :] = out.reshape(-1)
        self.hdr[2] = seq + 1          # x86-64 (TSO): the row's stores are globally visible before the counter's

    def done(self) -> int:
        return int(self.hdr[2])

    def wait_result(self, seq: int, stop_event=None, timeout: float = 60.0) -> Optional[np.ndarray]:
        t0 = time.perf_counter()
        spins = 0
        while int(self.hdr[2]) <= seq:
            if stop_event is not None and stop_event.is_set():
                return None
            spins += 1
            if spins > 200:
                time.sleep(10e-6)
            if time.perf_counter() - t0 > timeout:
                raise TimeoutError(f"result {seq} not published within {timeout}s")
        row = np.array(self.results[seq % self.ring], copy=True)
        self.hdr[6] = seq + 1          # row copied out: the publisher may reuse it
        return row

    def close(self):
        try:
            self.barrier()
        except Exception:
            pass
        self.hdr = None
        self.results = None
        try:
            self.shm.close()
            if self.rank == 0:
                self.shm.unlink()
        except Exception:
            pass
        if self._owns_group and self.dist.is_initialized():
            self.dist.destroy_process_group()
