"""Shared per-node state - the interface of the reference's ``NodeState``
(``src/node_state.py:6-41``) on a condition variable.

Same constructor and the same four attributes (``chunk_size`` read-only; ``next_node``, ``model``,
``weights`` settable), including the reference's "empty string means not set yet" sentinel
(``node_state.py:9-11``).  The reference's consumers poll these fields with ``time.sleep(5)``
(``src/node.py:32-33,95-96``); here every assignment notifies waiters, so ``wait_for`` returns as
soon as the field is published.  ``chunk_size`` only exists for interface parity - the NVLink hop
has no chunking.  The TCP framing helpers of the reference file (``socket_send`` / ``socket_recv``,
``node_state.py:43-101``) are provided further down for host-side compatibility; the hot path
does not use them (SURVEY.md 8f, rank 2).
"""
from __future__ import annotations

import threading
from typing import Any, Optional

_UNSET = ""          # the reference's sentinel


class _Published:
    """Data descriptor: a field guarded by the owner's condition variable; writes wake waiters."""

    def __init__(self, read_only: bool = False):
        self.read_only = read_only
        self.slot = ""

    def __set_name__(self, owner, name):
        self.slot = "_" + name

    def __get__(self, obj, objtype=None):
        if obj is None:
            return self
        with obj._cond:
            return getattr(obj, self.slot)

    def __set__(self, obj, value):
        if self.read_only:
            raise AttributeError(f"{self.slot[1:]} is read-only")
        with obj._cond:
            setattr(obj, self.slot, value)
            obj._cond.notify_all()


class NodeState:
    chunk_size = _Published(read_only=True)
    next_node = _Published()
    model = _Published()
    weights = _Published()

    def __init__(self, chunk_size) -> None:
        self._cond = threading.Condition(threading.Lock())
        self._chunk_size = chunk_size
        self._next_node: Any = _UNSET
        self._model: Any = _UNSET
        self._weights: Any = _UNSET

    def is_set(self, field: str) -> bool:
        v = getattr(self, field)
        return not (isinstance(v, str) and v == _UNSET)

    def wait_for(self, field: str, timeout: Optional[float] = None):
        """Block until ``field`` ('weights' | 'model' | 'next_node') has been published; return its value."""
        slot = "_" + field

        def published() -> bool:
            v = getattr(self, slot)
            return not (isinstance(v, str) and v == _UNSET)

        with self._cond:
            if not self._cond.wait_for(published, timeout=timeout):
                raise TimeoutError(f"NodeState.{field} not set within {timeout}s")
            return getattr(self, slot)


# ------------------------------------------------------------------------------------------------------
# Wire framing of the reference transport (``src/node_state.py:43-101``): an 8-byte
# big-endian length followed by the payload, written / read in slices of at most ``chunk_size`` bytes on
# a non-blocking socket, waiting with ``select`` whenever the kernel buffer is full / empty.  The GPU hot
# path never uses it (the hop is an NVLink store) - it exists so that host-side tooling can talk to
# reference-style peers (SURVEY.md 8f, rank 2) and so the two names of the reference module resolve.
# ------------------------------------------------------------------------------------------------------
import select as _select
import socket as _socket

_LEN_BYTES = 8
_WOULD_BLOCK = (BlockingIOError, InterruptedError)


def _send_all(sock: "_socket.socket", view: memoryview) -> None:
    sent = 0
    while sent < len(view):
        try:
            sent += sock.send(view[sent:])
        except _WOULD_BLOCK:
            _select.select([], [sock], [])
        except OSError as e:           # EAGAIN surfaces as OSError on some platforms
            if e.errno not in (_socket.EAGAIN, _socket.EWOULDBLOCK):
                raise
            _select.select([], [sock], [])


def socket_send(bytes, sock: "_socket.socket", chunk_size: int) -> None:  # noqa: A002 - reference's parameter name
    """Frame and send ``bytes``: 8-byte big-endian length, then the payload in ``chunk_size`` slices."""
    payload = memoryview(bytes).cast("B")
    if chunk_size < 1:
        raise ValueError("chunk_size must be positive")
    _send_all(sock, memoryview(len(payload).to_bytes(_LEN_BYTES, "big")))
    for off in range(0, len(payload), chunk_size):
        _send_all(sock, payload[off:off + chunk_size])


def _recv_exact(sock: "_socket.socket", out: memoryview, chunk_size: int) -> None:
    got = 0
    while got < len(out):
        want = min(len(out) - got, chunk_size)
        try:
            n = sock.recv_into(out[got:got + want], want)
        except _WOULD_BLOCK:
            _select.select([sock], [], [])
            continue
        except OSError as e:
            if e.errno not in (_socket.EAGAIN, _socket.EWOULDBLOCK):
                raise
            _select.select([sock], [], [])
            continue
        if n == 0:
            raise ConnectionError("peer closed the connection mid-frame")
        got += n


def socket_recv(sock: "_socket.socket", chunk_size: int) -> bytearray:
    """Receive one frame written by ``socket_send``; returns the payload as a ``bytearray``."""
    if chunk_size < 1:
        raise ValueError("chunk_size must be positive")
    header = bytearray(_LEN_BYTES)
    _recv_exact(sock, memoryview(header), _LEN_BYTES)
    size = int.from_bytes(header, "big")
    data = bytearray(size)
    if size:
        _recv_exact(sock, memoryview(data), chunk_size)
    return data
