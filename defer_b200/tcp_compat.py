"""Network-transport compatibility mode (SURVEY.md 8f, rank 2): the reference's TCP control and data plane, so that a
H100 stage can sit in a chain with reference-style peers (edge devices, other boxes) instead of - or next to - the NVLink hop.

What the reference does on the wire (``src/dispatcher.py:44-80``, ``src/node.py:20-108``), restated:

* three TCP ports per node: 5000 activations, 5001 architecture + next hop, 5002 weights (``src/dispatcher.py:18``);
* weights (``:5002``): an 8-byte big-endian array count, then one frame per array (``socket_send`` framing of
  ``src/node_state.py:43-69``: 8-byte big-endian length + payload in ``chunk_size`` slices), each payload an encoded array;
* architecture (``:5001``): one frame with the Keras JSON, one frame (sent with ``chunk_size=1``) with the next hop's
  address, then the node answers a single byte ``0x06`` once its model is built and the weights are set;
* activations (``:5000``): one frame per tensor, node -> next node -> ... -> dispatcher (the last node's next hop is the
  dispatcher itself, ``src/dispatcher.py:51-55``); strictly FIFO on one connection per hop.

Codec: the reference encodes every array as ``lz4.frame.compress(zfpy.compress_numpy(arr))`` (lossless: reversible ZFP).
``zfpy`` / ``lz4`` are not installable in this image, so the codec is pluggable: ``ZfpLz4Codec`` (used automatically when both
wheels import - wire-compatible with the reference) and ``RawCodec`` (a self-describing lossless container: dtype, shape,
raw bytes) for chains made of defer_b200 peers.  Either way the hop is lossless, like the NVLink copy.

This module is host-side only and never on the GPU hot path; the compute of a ``TcpNode`` is whatever ``predict`` callable it
is given (a ``StageRunner.predict`` on an H100, or any stand-in in tests).
"""
from __future__ import annotations

import queue
import select
import socket
import struct
import threading
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from .node_state import NodeState, socket_recv, socket_send

DATA_PORT, MODEL_PORT, WEIGHTS_PORT = 5000, 5001, 5002      # src/dispatcher.py:18, src/node.py:17
ACK = b"\x06"                                                 # src/node.py:41-42
CHUNK_SIZE = 512 * 1000                                       # src/dispatcher.py:24, src/node.py:111


# ----------------------------------------------------------------------------------------------------- codecs
class RawCodec:
    """Lossless self-describing container: magic, dtype string, rank, shape, raw C-order bytes."""
    MAGIC = b"DFRW"

    def encode(self, arr) -> bytes:
        a = np.asarray(arr)
        if not a.flags["C_CONTIGUOUS"]:
            a = np.ascontiguousarray(a)          # (never for 0-d arrays: ascontiguousarray would make them 1-d)
        dt = a.dtype.str.encode()
        head = self.MAGIC + struct.pack(">B", len(dt)) + dt + struct.pack(">B", a.ndim) + struct.pack(f">{a.ndim}Q", *a.shape)
        return head + a.tobytes()

    def decode(self, byts) -> np.ndarray:
        b = bytes(byts)
        if b[:4] != self.MAGIC:
            raise ValueError("not a RawCodec frame (is the peer using the zfp+lz4 codec?)")
        n = b[4]
        dt = np.dtype(b[5:5 + n].decode())
        off = 5 + n
        nd = b[off]
        shape = struct.unpack(f">{nd}Q", b[off + 1:off + 1 + 8 * nd])
        off += 1 + 8 * nd
        return np.frombuffer(b, dtype=dt, offset=off).reshape(shape).copy()


class ZfpLz4Codec:
    """The reference's codec, byte-compatible with it (needs the ``zfpy`` and ``lz4`` wheels)."""

    def __init__(self):
        import lz4.frame  # noqa: F401  (ImportError = codec unavailable)
        import zfpy  # noqa: F401
        self._lz4, self._zfpy = lz4.frame, zfpy

    def encode(self, arr) -> bytes:
        return self._lz4.compress(self._zfpy.compress_numpy(np.ascontiguousarray(arr)))     # src/node.py:76-77

    def decode(self, byts) -> np.ndarray:
        return self._zfpy.decompress_numpy(self._lz4.decompress(bytes(byts)))                # src/node.py:78-79


def default_codec():
    try:
        return ZfpLz4Codec()
    except ImportError:
        return RawCodec()


# ----------------------------------------------------------------------------------------------------- helpers
def _send_count(sock: socket.socket, n: int) -> None:
    """The bare 8-byte big-endian count that precedes the weight frames (``src/dispatcher.py:67-77``)."""
    view = memoryview(int(n).to_bytes(8, "big"))
    while len(view):
        try:
            view = view[sock.send(view):]
        except (BlockingIOError, InterruptedError):
            select.select([], [sock], [])


def _recv_count(sock: socket.socket) -> int:
    buf = bytearray()
    while len(buf) < 8:
        try:
            chunk = sock.recv(8 - len(buf))
        except (BlockingIOError, InterruptedError):
            select.select([sock], [], [])
            continue
        if not chunk:
            raise ConnectionError("peer closed the connection before the weight count")
        buf.extend(chunk)
    return int.from_bytes(buf, "big")


def _connect(addr: Tuple[str, int], timeout: float) -> socket.socket:
    s = socket.create_connection(addr, timeout=timeout)
    s.setsockopt(socket.IPPROTO_TCP, socket.TCP_NODELAY, 1)
    s.setblocking(False)
    return s


def _wait_state(state: NodeState, field: str, stop: threading.Event):
    """``NodeState.wait_for`` in slices, so a stopping node does not hang on a field that will never be published."""
    while not stop.is_set():
        try:
            return state.wait_for(field, timeout=0.2)
        except TimeoutError:
            continue
    return None


def _listen(port: int, host: str = "0.0.0.0") -> socket.socket:
    srv = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
    srv.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
    srv.bind((host, port))
    srv.listen(1)
    return srv


# ----------------------------------------------------------------------------------------------------- dispatcher side
class TcpDispatcher:
    """Dispatcher half of the wire protocol: ship stages, feed node 0, collect from the last node."""

    def __init__(self, codec=None, chunk_size: int = CHUNK_SIZE, timeout: float = 10.0):
        self.codec = codec or default_codec()
        self.chunk_size = chunk_size
        self.timeout = timeout

    def dispatch_stage(self, node_host: str, model_json: str, weights: Sequence[np.ndarray], next_node: str,
                       model_port: int = MODEL_PORT, weights_port: int = WEIGHTS_PORT) -> None:
        """``_dispatchModels`` for one node (``src/dispatcher.py:46-65``): weights first, then JSON + next hop, then wait
        for the 0x06 acknowledgement."""
        ws = _connect((node_host, weights_port), self.timeout)
        try:
            _send_count(ws, len(weights))
            for w in weights:
                socket_send(self.codec.encode(w), ws, self.chunk_size)
            ms = _connect((node_host, model_port), self.timeout)
            try:
                socket_send(model_json.encode(), ms, self.chunk_size)
                socket_send(next_node.encode(), ms, 1)                         # chunk_size = 1, as the reference does
                ready, _, _ = select.select([ms], [], [], max(self.timeout, 600.0))
                if not ready:
                    raise TimeoutError(f"node {node_host}:{model_port} did not acknowledge its stage")
                ms.setblocking(True)
                ack = ms.recv(1)
                if ack != ACK:
                    raise ConnectionError(f"node {node_host}:{model_port} answered {ack!r}, expected 0x06")
            finally:
                ms.close()
        finally:
            ws.close()

    def open_input(self, node_host: str, data_port: int = DATA_PORT) -> socket.socket:
        return _connect((node_host, data_port), self.timeout)                    # src/dispatcher.py:86-88

    def send_input(self, sock: socket.socket, x) -> None:
        socket_send(self.codec.encode(x), sock, self.chunk_size)                 # src/dispatcher.py:90-93

    def result_server(self, output: "queue.Queue", data_port: int = DATA_PORT, stop: Optional[threading.Event] = None,
                      ready: Optional[threading.Event] = None) -> None:
        """``_result_server`` (``src/dispatcher.py:95-105``): accept the last node, decode, ``output.put``."""
        srv = _listen(data_port)
        srv.settimeout(0.2)
        if ready is not None:
            ready.set()
        cli = None
        try:
            while cli is None:
                if stop is not None and stop.is_set():
                    return
                try:
                    cli = srv.accept()[0]
                except socket.timeout:
                    continue
            cli.setblocking(False)
            while stop is None or not stop.is_set():
                r, _, _ = select.select([cli], [], [], 0.2)
                if not r:
                    continue
                try:
                    data = socket_recv(cli, self.chunk_size)
                except ConnectionError:
                    return
                output.put(self.codec.decode(data))
        finally:
            if cli is not None:
                cli.close()
            srv.close()


# ----------------------------------------------------------------------------------------------------- node side
class TcpNode:
    """Node half: the reference's four threads (``src/node.py:110-124``) around a pluggable stage builder.

    ``build_stage(model_json, weights) -> predict`` is what replaces ``model_from_json`` + ``set_weights`` +
    ``_make_predict_function`` (``src/node.py:31-37``); on an H100 it is
    ``lambda j, w: StageRunner.from_wire(j, w, device=0, ...).predict``.
    """

    def __init__(self, build_stage: Callable[[str, List[np.ndarray]], Callable[[np.ndarray], np.ndarray]], codec=None,
                 ports: Tuple[int, int, int] = (DATA_PORT, MODEL_PORT, WEIGHTS_PORT), next_port: Optional[int] = None,
                 chunk_size: int = CHUNK_SIZE, host: str = "0.0.0.0"):
        self.build_stage = build_stage
        self.codec = codec or default_codec()
        self.data_port, self.model_port, self.weights_port = ports
        self.next_port = next_port if next_port is not None else DATA_PORT   # port of the next hop's data server
        self.host = host
        self.state = NodeState(chunk_size)
        self.to_send: "queue.Queue" = queue.Queue(1000)                      # src/node.py:114
        self.stop = threading.Event()
        self.listening = threading.Event()
        self._n_listening = 0
        self._lock = threading.Lock()
        self.error: Optional[BaseException] = None
        self.threads: List[threading.Thread] = []

    # -- helpers
    def _mark_listening(self):
        with self._lock:
            self._n_listening += 1
            if self._n_listening == 3:
                self.listening.set()

    def _accept(self, port: int) -> Optional[socket.socket]:
        srv = _listen(port, self.host)
        srv.settimeout(0.2)
        self._mark_listening()
        try:
            while not self.stop.is_set():
                try:
                    cli = srv.accept()[0]
                    cli.setblocking(False)
                    return cli
                except socket.timeout:
                    continue
            return None
        finally:
            srv.close()

    def _guard(self, fn):
        def run():
            try:
                fn()
            except BaseException as e:   # noqa: BLE001 - surfaced through .error, like the dispatcher's threads
                self.error = e
                self.stop.set()
        return run

    # -- the four roles
    def _weights_socket(self):                                               # src/node.py:45-75
        cli = self._accept(self.weights_port)
        if cli is None:
            return
        try:
            n = _recv_count(cli)
            self.state.weights = [self.codec.decode(socket_recv(cli, self.state.chunk_size)) for _ in range(n)]
        finally:
            cli.close()

    def _model_socket(self):                                                 # src/node.py:20-43
        cli = self._accept(self.model_port)
        if cli is None:
            return
        try:
            model_json = bytes(socket_recv(cli, self.state.chunk_size)).decode()
            next_node = bytes(socket_recv(cli, 1)).decode()
            weights = _wait_state(self.state, "weights", self.stop)          # condition variable, not a 5 s poll
            if weights is None:
                return
            self.state.model = self.build_stage(model_json, weights)
            self.state.next_node = next_node
            select.select([], [cli], [])
            cli.send(ACK)
        finally:
            cli.close()

    def _data_server(self):                                                  # src/node.py:80-91
        cli = self._accept(self.data_port)
        if cli is None:
            return
        try:
            while not self.stop.is_set():
                r, _, _ = select.select([cli], [], [], 0.2)
                if not r:
                    continue
                try:
                    data = socket_recv(cli, self.state.chunk_size)
                except ConnectionError:
                    return
                self.to_send.put(self.codec.decode(data))
        finally:
            cli.close()

    def _data_client(self):                                                  # src/node.py:93-108
        next_node = _wait_state(self.state, "next_node", self.stop)
        if next_node is None:
            return
        predict = self.state.model
        host, _, port = next_node.partition(":")                             # "ip" (reference) or "ip:port" (tests on one host)
        out = _connect((host, int(port) if port else self.next_port), 30.0)
        try:
            while not self.stop.is_set():
                try:
                    inpt = self.to_send.get(timeout=0.2)
                except queue.Empty:
                    continue
                socket_send(self.codec.encode(predict(inpt)), out, self.state.chunk_size)
        finally:
            out.close()

    def start(self) -> "TcpNode":
        for fn in (self._weights_socket, self._model_socket, self._data_server, self._data_client):
            t = threading.Thread(target=self._guard(fn), daemon=True, name=f"tcpnode-{fn.__name__}")
            t.start()
            self.threads.append(t)
        return self

    def run(self):
        """Blocking form, like the reference's ``Node.run`` (``src/node.py:110-124``)."""
        self.start()
        for t in self.threads:
            t.join()

    def close(self):
        self.stop.set()
        for t in self.threads:
            t.join(timeout=5)
