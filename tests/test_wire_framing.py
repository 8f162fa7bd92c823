"""The reference's TCP framing (src/node_state.py:43-101): 8-byte big-endian length + chunked payload on
non-blocking sockets.  Host-side compatibility helper; not on the GPU hot path."""
import socket
import threading

import numpy as np
import pytest

from defer_b200.node_state import socket_recv, socket_send


def _pair(nonblocking=True):
    a, b = socket.socketpair()
    if nonblocking:
        a.setblocking(False)
        b.setblocking(False)
    return a, b


@pytest.mark.parametrize("size,chunk", [(0, 512000), (1, 1), (17, 4), (512000, 512000), (3_211_264, 512000), (1000, 1)])
def test_roundtrip_sizes(size, chunk):
    a, b = _pair()
    payload = np.random.default_rng(size).integers(0, 256, size, dtype=np.uint8).tobytes()
    out = {}
    t = threading.Thread(target=lambda: out.setdefault("d", socket_recv(b, chunk)))
    t.start()
    socket_send(payload, a, chunk)
    t.join(timeout=30)
    assert not t.is_alive()
    assert bytes(out["d"]) == payload and isinstance(out["d"], bytearray)
    a.close(); b.close()


def test_frame_layout_matches_reference_format():
    a, b = _pair(nonblocking=False)
    socket_send(b"abc", a, 2)
    raw = b.recv(64)
    assert raw == (3).to_bytes(8, "big") + b"abc"
    # a frame produced by hand (what a reference node would send) is readable
    a.sendall((5).to_bytes(8, "big") + b"hello")
    assert bytes(socket_recv(b, 512000)) == b"hello"
    a.close(); b.close()


def test_back_to_back_frames_and_next_hop_chunk1():
    # the dispatcher sends the JSON with chunk 512000 and the next-hop string with chunk_size=1 (src/dispatcher.py:62-63)
    a, b = _pair()
    got = []
    t = threading.Thread(target=lambda: got.extend([socket_recv(b, 512000), socket_recv(b, 1)]))
    t.start()
    socket_send(b'{"class_name": "Model"}', a, 512000)
    socket_send("cuda:3".encode(), a, chunk_size=1)
    t.join(timeout=30)
    assert [bytes(g) for g in got] == [b'{"class_name": "Model"}', b"cuda:3"]
    a.close(); b.close()


def test_peer_close_mid_frame_raises():
    a, b = _pair(nonblocking=False)
    a.sendall((100).to_bytes(8, "big") + b"short")
    a.close()
    with pytest.raises(ConnectionError):
        socket_recv(b, 512000)
    b.close()
