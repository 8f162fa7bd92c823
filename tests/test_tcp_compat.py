"""Network-transport compatibility mode (SURVEY.md 8f rank 2): the reference's TCP handshake and data plane
(reference src/dispatcher.py:44-105, src/node.py:20-108) over real localhost sockets - weight count + framed
arrays on the weights port, JSON + next hop + 0x06 ACK on the model port, framed activations node -> node ->
dispatcher - with a 2-stage ResNet-style model whose stage compute is the CPU oracle (test infrastructure)."""
import queue
import socket
import threading

import numpy as np
import pytest

from defer_b200 import applications, dag_util, tcp_compat
from defer_b200.tcp_compat import ACK, RawCodec, TcpDispatcher, TcpNode


def _free_ports(n):
    socks = []
    for _ in range(n):
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        socks.append(s)
    ports = [s.getsockname()[1] for s in socks]
    for s in socks:
        s.close()
    return ports


def test_raw_codec_roundtrip_is_lossless():
    c = RawCodec()
    rng = np.random.default_rng(0)
    for shape, dt in [((1, 7, 7, 5), np.float32), ((3,), np.float64), ((2, 0, 4), np.float32), ((), np.int64)]:
        a = rng.standard_normal(shape).astype(dt) if np.dtype(dt).kind == "f" else np.array(7, dt)
        b = c.decode(c.encode(a))
        assert b.dtype == a.dtype and b.shape == a.shape and np.array_equal(a, b)
    with pytest.raises(ValueError):
        c.decode(b"\x04\x22M\x18 not ours")        # an lz4 frame magic, i.e. a reference-codec peer


def test_default_codec_falls_back_without_zfpy_lz4():
    c = tcp_compat.default_codec()
    assert isinstance(c, (RawCodec, tcp_compat.ZfpLz4Codec))


@pytest.mark.timeout(120)
def test_two_node_chain_over_tcp_matches_the_whole_model():
    from oracle.keras_ref import WireModel, predict
    m = applications.ResNet50(input_shape=(64, 64, 3))
    cut = "add_6"
    parts = [dag_util.construct_model(m, "input_1", cut, part_name="part1"),
             dag_util.construct_model(m, cut, m.output._keras_history[0].name, part_name="part2")]
    p = _free_ports(7)
    node_ports = [(p[0], p[1], p[2]), (p[3], p[4], p[5])]
    result_port = p[6]
    built = []

    def build_stage(model_json, weights):       # stands in for StageRunner.from_wire(...).predict on a GPU node
        ref = WireModel(model_json, weights)
        built.append(len(weights))
        return lambda x: ref.predict(np.asarray(x, np.float32))

    nodes = [TcpNode(build_stage, codec=RawCodec(), ports=node_ports[i], host="127.0.0.1").start() for i in range(2)]
    disp = TcpDispatcher(codec=RawCodec(), timeout=30.0)
    out_q, stop, ready = queue.Queue(), threading.Event(), threading.Event()
    rs = threading.Thread(target=disp.result_server, args=(out_q, result_port, stop, ready), daemon=True)
    rs.start()
    try:
        assert ready.wait(10) and all(n.listening.wait(10) for n in nodes)
        # the reference's placement loop: stage i -> node i, next hop = node i+1, the last one points back at the dispatcher
        for i, part in enumerate(parts):
            nxt = f"127.0.0.1:{node_ports[i + 1][0]}" if i == 0 else f"127.0.0.1:{result_port}"
            disp.dispatch_stage("127.0.0.1", part.to_json(), part.get_weights(), nxt, model_port=node_ports[i][1],
                                weights_port=node_ports[i][2])
        assert built == [len(parts[0].get_weights()), len(parts[1].get_weights())]      # both ACKed after building
        feed = disp.open_input("127.0.0.1", node_ports[0][0])
        xs = [applications.synthetic_input(1, shape=(64, 64, 3), seed=s) for s in range(4)]
        for x in xs:
            disp.send_input(feed, x)
        got = [out_q.get(timeout=60) for _ in xs]
        feed.close()
        for x, y in zip(xs, got):                                                        # FIFO, lossless hops
            want = predict(m.to_json(), m.get_weights(), x)
            assert y.shape == (1, 1000) and np.array_equal(y, want)
        assert all(n.error is None for n in nodes)
    finally:
        stop.set()
        for n in nodes:
            n.close()
        rs.join(timeout=5)


def test_ack_byte_and_ports_are_the_references():
    assert ACK == b"\x06" and (tcp_compat.DATA_PORT, tcp_compat.MODEL_PORT, tcp_compat.WEIGHTS_PORT) == (5000, 5001, 5002)
    assert tcp_compat.CHUNK_SIZE == 512 * 1000
