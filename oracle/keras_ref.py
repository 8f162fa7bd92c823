"""ORACLE - TEST INFRASTRUCTURE ONLY.  CPU restatement of the reference's stage arithmetic.

PARITY UNPINNED WITH RESPECT TO THE REFERENCE ITSELF: ANRGUSC/DEFER cannot be executed in this image - its
arithmetic lives in un-vendored, un-pinned third-party wheels (TensorFlow ~1.14 + keras_applications 1.0.8, zfpy,
lz4; call sites ``src/node.py:31,34,106``, ``src/dispatcher.py:49,57``, ``test/test.py:14``) that are
not installed and not installable offline, and none of its scripts compares a value (``test/test.py:34`` prints
shapes).  This file therefore restates the *published* Keras layer semantics those call sites rely on.

What pins it instead (round 2): an implementation we did not write.  ``tests/test_oracle_pin.py`` transplants the
seeded Keras-layout weights into ``torchvision.models.vgg16`` (arithmetically the Keras VGG16, 138 357 544 parameters)
and into ``torchvision.models.resnet50`` with the stride moved from the 3x3 to the first 1x1 convolution, conv biases
folded into the BatchNorm means and eps = 1e-3 (exactly the deltas between torchvision's v1.5 and keras_applications'
``resnet50.py``); this oracle and the model zoo's graph JSON must reproduce torchvision's class probabilities to 1e-9
(fp64) / 1e-5 (fp32), and an intermediate tensor (end of conv3_x) to 1e-9.  That removes the failure mode where the
builder's graph and the builder's oracle share a topology mistake.  Further pins: Keras' parameter counts for the three
nets, hand-computed known-answer cases and a pure-Python-loop convolution (``tests/test_oracle.py``), agreement with an
independent executor (``oracle/torch_cpu.py``), committed golden vectors (``tests/golden/``).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / reference legs may
import this module.  The product (``defer_b200``) never does.

What is restated
----------------
* ``tf.keras.Model.predict`` on a functional (sub-)model given its wire format - the JSON config
  and the flat weight list the dispatcher ships (``src/dispatcher.py:49,57``; ``src/node.py:31,34,106``).
  Layers: Conv2D (HWIO kernel, bias, valid/same, fused activation), BatchNormalization in inference
  mode ``gamma*(x-mean)/sqrt(var+eps)+beta``, Activation(relu|softmax), Add, ZeroPadding2D,
  MaxPooling2D(valid), GlobalAveragePooling2D, Flatten (H,W,C order), Dense.
* the partition rule of ``src/dag_util.py:9-31`` + ``src/dispatcher.py:27-42``: stage p holds the
  layers strictly after ``cuts[p-1]`` through ``cuts[p]``.
* the hop: ``lz4(zfp_reversible(arr))`` is lossless (``src/node.py:76-79``), i.e. identity on fp32.
"""
from __future__ import annotations

import json
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np


# --------------------------------------------------------------------------- layer arithmetic

def same_pad(size: int, k: int, s: int) -> Tuple[int, int]:
    """TF 'SAME' padding: total = max((ceil(size/s)-1)*s + k - size, 0); extra goes after."""
    out = -(-size // s)
    total = max((out - 1) * s + k - size, 0)
    return total // 2, total - total // 2


def conv2d(x: np.ndarray, w: np.ndarray, b: Optional[np.ndarray], strides=(1, 1), padding="valid") -> np.ndarray:
    """NHWC x HWIO convolution (cross-correlation, as Keras) via im2col + one matmul."""
    kh, kw, cin, cout = w.shape
    sh, sw = strides
    if padding == "same":
        pt, pb = same_pad(x.shape[1], kh, sh)
        pl, pr = same_pad(x.shape[2], kw, sw)
        x = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    n, h, wd, c = x.shape
    assert c == cin, (x.shape, w.shape)
    ho = (h - kh) // sh + 1
    wo = (wd - kw) // sw + 1
    if kh == 1 and kw == 1:
        cols = x[:, ::sh, ::sw, :][:, :ho, :wo, :].reshape(n * ho * wo, cin)
    else:
        s0, s1, s2, s3 = x.strides
        patches = np.lib.stride_tricks.as_strided(
            x, shape=(n, ho, wo, kh, kw, c), strides=(s0, s1 * sh, s2 * sw, s1, s2, s3), writeable=False)
        cols = patches.reshape(n * ho * wo, kh * kw * c)
    y = cols @ w.reshape(kh * kw * cin, cout)
    if b is not None:
        y = y + b
    return y.reshape(n, ho, wo, cout)


def conv2d_loops(x: np.ndarray, w: np.ndarray, b, strides=(1, 1), padding="valid") -> np.ndarray:
    """Pure-Python-loop convolution in float64 - small cases only; pins ``conv2d``."""
    kh, kw, cin, cout = w.shape
    sh, sw = strides
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    if padding == "same":
        pt, pb = same_pad(x.shape[1], kh, sh)
        pl, pr = same_pad(x.shape[2], kw, sw)
        x = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    n, h, wd, _ = x.shape
    ho = (h - kh) // sh + 1
    wo = (wd - kw) // sw + 1
    y = np.zeros((n, ho, wo, cout), np.float64)
    for bi in range(n):
        for i in range(ho):
            for j in range(wo):
                for co in range(cout):
                    acc = 0.0
                    for a in range(kh):
                        for bb in range(kw):
                            for ci in range(cin):
                                acc += x[bi, i * sh + a, j * sw + bb, ci] * w[a, bb, ci, co]
                    y[bi, i, j, co] = acc + (0.0 if b is None else float(b[co]))
    return y


def batchnorm(x, gamma, beta, mean, var, eps):
    dt = x.dtype
    inv = (gamma.astype(dt) / np.sqrt(var.astype(dt) + dt.type(eps)))
    return (x - mean.astype(dt)) * inv + beta.astype(dt)


def relu(x):
    return np.maximum(x, 0)


def softmax(x):
    z = x - x.max(axis=-1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(axis=-1, keepdims=True)


def maxpool2d(x, pool, strides):
    ph, pw = pool
    sh, sw = strides
    n, h, w, c = x.shape
    ho = (h - ph) // sh + 1
    wo = (w - pw) // sw + 1
    s0, s1, s2, s3 = x.strides
    win = np.lib.stride_tricks.as_strided(x, shape=(n, ho, wo, ph, pw, c),
                                          strides=(s0, s1 * sh, s2 * sw, s1, s2, s3), writeable=False)
    return win.max(axis=(3, 4))


def zeropad2d(x, padding):
    (t, b), (l, r) = padding
    return np.pad(x, ((0, 0), (t, b), (l, r), (0, 0)))


def apply_activation(y, act):
    if act in (None, "linear"):
        return y
    if act == "relu":
        return relu(y)
    if act == "softmax":
        return softmax(y)
    raise ValueError(act)


# --------------------------------------------------------------------------- wire-format executor

class WireModel:
    """A (sub-)model in wire format: Keras-style JSON config + flat weight list."""

    def __init__(self, json_text, weights: Sequence[np.ndarray]):
        if isinstance(json_text, (bytes, bytearray)):
            json_text = bytes(json_text).decode()
        cfg = json.loads(json_text)["config"]
        self.name = cfg.get("name", "")
        self.layers = cfg["layers"]
        self.input_name = cfg["input_layers"][0][0]
        self.output_name = cfg["output_layers"][0][0]
        self.by_name = {l["name"]: l for l in self.layers}
        # assign weights in layer order (Keras get_weights order)
        self.weights: Dict[str, List[np.ndarray]] = {}
        i = 0
        for l in self.layers:
            n = self._n_weights(l)
            self.weights[l["name"]] = [np.asarray(a) for a in weights[i:i + n]]
            i += n
        if i != len(weights):
            raise ValueError(f"{len(weights)} weight arrays given, {i} consumed")

    @staticmethod
    def _n_weights(l) -> int:
        cn, c = l["class_name"], l["config"]
        if cn in ("Conv2D", "Dense"):
            return 2 if c.get("use_bias", True) else 1
        if cn == "BatchNormalization":
            return 4
        return 0

    def inbound(self, name) -> List[str]:
        nodes = self.by_name[name]["inbound_nodes"]
        return [e[0] for e in nodes[0]] if nodes else []

    def topo_order(self) -> List[str]:
        order, seen = [], set()
        stack = [(self.output_name, False)]
        while stack:
            n, done = stack.pop()
            if done:
                order.append(n)
                continue
            if n in seen:
                continue
            seen.add(n)
            stack.append((n, True))
            for p in reversed(self.inbound(n)):
                if p not in seen:
                    stack.append((p, False))
        return order

    def predict(self, x: np.ndarray, dtype=np.float32, return_all: bool = False,
                final_activation: bool = True):
        """Keras ``predict`` semantics.  ``final_activation=False`` returns the pre-softmax logits
        when the output layer ends in a softmax (for non-saturated comparisons)."""
        dt = np.dtype(dtype)
        vals: Dict[str, np.ndarray] = {self.input_name: np.asarray(x, dt)}
        for name in self.topo_order():
            if name == self.input_name:
                continue
            l = self.by_name[name]
            cn, c = l["class_name"], l["config"]
            ins = [vals[p] for p in self.inbound(name)]
            w = [a.astype(dt) for a in self.weights[name]]
            last = name == self.output_name
            if cn == "Conv2D":
                y = conv2d(ins[0], w[0], w[1] if len(w) > 1 else None, tuple(c["strides"]), c["padding"])
                y = apply_activation(y, c.get("activation"))
            elif cn == "Dense":
                y = ins[0] @ w[0]
                if len(w) > 1:
                    y = y + w[1]
                act = c.get("activation")
                if last and not final_activation and act == "softmax":
                    act = None
                y = apply_activation(y, act)
            elif cn == "BatchNormalization":
                y = batchnorm(ins[0], w[0], w[1], w[2], w[3], c["epsilon"])
            elif cn == "Activation":
                act = c["activation"]
                if last and not final_activation and act == "softmax":
                    act = None
                y = apply_activation(ins[0], act)
            elif cn == "Add":
                y = ins[0]
                for t in ins[1:]:
                    y = y + t
            elif cn == "ZeroPadding2D":
                y = zeropad2d(ins[0], c["padding"])
            elif cn == "MaxPooling2D":
                y = maxpool2d(ins[0], tuple(c["pool_size"]), tuple(c["strides"]))
            elif cn == "GlobalAveragePooling2D":
                y = ins[0].mean(axis=(1, 2), dtype=dt)
            elif cn == "Flatten":
                y = ins[0].reshape(ins[0].shape[0], -1)
            else:
                raise ValueError(f"oracle: unsupported layer class {cn}")
            vals[name] = np.ascontiguousarray(y, dtype=dt)
        return vals if return_all else vals[self.output_name]


def predict(json_text, weights, x, dtype=np.float32, **kw):
    return WireModel(json_text, weights).predict(x, dtype=dtype, **kw)


# --------------------------------------------------------------------------- partition rule

def stage_layer_sets(json_text, cuts: Sequence[str]) -> List[List[str]]:
    """Layer names each stage computes under the reference rule (``src/dispatcher.py:30-41`` +
    ``src/dag_util.py:9-25``): walk back from ``end`` and stop at ``start``.  Independent of the
    product partitioner (works on the wire JSON)."""
    wm = WireModel(json_text, _dummy_weights(json_text))
    bounds = [wm.input_name] + list(cuts) + [wm.output_name]
    stages = []
    for p in range(len(bounds) - 1):
        start, end = bounds[p], bounds[p + 1]
        seen, stack = set(), [end]
        while stack:
            n = stack.pop()
            if n == start or n in seen:
                continue
            seen.add(n)
            prev = wm.inbound(n)
            if not prev:
                raise ValueError(f"cut {start!r} is not an articulation point (reached {n!r})")
            stack.extend(prev)
        stages.append(sorted(seen))
    return stages


def _dummy_weights(json_text):
    cfg = json.loads(json_text)["config"]
    return [np.zeros(1, np.float32)] * sum(WireModel._n_weights(l) for l in cfg["layers"])


def pipeline_predict(stage_wire: Sequence[Tuple[str, Sequence[np.ndarray]]], x, dtype=np.float32, **kw):
    """Chain of stages with the identity (lossless) hop between them."""
    y = x
    for i, (js, ws) in enumerate(stage_wire):
        last = i == len(stage_wire) - 1
        y = WireModel(js, ws).predict(y, dtype=dtype, **(kw if last else {}))
    return y


def rel_err(y, ref) -> float:
    """The parity figure of SURVEY.md 8d: max|y - ref| / max|ref|."""
    y = np.asarray(y, np.float64)
    ref = np.asarray(ref, np.float64)
    return float(np.max(np.abs(y - ref)) / max(np.max(np.abs(ref)), 1e-30))
