"""Keras-free layer-DAG IR exposing exactly the surface DEFER touches.

The reference partitions a ``tf.keras.Model`` (``src/dag_util.py:3-31``,
``src/dispatcher.py:27-42``) and ships ``to_json()`` + ``get_weights()`` to each node
(``src/dispatcher.py:49,57``; rebuilt with ``model_from_json`` + ``set_weights`` at
``src/node.py:31,34``).  TensorFlow is not installable here, so this module is a small
functional-API graph with the same attribute names:

* ``model.get_layer(name)``, ``layer.inbound_nodes[0].inbound_layers`` (a single layer when
  there is one inbound edge, a list otherwise - the case ``dag_util.get_previous`` checks for),
  ``layer.output``, ``tensor._keras_history[0].name`` (``src/dispatcher.py:32,37``);
* ``Input(tensor=..., name=...)``, ``layer(x)`` re-application with shared weights
  (``src/dag_util.py:23-24,28``), ``Model(inputs=, outputs=)`` (``src/dag_util.py:30``);
* ``to_json`` / ``model_from_json`` / ``get_weights`` / ``set_weights`` in Keras layer order.

It holds graph structure and host weights only; arithmetic lives in the CUDA library
(``defer_b200/csrc``) and, for tests, in ``oracle/``.
"""
from __future__ import annotations

import json
import re
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

# --------------------------------------------------------------------------- naming

_UIDS: Dict[str, int] = {}


def clear_session() -> None:
    """Reset auto-naming counters (tf.keras ``backend.clear_session`` analogue)."""
    _UIDS.clear()


def _to_snake_case(name: str) -> str:
    s = re.sub("(.)([A-Z][a-z0-9]+)", r"\1_\2", name)
    s = re.sub("([a-z])([A-Z])", r"\1_\2", s).lower()
    return s


def _unique_name(prefix: str, zero_based: bool) -> str:
    n = _UIDS.get(prefix, 0)
    _UIDS[prefix] = n + 1
    if zero_based:  # tf.keras: add, add_1, ...
        return prefix if n == 0 else f"{prefix}_{n}"
    return f"{prefix}_{n + 1}"  # input_1, input_2, ...


# --------------------------------------------------------------------------- graph objects

Shape = Tuple[Optional[int], ...]


class SymbolicTensor:
    """Placeholder for a layer output; carries shape and ``_keras_history``."""

    def __init__(self, shape: Shape, layer: "Layer", node_index: int, name: str):
        self.shape = tuple(shape)
        self._keras_history = (layer, node_index, 0)
        self.name = name

    def __repr__(self) -> str:
        return f"<SymbolicTensor {self.name} shape={self.shape}>"


class Node:
    """One application of a layer to input tensors (Keras ``Node``)."""

    def __init__(self, outbound_layer: "Layer", input_tensors: List[SymbolicTensor]):
        self.outbound_layer = outbound_layer
        self.input_tensors = list(input_tensors)
        self.output_tensor: Optional[SymbolicTensor] = None
        # recorded at creation, as Keras does: Input(tensor=...) later re-tags tensor histories
        self._inbound_layers = [t._keras_history[0] for t in self.input_tensors]

    @property
    def inbound_layers(self):
        layers = list(self._inbound_layers)
        # TF 1.14 returns the bare layer for a single inbound edge, a list otherwise;
        # dag_util.get_previous (reference src/dag_util.py:4-6) handles both.
        if len(layers) == 1:
            return layers[0]
        return layers

    def iterate_inbound(self):
        for t in self.input_tensors:
            layer, node_index, tensor_index = t._keras_history
            yield layer, node_index, tensor_index, t


class Layer:
    class_name = "Layer"
    auto_name_zero_based = True

    def __init__(self, name: Optional[str] = None):
        if name is None:
            name = _unique_name(_to_snake_case(type(self).__name__), self.auto_name_zero_based)
        self.name = name
        self._inbound_nodes: List[Node] = []
        self._weights: List[np.ndarray] = []
        self.built = False

    # -- graph wiring
    @property
    def inbound_nodes(self) -> List[Node]:
        return self._inbound_nodes

    @property
    def output(self) -> SymbolicTensor:
        if not self._inbound_nodes:
            raise AttributeError(f"Layer {self.name} has no inbound nodes")
        return self._inbound_nodes[0].output_tensor

    @property
    def input(self):
        node = self._inbound_nodes[0]
        return node.input_tensors[0] if len(node.input_tensors) == 1 else node.input_tensors

    def __call__(self, inputs):
        tensors = list(inputs) if isinstance(inputs, (list, tuple)) else [inputs]
        for t in tensors:
            if not isinstance(t, SymbolicTensor):
                raise TypeError(f"{self.name}: expected SymbolicTensor, got {type(t)}")
        in_shapes = [t.shape for t in tensors]
        if not self.built:
            self.build(in_shapes)
            self.built = True
        out_shape = self.compute_output_shape(in_shapes)
        node = Node(self, tensors)
        idx = len(self._inbound_nodes)
        node.output_tensor = SymbolicTensor(out_shape, self, idx, f"{self.name}/out:{idx}")
        self._inbound_nodes.append(node)
        return node.output_tensor

    # -- to be specialised
    def build(self, input_shapes: List[Shape]) -> None:
        pass

    def compute_output_shape(self, input_shapes: List[Shape]) -> Shape:
        return input_shapes[0]

    def get_config(self) -> dict:
        return {"name": self.name}

    # -- weights (Keras order, numpy float32)
    weight_names: Tuple[str, ...] = ()

    def weight_shapes(self) -> List[Tuple[int, ...]]:
        return []

    def get_weights(self) -> List[np.ndarray]:
        return list(self._weights)

    def set_weights(self, weights: Sequence[np.ndarray]) -> None:
        shapes = self.weight_shapes()
        if len(weights) != len(shapes):
            raise ValueError(f"{self.name}: expected {len(shapes)} weight arrays, got {len(weights)}")
        out = []
        for w, s in zip(weights, shapes):
            w = np.ascontiguousarray(w, dtype=np.float32)
            if tuple(w.shape) != tuple(s):
                raise ValueError(f"{self.name}: weight shape {w.shape} != expected {s}")
            out.append(w)
        self._weights = out

    def count_params(self) -> int:
        return int(sum(int(np.prod(s)) for s in self.weight_shapes()))

    def __repr__(self) -> str:
        return f"<{type(self).__name__} {self.name}>"


def _pair(v) -> Tuple[int, int]:
    if isinstance(v, (list, tuple)):
        return int(v[0]), int(v[1])
    return int(v), int(v)


def _conv_out(size: Optional[int], k: int, s: int, padding: str) -> Optional[int]:
    if size is None:
        return None
    if padding == "same":
        return (size + s - 1) // s
    return (size - k) // s + 1


class InputLayer(Layer):
    class_name = "InputLayer"
    auto_name_zero_based = False

    def __init__(self, batch_input_shape: Shape, name: Optional[str] = None,
                 input_tensor: Optional[SymbolicTensor] = None):
        if name is None:
            name = _unique_name("input", zero_based=False)
        super().__init__(name)
        self.batch_input_shape = tuple(batch_input_shape)
        self.built = True
        node = Node(self, [])
        if input_tensor is not None:
            # TF 1.x InputLayer(input_tensor=t) returns t itself and re-tags t._keras_history; here the
            # SAME tensor object is kept (so Model(inputs=start.output, ...) of src/dag_util.py:30 sees it)
            # and the new input layer is recorded as an alias instead of overwriting the history - the
            # original model stays intact and can be partitioned again.
            input_tensor._input_alias = (self, 0, 0)
            node.output_tensor = input_tensor
        else:
            node.output_tensor = SymbolicTensor(self.batch_input_shape, self, 0, f"{self.name}:0")
        self._inbound_nodes.append(node)

    def get_config(self):
        return {"name": self.name, "batch_input_shape": list(self.batch_input_shape), "dtype": "float32"}


def Input(shape: Optional[Sequence[int]] = None, tensor: Optional[SymbolicTensor] = None,
          name: Optional[str] = None) -> SymbolicTensor:
    """``tf.keras.Input``.  With ``tensor=`` the SAME tensor object is returned, standing for the output
    of a new ``InputLayer`` named ``name`` - what reference ``src/dag_util.py:28,30`` relies on
    (``Model(inputs=model.get_layer(start).output, ...)`` passes the original tensor)."""
    if tensor is not None:
        layer = InputLayer(tensor.shape, name=name, input_tensor=tensor)
        return layer.output
    if shape is None:
        raise ValueError("Input needs shape= or tensor=")
    layer = InputLayer((None,) + tuple(shape), name=name)
    return layer.output


class Conv2D(Layer):
    class_name = "Conv2D"

    def __init__(self, filters, kernel_size, strides=(1, 1), padding="valid", activation=None,
                 use_bias=True, name=None, **_ignored):
        super().__init__(name)
        self.filters = int(filters)
        self.kernel_size = _pair(kernel_size)
        self.strides = _pair(strides)
        self.padding = str(padding).lower()
        if self.padding not in ("valid", "same"):
            raise ValueError(f"{self.name}: padding {padding!r}")
        self.activation = activation if activation not in ("linear",) else None
        self.use_bias = bool(use_bias)
        self.in_channels: Optional[int] = None

    def build(self, input_shapes):
        self.in_channels = int(input_shapes[0][-1])
        if not self._weights:
            self._weights = [np.zeros(s, np.float32) for s in self.weight_shapes()]

    def weight_shapes(self):
        kh, kw = self.kernel_size
        s = [(kh, kw, self.in_channels, self.filters)]  # HWIO
        if self.use_bias:
            s.append((self.filters,))
        return s

    def compute_output_shape(self, input_shapes):
        n, h, w, _ = input_shapes[0]
        return (n, _conv_out(h, self.kernel_size[0], self.strides[0], self.padding),
                _conv_out(w, self.kernel_size[1], self.strides[1], self.padding), self.filters)

    def get_config(self):
        return {"name": self.name, "filters": self.filters, "kernel_size": list(self.kernel_size),
                "strides": list(self.strides), "padding": self.padding,
                "activation": self.activation or "linear", "use_bias": self.use_bias,
                "data_format": "channels_last"}


class Dense(Layer):
    class_name = "Dense"

    def __init__(self, units, activation=None, use_bias=True, name=None, **_ignored):
        super().__init__(name)
        self.units = int(units)
        self.activation = activation if activation not in ("linear",) else None
        self.use_bias = bool(use_bias)
        self.in_features: Optional[int] = None

    def build(self, input_shapes):
        self.in_features = int(input_shapes[0][-1])
        if not self._weights:
            self._weights = [np.zeros(s, np.float32) for s in self.weight_shapes()]

    def weight_shapes(self):
        s = [(self.in_features, self.units)]
        if self.use_bias:
            s.append((self.units,))
        return s

    def compute_output_shape(self, input_shapes):
        return tuple(input_shapes[0][:-1]) + (self.units,)

    def get_config(self):
        return {"name": self.name, "units": self.units, "activation": self.activation or "linear",
                "use_bias": self.use_bias}


class BatchNormalization(Layer):
    """Inference-mode BN: y = gamma * (x - mean) / sqrt(var + eps) + beta (moving stats)."""
    class_name = "BatchNormalization"

    def __init__(self, axis=-1, epsilon=1e-3, name=None, **_ignored):
        super().__init__(name)
        self.axis = int(axis)
        self.epsilon = float(epsilon)
        self.channels: Optional[int] = None

    def build(self, input_shapes):
        rank = len(input_shapes[0])
        if self.axis not in (-1, rank - 1):
            raise ValueError(f"{self.name}: only channels_last BN is supported")
        self.channels = int(input_shapes[0][-1])
        if not self._weights:
            c = self.channels
            self._weights = [np.ones(c, np.float32), np.zeros(c, np.float32),
                             np.zeros(c, np.float32), np.ones(c, np.float32)]

    def weight_shapes(self):
        return [(self.channels,)] * 4  # gamma, beta, moving_mean, moving_variance

    def get_config(self):
        return {"name": self.name, "axis": -1, "epsilon": self.epsilon}


class Activation(Layer):
    class_name = "Activation"

    def __init__(self, activation, name=None):
        super().__init__(name)
        self.activation = str(activation)
        if self.activation not in ("relu", "softmax", "linear"):
            raise ValueError(f"{self.name}: unsupported activation {activation!r}")

    def get_config(self):
        return {"name": self.name, "activation": self.activation}


class Add(Layer):
    class_name = "Add"

    def compute_output_shape(self, input_shapes):
        if len(input_shapes) < 2:
            raise ValueError(f"{self.name}: Add needs at least 2 inputs")
        for s in input_shapes[1:]:
            if tuple(s) != tuple(input_shapes[0]):
                raise ValueError(f"{self.name}: shape mismatch {input_shapes}")
        return input_shapes[0]


class ZeroPadding2D(Layer):
    class_name = "ZeroPadding2D"

    def __init__(self, padding=(1, 1), name=None):
        super().__init__(name)
        if isinstance(padding, int):
            p = ((padding, padding), (padding, padding))
        else:
            a, b = padding
            p = (_pair(a) if isinstance(a, (list, tuple)) else (int(a), int(a)),
                 _pair(b) if isinstance(b, (list, tuple)) else (int(b), int(b)))
        self.padding = p

    def compute_output_shape(self, input_shapes):
        n, h, w, c = input_shapes[0]
        (t, b), (l, r) = self.padding
        return (n, None if h is None else h + t + b, None if w is None else w + l + r, c)

    def get_config(self):
        return {"name": self.name, "padding": [list(self.padding[0]), list(self.padding[1])],
                "data_format": "channels_last"}


class MaxPooling2D(Layer):
    class_name = "MaxPooling2D"

    def __init__(self, pool_size=(2, 2), strides=None, padding="valid", name=None):
        super().__init__(name)
        self.pool_size = _pair(pool_size)
        self.strides = _pair(strides) if strides is not None else self.pool_size
        self.padding = str(padding).lower()
        if self.padding != "valid":
            raise ValueError(f"{self.name}: only 'valid' max-pooling occurs in the supported nets")

    def compute_output_shape(self, input_shapes):
        n, h, w, c = input_shapes[0]
        return (n, _conv_out(h, self.pool_size[0], self.strides[0], "valid"),
                _conv_out(w, self.pool_size[1], self.strides[1], "valid"), c)

    def get_config(self):
        return {"name": self.name, "pool_size": list(self.pool_size), "strides": list(self.strides),
                "padding": self.padding, "data_format": "channels_last"}


class GlobalAveragePooling2D(Layer):
    class_name = "GlobalAveragePooling2D"

    def compute_output_shape(self, input_shapes):
        n, _, _, c = input_shapes[0]
        return (n, c)


class Flatten(Layer):
    """Row-major (H, W, C) flatten - fc1 rows of VGG16 follow this order."""
    class_name = "Flatten"

    def compute_output_shape(self, input_shapes):
        s = input_shapes[0]
        if any(d is None for d in s[1:]):
            raise ValueError(f"{self.name}: cannot flatten unknown dims {s}")
        return (s[0], int(np.prod(s[1:])))


LAYER_CLASSES = {c.class_name: c for c in (InputLayer, Conv2D, Dense, BatchNormalization, Activation, Add,
                                           ZeroPadding2D, MaxPooling2D, GlobalAveragePooling2D, Flatten)}


# --------------------------------------------------------------------------- Model

class Model:
    """Functional model: the sub-graph between ``inputs`` and ``outputs``.

    Layer order follows Keras' ``_map_graph_network`` (depth-descending, ties by first visit in a
    DFS from the outputs) so ``get_weights()`` lists arrays in the order Keras would.
    Each entry of ``self.nodes`` is ``(layer, node_index)`` in execution order.
    """

    def __init__(self, inputs, outputs, name: Optional[str] = None):
        self.inputs: List[SymbolicTensor] = list(inputs) if isinstance(inputs, (list, tuple)) else [inputs]
        self.outputs: List[SymbolicTensor] = list(outputs) if isinstance(outputs, (list, tuple)) else [outputs]
        if len(self.inputs) != 1 or len(self.outputs) != 1:
            raise ValueError("DEFER partitions single-input single-output chains (src/dispatcher.py:32,37)")
        self.name = name or _unique_name("model", zero_based=True)
        self._map_graph()

    # Keras attribute names used by the dispatcher
    @property
    def input(self) -> SymbolicTensor:
        return self.inputs[0]

    @property
    def output(self) -> SymbolicTensor:
        return self.outputs[0]

    def _map_graph(self) -> None:
        input_ids = {id(t) for t in self.inputs}
        layer_indices: Dict[Layer, int] = {}
        order: List[Tuple[Layer, int]] = []      # nodes, producers first (post-order)
        finished = set()
        in_progress = set()
        node_inputs: Dict[Tuple[int, int], List[SymbolicTensor]] = {}

        def hist(t: SymbolicTensor):
            # a model input given as Input(tensor=t) is produced by its alias InputLayer in THIS model
            if id(t) in input_ids and getattr(t, "_input_alias", None) is not None:
                return t._input_alias
            return t._keras_history

        def build_map(tensor: SymbolicTensor) -> None:
            # iterative DFS: recursion depth would exceed Python's limit on ResNet152
            stack = [(tensor, 0)]
            while stack:
                t, state = stack.pop()
                layer, node_index, _ = hist(t)
                key = (id(layer), node_index)
                if state == 0:
                    if key in finished:
                        continue
                    if key in in_progress:
                        raise ValueError(f"cycle at layer {layer.name}")
                    if layer not in layer_indices:
                        layer_indices[layer] = len(layer_indices)
                    in_progress.add(key)
                    stack.append((t, 1))
                    if id(t) in input_ids:
                        node_inputs[key] = []
                        continue
                    node = layer._inbound_nodes[node_index]
                    if isinstance(layer, InputLayer):
                        raise ValueError(
                            f"graph reaches InputLayer {layer.name} which is not a model input "
                            "(cut layer is not an articulation point?)")
                    node_inputs[key] = list(node.input_tensors)
                    for it in reversed(node.input_tensors):
                        stack.append((it, 0))
                else:
                    in_progress.discard(key)
                    if key not in finished:
                        finished.add(key)
                        order.append((layer, node_index))

        for o in self.outputs:
            build_map(o)

        # depths (Keras: outputs depth 0, producers deeper)
        node_depth: Dict[Tuple[int, int], int] = {}
        layer_depth: Dict[Layer, int] = {}
        for layer, node_index in reversed(order):
            key = (id(layer), node_index)
            d = max(node_depth.get(key, 0), layer_depth.get(layer, 0))
            node_depth[key] = d
            layer_depth[layer] = d
            for it in node_inputs[key]:
                il, ini, _ = hist(it)
                ikey = (id(il), ini)
                node_depth[ikey] = max(d + 1, node_depth.get(ikey, 0))
        # the model's input tensors are represented by (possibly synthetic) input layers at max depth
        self._input_keys = {(id(hist(t)[0]), hist(t)[1]) for t in self.inputs}
        # frozen now: a later Input(tensor=...) on the same tensor (another partition) changes its alias
        self._input_layers = [hist(t)[0] for t in self.inputs]
        self._output_layers = [t._keras_history[0] for t in self.outputs]
        max_d = max(layer_depth.values()) if layer_depth else 0
        for l in self._input_layers:
            layer_depth[l] = max_d

        layers = sorted(layer_depth.keys(), key=lambda l: (-layer_depth[l], layer_indices[l]))
        self._node_order = order
        self._node_inputs = node_inputs
        self._node_input_names = {k: [hist(t)[0].name for t in v] for k, v in node_inputs.items()}
        self._layer_depth = layer_depth
        # Layers whose *output* is the model input stand in as the InputLayer of this model.
        self.layers: List[Layer] = layers
        names = [l.name for l in layers]
        if len(set(names)) != len(names):
            raise ValueError("duplicate layer names in model")
        self._by_name = {l.name: l for l in layers}

    def get_layer(self, name: str) -> Layer:
        try:
            return self._by_name[name]
        except KeyError:
            raise ValueError(f"No such layer: {name}") from None

    # -- execution-ordered description (used by planner and oracle via JSON)
    def iter_nodes(self):
        """Yield ``(layer, input_layer_names)`` producers-first; model inputs yield ``(layer, None)``."""
        for layer, node_index in self._node_order:
            key = (id(layer), node_index)
            if key in self._input_keys:
                yield layer, None
            else:
                yield layer, list(self._node_input_names[key])

    # -- weights
    def _weighted_layers(self) -> List[Layer]:
        inputs = set(self._input_layers)
        return [l for l in self.layers if l not in inputs and l.weight_shapes()]

    def get_weights(self) -> List[np.ndarray]:
        out: List[np.ndarray] = []
        for l in self._weighted_layers():
            out.extend(l.get_weights())
        return out

    def set_weights(self, weights: Sequence[np.ndarray]) -> None:
        i = 0
        for l in self._weighted_layers():
            n = len(l.weight_shapes())
            l.set_weights(weights[i:i + n])
            i += n
        if i != len(weights):
            raise ValueError(f"set_weights: {len(weights)} arrays given, {i} consumed")

    def count_params(self) -> int:
        return sum(l.count_params() for l in self._weighted_layers())

    # -- serialisation (stage wire format, reference src/dispatcher.py:49 / src/node.py:31)
    def get_config(self) -> dict:
        input_layers = set(self._input_layers)
        layer_cfgs = []
        inbound: Dict[str, List[str]] = {}
        for layer, ins in self.iter_nodes():
            inbound[layer.name] = ins if ins is not None else []
        for l in self.layers:
            if l in input_layers:
                shape = l.output.shape if l._inbound_nodes else None
                # the input tensor of a sub-model is the output of the cut layer: serialise as InputLayer
                t = self.inputs[self._input_layers.index(l)]
                layer_cfgs.append({"name": l.name, "class_name": "InputLayer",
                                   "config": {"name": l.name, "batch_input_shape": list(t.shape),
                                              "dtype": "float32"},
                                   "inbound_nodes": []})
            else:
                layer_cfgs.append({"name": l.name, "class_name": l.class_name, "config": l.get_config(),
                                   "inbound_nodes": [[[n, 0, 0, {}] for n in inbound[l.name]]]})
        return {"name": self.name, "layers": layer_cfgs,
                "input_layers": [[l.name, 0, 0] for l in self._input_layers],
                "output_layers": [[l.name, 0, 0] for l in self._output_layers]}

    def to_json(self) -> str:
        return json.dumps({"class_name": "Model", "config": self.get_config(),
                           "backend": "defer_b200", "keras_version": "defer_b200-ir-1"})

    def summary_lines(self) -> List[str]:
        lines = []
        for layer, ins in self.iter_nodes():
            lines.append(f"{layer.name:28s} {layer.class_name:24s} <- {ins}")
        return lines

    # -- execution: the product path is the CUDA engine (never the oracle)
    def predict(self, x, dtype: str = "float32", device: Union[int, str] = 0):
        """Run the whole model as ONE stage on a GPU through the C-ABI (reference
        ``test/local_infer.py:21``).  Raises if the CUDA library / a GPU is missing."""
        from .node import StageRunner  # local import: keeps IR importable without CUDA
        runner = getattr(self, "_runner", None)
        key = (dtype, str(device), int(np.asarray(x).shape[0]))
        if runner is None or getattr(self, "_runner_key", None) != key:
            if runner is not None:
                runner.close()
            runner = StageRunner.from_model(self, device=device, dtype=dtype, max_batch=key[2])
            self._runner, self._runner_key = runner, key
        return runner.predict(np.asarray(x, dtype=np.float32))


def model_from_json(text: Union[str, bytes]) -> Model:
    """Rebuild a functional model from ``Model.to_json()`` (reference ``src/node.py:31``)."""
    if isinstance(text, (bytes, bytearray)):
        text = bytes(text).decode()
    doc = json.loads(text)
    cfg = doc["config"]
    tensors: Dict[str, SymbolicTensor] = {}
    pending = list(cfg["layers"])
    # layers are stored depth-sorted; resolve by dependency to be order-agnostic
    progress = True
    while pending and progress:
        progress = False
        rest = []
        for lc in pending:
            cls = LAYER_CLASSES[lc["class_name"]]
            c = dict(lc["config"])
            if cls is InputLayer:
                layer = InputLayer(tuple(c["batch_input_shape"]), name=c["name"])
                tensors[layer.name] = layer.output
                progress = True
                continue
            ins = [e[0] for e in lc["inbound_nodes"][0]]
            if not all(n in tensors for n in ins):
                rest.append(lc)
                continue
            c.pop("data_format", None)
            c.pop("dtype", None)
            layer = cls(**c)
            args = [tensors[n] for n in ins]
            tensors[layer.name] = layer(args if len(args) > 1 else args[0])
            progress = True
        pending = rest
    if pending:
        raise ValueError(f"model_from_json: unresolved layers {[l['name'] for l in pending]}")
    inputs = [tensors[e[0]] for e in cfg["input_layers"]]
    outputs = [tensors[e[0]] for e in cfg["output_layers"]]
    return Model(inputs if len(inputs) > 1 else inputs[0], outputs if len(outputs) > 1 else outputs[0],
                 name=cfg.get("name"))
