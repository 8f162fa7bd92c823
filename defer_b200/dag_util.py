"""Graph partitioner with the reference's signatures (``src/dag_util.py:3-31``).

``construct_model(model, start, end, part_name)`` returns the sub-model that computes every layer
strictly after ``start`` through ``end``; its input *is* ``start``'s output tensor.  The walk is the
reference's backward recursion from ``end`` to ``start`` re-applying each (shared) layer on the new
input, with two deliberate differences (SURVEY.md 3.1):

* memoised - the reference re-instantiates the earliest residual block 2^(m-1) times for a stage
  with m blocks (both ``Add`` inputs recurse to the same predecessor, ``src/dag_util.py:16-17``);
* iterative - ResNet152 stages exceed Python's recursion limit.

Numerically the result is identical: the same layer objects (same weights) applied to the same
tensors once.
"""
from __future__ import annotations

from typing import Dict, List, Optional

from . import keras_like as K


def get_previous(model, name: str) -> List[str]:
    """Names of the layers feeding ``name`` (reference ``src/dag_util.py:3-7``)."""
    inbound = model.get_layer(name).inbound_nodes[0].inbound_layers
    if type(inbound) != list:  # noqa: E721 - same check as the reference
        inbound = [inbound]
    return [layer.name for layer in inbound]


def traverse(model, name: str, start: str, part_name: str, inpt, _memo: Optional[Dict[str, object]] = None):
    """Output tensor of layer ``name`` recomputed from ``inpt`` standing for ``start``'s output
    (reference ``src/dag_util.py:9-25``)."""
    memo: Dict[str, object] = _memo if _memo is not None else {}
    stack = [(name, False)]
    while stack:
        cur, expanded = stack.pop()
        if cur in memo:
            continue
        # base case: reached the cut layer (or the freshly defined input layer)
        if cur == start or cur == part_name:
            memo[cur] = inpt
            continue
        prev = get_previous(model, cur)
        if not expanded:
            if not prev:
                raise ValueError(
                    f"traverse reached source layer {cur!r} without meeting start={start!r}: "
                    "the cut is not an articulation point of the graph")
            stack.append((cur, True))
            for n in reversed(prev):
                if n not in memo:
                    stack.append((n, False))
            continue
        output = [memo[n] for n in prev]
        if len(output) == 1:  # DAG node with one previous connection (src/dag_util.py:20-21)
            output = output[0]
        layer = model.get_layer(cur)
        memo[cur] = layer(output)
    return memo[name]


def construct_model(model, start: str, end: str, part_name: str = "part_begin"):
    """Sub-model ``(start, end]`` (reference ``src/dag_util.py:27-31``)."""
    inpt = K.Input(tensor=model.get_layer(start).output, name=part_name)
    output = traverse(model, end, start, part_name, inpt)
    part = K.Model(inputs=model.get_layer(start).output, outputs=output)
    return part
