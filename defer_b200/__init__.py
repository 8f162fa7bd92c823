"""defer_b200 - Hopper-native (H100) pipeline-partitioned inference with the DEFER API.

Public surface mirrors the reference (``src``): ``DEFER`` (dispatcher), ``Node``,
``NodeState``, ``dag_util.construct_model``; model builders stand in for ``keras.applications``.
"""
from . import keras_like, applications, dag_util  # noqa: F401
from .node_state import NodeState  # noqa: F401

__all__ = ["keras_like", "applications", "dag_util", "NodeState", "DEFER", "Node"]


def __getattr__(name):
    # DEFER / Node pull in ctypes + the CUDA library lazily so the IR stays importable anywhere
    if name == "DEFER":
        from .dispatcher import DEFER
        return DEFER
    if name == "Node":
        from .node import Node
        return Node
    raise AttributeError(name)
