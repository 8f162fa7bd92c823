"""ORACLE - TEST / BASELINE INFRASTRUCTURE ONLY.  Second, independent CPU executor of the same wire
format built on ``torch.nn.functional`` (oneDNN/MKL, all host cores).

Used (a) to cross-check ``oracle/keras_ref.py`` and (b) as the *timed* CPU stand-in for the
reference's TensorFlow-CPU ``model.predict`` (``test/local_infer.py:16-23``,
``src/node.py:105-106``) in ``bench.py``'s ``cpu_baseline`` and ``--impl reference`` legs:
TensorFlow is not installable here, so the baseline is a port (``cpu_baseline.kind = "port"``).
PARITY UNPINNED - see ``oracle/keras_ref.py``.  Never imported by the product.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from .keras_ref import WireModel, same_pad


class TorchCpuModel:
    def __init__(self, json_text, weights: Sequence[np.ndarray], dtype=torch.float32):
        self.wm = WireModel(json_text, weights)
        self.dtype = dtype
        self.order = [n for n in self.wm.topo_order() if n != self.wm.input_name]
        self.params: Dict[str, List[torch.Tensor]] = {}
        for name in self.order:
            l = self.wm.by_name[name]
            w = [torch.from_numpy(np.ascontiguousarray(a)).to(dtype) for a in self.wm.weights[name]]
            if l["class_name"] == "Conv2D":
                w[0] = w[0].permute(3, 2, 0, 1).contiguous(memory_format=torch.channels_last)  # HWIO -> OIHW
            elif l["class_name"] == "Dense":
                w[0] = w[0].t().contiguous()
            self.params[name] = w

    @torch.no_grad()
    def predict(self, x: np.ndarray, final_activation: bool = True) -> np.ndarray:
        wm = self.wm
        t = torch.from_numpy(np.ascontiguousarray(x)).to(self.dtype)
        if t.dim() == 4:
            t = t.permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)  # NHWC data, NCHW view
        vals = {wm.input_name: t}
        for name in self.order:
            l = wm.by_name[name]
            cn, c = l["class_name"], l["config"]
            ins = [vals[p] for p in wm.inbound(name)]
            w = self.params[name]
            last = name == wm.output_name
            if cn == "Conv2D":
                xi = ins[0]
                kh, kw = c["kernel_size"]
                sh, sw = c["strides"]
                if c["padding"] == "same":
                    pt, pb = same_pad(xi.shape[2], kh, sh)
                    pl, pr = same_pad(xi.shape[3], kw, sw)
                    if pt == pb and pl == pr:
                        y = F.conv2d(xi, w[0], w[1] if len(w) > 1 else None, stride=(sh, sw), padding=(pt, pl))
                    else:
                        y = F.conv2d(F.pad(xi, (pl, pr, pt, pb)), w[0], w[1] if len(w) > 1 else None, stride=(sh, sw))
                else:
                    y = F.conv2d(xi, w[0], w[1] if len(w) > 1 else None, stride=(sh, sw))
                if c.get("activation") == "relu":
                    y = F.relu(y)
            elif cn == "Dense":
                y = F.linear(ins[0], w[0], w[1] if len(w) > 1 else None)
                act = c.get("activation")
                if act == "relu":
                    y = F.relu(y)
                elif act == "softmax" and (final_activation or not last):
                    y = F.softmax(y, dim=-1)
            elif cn == "BatchNormalization":
                y = F.batch_norm(ins[0], w[2], w[3], w[0], w[1], training=False, eps=c["epsilon"])
            elif cn == "Activation":
                a = c["activation"]
                if a == "relu":
                    y = F.relu(ins[0])
                elif a == "softmax" and (final_activation or not last):
                    y = F.softmax(ins[0], dim=-1)
                else:
                    y = ins[0]
            elif cn == "Add":
                y = ins[0]
                for o in ins[1:]:
                    y = y + o
            elif cn == "ZeroPadding2D":
                (pt, pb), (pl, pr) = c["padding"]
                y = F.pad(ins[0], (pl, pr, pt, pb))
            elif cn == "MaxPooling2D":
                y = F.max_pool2d(ins[0], tuple(c["pool_size"]), tuple(c["strides"]))
            elif cn == "GlobalAveragePooling2D":
                y = ins[0].mean(dim=(2, 3))
            elif cn == "Flatten":
                y = ins[0].permute(0, 2, 3, 1).reshape(ins[0].shape[0], -1)  # H,W,C order
            else:
                raise ValueError(cn)
            vals[name] = y
        out = vals[wm.output_name]
        if out.dim() == 4:
            out = out.permute(0, 2, 3, 1)
        return out.contiguous().to(torch.float32).numpy()
