"""Run one coalesced microbatch of a model through a single stage twice; the second pass sits between
cudaProfilerStart/Stop, so a profiler that honours that capture range records exactly one launch of every kernel of the
step.
usage: run_stage_once.py [model] [dtype] [batch] [cuts,comma,separated]   (cuts -> a pipeline on one GPU, exercising the
standalone element-wise kernels and the hop)"""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from defer_b200 import _cabi  # noqa: E402

_cabi.load()
import numpy as np  # noqa: E402
import torch  # noqa: E402
from defer_b200 import applications, dag_util  # noqa: E402
from defer_b200.node import StageRunner  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "resnet50"
dtype = sys.argv[2] if len(sys.argv) > 2 else "float32"
batch = int(sys.argv[3]) if len(sys.argv) > 3 else 32
cuts = [c for c in (sys.argv[4].split(",") if len(sys.argv) > 4 else []) if c]
model = {"resnet50": applications.ResNet50, "resnet152": applications.ResNet152, "vgg16": applications.VGG16}[name]()
x = applications.synthetic_input(batch)
names = [model.input._keras_history[0].name] + cuts + [model.output._keras_history[0].name]
parts = [dag_util.construct_model(model, names[i], names[i + 1], part_name=f"part{i+1}") for i in range(len(names) - 1)]
n = len(parts)
runners = [StageRunner.from_wire(p.to_json(), p.get_weights(), device=0, dtype=dtype, max_batch=batch, depth=1,
                                 is_first=(i == 0), is_last=(i == n - 1), finalize=False) for i, p in enumerate(parts)]
for i in range(n - 1):
    runners[i].link_to(runners[i + 1])
for r in runners:
    r.finalize()


def once(seq):
    runners[0].submit(seq, x)
    for r in runners:
        r.step(seq)
    return runners[-1].result(seq)


once(0)
torch.cuda.synchronize()
torch.cuda.profiler.start()
y = once(1)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("probs sum", float(np.asarray(y).sum()), "kernels/step", sum(r.num_kernels() for r in runners))
for r in runners:
    r.sync()
for r in runners:
    r.unlink()
for r in runners:
    r.close()
