#!/usr/bin/env python
"""One eager (non-graph) generator step between cudaProfilerStart/Stop, for a profiler that honours them, e.g.
   ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file X python tools/profile_step.py
The program's launch order (one ffcb call name per line) goes to stderr.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

math = sys.argv[1] if len(sys.argv) > 1 else "bf16x3"
batch = int(sys.argv[2]) if len(sys.argv) > 2 else 32
os.environ["LAMA_B200_MATH"] = math
os.environ["LAMA_B200_STRICT"] = "1"
from lama_b200 import _lib as L, engine as E, modules as M  # noqa: E402
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask, generator_input  # noqa: E402

dev = torch.device("cuda:0")
gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to(dev)
img, mask = synthetic_image_mask(batch, 512, 0)
x = generator_input(img, mask).to(dev)
ex = E.get_executor(gen, "generator", (x,), math={"fp32": L.MATH_FP32, "bf16x3": L.MATH_BF16X3}[math])
for _ in range(2):
    ex.run({"x0": x})
torch.cuda.synchronize()
for name, _f, _a in ex.calls:
    sys.stderr.write(name + "\n")
torch.cuda.profiler.start()
ex.run({"x0": x})
torch.cuda.synchronize()
torch.cuda.profiler.stop()
