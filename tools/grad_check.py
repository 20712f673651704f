#!/usr/bin/env python
"""dL/dx of one FFCResnetBlock: the native forward+backward program vs float64 autograd through the torch-CPU oracle
(oracle/ffc_torch_cpu.py).  Prints relative 2-norm errors per shape.

For comparison it also prints the torch composition of the same module on the same GPU (fp32, TF32 off, cuFFT) against
that oracle ("torch_gpu_*").  Its FourierUnit inverse transforms a spectrum that is not Hermitian (the spectral ReLU
breaks the symmetry); cuFFT's C2R gives such input a meaning of its own on some shapes, e.g. 128-wide planes with 64 or
more planes per call, so that arm is no yardstick there."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from lama_b200 import modules as M  # noqa: E402
from lama_b200.testing import seeded_parameters_  # noqa: E402
from oracle import ffc_torch_cpu as otc  # noqa: E402

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda:0")
rel = lambda x, y: float((x.double() - y).norm() / y.norm())  # noqa: E731
out = {}
for (b, h, w) in ((1, 64, 64), (1, 128, 128), (1, 17, 25), (1, 96, 128), (1, 256, 256)):
    blk = seeded_parameters_(M.FFCResnetBlock(512, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                              activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                              enable_lfu=False).eval(), 4, gain=1.0)
    sd = {k: v.double() for k, v in blk.state_dict().items()}
    blk = blk.to(dev)
    for p in blk.parameters():
        p.requires_grad_(False)
    g = torch.Generator().manual_seed(h)
    xl, xg = torch.randn(b, 128, h, w, generator=g), torch.randn(b, 384, h, w, generator=g)
    gl, gg = torch.randn(b, 128, h, w, generator=g), torch.randn(b, 384, h, w, generator=g)
    a, c = xl.double().requires_grad_(True), xg.double().requires_grad_(True)
    o_l, o_g = otc.ffc_resnet_block(a, c, sd, "", ratio_gout=0.75)
    ((o_l * gl.double()).sum() + (o_g * gg.double()).sum()).backward()
    want = (o_l.detach(), o_g.detach(), a.grad, c.grad)
    row = {}
    for mode, tag in (("1", ""), ("0", "torch_gpu_")):
        os.environ["LAMA_B200_NATIVE_GRAD"] = mode
        os.environ["LAMA_B200_STRICT"] = "0"
        a, c = xl.to(dev).requires_grad_(True), xg.to(dev).requires_grad_(True)
        o_l, o_g = blk((a, c))
        ((o_l * gl.to(dev)).sum() + (o_g * gg.to(dev)).sum()).backward()
        got = (o_l.detach(), o_g.detach(), a.grad, c.grad)
        for k, x, y in zip(("fwd_l", "fwd_g", "dx_l", "dx_g"), got, want):
            row[tag + k] = rel(x.cpu(), y)
    out[f"{h}x{w}"] = row
print(json.dumps(out))
