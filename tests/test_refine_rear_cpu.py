"""The generator's rear as one forward + input-gradient program (engine.build_rear_grad_program: residual blocks,
up-sampling tail, head — what the refinement loop back-propagates through, evaluation/refinement.py:137-167) checked
on the CPU: interpreted in float64 by tests/spec_interp.py against float64 autograd through the oracle composition,
its support predicate, and its buffer liveness / storage."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs
from oracle import ffc_torch_cpu as otc
from spec_interp import SpecInterpreter, check_liveness


def rear_oracle_grads(gen, z1, z2, g0, kw):
    """(pred, dL/dz1, dL/dz2) in float64 autograd with L = sum(pred * g0)."""
    sd = {k: v.detach().double().cpu() for k, v in gen.state_dict().items()}
    a, b = z1.double().cpu().requires_grad_(True), z2.double().cpu().requires_grad_(True)
    y = otc.generator_rear(a, b, sd, kw)
    (y * g0.double().cpu()).sum().backward()
    return y.detach(), a.grad, b.grad


def _close(got, ref, rel=1e-6):
    scale = float(ref.abs().max()) or 1.0
    err = float((got.double() - ref.double()).abs().max())
    assert err <= rel * scale, f"{err:.3e} > {rel:g}*{scale:.3e}"


def _gen(act="sigmoid", **kw):
    kw = dict(small_lama_kwargs(**kw), add_out_act=act)
    return seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 5, gain=1.0), kw


@pytest.mark.parametrize("math", [L.MATH_FP32, L.MATH_BF16X3])
@pytest.mark.parametrize("b,h,w,act", [(2, 6, 10, "sigmoid"), (1, 5, 7, "sigmoid"), (1, 6, 10, "tanh"),
                                       (1, 5, 7, False)])
def test_rear_program_matches_autograd(b, h, w, act, math):
    """y0, dx0, dx1 of the interpreted program vs float64 autograd through the oracle to 1e-6 of their range: the ConvT
    adjoint as a stride-2 zero-border contraction with the BN scale on its input axis, the head adjoint with its
    reflect fold, the ReLU masks of every up stage, the Y2-before-the-add masks of the blocks.  The split-bf16 arm's
    program differs in its head (row contraction + gather) and rings, not in its arithmetic here."""
    gen, kw = _gen(act, ngf=8, n_blocks=2)
    cl, cg = 16, 48
    assert E.rear_grad_supported(gen, (b, cl, h, w), (b, cg, h, w))
    g = torch.Generator().manual_seed(3)
    z1, z2 = torch.randn(b, cl, h, w, generator=g), torch.randn(b, cg, h, w, generator=g)
    g0 = torch.randn(b, 3, 8 * h, 8 * w, generator=g)
    with torch.no_grad():
        prog = E.build_module_program(gen, "generator_rear_grad", ((b, cl, h, w), (b, cg, h, w)), math)
    assert prog.math == math
    assert any(isinstance(op, E.HeadBwdOp) for op in prog.ops) and sum(isinstance(op, E.AddOp) for op in prog.ops) == 2
    out = SpecInterpreter(prog).run(dict(x0=z1, x1=z2, g0=g0))
    y, d1, d2 = rear_oracle_grads(gen, z1, z2, g0, kw)
    _close(out["y0"], y)
    _close(out["dx0"], d1)
    _close(out["dx1"], d2)


def test_rear_grad_supported():
    big = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    assert E.rear_grad_supported(big, (1, 128, 64, 64), (1, 384, 64, 64))
    assert E.rear_grad_supported(big, (1, 128, 168, 168), (1, 384, 168, 168))
    n = E.BLOCK_GRAD_MAX_PLANE + 8
    assert not E.rear_grad_supported(big, (1, 128, n, 64), (1, 384, n, 64))
    assert not E.rear_grad_supported(big, (1, 128, 64, 64), (1, 256, 64, 64))          # channel split mismatch
    kw = small_lama_kwargs(ngf=16, n_blocks=1, n_downsampling=2)
    kw.update(out_ffc=True, out_ffc_kwargs=dict(ratio_gin=0.5, ratio_gout=0.5, enable_lfu=False))
    assert not E.rear_grad_supported(M.FFCResNetGenerator(**kw).eval(), (1, 16, 8, 8), (1, 48, 8, 8))
    for opt in (dict(enable_lfu=True), dict(gated=True)):
        kw = small_lama_kwargs(ngf=8, n_blocks=1)
        kw["resnet_conv_kwargs"] = dict(kw["resnet_conv_kwargs"], **opt)
        assert not E.rear_grad_supported(M.FFCResNetGenerator(**kw).eval(), (1, 16, 8, 8), (1, 48, 8, 8)), opt
    g = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval()
    assert E.rear_grad_supported(g, (1, 16, 8, 8), (1, 48, 8, 8))
    g.model[-1] = torch.nn.ReLU()                                                       # a head activation without adjoint
    assert not E.rear_grad_supported(g, (1, 16, 8, 8), (1, 48, 8, 8))


def test_rear_program_storage_is_live_and_smaller_than_per_block_programs():
    """Liveness of the pooled storage on the rear program (every Y1 / Y2 / t / z of the forward stays allocated until
    its backward read), and big-lama at the last refinement scale (168x168 bottleneck, 1344x1344 image): one rear
    program holds less than the 18 per-block forward+backward programs of the module path (DESIGN.md section 5)."""
    gen, _ = _gen("sigmoid", ngf=8, n_blocks=2)
    with torch.no_grad():
        small = E.build_module_program(gen, "generator_rear_grad", ((2, 16, 6, 10), (2, 48, 6, 10)), L.MATH_BF16X3)
    check_liveness(small)
    big = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    sl, sg = (1, 128, 168, 168), (1, 384, 168, 168)
    with torch.no_grad():
        rear = E.build_module_program(big, "generator_rear_grad", (sl, sg), L.MATH_BF16X3)
        blk = E.build_module_program(big.model[5], "resnet_block_grad", (sl, sg), L.MATH_BF16X3)
    rear_bytes = check_liveness(rear)
    blk_bytes = check_liveness(blk)
    print(f"rear program {rear_bytes / 1e9:.2f} GB, 18 block programs {18 * blk_bytes / 1e9:.2f} GB")
    assert rear_bytes < 18 * blk_bytes
