"""The generator's rear as one forward + input-gradient program (engine.build_rear_grad_program: residual blocks,
up-sampling tail, head — what the refinement loop back-propagates through, evaluation/refinement.py:137-167) checked
on the CPU: interpreted in float64 by tests/spec_interp.py (with the two rear-only ops restated below) against float64 autograd through the oracle composition,
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
from spec_interp import SpecInterpreter


class RearSpecInterpreter(SpecInterpreter):
    """SpecInterpreter plus float64 restatements of the two ops only the rear program has: ffcb_add and ffcb_head_bwd7
    (include/ffc_b200.h); every other op goes to the base interpreter."""

    def step(self, op, inputs, out):
        if isinstance(op, E.AddOp):
            self.write(op.out, self.read(op.a) + self.read(op.b))
        elif isinstance(op, E.HeadBwdOp):
            y, dy = out[op.y].double(), inputs[op.dy].double().to(out[op.y].device)
            d = {L.ACT_NONE: dy, L.ACT_SIGMOID: dy * y * (1 - y), L.ACT_TANH: dy * (1 - y * y)}[op.act]
            w = op.w.double().to(d.device).reshape(op.n_out, 7, 7, -1).permute(0, 3, 1, 2)      # [N, C, 7, 7]
            gp = F.conv_transpose2d(d, w)                                                     # [B, C, H+6, W+6]
            h, wd = gp.shape[2] - 6, gp.shape[3] - 6
            # Fold3: padded row / column p came from interior reflect(p - 3)
            ry = (torch.arange(h + 6, device=gp.device) - 3).abs(); ry = torch.where(ry >= h, 2 * h - 2 - ry, ry)
            rx = (torch.arange(wd + 6, device=gp.device) - 3).abs(); rx = torch.where(rx >= wd, 2 * wd - 2 - rx, rx)
            g = torch.zeros(gp.shape[0], gp.shape[1], h, wd + 6, dtype=gp.dtype, device=gp.device).index_add_(2, ry, gp)
            g = torch.zeros(gp.shape[0], gp.shape[1], h, wd, dtype=gp.dtype, device=gp.device).index_add_(3, rx, g)
            m = self.read(op.mask)
            self.write(op.out, g.permute(0, 2, 3, 1).to(m.device) * (m > 0))
        else:
            super().step(op, inputs, out)


def rear_oracle(z1, z2, sd, kw):
    """``generator.model[first_block:]`` composed from the oracle: ffc_resnet_block per block, then ConvTranspose2d +
    eval BN + ReLU per up stage, then reflect pad 3 + 7x7 conv + the head activation (ffc.py:345-363)."""
    nd, nb = kw["n_downsampling"], kw["n_blocks"]
    i = 2 + nd
    z_l, z_g = z1, z2
    for _ in range(nb):
        z_l, z_g = otc.ffc_resnet_block(z_l, z_g, sd, f"model.{i}.", ratio_gout=0.75); i += 1
    h = torch.cat((z_l, z_g), dim=1); i += 1
    for _ in range(nd):
        h = F.conv_transpose2d(h, sd[f"model.{i}.weight"], sd[f"model.{i}.bias"], stride=2, padding=1,
                               output_padding=1)
        h = torch.relu(otc._bn(h, sd, f"model.{i + 1}.")); i += 3
    h = F.conv2d(F.pad(h, (3, 3, 3, 3), mode="reflect"), sd[f"model.{i + 1}.weight"], sd[f"model.{i + 1}.bias"])
    act = kw.get("add_out_act", True)
    if act is True or act == "tanh":
        return torch.tanh(h)
    return torch.sigmoid(h) if act == "sigmoid" else h


def rear_oracle_grads(gen, z1, z2, g0, kw):
    """(pred, dL/dz1, dL/dz2) in float64 autograd with L = sum(pred * g0)."""
    sd = {k: v.detach().double().cpu() for k, v in gen.state_dict().items()}
    a, b = z1.double().cpu().requires_grad_(True), z2.double().cpu().requires_grad_(True)
    y = rear_oracle(a, b, sd, kw)
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
    out = RearSpecInterpreter(prog).run(dict(x0=z1, x1=z2, g0=g0))
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


def _nbytes(b):
    if b.tile:
        return -(-(b.B * b.H * b.W) // 128) * 128 * b.C * 4
    if b.cg:
        return b.B * b.H * b.W * b.C * 4
    return b.B * (b.H + 2 * b.pad) * (b.W + 2 * b.pad) * b.C * 4


def _check_liveness(prog):
    """No two buffers of one storage slot are live at once (a forward write must survive to its backward read); returns
    the pooled storage in bytes."""
    slots = E.assign_storage_slots(prog)
    first, last = {}, {}
    for i, op in enumerate(prog.ops):
        r, w = E.op_views(op)
        for tv in r + w:
            first.setdefault(tv.buf.name, i)
            last[tv.buf.name] = i
    by_slot = {}
    for b in prog.bufs:
        by_slot.setdefault(slots[b.name], []).append(b)
    for members in by_slot.values():
        assert len({E.storage_key(b) for b in members}) == 1
        members = sorted(members, key=lambda b: first.get(b.name, -1))
        for a, b in zip(members, members[1:]):
            assert last[a.name] < first[b.name], (a.name, b.name)
    return sum(_nbytes(m[0]) for m in by_slot.values())


def test_rear_program_storage_is_live_and_smaller_than_per_block_programs():
    """Liveness of the pooled storage on the rear program (every Y1 / Y2 / t / z of the forward stays allocated until
    its backward read), and big-lama at the last refinement scale (168x168 bottleneck, 1344x1344 image): one rear
    program holds less than the 18 per-block forward+backward programs of the module path (DESIGN.md section 5)."""
    gen, _ = _gen("sigmoid", ngf=8, n_blocks=2)
    with torch.no_grad():
        small = E.build_module_program(gen, "generator_rear_grad", ((2, 16, 6, 10), (2, 48, 6, 10)), L.MATH_BF16X3)
    _check_liveness(small)
    big = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    sl, sg = (1, 128, 168, 168), (1, 384, 168, 168)
    with torch.no_grad():
        rear = E.build_module_program(big, "generator_rear_grad", (sl, sg), L.MATH_BF16X3)
        blk = E.build_module_program(big.model[5], "resnet_block_grad", (sl, sg), L.MATH_BF16X3)
    rear_bytes = _check_liveness(rear)
    blk_bytes = _check_liveness(blk)
    print(f"rear program {rear_bytes / 1e9:.2f} GB, 18 block programs {18 * blk_bytes / 1e9:.2f} GB")
    assert rear_bytes < 18 * blk_bytes
