"""The whole generator as one forward + input-gradient program (kind ``generator_grad``, lama_b200/generator_grad.py)
checked on the CPU: interpreted in float64 against float64 autograd through the oracle composition (FFC) and the
drop-in's torch composition (LaMa-Regular), the stem adjoint's restatement against autograd, the support gate, buffer
liveness and the program's storage."""
import pytest
import torch
import torch.nn.functional as F

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import generator_grad as GG
from lama_b200 import modules as M
from lama_b200 import pix2pixhd as PX
from lama_b200.testing import (BIG_LAMA_KWARGS, LAMA_REGULAR_KWARGS, seeded_parameters_, small_lama_kwargs,
                               small_regular_kwargs)
from oracle import ffc_torch_cpu as otc
from spec_interp import SpecInterpreter, check_liveness


def stem_adjoint_f64(g, w, cin):
    """ffcb_stem_bwd7 restated: g [B, N, H, W], w [N][49][Cin] -> Fold3(Conv7^T(g)) [B, Cin, H, W]."""
    wk = w.double().reshape(w.shape[0], 7, 7, cin).permute(0, 3, 1, 2)
    gp = F.conv_transpose2d(g.double(), wk)                                     # [B, Cin, H+6, W+6]
    h, wd = gp.shape[2] - 6, gp.shape[3] - 6
    ry = (torch.arange(h + 6) - 3).abs(); ry = torch.where(ry >= h, 2 * h - 2 - ry, ry)
    rx = (torch.arange(wd + 6) - 3).abs(); rx = torch.where(rx >= wd, 2 * wd - 2 - rx, rx)
    t = torch.zeros(gp.shape[0], cin, h, wd + 6, dtype=gp.dtype).index_add_(2, ry, gp)
    return torch.zeros(gp.shape[0], cin, h, wd, dtype=gp.dtype).index_add_(3, rx, t)


class Interp(SpecInterpreter):
    """The interpreter with the op type of the generator-gradient program."""

    def StemBwdOp(self, op, ext):
        ext[op.dst] = stem_adjoint_f64(self.read(op.g).permute(0, 3, 1, 2), op.w, op.cin)


def ffc_generator_f64(gen, kw, x):
    """FFCResNetGenerator composed from the oracle in float64 (differentiable): stem, downs, ``generator_rear``."""
    sd = {k: v.detach().to(x.device, torch.float64) for k, v in gen.state_dict().items()}
    nd = kw["n_downsampling"]
    l, g = otc.ffc_bn_act(F.pad(x, (3, 3, 3, 3), mode="reflect"), 0, sd, "model.1.", ratio_gout=0)
    for d in range(nd):
        rg = kw["resnet_conv_kwargs"]["ratio_gin"] if d == nd - 1 else 0
        l, g = otc.ffc_bn_act(l, g, sd, f"model.{2 + d}.", ratio_gout=rg, stride=2, padding=1)
    return otc.generator_rear(l, g, sd, kw)


def regular_generator_f64(gen, x):
    """GlobalGenerator in float64 with each ReLU an oracle site (``otc.relu``: pinnable), named by the state-dict
    prefix of the BN before it; otherwise the drop-in's own torch composition."""
    mods = list(gen.model)
    h = x
    for i, m in enumerate(mods):
        if isinstance(m, torch.nn.ReLU):
            h = otc.relu(h, f"model.{i - 1}.")
        elif isinstance(m, PX.ResnetBlock):
            cb = list(m.conv_block)
            t = h
            for j, c in enumerate(cb):
                t = otc.relu(t, f"model.{i}.conv_block.{j - 1}.") if isinstance(c, torch.nn.ReLU) else c(t)
            h = h + t
        else:
            h = m(h)
    return h


def oracle_grads(gen, kw, x, g0):
    """(y, dL/dx) in float64 autograd with L = sum(y * g0)."""
    gd = gen.double() if kw is None else gen
    a = x.detach().double().requires_grad_(True)
    y = regular_generator_f64(gd, a) if kw is None else ffc_generator_f64(gen, kw, a)
    (y * g0.double()).sum().backward()
    return y.detach(), a.grad


def _close(got, ref, rel=1e-6):
    scale = float(ref.abs().max()) or 1.0
    err = float((got.double() - ref.double()).abs().max())
    assert err <= rel * scale, f"{err:.3e} > {rel:g}*{scale:.3e}"


def _ffc(n_down, act, ngf=8, n_blocks=2):
    kw = dict(small_lama_kwargs(ngf=ngf, n_blocks=n_blocks, n_downsampling=n_down), add_out_act=act)
    return seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 5, gain=1.0).requires_grad_(False), kw


def _regular(n_down, act, ngf=8, n_blocks=2):
    kw = dict(small_regular_kwargs(ngf=ngf, n_blocks=n_blocks, n_downsampling=n_down), add_out_act=act)
    return seeded_parameters_(PX.GlobalGenerator(**kw).eval(), 5, gain=1.0).requires_grad_(False)


CASES = [(1, (24, 32), "sigmoid"), (2, (40, 72), "tanh"), (3, (24, 32), False), (3, (40, 72), "sigmoid")]


@pytest.mark.parametrize("math", [L.MATH_FP32, L.MATH_BF16X3])
@pytest.mark.parametrize("kind", ["ffc", "regular"])
@pytest.mark.parametrize("n_down,hw,act", CASES)
def test_generator_grad_program_matches_autograd(kind, n_down, hw, act, math):
    """y0 and dx0 of the interpreted program vs float64 autograd to 1e-6 of their range: the stem adjoint's reflect
    fold, the stride-2 adjoints as phase contractions (reflect: onto the padded plane, then the fold; zero: the
    interior), the ReLU masks of the stem, every down and every block, and the rear's backward."""
    # one down at ngf 8 leaves 16 bottleneck channels, a FourierUnit too narrow for the native blocks: ngf 16 there
    gen, kw = _ffc(n_down, act, ngf=8 if n_down > 1 else 16) if kind == "ffc" else (_regular(n_down, act), None)
    b, (h, w) = 2, hw
    shape = (b, 4, h, w)
    assert GG.generator_grad_supported(gen, shape)
    g = torch.Generator().manual_seed(h + n_down)
    x, g0 = torch.randn(shape, generator=g), torch.randn(b, 3, h, w, generator=g)
    with torch.no_grad():
        prog = E.build_module_program(gen, "generator_grad", (shape,), math)
    assert sum(isinstance(op, GG.StemBwdOp) for op in prog.ops) == 1
    out = Interp(prog).run(dict(x0=x, g0=g0))
    y, dx = oracle_grads(gen, kw, x, g0)
    _close(out["y0"], y)
    _close(out["dx0"], dx)
    check_liveness(prog)


@pytest.mark.parametrize("cin", [1, 4, 8])
def test_stem_adjoint_restatement_is_autograd(cin):
    """The restatement of ffcb_stem_bwd7 equals autograd of ReflectionPad2d(3) + conv7 exactly (integer operands) for
    every plane of 4..9 rows and columns: every combination of the top / bottom / left / right folds."""
    g = torch.Generator().manual_seed(cin)
    n = 8
    w = torch.randint(-4, 5, (n, cin, 7, 7), generator=g).double()
    wk = w.permute(0, 2, 3, 1).reshape(n, 49, cin)
    for h in range(4, 10):
        for wd in range(4, 10):
            x = torch.zeros(2, cin, h, wd, dtype=torch.float64, requires_grad=True)
            gy = torch.randint(-3, 4, (2, n, h, wd), generator=g).double()
            (F.conv2d(F.pad(x, (3, 3, 3, 3), mode="reflect"), w) * gy).sum().backward()
            assert torch.equal(stem_adjoint_f64(gy, wk, cin), x.grad), (h, wd)


def test_generator_grad_gate():
    """Refused: LFU, gated and out_ffc generators, trainable weights, training mode, planes the no-grad program
    rejects, a head activation without adjoint; accepted: frozen big-lama and lama-regular in eval mode."""
    big = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval().requires_grad_(False)
    assert GG.generator_grad_supported(big, (1, 4, 512, 512))
    assert E.generator_grad_supported(big, (2, 4, 1080, 1920))
    assert not GG.generator_grad_supported(big, (1, 4, 516, 512))             # not a multiple of 8
    big.model[2].ffc.convl2l.weight.requires_grad_(True)
    assert not GG.generator_grad_supported(big, (1, 4, 512, 512))             # one trainable weight
    big.requires_grad_(False).train()
    assert not GG.generator_grad_supported(big, (1, 4, 512, 512))             # training mode
    for opt in (dict(enable_lfu=True), dict(gated=True)):
        kw = small_lama_kwargs(ngf=8, n_blocks=1)
        kw["resnet_conv_kwargs"] = dict(kw["resnet_conv_kwargs"], **opt)
        gen = M.FFCResNetGenerator(**kw).eval().requires_grad_(False)
        assert not GG.generator_grad_supported(gen, (1, 4, 64, 64)), opt
    kw = small_lama_kwargs(ngf=16, n_blocks=1, n_downsampling=2)
    kw.update(out_ffc=True, out_ffc_kwargs=dict(ratio_gin=0.5, ratio_gout=0.5, enable_lfu=False))
    assert not GG.generator_grad_supported(M.FFCResNetGenerator(**kw).eval().requires_grad_(False), (1, 4, 32, 32))
    gen = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval().requires_grad_(False)
    assert GG.generator_grad_supported(gen, (1, 4, 64, 64))
    gen.model[-1] = torch.nn.ReLU()
    assert not GG.generator_grad_supported(gen, (1, 4, 64, 64))
    reg = PX.GlobalGenerator(**LAMA_REGULAR_KWARGS).eval().requires_grad_(False)
    assert GG.generator_grad_supported(reg, (1, 4, 512, 512))
    assert not GG.generator_grad_supported(reg, (1, 4, 512, 508))
    reg.train()
    assert not GG.generator_grad_supported(reg, (1, 4, 512, 512))
    reg.eval().model[2].weight.requires_grad_(True)
    assert not GG.generator_grad_supported(reg, (1, 4, 512, 512))


# program_storage_bytes (computed from the buffer shapes and storage slots, not measured) of the split-bf16 programs
STORAGE = {
    ("big-lama", 512, 512): 1330010624,
    ("big-lama", 2160, 3840): 41278461440,
    ("lama-regular", 512, 512): 714432016,
    ("lama-regular", 2160, 3840): 22325022224,
}


@pytest.mark.parametrize("model,h,w", list(STORAGE))
def test_generator_grad_storage(model, h, w):
    """The pooled storage of the batch-1 program, pinned; printed next to the no-grad program's."""
    if model == "big-lama":
        gen = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval().requires_grad_(False)
    else:
        gen = PX.GlobalGenerator(**LAMA_REGULAR_KWARGS).eval().requires_grad_(False)
    shape = (1, 4, h, w)
    with torch.no_grad():
        prog = E.build_module_program(gen, "generator_grad", (shape,), L.MATH_BF16X3)
        fwd = E.build_module_program(gen, "generator", (shape,), L.MATH_BF16X3)
    assert prog.math == L.MATH_BF16X3
    got, fwd_bytes = E.program_storage_bytes(prog), E.program_storage_bytes(fwd)
    print(f"{model} {h}x{w}: generator_grad {got} B ({got / 1e9:.2f} GB), generator {fwd_bytes / 1e9:.2f} GB")
    assert got == STORAGE[(model, h, w)]
