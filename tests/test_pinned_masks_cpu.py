"""Pinned ReLU masks on the CPU: the float64 oracle with the masks of another run (``otc.pinned_relu_masks``), and the
ReLU outputs the block-gradient and rear programs keep, named by the oracle's sites (``device_state.MaskCapture``).

A gradient program is linear once its ReLU masks are fixed.  Run with the masks a device run read, the oracle differs
from that run by arithmetic round-off alone, so tests/test_gpu_pinned_grads.py can hold every element to the op-level
tolerance.  These tests show, without a GPU, that the hook changes nothing but the masks, that every kept output maps
onto exactly one oracle site, and that masks captured from an interpreted run reproduce that run's input gradients."""
import pytest
import torch

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs
from oracle import ffc_torch_cpu as otc
from device_state import MaskCapture, covers, mask_view, relu_sites
from spec_interp import SpecInterpreter


def _block(dim, seed=4):
    return seeded_parameters_(M.FFCResnetBlock(dim, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                               activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                               enable_lfu=False).eval(), seed, gain=1.0)


def _gen(kw, act="sigmoid", seed=5):
    kw = dict(kw, add_out_act=act)
    return seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), seed, gain=1.0), kw


def _randn(*shape, g):
    return torch.randn(*shape, generator=g, dtype=torch.float64)


def block_oracle(blk, xl, xg, gl, gg):
    """(y_l, y_g, dx_l, dx_g) of FFCResnetBlock in float64 autograd with L = sum(out * g): y = conv2(conv1(x)) without
    the identity (what the block-gradient program writes as y0 / y1), dx with it."""
    sd = {k: v.detach().to(xl.device, torch.float64) for k, v in blk.state_dict().items()}
    a, b = xl.detach().double().requires_grad_(True), xg.detach().double().requires_grad_(True)
    kw = dict(ratio_gout=0.75, padding=1)
    y1 = otc.ffc_bn_act(a, b, sd, "conv1.", **kw)
    y_l, y_g = otc.ffc_bn_act(*y1, sd, "conv2.", **kw)
    (((a + y_l) * gl.double()).sum() + ((b + y_g) * gg.double()).sum()).backward()
    return y_l.detach(), y_g.detach(), a.grad, b.grad


def rear_oracle(gen, kw, z1, z2, g0):
    """(pred, dz1, dz2) of the generator's rear in float64 autograd with L = sum(pred * g0)."""
    sd = {k: v.detach().to(z1.device, torch.float64) for k, v in gen.state_dict().items()}
    a, b = z1.detach().double().requires_grad_(True), z2.detach().double().requires_grad_(True)
    y = otc.generator_rear(a, b, sd, kw)
    (y * g0.double()).sum().backward()
    return y.detach(), a.grad, b.grad


def _own_masks(fn):
    """Run ``fn`` unhooked and return its result and the mask (output > 0) of every ReLU site it passed."""
    with otc.recorded_relu_masks() as masks:
        out = fn()
    return out, masks


def _equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def test_pinned_with_its_own_masks_is_bit_identical_to_autograd():
    """Block and rear: the oracle hooked with the masks of its own float64 forward reproduces unhooked autograd bit for
    bit (forward and input gradients), and serves every site it passed."""
    g = torch.Generator().manual_seed(1)
    blk = _block(128)
    xl, xg, gl, gg = _randn(2, 32, 9, 13, g=g), _randn(2, 96, 9, 13, g=g), _randn(2, 32, 9, 13, g=g), \
        _randn(2, 96, 9, 13, g=g)
    want, masks = _own_masks(lambda: block_oracle(blk, xl, xg, gl, gg))
    assert len(masks) == 8          # per FFC_BN_ACT: bn_l, bn_g, st.conv1's BN, fu.bn
    with otc.pinned_relu_masks(masks) as served:
        got = block_oracle(blk, xl, xg, gl, gg)
    assert served == set(masks)
    assert _equal(got, want)

    gen, kw = _gen(small_lama_kwargs(ngf=8, n_blocks=2))
    z1, z2, g0 = _randn(1, 16, 5, 7, g=g), _randn(1, 48, 5, 7, g=g), _randn(1, 3, 40, 56, g=g)
    want, masks = _own_masks(lambda: rear_oracle(gen, kw, z1, z2, g0))
    assert len(masks) == 2 * 8 + 3
    with otc.pinned_relu_masks(masks) as served:
        got = rear_oracle(gen, kw, z1, z2, g0)
    assert served == set(masks)
    assert _equal(got, want)


def test_pinned_masks_are_used_and_required():
    """The hook really replaces the masks (all-ones masks make the block linear in x), and a missing site or a mask of
    the wrong shape raises."""
    g = torch.Generator().manual_seed(2)
    blk = _block(128)
    xl, xg, gl, gg = _randn(1, 32, 6, 10, g=g), _randn(1, 96, 6, 10, g=g), _randn(1, 32, 6, 10, g=g), \
        _randn(1, 96, 6, 10, g=g)
    prog = E.build_module_program(blk, "resnet_block_grad", ((1, 32, 6, 10), (1, 96, 6, 10)), L.MATH_FP32)
    ones = {s: torch.ones(v.batch, v.channels, *v.hw, dtype=torch.bool) for s, v in relu_sites(prog, blk).items()}
    with otc.pinned_relu_masks(ones):
        ys = [block_oracle(blk, k * xl, k * xg, gl, gg) for k in (1, 2, 3)]
    for i in range(2):                                            # affine in x: y(x) + y(3x) = 2 y(2x)
        _close(ys[0][i] + ys[2][i], 2 * ys[1][i], 1e-12)
    assert _equal(ys[0][2:], ys[1][2:])                           # so its gradient does not depend on x
    free = block_oracle(blk, xl, xg, gl, gg)
    assert float((free[2] - ys[0][2]).abs().max()) > 1e-3 * float(free[2].abs().max())
    site = sorted(ones)[0]
    with pytest.raises(KeyError), otc.pinned_relu_masks({k: v for k, v in ones.items() if k != site}):
        block_oracle(blk, xl, xg, gl, gg)
    with pytest.raises(ValueError), otc.pinned_relu_masks(dict(ones, **{site: ones[site][..., :-1]})):
        block_oracle(blk, xl, xg, gl, gg)


def _programs():
    small_gen, small_kw = _gen(small_lama_kwargs(ngf=8, n_blocks=2))
    big_gen, big_kw = _gen(BIG_LAMA_KWARGS)
    return {"small": (_block(128), (32, 96), small_gen, small_kw, (16, 48)),
            "big": (_block(512), (128, 384), big_gen, big_kw, (128, 384))}


@pytest.mark.parametrize("math", [L.MATH_FP32, L.MATH_BF16X3])
@pytest.mark.parametrize("layout", ["small", "big"])
def test_kept_relu_outputs_map_one_to_one_onto_oracle_sites(layout, math):
    """Block-gradient and rear programs of the small and big-lama layouts (the big block also at 64x64, the split-bf16
    arm's planar chain): every kept ReLU output names an oracle site with its shape, the oracle passes exactly these
    sites, and exactly one ReLU backward (ReluBwdOp / HeadBwdOp) reads each of them."""
    blk, bch, gen, kw, gch = _programs()[layout]
    planes = [(6, 10)] + ([(64, 64)] if layout == "big" else [])
    cases = [("resnet_block_grad", blk, bch, hw) for hw in planes] + [("generator_rear_grad", gen, gch, (5, 7))]
    for kind, module, (cl, cg), (h, w) in cases:
        with torch.no_grad():
            prog = E.build_module_program(module, kind, ((1, cl, h, w), (1, cg, h, w)), math)
        assert prog.math == math
        sites = relu_sites(prog, module)
        ones = {s: torch.ones(v.batch, v.channels, *v.hw, dtype=torch.float64) for s, v in sites.items()}
        z = torch.zeros(1, cl, h, w, dtype=torch.float64), torch.zeros(1, cg, h, w, dtype=torch.float64)
        with otc.pinned_relu_masks(ones) as served:
            if kind == "resnet_block_grad":
                block_oracle(blk, *z, *z)
            else:
                rear_oracle(gen, kw, *z, torch.zeros(1, 3, 8 * h, 8 * w))
        assert served == set(sites), (kind, sorted(set(sites) ^ served))
        n_blocks = 1 if kind == "resnet_block_grad" else kw["n_blocks"]
        assert len(sites) == 8 * n_blocks + (kw["n_downsampling"] if kind != "resnet_block_grad" else 0)
        if (h, w) == (64, 64) and math == L.MATH_BF16X3:
            assert any(v.buf.cg for v in sites.values()), "expected the channel-group planar chain at 64x64"
        readers = {s: [i for i, op in enumerate(prog.ops) if mask_view(op) is not None and covers(mask_view(op), v)]
                   for s, v in sites.items()}
        assert all(len(r) == 1 for r in readers.values()), readers


@torch.no_grad()
def _dyadic_(module):
    """Parameters the engine's fp32 packing keeps exactly: float64, conv weights and biases on a 2^-8 grid, every BN
    an exact scale on a 2^-4 grid (running_var + eps == 1) with mean and beta on a 2^-8 grid.  The interpreter then
    runs the oracle's own weights, and the two differ by float64 round-off alone."""
    module.double()
    for m in module.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_var.fill_(1 - m.eps)
            m.weight.copy_(torch.where(m.weight.abs() < 1 / 16, torch.full_like(m.weight, 0.5),
                                       (m.weight * 16).round() / 16))
            for t in (m.bias, m.running_mean):
                t.copy_((t * 256).round() / 256)
        elif isinstance(m, (torch.nn.Conv2d, torch.nn.ConvTranspose2d)):
            for t in (m.weight, m.bias):
                if t is not None:
                    t.copy_((t * 256).round() / 256)
    return module


def _interp_masks(prog, blk_or_gen, feed):
    """Run the interpreter op by op, capturing the masks its backward reads."""
    interp = SpecInterpreter(prog)
    cap = MaskCapture(prog, blk_or_gen)
    out = {}
    for op in prog.ops:
        cap.before(op, lambda b: interp.mem[b.name])
        interp.step(op, feed, out)
    cap.assert_complete()
    return out, cap.masks


def _close(got, want, rel):
    scale = float(want.abs().max())
    err = float((got.double() - want.double()).abs().max())
    assert err <= rel * scale, f"{err:.3e} > {rel:g} * {scale:.3e}"


def test_masks_captured_from_the_interpreter_reproduce_its_input_gradients():
    """Masks captured from a SpecInterpreter run of the block-gradient and the rear program (parameters the packing keeps
    exactly, ``_dyadic_``): the pinned oracle's y, dx0 and dx1 equal the interpreter's to 1e-10 of their range — the
    engine's transposed, BN-folded decomposition is the gradient of the oracle's forward at those masks, with the
    Hermitian weights of the FFT pair and the reflect folds."""
    g = torch.Generator().manual_seed(3)
    blk = _dyadic_(_block(128))
    b, cl, cg, h, w = 2, 32, 96, 7, 11
    feed = dict(x0=_randn(b, cl, h, w, g=g), x1=_randn(b, cg, h, w, g=g), g0=_randn(b, cl, h, w, g=g),
                g1=_randn(b, cg, h, w, g=g))
    with torch.no_grad():
        prog = E.build_module_program(blk, "resnet_block_grad", ((b, cl, h, w), (b, cg, h, w)), L.MATH_FP32)
    out, masks = _interp_masks(prog, blk, feed)
    with otc.pinned_relu_masks(masks):
        y_l, y_g, d_l, d_g = block_oracle(blk, feed["x0"], feed["x1"], feed["g0"], feed["g1"])
    for k, want in (("y0", y_l), ("y1", y_g), ("dx0", d_l), ("dx1", d_g)):
        _close(out[k], want, 1e-10)

    gen, kw = _gen(small_lama_kwargs(ngf=8, n_blocks=2), act="tanh")
    _dyadic_(gen)
    b, h, w = 1, 5, 7
    feed = dict(x0=_randn(b, 16, h, w, g=g), x1=_randn(b, 48, h, w, g=g), g0=_randn(b, 3, 8 * h, 8 * w, g=g))
    with torch.no_grad():
        prog = E.build_module_program(gen, "generator_rear_grad", ((b, 16, h, w), (b, 48, h, w)), L.MATH_FP32)
    out, masks = _interp_masks(prog, gen, feed)
    with otc.pinned_relu_masks(masks):
        y, d1, d2 = rear_oracle(gen, kw, feed["x0"], feed["x1"], feed["g0"])
    for k, want in (("y0", y), ("dx0", d1), ("dx1", d2)):
        _close(out[k], want, 1e-10)
