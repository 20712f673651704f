"""Input gradients on the GPU, every element, against float64 autograd run with the kernels' own ReLU masks.

A gradient program is linear once its ReLU masks are fixed.  Each case issues the block-gradient or rear program one
call at a time (``device_state.DeviceRun``), reads every mask its backward uses from the device right before the ReLU
backward that reads it (``device_state.MaskCapture``), and runs the float64 oracle with those masks
(``otc.pinned_relu_masks``).  The reference then differs from the device by arithmetic round-off alone, so every
element of the forward outputs and of dx0 / dx1 is held to the op-level tolerance of the op-by-op harness
(``device_state.op_tol`` of a contraction): |got - want| <= tau * max|want|, tau = 2e-5 on the fp32 arm and 2e-4 on the
split-bf16 arm.  Per site, the number of mask elements that differ from the unpinned float64 forward is printed: those
flips are what the statistical tests against unpinned autograd (``_bulk_close`` in test_gpu_refine_large_planes.py)
have to absorb.

The float64 oracle runs on the GPU (cuDNN / cuFFT in float64): it is a reference, not a product path."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200.testing import seeded_parameters_, small_lama_kwargs  # noqa: E402
from oracle import ffc_torch_cpu as otc              # noqa: E402
from device_state import DEV, DeviceRun, MaskCapture, max_rel  # noqa: E402
from test_pinned_masks_cpu import block_oracle, rear_oracle    # noqa: E402

MATHS = {"fp32": L.MATH_FP32, "bf16x3": L.MATH_BF16X3}
TAU = {"fp32": 2e-5, "bf16x3": 2e-4}                 # op_tol of a contraction in device_state.py


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


@pytest.fixture(autouse=True)
def _strict_env():
    os.environ["LAMA_B200_STRICT"] = "1"
    yield
    os.environ.pop("LAMA_B200_STRICT", None)


def _block(dim, seed=4):
    return seeded_parameters_(M.FFCResnetBlock(dim, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                               activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                               enable_lfu=False).eval(), seed, gain=1.0)


def _randn(*shape, g):
    return torch.randn(*shape, generator=g)


def _rel2(got, want) -> float:
    return float((got - want).pow(2).sum().sqrt() / want.pow(2).sum().sqrt())


def run_pinned(module, kind, shapes, feed, math, after=None):
    """Run the program of ``module`` on the GPU one call at a time, capturing its ReLU masks; ``after(i, op, run)`` runs
    after each call.  Returns (program, device outputs on DEV as float64, masks on DEV)."""
    with torch.no_grad():
        prog = E.build_module_program(module, kind, shapes, MATHS[math])
    assert prog.math == MATHS[math], "the program fell back to the other arithmetic"
    run = DeviceRun(prog, feed)
    cap = MaskCapture(prog, module)
    run.run(before=lambda i, op: cap.before(op, run.dec),
            after=(lambda i, op: after(i, op, run)) if after is not None else None)
    cap.assert_complete()
    out = {k: v.to(DEV).double() for k, v in run.ex.outputs.items()}
    return prog, out, {k: v.to(DEV) for k, v in cap.masks.items()}


def check_pinned(label, out, masks, oracle, names, math):
    """``oracle()`` -> the reference of the outputs ``names`` in order.  Runs it unpinned (recording the float64
    forward's masks) and pinned to ``masks``; prints per site the mask elements that differ and per output the
    max-abs and 2-norm errors; returns {output: (pinned max-abs error, unpinned reference)}."""
    with otc.recorded_relu_masks() as free_masks:
        free = oracle()
    with otc.pinned_relu_masks(masks) as served:
        pinned = oracle()
    assert served == set(masks)
    print(f"\n  {label} ({math})")
    for site in sorted(masks):
        flips = int((masks[site] != free_masks[site]).sum())
        print(f"    mask {site}: {flips} of {masks[site].numel()} differ from the float64 forward")
    res = {}
    for name, want, ref in zip(names, pinned, free):
        got = out[name]
        err = max_rel(got, want)
        print(f"    {name}: max-abs {err:.2e} (tau {TAU[math]:g}), 2-norm {_rel2(got, want):.2e}; "
              f"unpinned: max-abs {max_rel(got, ref):.2e}, 2-norm {_rel2(got, ref):.2e}")
        res[name] = (err, ref)
    return res


def _assert_within(res, math):
    bad = {k: e for k, (e, _) in res.items() if not e <= TAU[math]}
    assert not bad, f"beyond tau = {TAU[math]:g} of the range: " + ", ".join(f"{k} {e:.2e}" for k, e in bad.items())


def _block_case(cl, cg, h, w, math, b=1, after=None):
    blk = _block(cl + cg).to(DEV)
    g = torch.Generator().manual_seed(h * 1000 + w)
    xl, xg, gl, gg = (_randn(b, ch, h, w, g=g) for ch in (cl, cg, cl, cg))
    shapes = ((b, cl, h, w), (b, cg, h, w))
    prog, out, masks = run_pinned(blk, "resnet_block_grad", shapes, dict(x0=xl, x1=xg, g0=gl, g1=gg), math, after)
    args = [t.to(DEV) for t in (xl, xg, gl, gg)]
    res = check_pinned(f"block {cl}+{cg} at {b}x{h}x{w}", out, masks, lambda: block_oracle(blk, *args),
                       ("y0", "y1", "dx0", "dx1"), math)
    return prog, out, res


# ------------------------------------------------------------------------------------------------ block gradients
BIG = [(128, 128), (270, 480), (108, 259), (211, 251), (128, 1024), (1024, 96)]


@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
@pytest.mark.parametrize("h,w", BIG)
def test_big_lama_block_gradients_pinned(h, w, math):
    """big-lama's block (128 + 384 channels): 128-wide planes, 8-channel FFT lengths (270x480: rows of 480, 128x1024),
    Bluestein lengths (108x259, 211x251) and a tall rectangular plane (1024x96)."""
    _assert_within(_block_case(128, 384, h, w, math)[2], math)


def test_big_lama_block_gradients_pinned_planar_chain():
    """64x64 on the split-bf16 arm: the FourierUnit chain in channel-group planar, tile-blocked storage."""
    prog, _, res = _block_case(128, 384, 64, 64, "bf16x3")
    assert any(b.cg for b in prog.bufs), "expected the channel-group planar chain at 64x64"
    _assert_within(res, "bf16x3")


@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
@pytest.mark.parametrize("b,h,w", [(2, 17, 25), (1, 16, 1021), (1, 1021, 16)])
def test_small_block_gradients_pinned(b, h, w, math):
    """A small block (32 + 96 channels): ragged mixed-radix planes with a batch of 2, and Bluestein axes of 1021
    points (m = 2048) along the rows and along the columns."""
    _assert_within(_block_case(32, 96, h, w, math, b=b)[2], math)


# ------------------------------------------------------------------------------------------------ rear program
@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
@pytest.mark.parametrize("b,h,w,act", [(2, 17, 25, "sigmoid"), (2, 17, 25, "tanh"), (2, 17, 25, False),
                                       (1, 108, 259, "sigmoid"), (1, 127, 256, "sigmoid")])
def test_rear_gradients_pinned(b, h, w, act, math):
    """The rear program of a small generator (2 blocks, 3 up stages, ngf 8): each head activation, a Bluestein
    bottleneck (108x259 -> 864x2072) and a rectangular one (127x256 -> 1016x2048).  Sites: the blocks' four ReLUs each,
    and every up stage (the last one's mask is read by the head adjoint)."""
    kw = dict(small_lama_kwargs(ngf=8, n_blocks=2), add_out_act=act)
    gen = seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 5, gain=1.0).to(DEV)
    cl, cg = 16, 48
    g = torch.Generator().manual_seed(h * 1000 + w)
    z1, z2, g0 = _randn(b, cl, h, w, g=g), _randn(b, cg, h, w, g=g), _randn(b, 3, 8 * h, 8 * w, g=g)
    assert E.rear_grad_supported(gen, (b, cl, h, w), (b, cg, h, w))
    _, out, masks = run_pinned(gen, "generator_rear_grad", ((b, cl, h, w), (b, cg, h, w)),
                               dict(x0=z1, x1=z2, g0=g0), math)
    assert len(masks) == 2 * 8 + 3
    args = [t.to(DEV) for t in (z1, z2, g0)]
    res = check_pinned(f"rear {act} at {b}x{h}x{w}", out, masks, lambda: rear_oracle(gen, kw, *args),
                       ("y0", "dx0", "dx1"), math)
    _assert_within(res, math)


# ------------------------------------------------------------------------------------------------ sensitivity
def test_pinned_check_flags_what_the_bulk_statistics_pass():
    """Scale one 4-channel group of the block backward's last fold (the 4 global channels of dx with the largest
    values) by 1 + 2^-10 on the device right after its call, as test_harness_flags_a_corrupted_op does.  The pinned
    check fails on it; the statistics of the tests against unpinned autograd (fewer than half the elements beyond tol,
    median below tol, 2-norm below 20 tol; tol = 5e-4 on the split-bf16 arm) pass on the same output."""
    math, cl, cg, h, w = "bf16x3", 128, 384, 128, 128
    hit = []

    def after(i, op, run):
        if op is not [o for o in run.prog.ops if isinstance(o, E.FoldOp)][-1]:
            return
        b = op.out.buf
        assert b.fmt == L.F32 and not b.pad and not b.cg
        storage = run.ex.storage[b.name]
        v = storage.reshape(-1)[:b.B * b.H * b.W * b.C].view(b.B, b.H, b.W, b.C)
        assert v.data_ptr() == storage.data_ptr()
        peak = v[..., cl:].abs().amax(dim=(0, 1, 2)).view(-1, 4).amax(dim=1)
        c0 = cl + 4 * int(peak.argmax())
        v[..., c0:c0 + 4].mul_(1 + 2 ** -10)
        hit.append(c0 - cl)

    _, out, res = _block_case(cl, cg, h, w, math, after=after)
    assert len(hit) == 1, "the last fold was not corrupted exactly once"
    err, ref = res["dx1"]
    got, tol = out["dx1"], 5e-4
    d = (got - ref).abs()
    scale = float(ref.abs().max())
    off, med, l2 = float((d > tol * scale).double().mean()), float(d.median()) / scale, _rel2(got, ref)
    print(f"  dx1 channels {hit[0]}..{hit[0] + 3} scaled by 1 + 2^-10: pinned max-abs {err:.2e} (tau {TAU[math]:g}); "
          f"unpinned: beyond {tol:g} {off:.3f}, median {med:.2e}, 2-norm {l2:.2e} (limits 0.5, {tol:g}, {20 * tol:g})")
    assert err > TAU[math], "the pinned check missed the scaled channels"
    assert off < 0.5 and med < tol and l2 < 20 * tol, "the bulk statistics flag the scaled channels too"
