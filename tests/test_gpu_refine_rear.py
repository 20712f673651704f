"""The generator's rear (residual blocks, up-sampling tail, head) as one native forward + input-gradient program on the
GPU (``pytest -m gpu``, an H100): the two kernels it adds (ffcb_head_bwd7, ffcb_add) and the ConvTranspose adjoint
contraction alone, the whole program against float64 autograd through the oracle and against the per-module path,
no library kernels outside the project, and the refinement loop end to end."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200 import packing as P                   # noqa: E402
from lama_b200 import refine as R                    # noqa: E402
from lama_b200.testing import (BIG_LAMA_KWARGS, generator_input, seeded_parameters_,  # noqa: E402
                               small_lama_kwargs, synthetic_image_mask)
from test_refine_rear_cpu import rear_oracle_grads   # noqa: E402

DEV = "cuda:0"
TOL = {L.MATH_FP32: 2e-5, L.MATH_BF16X3: 2e-4}
MATHS = [L.MATH_FP32, L.MATH_BF16X3]


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


@pytest.fixture(params=["fp32", "bf16x3"])
def math_mode(request):
    os.environ["LAMA_B200_MATH"] = request.param
    os.environ["LAMA_B200_STRICT"] = "1"
    yield request.param
    os.environ.pop("LAMA_B200_MATH", None)
    os.environ.pop("LAMA_B200_STRICT", None)


def _rel(got, want):
    want = want.double().cpu()
    return float((got.double().cpu() - want).abs().max()) / (float(want.abs().max()) or 1.0)


def _bulk_close(got, want, tol, frac=0.25):
    """The rule of test_gpu_parity.py::test_resnet_block_input_gradients_vs_autograd_oracle: an activation within
    round-off of zero can fall on the other side of a ReLU in two implementations, so the bulk of the elements agrees to
    ``tol`` of the range (all but ``frac``), the median is below it, and the 2-norm error is small."""
    got, want = got.double().cpu(), want.double().cpu()
    d = (got - want).abs()
    scale = float(want.abs().max())
    off, med = float((d > tol * scale).double().mean()), float(d.median()) / scale
    l2 = float(d.pow(2).sum().sqrt() / want.pow(2).sum().sqrt())
    print(f"  beyond {tol:g}: {off:.3f}, median {med:.2e}, 2-norm {l2:.2e} (of the range / norm)")
    assert off < frac, "too many elements off"
    assert med < tol
    assert l2 < 20 * tol


def _run(prog, feed):
    ex = E.CudaExecutor(prog, torch.device(DEV))
    return ex, ex.run({k: v.to(DEV).contiguous() for k, v in feed.items()})


# ------------------------------------------------------------------------------------------------ kernels alone
@pytest.mark.parametrize("shape", [(1, 64, 17, 25), (2, 64, 100, 136), (1, 64, 4, 4), (1, 8, 33, 64)])
@pytest.mark.parametrize("act", [L.ACT_SIGMOID, L.ACT_TANH, L.ACT_NONE])
@pytest.mark.parametrize("math", MATHS)
def test_head_bwd7_matches_autograd(shape, act, math):
    """ffcb_head_bwd7 = [up > 0] * Fold3(Conv7^T(act'(y) * dy)) vs float64 autograd of pad3 + conv7 + act through a
    ReLU.  The split-bf16 program stores the ReLU output with a ring of 3 and the gradient in split bf16; the fp32
    program both in float32."""
    b, c, h, w = shape
    n = 3
    g = torch.Generator().manual_seed(h * w + act)
    u = torch.randn(b, c, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(n, c, 7, 7, generator=g, dtype=torch.float64) * (0.5 / c ** 0.5)
    bias = torch.randn(n, generator=g, dtype=torch.float64) * 0.1
    dy = torch.randn(b, n, h, w, generator=g, dtype=torch.float64)
    prog = E.Program("head_bwd7_test", math)
    U = prog.buf("up", b, h, w, c, gemm=True, halo=True, halo_px=3)
    D = prog.buf("dup", b, h, w, c, gemm=True)
    wh, bh = P.pack_head(wt.float(), bias.float())
    prog.inputs = {"x0": (b, c, h, w), "g0": (b, n, h, w)}
    prog.outputs = {"y0": (b, n, h, w), "dx0": (b, c, h, w)}
    prog.ops = [E.ToNHWC("x0", E.TV(U)), E.HeadOp(E.TV(U), wh, bh, n, act, "y0"),
                E.HeadBwdOp("y0", "g0", wh, n, act, E.TV(U), E.TV(D)), E.ToNCHW(E.TV(D), "dx0")]
    assert (U.fmt, U.pad) == ((L.BF16X2, 3) if math == L.MATH_BF16X3 else (L.F32, 0))
    _, out = _run(prog, {"x0": torch.relu(u).float(), "g0": dy.float()})
    a = u.clone().requires_grad_(True)
    y = F.conv2d(F.pad(torch.relu(a), (3, 3, 3, 3), mode="reflect"), wt, bias)
    y = {L.ACT_SIGMOID: torch.sigmoid, L.ACT_TANH: torch.tanh, L.ACT_NONE: lambda t: t}[act](y)
    (y * dy).sum().backward()
    tol = 1e-5 if math == L.MATH_FP32 else 5e-5          # split bf16: 2^-17 per stored element
    assert _rel(out["y0"], y.detach()) < tol
    assert _rel(out["dx0"], a.grad) < tol, _rel(out["dx0"], a.grad)


@pytest.mark.parametrize("math", MATHS)
def test_add_sums_interior_and_ring(math):
    """ffcb_add in place on a ringed buffer: the values are a + b, and on the split-bf16 arm the 1-pixel ring of the
    result is bit for bit the reflection of its interior (no ring refresh needed after the add)."""
    b, c, h, w = 2, 64, 13, 21
    g = torch.Generator().manual_seed(7)
    x, y = torch.randn(b, c, h, w, generator=g), torch.randn(b, c, h, w, generator=g)
    prog = E.Program("add_test", math)
    X = prog.buf("x", b, h, w, c, gemm=True, halo=True)
    Y = prog.buf("y", b, h, w, c, gemm=True, halo=True)
    prog.inputs = {"x0": (b, c, h, w), "x1": (b, c, h, w)}
    prog.outputs = {"y0": (b, c, h, w)}
    prog.ops = [E.ToNHWC("x0", E.TV(X)), E.ToNHWC("x1", E.TV(Y)), E.AddOp(E.TV(X), E.TV(Y), E.TV(X)),
                E.ToNCHW(E.TV(X), "y0")]
    E.insert_border_ops(prog)
    assert sum(isinstance(op, E.BorderOp) for op in prog.ops) == (2 if math == L.MATH_BF16X3 else 0)
    ex, out = _run(prog, {"x0": x, "x1": y})
    assert _rel(out["y0"], x.double() + y.double()) < (1e-7 if math == L.MATH_FP32 else 1e-5)
    if math == L.MATH_BF16X3:
        s = ex.storage[X.name]                       # [2][B][H+2][W+2][C] bf16
        assert tuple(s.shape) == (2, b, h + 2, w + 2, c)
        assert torch.equal(s[:, :, 0], s[:, :, 2]) and torch.equal(s[:, :, h + 1], s[:, :, h - 1])
        assert torch.equal(s[:, :, :, 0], s[:, :, :, 2]) and torch.equal(s[:, :, :, w + 1], s[:, :, :, w - 1])


@pytest.mark.parametrize("cin,cout", [(512, 256), (256, 128), (128, 64)])
@pytest.mark.parametrize("hw", [(6, 10), (5, 13)])
@pytest.mark.parametrize("math", MATHS)
def test_convtranspose_adjoint_contraction(cin, cout, hw, math):
    """The adjoint of ConvTranspose2d(k3, s2, p1, op1) as the rear program emits it — ffcb_conv, stride 2, zero border,
    taps at -1..1, the transposed conv's own weight [Cin, Cout, 3, 3] — vs F.conv2d(stride=2, padding=1) in float64
    (big-lama's three tail channel pairs, a ragged width)."""
    h, w = hw
    g = torch.Generator().manual_seed(cin + h)
    wt = torch.randn(cin, cout, 3, 3, generator=g, dtype=torch.float64) / (3 * cout ** 0.5)
    d = torch.randn(1, cout, 2 * h, 2 * w, generator=g)
    prog = E.Program("convt_adjoint_test", math)
    Din = prog.buf("d", 1, 2 * h, 2 * w, cout, gemm=True)
    O = prog.buf("o", 1, h, w, cin)
    pk = P.pack_conv([(wt, 0, 0, 1)], None, None, stride=2, border=L.BORDER_ZERO)
    prog.inputs, prog.outputs = {"x0": (1, cout, 2 * h, 2 * w)}, {"y0": (1, cin, h, w)}
    prog.ops = [E.ToNHWC("x0", E.TV(Din)), E.ConvOp(pk, [E.TV(Din), None], E.TV(O)), E.ToNCHW(E.TV(O), "y0")]
    _, out = _run(prog, {"x0": d})
    want = F.conv2d(d.double(), wt, stride=2, padding=1)
    assert _rel(out["y0"], want) < TOL[math]


# ------------------------------------------------------------------------------------------------ whole program
def _frozen(gen):
    for p_ in gen.parameters():
        p_.requires_grad_(False)
    return gen


def test_rear_program_gradients_vs_autograd_oracle(math_mode):
    """dL/dz1, dL/dz2 through the native rear (small generator, 136x200 image, 17x25 bottleneck) vs float64 CPU
    autograd through the oracle composition; pred to the op-level tolerance."""
    kw = small_lama_kwargs(ngf=16, n_blocks=3)
    gen = _frozen(seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 2, gain=1.0)).to(DEV)
    g = torch.Generator().manual_seed(4)
    z1, z2 = torch.randn(1, 32, 17, 25, generator=g), torch.randn(1, 96, 17, 25, generator=g)
    g0 = torch.randn(1, 3, 136, 200, generator=g)
    assert E.rear_grad_supported(gen, z1.shape, z2.shape)
    a, b = z1.to(DEV).requires_grad_(True), z2.to(DEV).requires_grad_(True)
    pred = E.generator_rear_with_input_grad(gen, a, b)
    (pred * g0.to(DEV)).sum().backward()
    y, d1, d2 = rear_oracle_grads(gen, z1, z2, g0, kw)
    tol = 1e-4 if math_mode == "fp32" else 5e-4
    assert _rel(pred.detach(), y) < tol
    # measured on an H100: fp32 arm 2-norm 9e-7 (no flips); split-bf16 arm 35-43 % of the elements beyond 5e-4, median
    # 4e-4, 2-norm 7.6e-3 — three blocks of spectral ReLU masks whose flips each move a whole plane.  The module slice
    # (torch tail under TF32) measures 90 % / 3e-3 / 2.6e-2 against the same oracle on either arm.
    frac = 0.25 if math_mode == "fp32" else 0.5
    _bulk_close(a.grad, d1, tol, frac)
    _bulk_close(b.grad, d2, tol, frac)


def _front(gen, x):
    front, _ = R.split_generator(gen.model)
    with torch.no_grad():
        return front(x)


def test_big_lama_rear_matches_generator_program_and_module_path(math_mode):
    """big-lama at 512x512 (64x64 bottleneck, planar FourierUnit chain): pred of the rear program vs the generator
    program on the same input (they differ only by the rounding of Y2 before the identity add), and its gradients vs
    the per-module path (native block gradients, torch tail with TF32 off)."""
    gen = _frozen(seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0)).to(DEV)
    img, mask = synthetic_image_mask(1, 512, 3)
    x = generator_input(img, mask).to(DEV)
    with torch.no_grad():
        want = gen(x)
    z1, z2 = _front(gen, x)
    a, b = z1.detach().clone().requires_grad_(True), z2.detach().clone().requires_grad_(True)
    pred = E.generator_rear_with_input_grad(gen, a, b)
    diff = float((pred.detach() - want).abs().max())
    print(f"\nbig-lama 512x512 {math_mode}: rear program vs generator program max-abs {diff:.2e}")
    assert diff < 1e-3
    g0 = torch.randn(pred.shape, generator=torch.Generator().manual_seed(1)).to(DEV)
    (pred * g0).sum().backward()
    _, rear_mods = R.split_generator(gen.model)
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        c, d = z1.detach().clone().requires_grad_(True), z2.detach().clone().requires_grad_(True)
        os.environ["LAMA_B200_STRICT"] = "0"                  # the tail's plain nn modules run in torch
        (rear_mods((c, d)) * g0).sum().backward()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
        os.environ["LAMA_B200_STRICT"] = "1"
    tol = 1e-4 if math_mode == "fp32" else 5e-4
    # split-bf16 arm: the rear keeps X in split bf16 between the 18 blocks where the module slice adds in float32, so
    # ReLU masks near zero flip between the two (measured: 46 % of the elements beyond 5e-4 of the range)
    frac = 0.25 if math_mode == "fp32" else 0.6
    _bulk_close(a.grad, c.grad, tol, frac)
    _bulk_close(b.grad, d.grad, tol, frac)


def test_rear_launches_only_project_kernels(math_mode):
    """A rear forward + backward issues no cuDNN / cuFFT / cuBLAS kernel, and the library counts exactly the launches
    of one full replay of the program."""
    gen = _frozen(seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=16, n_blocks=2)).eval(), 1)).to(DEV)
    g = torch.Generator().manual_seed(5)
    z1, z2 = torch.randn(1, 32, 16, 24, generator=g).to(DEV), torch.randn(1, 96, 16, 24, generator=g).to(DEV)
    g0 = torch.randn(1, 3, 128, 192, generator=g).to(DEV)
    a, b = z1.clone().requires_grad_(True), z2.clone().requires_grad_(True)
    (E.generator_rear_with_input_grad(gen, a, b) * g0).sum().backward()       # builds + warms the executor
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        (E.generator_rear_with_input_grad(gen, a, b) * g0).sum().backward()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    banned = [n for n in names if "ffcb" not in n and any(k in n.lower() for k in ("cudnn", "fft", "xmma", "gemm",
                                                                                    "cutlass"))]
    assert not banned, banned
    assert any("head_bwd7" in n for n in names) and any("add_kernel" in n for n in names)
    ex = E.get_executor(gen, "generator_rear_grad", (z1, z2))
    ex.run({"x0": z1, "x1": z2, "g0": g0})
    lib = L.get_lib()
    lib.ffcb_reset_launch_count()
    ex.run({"x0": z1, "x1": z2}, part=0)
    ex.run({"g0": g0}, part=1)
    assert lib.ffcb_launch_count() == ex.launches_per_run >= len(ex.calls)


def _refine_with(rear_of, img, mask, generator, *, modulo, n_iters, lr, min_side, max_scales, px_budget):
    """refine_predict's scale loop with an explicit rear callable."""
    front, rear_mods = R.split_generator(generator.model)
    rear = rear_of(rear_mods)
    images, masks = R.image_mask_pyramid(img, mask, min_side, max_scales, px_budget)
    result = None
    for im, mk in zip(images, masks):
        orig = tuple(im.shape[2:])
        im_p, mk_p = R._pad_to_modulo(im, modulo).to(DEV), R._pad_to_modulo(mk, modulo).to(DEV)
        mk_p = (mk_p >= 1e-8).to(mk_p.dtype)
        result = R.infer_scale(im_p, mk_p, front, rear, result, orig, n_iters, lr)[:, :, :orig[0], :orig[1]]
    return result.cpu()


def test_refinement_native_rear_matches_module_path():
    """refine_predict (native rear program at every scale) vs the same loop driven by the module slice (native block
    gradients, torch tail): the bounds of test_gpu_parity.py's refinement test.  A second rear forward of the same
    shape before the backward raises instead of returning gradients of overwritten activations."""
    os.environ["LAMA_B200_MATH"] = "bf16x3"
    try:
        g = seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=16, n_blocks=3)).eval(), 2, gain=1.0).to(DEV)
        gen = torch.Generator().manual_seed(0)
        img = torch.rand(1, 3, 136, 200, generator=gen)
        mask = torch.zeros(1, 1, 136, 200); mask[..., 30:90, 50:150] = 1
        kw = dict(modulo=8, n_iters=4, lr=0.002, min_side=64, max_scales=2, px_budget=10 ** 7)
        native = R.refine_predict(img, mask, g, **kw)
        assert any(k[0] == "generator_rear_grad" for k in E._PROGRAMS.get(g, {})), "the native rear did not run"
        ref = _refine_with(lambda mods: mods, img, mask, g, **kw)
        assert torch.isfinite(native).all()
        assert float((native - ref).abs().max()) < 5e-3
        assert float((native - ref).abs().mean()) < 2e-4
        z1 = torch.randn(1, 32, 17, 25, device=DEV, requires_grad=True)
        z2 = torch.randn(1, 96, 17, 25, device=DEV, requires_grad=True)
        p1 = E.generator_rear_with_input_grad(g, z1, z2)
        E.generator_rear_with_input_grad(g, z1, z2)
        with pytest.raises(RuntimeError, match="ran forward again"):
            p1.sum().backward()
    finally:
        os.environ.pop("LAMA_B200_MATH", None)
