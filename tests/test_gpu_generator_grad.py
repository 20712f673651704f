"""Input gradients through the whole generator on the GPU (kind ``generator_grad``, lama_b200/generator_grad.py).

* ``ffcb_stem_bwd7`` bit for bit against float64 on exactly representable operands (small integers times powers of two:
  every product and partial sum is exact in float32, so any summation order gives the float64 value).
* The stride-2 down adjoints (reflect: phases onto the padded plane + fold; zero border: interior phases) op by op
  against float64 autograd, within tau of max|want| (tau = 2e-5 fp32 arm, 2e-4 split-bf16 arm).
* Whole-program y0 / dx0 element by element against the float64 oracle run with the device's own ReLU masks
  (``otc.pinned_relu_masks``; see tests/test_gpu_pinned_grads.py), within the same tau, on both arms.
* The drop-in modules under autograd."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import generator_grad as GG           # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200 import pix2pixhd as PX                # noqa: E402
from lama_b200.testing import (BIG_LAMA_KWARGS, LAMA_REGULAR_KWARGS, seeded_parameters_,  # noqa: E402
                               small_lama_kwargs)
from oracle import ffc_torch_cpu as otc              # noqa: E402
from device_state import DEV, DeviceRun, MaskCapture, max_rel  # noqa: E402
from test_generator_grad_cpu import ffc_generator_f64, regular_generator_f64  # noqa: E402

MATHS = {"fp32": L.MATH_FP32, "bf16x3": L.MATH_BF16X3}
TAU = {"fp32": 2e-5, "bf16x3": 2e-4}


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


@pytest.fixture(autouse=True)
def _strict_env():
    os.environ["LAMA_B200_STRICT"] = "1"
    yield
    os.environ.pop("LAMA_B200_STRICT", None)


def _nhwc_tensor(v: torch.Tensor, fmt: int):
    """(descriptor, storage) of a channels-last [B, H, W, C] device view of ``v``: float32, or split bf16 whose hi
    plane holds ``v`` (exact in bf16) and whose lo plane is zero."""
    b, h, w, c = v.shape
    t = L.Tensor()
    if fmt == L.F32:
        st = v.float().contiguous().to(DEV)
        t.lo_off = 0
    else:
        st = torch.stack([v.bfloat16(), torch.zeros_like(v, dtype=torch.bfloat16)]).contiguous().to(DEV)
        t.lo_off = b * h * w * c
    t.ptr, t.sb, t.sy, t.sx = st.data_ptr(), h * w * c, w * c, c
    t.B, t.H, t.W, t.C, t.fmt, t.pad, t.reflect_border = b, h, w, c, fmt, 0, 0
    return t, st


# ------------------------------------------------------------------------------------------------ stem adjoint
@pytest.mark.parametrize("fmt", [L.F32, L.BF16X2])
@pytest.mark.parametrize("cin", [4, 8])
@pytest.mark.parametrize("h,w", [(8, 8), (13, 21), (40, 33), (65, 130)])
def test_stem_bwd7_exact(h, w, cin, fmt):
    g = torch.Generator().manual_seed(h * 131 + w + cin)
    n, b = 24, 2                                   # 3 chunks of 8 gradient channels
    wt = torch.randint(-16, 17, (n, cin, 7, 7), generator=g).double() / 64
    gy = torch.randint(-8, 9, (b, n, h, w), generator=g).double()
    x = torch.zeros(b, cin, h, w, dtype=torch.float64, requires_grad=True)
    (F.conv2d(F.pad(x, (3, 3, 3, 3), mode="reflect"), wt) * gy).sum().backward()
    want = x.grad
    desc, _keep = _nhwc_tensor(gy.permute(0, 2, 3, 1), fmt)
    wk = wt.permute(0, 2, 3, 1).reshape(n, 49, cin).float().contiguous().to(DEV)
    dx = torch.full((b, cin, h, w), float("nan"), device=DEV)
    lib = L.get_lib()
    L.check(lib.ffcb_stem_bwd7(desc, wk.data_ptr(), cin, dx.data_ptr(), torch.cuda.current_stream().cuda_stream),
            "ffcb_stem_bwd7")
    torch.cuda.synchronize()
    got = dx.double().cpu()
    if not torch.equal(got, want):
        i = (got != want).nonzero()[0].tolist()
        pytest.fail(f"first mismatch at {i}: got {got[tuple(i)]}, want {want[tuple(i)]}")


# ------------------------------------------------------------------------------------------------ down adjoints
@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
@pytest.mark.parametrize("padded", [True, False], ids=["reflect", "zero"])
@pytest.mark.parametrize("n,c,h,w", [(128, 64, 64, 64), (64, 32, 40, 72), (512, 256, 128, 96)])
def test_down_adjoint_op_by_op(n, c, h, w, padded, math):
    """gradient w.r.t. x of scale * conv3x3_s2(pad(x)), from g = dL/dy (h/2 x w/2): the four phase contractions (and
    the fold for the reflect border) against float64 autograd."""
    gen = torch.Generator().manual_seed(n + h)
    b = 2
    wt = torch.randn(n, c, 3, 3, generator=gen) / (3 * c ** 0.5)
    sc = 0.5 + torch.rand(n, generator=gen)
    gy = torch.randn(b, n, h // 2, w // 2, generator=gen)
    prog = E.Program("down_adjoint", MATHS[math])
    D = prog.buf("g", b, h // 2, w // 2, n, gemm=True)
    Y = prog.buf("y", b, h // 2, w // 2, n, gemm=True, halo=True)
    X = prog.buf("x", b, h, w, c, gemm=True, halo=True)
    prog.inputs = {"x0": (b, n, h // 2, w // 2)}
    prog.ops.append(E.ToNHWC("x0", E.TV(D)))
    DX = GG.emit_down_adjoint(prog, Y, D, wt.to(DEV), sc.double().to(DEV), X, padded)
    prog.ops = [op for op in prog.ops if not isinstance(op, E.ReluBwdOp)]       # the contractions (and fold) alone
    for op in prog.ops:
        if isinstance(op, E.ConvOp):
            op.ins[0] = E.TV(D)
    prog.ops.append(E.ToNCHW(E.TV(DX), "y0"))
    prog.outputs = {"y0": (b, c, h, w)}
    E.insert_border_ops(prog)
    out = E.CudaExecutor(prog, torch.device(DEV)).run({"x0": gy.to(DEV)})["y0"].double().cpu()
    x = torch.zeros(b, c, h, w, dtype=torch.float64, requires_grad=True)
    xp = F.pad(x, (1, 1, 1, 1), mode="reflect" if padded else "constant")
    (F.conv2d(xp, wt.double() * sc.double()[:, None, None, None], stride=2) * gy.double()).sum().backward()
    err = max_rel(out, x.grad)
    print(f"down adjoint {n}->{c} {h}x{w} {'reflect' if padded else 'zero'} {math}: {err:.2e}")
    assert err <= TAU[math]


# ------------------------------------------------------------------------------------------------ whole program
def _pinned_case(gen, shape, math, oracle):
    """Run the program one call at a time capturing its masks, then the float64 oracle (``oracle(x, g0)`` -> y) pinned
    to them; returns {y0, dx0: max |got - want| / max |want|}."""
    g = torch.Generator().manual_seed(shape[2] + shape[3])
    x = torch.randn(shape, generator=g)
    g0 = torch.randn(shape[0], 3, shape[2], shape[3], generator=g)
    with torch.no_grad():
        prog = E.build_module_program(gen, "generator_grad", (shape,), MATHS[math])
    assert prog.math == MATHS[math], "the program fell back to the other arithmetic"
    run = DeviceRun(prog, dict(x0=x, g0=g0))
    cap = MaskCapture(prog, gen)
    run.run(before=lambda i, op: cap.before(op, run.dec))
    cap.assert_complete()
    out = {k: v.double() for k, v in run.ex.outputs.items()}
    del run
    masks = {k: v.to(DEV) for k, v in cap.masks.items()}
    a = x.to(DEV).double().requires_grad_(True)
    with otc.pinned_relu_masks(masks):
        y = oracle(a)
        (y * g0.to(DEV).double()).sum().backward()
    res = {"y0": max_rel(out["y0"], y.detach()), "dx0": max_rel(out["dx0"], a.grad)}
    print(f"\n  {type(gen).__name__} {shape} {math}: " + ", ".join(f"{k} {v:.2e}" for k, v in res.items()))
    return res


def _ffc_case(kw, shape, math, seed=0):
    gen = seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), seed).requires_grad_(False).to(DEV)
    res = _pinned_case(gen, shape, math, lambda a: ffc_generator_f64(gen, kw, a))
    assert all(v <= TAU[math] for v in res.values()), res


def _regular_case(shape, math):
    gen = seeded_parameters_(PX.GlobalGenerator(**LAMA_REGULAR_KWARGS).eval(), 0).requires_grad_(False).to(DEV)
    gd = PX.GlobalGenerator(**LAMA_REGULAR_KWARGS).eval().double().to(DEV)
    gd.load_state_dict(gen.state_dict())
    res = _pinned_case(gen, shape, math, lambda a: regular_generator_f64(gd, a))
    assert all(v <= TAU[math] for v in res.values()), res


@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
def test_big_lama_512_batch2_pinned(math):
    _ffc_case(BIG_LAMA_KWARGS, (2, 4, 512, 512), math)


@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
def test_big_lama_1080x1920_pinned(math):
    """A 135 x 240 bottleneck."""
    _ffc_case(BIG_LAMA_KWARGS, (1, 4, 1080, 1920), math)


@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
def test_bluestein_bottleneck_pinned(math):
    """A 211 x 251 bottleneck: both FFT axes are Bluestein lengths."""
    _ffc_case(small_lama_kwargs(ngf=8, n_blocks=2), (1, 4, 8 * 211, 8 * 251), math)


@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
@pytest.mark.parametrize("h,w", [(512, 512), (1024, 768)])
def test_lama_regular_pinned(h, w, math):
    _regular_case((1, 4, h, w), math)


# ------------------------------------------------------------------------------------------------ module wiring
def _big(seed=0):
    return seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), seed).requires_grad_(False).to(DEV)


@pytest.mark.parametrize("kind", ["big-lama", "lama-regular"])
def test_module_autograd_takes_the_native_program(kind):
    """``torch.autograd.grad(generator(x).sum(), x)`` runs the native program (LAMA_B200_STRICT=1 raises on a torch
    fallback), its y is within 3e-4 of the no-grad output, image i alone and inside a batch get bit-identical dx,
    and a second forward before the backward raises."""
    gen = _big() if kind == "big-lama" else seeded_parameters_(
        PX.GlobalGenerator(**LAMA_REGULAR_KWARGS).eval(), 0).requires_grad_(False).to(DEV)
    g = torch.Generator().manual_seed(7)
    x = torch.rand(3, 4, 256, 384, generator=g).to(DEV)
    xr = x.clone().requires_grad_(True)
    y = gen(xr)
    assert y.grad_fn is not None and "SplitProgramFn" in type(y.grad_fn).__name__
    (dx,) = torch.autograd.grad(y.sum(), xr)
    with torch.no_grad():
        y_ref = gen(x)
    assert float((y.detach() - y_ref).abs().max()) <= 3e-4
    x1 = x[1:2].clone().requires_grad_(True)
    (dx1,) = torch.autograd.grad(gen(x1).sum(), x1)
    assert torch.equal(dx1, dx[1:2])
    with torch.enable_grad():
        z = x.clone().requires_grad_(True)
        y1 = gen(z)
        gen(z)
        with pytest.raises(RuntimeError, match="ran forward again"):
            y1.sum().backward()
    y2 = gen(x)                                     # no input gradient wanted: the no-grad generator program
    assert not y2.requires_grad and torch.equal(y2, y_ref)


def test_trainable_weights_keep_the_torch_composition():
    os.environ.pop("LAMA_B200_STRICT", None)
    gen = _big()
    gen.model[-2].weight.requires_grad_(True)
    x = torch.rand(1, 4, 128, 128, device=DEV, requires_grad=True)
    y = gen(x)
    assert "SplitProgramFn" not in type(y.grad_fn).__name__
    y.sum().backward()
    assert gen.model[-2].weight.grad is not None and x.grad is not None
