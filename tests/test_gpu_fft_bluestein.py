"""GPU tests of the Bluestein (chirp-z) mode of the two-pass FFT kernels (``pytest -m gpu``): axes whose length has a
large prime factor (the bottlenecks of e.g. 3832x2160 -> 270x479 and 4016x2008 -> 251x502 photos; 211, 251, 263,
479, 502, 1021 all take Bluestein, 270 keeps its runtime plan).  Checkers: numpy
float64 (oracle/ffc_numpy.py) and the torch-CPU oracle port (oracle/ffc_torch_cpu.py), with the bounds of
tests/test_gpu_large_planes.py; FFCB_FFT_BLUESTEIN=0 (the runtime plans) as the cross-check of the lengths that keep
their plan."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200.testing import (BIG_LAMA_KWARGS, generator_input, seeded_parameters_,  # noqa: E402
                               small_lama_kwargs, synthetic_image_mask)
from oracle import ffc_numpy as onp                  # noqa: E402
from oracle import ffc_torch_cpu as otc              # noqa: E402

DEV = "cuda:0"
TOL = {"fp32": 2e-5, "bf16x3": 2e-4}


@pytest.fixture(autouse=True)
def _strict_env():
    os.environ["LAMA_B200_STRICT"] = "1"
    yield
    os.environ.pop("LAMA_B200_STRICT", None)
    os.environ.pop("FFCB_FFT_BLUESTEIN", None)


@pytest.fixture(params=["fp32", "bf16x3"])
def math_mode(request):
    os.environ["LAMA_B200_MATH"] = request.param
    yield request.param
    os.environ.pop("LAMA_B200_MATH", None)


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


def _rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max()) / (float(np.abs(ref).max()) or 1.0)


def _fft_program(b, c, h, w, split, out_c0):
    """rfft2 of x0 -> y0; irfft2 of x1 plus the residual x2 into channels [out_c0, out_c0 + c) of o -> y1."""
    wf = w // 2 + 1
    prog = E.Program("fft_test", L.MATH_BF16X3 if split else L.MATH_FP32)
    X = prog.buf("x", b, h, w, c); S = prog.buf("s", b, h, wf, 2 * c, gemm=split)
    Zin = prog.buf("z", b, h, wf, 2 * c); R = prog.buf("r", b, h, w, c)
    O = prog.buf("o", b, h, w, out_c0 + c, gemm=split)
    prog.inputs = {"x0": (b, c, h, w), "x1": (b, 2 * c, h, wf), "x2": (b, c, h, w)}
    prog.ops += [E.ToNHWC("x0", E.TV(X)), E.RfftOp(E.TV(X), E.TV(S)), E.ToNCHW(E.TV(S), "y0"),
                 E.ToNHWC("x1", E.TV(Zin)), E.ToNHWC("x2", E.TV(R)),
                 E.IrfftOp(E.TV(Zin), E.TV(R), E.TV(O, out_c0, c)), E.ToNCHW(E.TV(O, out_c0, c), "y1")]
    prog.outputs = {"y0": (b, 2 * c, h, wf), "y1": (b, c, h, w)}
    return prog


def _inputs(b, c, h, w):
    rng = np.random.default_rng(h * 1000 + w)
    x = rng.standard_normal((b, c, h, w)).astype(np.float32)
    z = np.maximum(rng.standard_normal((b, 2 * c, h, w // 2 + 1)), 0).astype(np.float32)
    res = rng.standard_normal((b, c, h, w)).astype(np.float32)
    return x, z, res


def _run(ex, x, z, res):
    return {k: v.cpu() for k, v in ex.run({"x0": torch.from_numpy(x).to(DEV), "x1": torch.from_numpy(z).to(DEV),
                                           "x2": torch.from_numpy(res).to(DEV)}).items()}


# ------------------------------------------------------------------------------------ FFT kernels
@pytest.mark.parametrize("split,out_c0", [(False, 0), (True, 0), (True, 4)])
@pytest.mark.parametrize("b,c,h,w", [(1, 4, 479, 270), (1, 8, 270, 479), (2, 12, 251, 502), (1, 36, 211, 263),
                                     (1, 4, 1021, 1021)])
def test_bluestein_fft_pair_against_numpy(b, c, h, w, split, out_c0):
    """ffcb_rfft2 / ffcb_irfft2 (two launches each) on planes with a Bluestein row or column axis vs numpy float64: the
    forward spectrum, and the inverse of a ReLU'd (non-Hermitian) spectrum plus the residual, in fp32 (2e-6 of max
    |ref|) and split bf16 (2e-5), the inverse also into channels [4, 4 + c) of a wider split-bf16 buffer.  36 channels
    leave dead lanes in the last CTA; m = 512 (211, 251), 1024 (263, 479, 502) and 2048 (1021, 4 channels per CTA)."""
    x, z, res = _inputs(b, c, h, w)
    wf = w // 2 + 1
    ex = E.CudaExecutor(_fft_program(b, c, h, w, split, out_c0), torch.device(DEV))
    out = _run(ex, x, z, res)
    spec = onp.rfft2_ortho(x.astype(np.float64))
    want_s = np.stack((spec.real, spec.imag), axis=2).reshape(b, 2 * c, h, wf)
    zc = z.astype(np.float64).reshape(b, c, 2, h, wf)
    want_y = onp.irfft2_explicit(zc[:, :, 0] + 1j * zc[:, :, 1], h, w) + res
    ef, ei = _rel_err(out["y0"].numpy(), want_s), _rel_err(out["y1"].numpy(), want_y)
    print(f"bluestein fft {b}x{c}x{h}x{w} {'split' if split else 'fp32'} c0={out_c0}: fwd {ef:.2e} inv {ei:.2e}")
    tol = 2e-5 if split else 2e-6
    assert ef < tol and ei < tol, (ef, ei)
    lib, stream = L.get_lib(), torch.cuda.current_stream().cuda_stream
    got = []
    for name, fn, args in ex.calls:
        if name in ("ffcb_rfft2", "ffcb_irfft2"):
            lib.ffcb_reset_launch_count()
            L.check(fn(*args, stream), name)
            got.append(int(lib.ffcb_launch_count()))
    torch.cuda.synchronize()
    assert got == [2, 2], got


def test_bluestein_round_trip_and_parseval_at_270x479():
    """big-lama's spectral planes on a 3832x2160 photo (192 channels, 270x479): irfft2(rfft2(x)) == x and Parseval."""
    b, c, h, w = 1, 192, 270, 479
    wf = w // 2 + 1
    x = torch.randn(b, c, h, w, generator=torch.Generator().manual_seed(7))
    prog = E.Program("fft_rt", L.MATH_FP32)
    X = prog.buf("x", b, h, w, c); S = prog.buf("s", b, h, wf, 2 * c); O = prog.buf("o", b, h, w, c)
    prog.inputs = {"x0": (b, c, h, w)}
    prog.ops += [E.ToNHWC("x0", E.TV(X)), E.RfftOp(E.TV(X), E.TV(S)), E.ToNCHW(E.TV(S), "y0"),
                 E.IrfftOp(E.TV(S), None, E.TV(O)), E.ToNCHW(E.TV(O), "y1")]
    prog.outputs = {"y0": (b, 2 * c, h, wf), "y1": (b, c, h, w)}
    out = {k: v.cpu() for k, v in E.CudaExecutor(prog, torch.device(DEV)).run({"x0": x.to(DEV)}).items()}
    assert float((out["y1"] - x).abs().max()) < 5e-6 * float(x.abs().max())
    p = (out["y0"].double().reshape(b, c, 2, h, wf) ** 2).sum(dim=2)
    wgt = torch.full((wf,), 2.0, dtype=torch.float64); wgt[0] = 1.0                  # odd width: no Nyquist bin
    assert abs(float((p * wgt).sum()) / float((x.double() ** 2).sum()) - 1.0) < 1e-5


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("b,c,h,w", [(1, 40, 270, 480), (1, 16, 375, 500), (2, 36, 64, 64)])
def test_lengths_that_keep_their_plan_are_bit_identical(b, c, h, w, split):
    """Planes whose lengths keep their runtime or compile-time plan (64x64 through the two-pass kernels) give the same
    bits with and without FFCB_FFT_BLUESTEIN=0."""
    x, z, res = _inputs(b, c, h, w)
    ex = E.CudaExecutor(_fft_program(b, c, h, w, split, 0), torch.device(DEV))
    os.environ["FFCB_FFT_TWO_PASS"] = "1"
    try:
        on = _run(ex, x, z, res)
        os.environ["FFCB_FFT_BLUESTEIN"] = "0"
        off = _run(ex, x, z, res)
    finally:
        os.environ.pop("FFCB_FFT_TWO_PASS", None)
        os.environ.pop("FFCB_FFT_BLUESTEIN", None)
    for k in ("y0", "y1"):
        assert torch.equal(on[k], off[k]), k


def test_bluestein_and_runtime_plans_agree_at_a_prime_width():
    """Sanity of the switch: at 270x479 the Bluestein pair and the direct DFT (FFCB_FFT_BLUESTEIN=0) agree to
    round-off, and both launch two kernels per direction."""
    b, c, h, w = 1, 16, 270, 479
    x, z, res = _inputs(b, c, h, w)
    ex = E.CudaExecutor(_fft_program(b, c, h, w, False, 0), torch.device(DEV))
    on = _run(ex, x, z, res)
    os.environ["FFCB_FFT_BLUESTEIN"] = "0"
    off = _run(ex, x, z, res)
    for k in ("y0", "y1"):
        assert _rel_err(on[k].numpy(), off[k].numpy()) < 2e-6, k
    assert not torch.equal(on["y0"], off["y0"]), "FFCB_FFT_BLUESTEIN=0 did not change the plan at 479 points"


# ------------------------------------------------------------------------------------ generators
_ORACLE = {}


def test_big_lama_at_2160x3832_against_oracle(math_mode):
    """big-lama on a 3832x2160 photo (bottleneck 270x479, rows through Bluestein) against the CPU fp32 oracle port, with
    the bounds of the 2160x3840 test: 5e-5 on the fp32 arm, 5e-4 on the split-bf16 arm."""
    seed = 0
    g = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), seed)
    sd = {k: v.clone() for k, v in g.state_dict().items()}
    img, mask = synthetic_image_mask(1, 2160, seed, width=3832)
    x = generator_input(img, mask)
    with torch.no_grad():
        y = g.to(DEV)(x.to(DEV)).cpu()
    E.invalidate(g)
    del g
    torch.cuda.empty_cache()
    if "big" not in _ORACLE:
        with torch.no_grad():
            _ORACLE["big"] = otc.ffc_resnet_generator(x, sd, **BIG_LAMA_KWARGS)
    ref = _ORACLE["big"]
    err = float((y - ref).abs().max())
    print(f"big-lama 2160x3832 ({math_mode}): max-abs {err:.2e}")
    assert ref.std() > 0.05 and err < (5e-5 if math_mode == "fp32" else 5e-4), err


def test_small_generator_at_2008x4016(math_mode):
    """A 251x502 bottleneck (both axes through Bluestein) against the float64 oracle (torch CPU in double)."""
    kw = small_lama_kwargs(ngf=8, n_blocks=2)
    g = seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 5)
    sd = {k: v.double() for k, v in g.state_dict().items()}
    img, mask = synthetic_image_mask(1, 2008, 5, width=4016)
    x = generator_input(img, mask)
    with torch.no_grad():
        y = g.to(DEV)(x.to(DEV)).cpu()
        ref = otc.ffc_resnet_generator(x.double(), sd, **kw)
    E.invalidate(g)
    err = float((y.double() - ref).abs().max())
    print(f"small generator 2008x4016 ({math_mode}): max-abs {err:.2e}")
    assert err < 3e-4, err


# ------------------------------------------------------------------------------------ gradients
def test_resnet_block_input_gradients_at_211x251(math_mode):
    """Native input gradients of big-lama's FFCResnetBlock on a 211x251 plane (both lengths prime, Bluestein in both
    directions; the FFT pair is its own adjoint) vs float64 autograd through the torch-CPU oracle, with the statistics
    of the native block-gradient tests on wide planes."""
    h, w, cl, cg = 211, 251, 128, 384
    blk = seeded_parameters_(M.FFCResnetBlock(cl + cg, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                              activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                              enable_lfu=False).eval(), 4, gain=1.0)
    sd = {k: v.clone() for k, v in blk.state_dict().items()}
    for p_ in blk.parameters():
        p_.requires_grad_(False)
    blk = blk.to(DEV)
    gen = torch.Generator().manual_seed(1)
    xl, xg, gl, gg = (torch.randn(1, ch, h, w, generator=gen) for ch in (cl, cg, cl, cg))
    a_l, a_g = xl.to(DEV).requires_grad_(True), xg.to(DEV).requires_grad_(True)
    L.get_lib().ffcb_reset_launch_count()
    o_l, o_g = blk((a_l, a_g))
    assert L.get_lib().ffcb_launch_count() > 10, "the native forward+backward program did not run"
    ((o_l * gl.to(DEV)).sum() + (o_g * gg.to(DEV)).sum()).backward()
    r_l, r_g = xl.double().requires_grad_(True), xg.double().requires_grad_(True)
    q_l, q_g = otc.ffc_resnet_block(r_l, r_g, {k: v.double() for k, v in sd.items()}, "", ratio_gout=0.75)
    ((q_l * gl.double()).sum() + (q_g * gg.double()).sum()).backward()
    assert _rel_err(o_l.detach().cpu().numpy(), q_l.detach().numpy()) < TOL[math_mode]
    assert _rel_err(o_g.detach().cpu().numpy(), q_g.detach().numpy()) < TOL[math_mode]
    tol = 1e-4 if math_mode == "fp32" else 5e-4
    for got, want in ((a_l.grad.cpu(), r_l.grad), (a_g.grad.cpu(), r_g.grad)):
        d = (got.double() - want.double()).abs()
        scale = float(want.abs().max())
        assert float((d > tol * scale).double().mean()) < 0.5, "too many elements off"
        assert float(d.median()) < tol * scale
        assert float(d.pow(2).sum().sqrt() / want.double().pow(2).sum().sqrt()) < 20 * tol
