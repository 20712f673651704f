"""GPU parity tests (run on an H100: ``pytest -m gpu``).  Everything goes through the C ABI of
libffc_b200.so (via the drop-in modules / lama_b200.engine); the checker is the oracle
(oracle/ffc_numpy.py float64, oracle/ffc_torch_cpu.py) and the committed goldens generated from the
unmodified reference.  /root/reference is NOT read here.

Tolerances (floating point path, stated per test):
  * op level, fp32 math:       max-abs <= 2e-5 * max|ref|   (fp32 round-off of FFT + 512-term dot products)
  * generator, any math mode:  max-abs <= 1e-3 on the sigmoid output (north_star), and we also assert the
                               tighter 5e-5 that the fp32 / bf16x3 arithmetic actually achieves.
"""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200 import packing as P                   # noqa: E402
from lama_b200.testing import (BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs,  # noqa: E402
                               synthetic_image_mask, generator_input)
from oracle import ffc_numpy as onp                  # noqa: E402
from oracle import ffc_torch_cpu as otc              # noqa: E402

DEV = "cuda:0"
MATHS = [L.MATH_FP32, L.MATH_BF16X3]
# op-level tolerance relative to max|ref|: fp32 round-off vs. split-bf16 operands (2^-16 per operand)
TOL = {"fp32": 2e-5, "bf16x3": 2e-4}


@pytest.fixture(autouse=True)
def _strict_env():
    """An unexpected torch fallback is a test failure; tests that do not depend on the arithmetic mode (the kernel
    level ones: they pick formats / math per program) run once, with the library default left alone."""
    os.environ["LAMA_B200_STRICT"] = "1"
    yield
    os.environ.pop("LAMA_B200_STRICT", None)


@pytest.fixture(params=["fp32", "bf16x3"])
def math_mode(request):
    """Module-level tests request this fixture and run in both arithmetic modes of the library (LAMA_B200_MATH)."""
    os.environ["LAMA_B200_MATH"] = request.param
    yield request.param
    os.environ.pop("LAMA_B200_MATH", None)


@pytest.fixture
def tc_math():
    """Tests of things that exist on the tensor-core arm only (uint8 front / back end, planar chain): run once, in that mode."""
    os.environ["LAMA_B200_MATH"] = "bf16x3"
    yield "bf16x3"
    os.environ.pop("LAMA_B200_MATH", None)


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


def _load(module, sd):
    missing, unexpected = module.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    assert not unexpected and all(k.endswith("num_batches_tracked") for k in missing)
    return module.eval().to(DEV)


def _rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max()) / (float(np.abs(ref).max()) or 1.0)


def _run_program(prog, feed):
    ex = E.CudaExecutor(prog, torch.device(DEV))
    out = ex.run({k: v.to(DEV).contiguous() for k, v in feed.items()})
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


# ------------------------------------------------------------------------------------ FFT kernels
@pytest.mark.parametrize("b,c,h,w", [(2, 8, 16, 16), (1, 32, 64, 64), (1, 4, 8, 32), (3, 36, 32, 32),
                                     (1, 8, 128, 128), (1, 4, 256, 256), (1, 4, 15, 15), (2, 4, 6, 9),
                                     (1, 4, 20, 24), (1, 8, 125, 188), (1, 4, 5, 2), (1, 40, 64, 4)])
def test_rfft2_irfft2_against_numpy(b, c, h, w):
    _check_fft_pair(b, c, h, w)


@pytest.mark.parametrize("mixed", ["0", "1"])
@pytest.mark.parametrize("b,c,h,w", [(1, 4, 15, 15), (2, 4, 6, 9), (1, 8, 125, 188), (1, 36, 96, 128),
                                     (1, 4, 135, 240), (2, 8, 47, 94), (1, 4, 7, 250), (1, 4, 3, 2)])
def test_fft_lengths_without_compile_time_plan(b, c, h, w, mixed, monkeypatch):
    """SURVEY.md row f2 (bin/predict.py pads to multiples of 8 only -> 96x128, 135x240, 125x188 ... bottleneck
    planes): runtime mixed-radix Stockham (FFCB_FFT_MIXED_RADIX=1) and the O(n^2) direct DFT (=0) against numpy —
    composite, prime-power, prime and large-prime-factor lengths."""
    monkeypatch.setenv("FFCB_FFT_MIXED_RADIX", mixed)
    _check_fft_pair(b, c, h, w)


def test_two_pass_fft_kernels_at_64x64(monkeypatch):
    """64x64 planes normally take the fused whole-plane kernels (fft_plane.cu); keep the general
    row/column kernels covered at that size too."""
    monkeypatch.setenv("FFCB_FFT_TWO_PASS", "1")
    _check_fft_pair(2, 40, 64, 64, launches=(2, 2))


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("residual", [True, False])
def test_plane_kernels_in_every_format(split, residual):
    """The 64x64 channels-last plane pair, one launch per direction: the forward in both spectrum formats, and all
    four format / residual instantiations of the inverse (32-bit in-plane offsets, channels-last vector epilogue
    staged in place of the half spectrum)."""
    _check_fft_pair(3, 40, 64, 64, split=split, residual=residual, launches=(1, 1))


def test_inverse_views_the_plane_kernel_refuses_take_two_pass():
    """A split-bf16 output at channel offset 4 is only 8-byte aligned, too little for the plane kernel's 16-byte
    stores: the inverse runs the two row / column kernels instead, and its result still matches numpy."""
    _check_fft_pair(2, 40, 64, 64, split=True, out_c0=4, launches=(1, 2))


def _check_fft_pair(b, c, h, w, split=False, residual=True, out_c0=0, launches=None):
    """ffcb_rfft2 / ffcb_irfft2 vs numpy (float64): forward spectrum, and the inverse of a NON-Hermitian
    (ReLU'd) spectrum with the residual add — pow2 Stockham and direct-DFT sizes.  ``split``: the formats of the
    generator program (forward spectrum and inverse output stored as split bf16, 2^-16 per value).  ``out_c0``: the
    inverse writes channels [out_c0, out_c0 + c) of a wider buffer.  ``launches``: the kernel launches expected of
    (ffcb_rfft2, ffcb_irfft2), i.e. which path each ran."""
    rng = np.random.default_rng(h * 1000 + w)
    x = rng.standard_normal((b, c, h, w)).astype(np.float32)
    wf = w // 2 + 1
    prog = E.Program("fft_test", L.MATH_BF16X3 if split else L.MATH_FP32)
    X = prog.buf("x", b, h, w, c); S = prog.buf("s", b, h, wf, 2 * c, gemm=split)
    Zin = prog.buf("z", b, h, wf, 2 * c); R = prog.buf("r", b, h, w, c); O = prog.buf("o", b, h, w, out_c0 + c, gemm=split)
    assert S.fmt == O.fmt == (L.BF16X2 if split else L.F32) and Zin.fmt == R.fmt == X.fmt == L.F32
    prog.inputs = {"x0": (b, c, h, w), "x1": (b, 2 * c, h, wf), "x2": (b, c, h, w)}
    prog.ops += [E.ToNHWC("x0", E.TV(X)), E.RfftOp(E.TV(X), E.TV(S)), E.ToNCHW(E.TV(S), "y0"),
                 E.ToNHWC("x1", E.TV(Zin)), E.ToNHWC("x2", E.TV(R)),
                 E.IrfftOp(E.TV(Zin), E.TV(R) if residual else None, E.TV(O, out_c0, c)), E.ToNCHW(E.TV(O, out_c0, c), "y1")]
    prog.outputs = {"y0": (b, 2 * c, h, wf), "y1": (b, c, h, w)}
    z = np.maximum(rng.standard_normal((b, 2 * c, h, wf)), 0).astype(np.float32)
    res = rng.standard_normal((b, c, h, w)).astype(np.float32)
    ex = E.CudaExecutor(prog, torch.device(DEV))
    out = {k: v.cpu() for k, v in ex.run({"x0": torch.from_numpy(x).to(DEV), "x1": torch.from_numpy(z).to(DEV),
                                          "x2": torch.from_numpy(res).to(DEV)}).items()}
    tol = 2e-5 if split else 2e-6
    spec = onp.rfft2_ortho(x.astype(np.float64))
    want_s = np.stack((spec.real, spec.imag), axis=2).reshape(b, 2 * c, h, wf)
    assert _rel_err(out["y0"].numpy(), want_s) < tol
    zc = z.astype(np.float64).reshape(b, c, 2, h, wf)
    want_y = onp.irfft2_explicit(zc[:, :, 0] + 1j * zc[:, :, 1], h, w) + (res if residual else 0.0)
    assert _rel_err(out["y1"].numpy(), want_y) < tol
    if launches is not None:       # replay each FFT call alone; the library counts the kernels it launches
        lib, stream = L.get_lib(), torch.cuda.current_stream().cuda_stream
        got = []
        for name, fn, args in ex.calls:
            if name in ("ffcb_rfft2", "ffcb_irfft2"):
                lib.ffcb_reset_launch_count()
                L.check(fn(*args, stream), name)
                got.append(int(lib.ffcb_launch_count()))
        torch.cuda.synchronize()
        assert tuple(got) == launches, got


def test_fft_round_trip_full_size():
    """Size-independent property at the BASELINE shape (32 x 192 x 64 x 64): irfft2(rfft2(x)) == x and
    Parseval (ortho norm; half spectrum counted twice except the k_w = 0 and Nyquist columns)."""
    b, c, h, w = 32, 192, 64, 64
    wf = w // 2 + 1
    x = torch.randn(b, c, h, w, generator=torch.Generator().manual_seed(7))
    prog = E.Program("fft_rt", L.MATH_FP32)
    X = prog.buf("x", b, h, w, c); S = prog.buf("s", b, h, wf, 2 * c); O = prog.buf("o", b, h, w, c)
    prog.inputs = {"x0": (b, c, h, w)}
    prog.ops += [E.ToNHWC("x0", E.TV(X)), E.RfftOp(E.TV(X), E.TV(S)), E.ToNCHW(E.TV(S), "y0"),
                 E.IrfftOp(E.TV(S), None, E.TV(O)), E.ToNCHW(E.TV(O), "y1")]
    prog.outputs = {"y0": (b, 2 * c, h, wf), "y1": (b, c, h, w)}
    out = _run_program(prog, {"x0": x})
    assert float((out["y1"] - x).abs().max()) < 5e-6 * float(x.abs().max())
    s = out["y0"].double().reshape(b, c, 2, h, wf)
    p = (s ** 2).sum(dim=2)
    wgt = torch.full((wf,), 2.0, dtype=torch.float64); wgt[0] = 1.0; wgt[-1] = 1.0
    assert abs(float((p * wgt).sum()) / float((x.double() ** 2).sum()) - 1.0) < 1e-5


# ------------------------------------------------------------------------------------ conv kernel
_CONV_CASES = ["k3_reflect", "k3_s2", "k1_two_src", "k7_nopad", "zero_border_phase", "ragged"]
# (the tensor-core arm requires 64-channel K segments: "k7_nopad" and "ragged" exist for the CUDA-core arm only)
_CONV_PARAMS = [(c, m) for m in MATHS for c in _CONV_CASES
                if not (m == L.MATH_BF16X3 and c in ("k7_nopad", "ragged"))]


@pytest.mark.parametrize("case,math", _CONV_PARAMS)
def test_conv_contract(case, math):
    """ffcb_conv vs the torch restatement of its contract (packing.apply_packed_reference), covering
    reflect / zero borders, stride 2, two sources, addend before/after the activation, sub-pixel
    output phases and sizes that are not multiples of the CTA tile."""
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    post = False
    if case == "k3_reflect":
        b, h, w, cin, n = 2, 16, 16, 64, 128
        pk = P.pack_conv([(rn(n, cin, 3, 3) * 0.1, 0, 0, 1)], rn(n).abs() + 0.5, rn(n), act=L.ACT_RELU)
        ins, out_hw, add, post = [rn(b, h, w, cin), None], (h, w), rn(b, h, w, n), True
    elif case == "k3_s2":
        b, h, w, cin, n = 1, 32, 32, 64, 64
        pk = P.pack_conv([(rn(n, cin, 3, 3) * 0.1, 0, 0, 1)], None, rn(n), stride=2, act=L.ACT_RELU)
        ins, out_hw, add = [rn(b, h, w, cin), None], (16, 16), None
    elif case == "k1_two_src":
        b, h, w, n = 2, 8, 8, 64
        pk = P.pack_conv([(rn(n, 64, 3, 3) * 0.1, 0, 64, 1), (rn(n, 128, 1, 1) * 0.1, 1, 0, 0)], rn(n).abs(), rn(n),
                         act=L.ACT_NONE)
        ins, out_hw, add = [rn(b, h, w, 128), rn(b, h, w, 128)], (h, w), rn(b, h, w, n)
    elif case == "k7_nopad":
        b, h, w, cin, n = 1, 22, 22, 4, 8
        pk = P.pack_conv([(rn(n, cin, 7, 7) * 0.1, 0, 0, 0)], None, None, act=L.ACT_SIGMOID)
        ins, out_hw, add = [rn(b, h, w, cin), None], (16, 16), None
    elif case == "zero_border_phase":
        b, h, w, cin, n = 2, 8, 8, 64, 64
        wt = rn(cin, n, 3, 3) * 0.1
        phases = P.pack_conv_transpose_phases(wt, rn(n), rn(n).abs() + 0.5, rn(n), act=L.ACT_RELU)
        x = rn(b, h, w, cin)
        prog = E.Program("convT", math)
        X = prog.buf("x", b, h, w, cin, gemm=True, halo=True); Y = prog.buf("y", b, 2 * h, 2 * w, n)
        prog.inputs = {"x0": (b, cin, h, w)}
        prog.ops.append(E.ToNHWC("x0", E.TV(X)))
        for a, bb, pk in phases:
            prog.ops.append(E.ConvOp(pk, [E.TV(X), None], E.TV(Y, phase=(a, bb))))
        prog.ops.append(E.ToNCHW(E.TV(Y), "y0")); prog.outputs = {"y0": (b, n, 2 * h, 2 * w)}
        _finish_borders(prog)
        out = _run_program(prog, {"x0": x.permute(0, 3, 1, 2).contiguous()})
        want = torch.zeros(b, 2 * h, 2 * w, n, dtype=torch.float64)
        for a, bb, pk in phases:
            want[:, a::2, bb::2] = P.apply_packed_reference(pk, [x, None], (h, w))
        tol = 2e-5 if math == L.MATH_FP32 else 2e-4
        assert _rel_err(out["y0"].permute(0, 2, 3, 1).numpy(), want.numpy()) < tol
        return
    else:  # ragged: M not a multiple of 128, N not a multiple of 64, K tail of 4
        b, h, w, cin, n = 3, 7, 9, 20, 24
        pk = P.pack_conv([(rn(n, cin, 3, 3) * 0.1, 0, 0, 1)], None, rn(n), act=L.ACT_RELU)
        ins, out_hw, add = [rn(b, h, w, cin), None], (h, w), None
    prog = E.Program("conv", math)
    bufs, tvs = [], []
    feed = {}
    for i, t in enumerate(ins):
        if t is None:
            tvs.append(None); continue
        bb = prog.buf(f"in{i}", *t.shape, gemm=True, halo=True)
        prog.inputs[f"x{i}"] = (t.shape[0], t.shape[3], t.shape[1], t.shape[2])
        prog.ops.append(E.ToNHWC(f"x{i}", E.TV(bb)))
        feed[f"x{i}"] = t.permute(0, 3, 1, 2).contiguous()
        tvs.append(E.TV(bb))
    Y = prog.buf("y", ins[0].shape[0], out_hw[0], out_hw[1], pk.n_out)
    atv = None
    if add is not None:
        A = prog.buf("add", *add.shape)
        prog.inputs["xa"] = (add.shape[0], add.shape[3], add.shape[1], add.shape[2])
        prog.ops.append(E.ToNHWC("xa", E.TV(A)))
        feed["xa"] = add.permute(0, 3, 1, 2).contiguous()
        atv = E.TV(A)
    prog.ops.append(E.ConvOp(pk, tvs, E.TV(Y), addend=atv, addend_post=post))
    prog.ops.append(E.ToNCHW(E.TV(Y), "y0"))
    prog.outputs = {"y0": (ins[0].shape[0], pk.n_out, out_hw[0], out_hw[1])}
    _finish_borders(prog)
    out = _run_program(prog, feed)
    want = P.apply_packed_reference(pk, ins, out_hw, addend=add, addend_post=post)
    tol = 2e-5 if math == L.MATH_FP32 else 2e-4
    assert _rel_err(out["y0"].permute(0, 2, 3, 1).numpy(), want.numpy()) < tol



@pytest.mark.parametrize("b,h,w,cin,n,c0", [(2, 64, 64, 64, 128, 0), (3, 9, 20, 64, 40, 0), (1, 32, 32, 128, 64, 64),
                                            (2, 4, 4, 64, 64, 0)])
def test_conv_tc_writes_the_reflected_ring_of_its_output(b, h, w, cin, n, c0):
    """conv_tc.cu (TcParams::ring): a whole-plane output with a 1-pixel reflected ring gets its ring from the
    contraction's own epilogue — no ffcb_fill_reflect_border launch in the program — bit-identical to reflecting the
    interior (split-bf16 storage: the mirrored pixels are copies).  Covers a channel slice of a wider buffer, a ragged
    plane and the smallest plane the rule covers; then a 3x3 reflect contraction consumes the ring."""
    g = torch.Generator().manual_seed(b * 1000 + h)
    x = torch.randn(b, h, w, cin, generator=g)
    pk1 = P.pack_conv([(torch.randn(n, cin, 1, 1, generator=g) * 0.1, 0, 0, 0)], None, torch.randn(n, generator=g), act=L.ACT_RELU)
    pk3 = P.pack_conv([(torch.randn(64, c0 + n, 3, 3, generator=g) * 0.05, 0, 0, 1)], None, torch.randn(64, generator=g), act=L.ACT_NONE)
    prog = E.Program("conv", L.MATH_BF16X3)
    X = prog.buf("x", b, h, w, cin, gemm=True)
    Y = prog.buf("y", b, h, w, c0 + n, gemm=True, halo=True)
    Z = prog.buf("z", b, h, w, 64)
    prog.inputs["x0"] = (b, cin, h, w)
    prog.ops.append(E.ToNHWC("x0", E.TV(X)))
    if c0:
        pk0 = P.pack_conv([(torch.randn(c0, cin, 1, 1, generator=g) * 0.1, 0, 0, 0)], None, torch.randn(c0, generator=g), act=L.ACT_NONE)
        prog.ops.append(E.ConvOp(pk0, [E.TV(X), None], E.TV(Y, 0, c0)))
    prog.ops.append(E.ConvOp(pk1, [E.TV(X), None], E.TV(Y, c0, n)))
    prog.ops.append(E.ConvOp(pk3, [E.TV(Y), None], E.TV(Z)))
    prog.ops.append(E.ToNCHW(E.TV(Z), "y0"))
    prog.outputs = {"y0": (b, 64, h, w)}
    E.insert_border_ops(prog)
    assert not any(isinstance(o, E.BorderOp) for o in prog.ops), "the producing contractions own the ring"
    ex = E.CudaExecutor(prog, torch.device(DEV))
    out = ex.run({"x0": x.permute(0, 3, 1, 2).contiguous().to(DEV)})
    torch.cuda.synchronize()
    st = ex.storage[Y.name].cpu()                                   # [2][B][H+2][W+2][C] bf16 hi|lo
    inner = st[:, :, 1:-1, 1:-1].float().permute(0, 1, 4, 2, 3).reshape(-1, c0 + n, h, w)
    want_ring = torch.nn.functional.pad(inner, (1, 1, 1, 1), mode="reflect")
    got = st.float().permute(0, 1, 4, 2, 3).reshape(-1, c0 + n, h + 2, w + 2)
    assert torch.equal(got, want_ring), "ring != reflection of the interior"
    y = P.apply_packed_reference(pk1, [x, None], (h, w))
    if c0:
        y = torch.cat([P.apply_packed_reference(pk0, [x, None], (h, w)), y], dim=-1)
    want = P.apply_packed_reference(pk3, [y, None], (h, w))
    assert _rel_err(out["y0"].cpu().permute(0, 2, 3, 1).numpy(), want.numpy()) < 2e-4


# ------------------------------------------------------------------ channel-group planar FourierUnit chain (round 2)
@pytest.mark.parametrize("residual", [True, False])
@pytest.mark.parametrize("b,c,h", [(2, 8, 64), (3, 24, 64), (1, 192, 64), (3, 8, 32), (2, 40, 32)])
def test_plane_fft_pair_channel_group_planar(b, c, h, residual):
    """fft_plane_cg.cu: the 64x64 plane kernels on [C/cg][B][H][W][cg] tensors — float32 cg=4 real planes in, split
    bf16 cg=8 spectrum out (GEMM operand format); float32 cg=8 spectrum + cg=4 residual in, split bf16 cg=8 and
    float32 cg=4 real planes out.  Checker: numpy float64 (oracle/ffc_numpy.py), incl. the C2R rule on a ReLU'd
    (non-Hermitian) spectrum."""
    w = h
    wf = w // 2 + 1
    rng = np.random.default_rng(b * 100 + c)
    x = rng.standard_normal((b, c, h, w)).astype(np.float32)
    z = np.maximum(rng.standard_normal((b, 2 * c, h, wf)), 0).astype(np.float32)
    res = rng.standard_normal((b, c, h, w)).astype(np.float32)
    prog = E.Program("fft_cg", L.MATH_BF16X3)
    X = prog.buf("x", b, h, w, c, cg=4); S = prog.buf("s", b, h, wf, 2 * c, gemm=True, cg=8)
    Z = prog.buf("z", b, h, wf, 2 * c, cg=8); R = prog.buf("r", b, h, w, c, cg=4)
    O = prog.buf("o", b, h, w, c, gemm=True, cg=8) if c % 8 == 0 else None
    O32 = prog.buf("o32", b, h, w, c, cg=4)
    prog.inputs = {"x0": (b, c, h, w), "x1": (b, 2 * c, h, wf), "x2": (b, c, h, w)}
    rtv = E.TV(R) if residual else None
    prog.ops += [E.ToNHWC("x0", E.TV(X)), E.RfftOp(E.TV(X), E.TV(S)), E.ToNCHW(E.TV(S), "y0"),
                 E.ToNHWC("x1", E.TV(Z)), E.ToNHWC("x2", E.TV(R)),
                 E.IrfftOp(E.TV(Z), rtv, E.TV(O32)), E.ToNCHW(E.TV(O32), "y2")]
    prog.outputs = {"y0": (b, 2 * c, h, wf), "y2": (b, c, h, w)}
    if O is not None:
        prog.ops += [E.IrfftOp(E.TV(Z), rtv, E.TV(O)), E.ToNCHW(E.TV(O), "y1")]
        prog.outputs["y1"] = (b, c, h, w)
    out = _run_program(prog, {"x0": torch.from_numpy(x), "x1": torch.from_numpy(z), "x2": torch.from_numpy(res)})
    spec = onp.rfft2_ortho(x.astype(np.float64))
    want_s = np.stack((spec.real, spec.imag), axis=2).reshape(b, 2 * c, h, wf)
    assert _rel_err(out["y0"].numpy(), want_s) < 2e-5
    zc = z.astype(np.float64).reshape(b, c, 2, h, wf)
    want_y = onp.irfft2_explicit(zc[:, :, 0] + 1j * zc[:, :, 1], h, w) + (res if residual else 0.0)
    assert _rel_err(out["y2"].numpy(), want_y) < 2e-6
    if O is not None:
        assert _rel_err(out["y1"].numpy(), want_y) < 2e-5


def test_planar_chain_startup_check_passes():
    """engine.planar_selftest gates the default layout of the SpectralTransform chain; a failure there silently costs
    the round-2 speed-up (the process keeps the channels-last chain), so it must be a visible test failure."""
    E._PLANAR_OK.clear()
    assert E.planar_selftest(torch.device(DEV)) is True


@pytest.mark.parametrize("case", ["flat_interleaved_to_planar8", "nhwc_to_planar4", "spatial_taps_plus_interleaved",
                                  "flat_ragged_m"])
def test_conv_tc_channel_group_planar_operands(case):
    """conv_tc.cu with the FourierUnit chain's layouts: [K/8][pixel][8] ("interleaved", no-swizzle descriptor, 1-D
    bulk copies) A operands and channel-group planar float32 outputs, against the torch restatement of ffcb_conv."""
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    prog = E.Program("conv_cg", L.MATH_BF16X3)
    feed = {}

    def inp(name, t, **kw):
        bb = prog.buf(name, *t.shape, gemm=True, **kw)
        prog.inputs[name] = (t.shape[0], t.shape[3], t.shape[1], t.shape[2])
        prog.ops.append(E.ToNHWC(name, E.TV(bb)))
        feed[name] = t.permute(0, 3, 1, 2).contiguous()
        return bb
    if case == "flat_interleaved_to_planar8":        # the spectral GEMM: S (cg 8) -> Z (cg 8 float32), ReLU
        b, h, w, k, n = 2, 64, 33, 128, 192
        x0 = rn(b, h, w, k)
        pk = P.pack_conv([(rn(n, k, 1, 1) * 0.1, 0, 0, 0)], rn(n).abs() + 0.5, rn(n), act=L.ACT_RELU)
        ins, tvs = [x0, None], [E.TV(inp("x0", x0, cg=8)), None]
        Y = prog.buf("y", b, h, w, n, cg=8)
    elif case == "flat_ragged_m":                     # M = 2*5*33 = 330: a partial last tile of interleaved rows
        b, h, w, k, n = 2, 5, 33, 64, 64
        x0 = rn(b, h, w, k)
        pk = P.pack_conv([(rn(n, k, 1, 1) * 0.1, 0, 0, 0)], None, rn(n), act=L.ACT_NONE)
        ins, tvs = [x0, None], [E.TV(inp("x0", x0, cg=8)), None]
        Y = prog.buf("y", b, h, w, n, cg=8)
    elif case == "nhwc_to_planar4":                   # SpectralTransform.conv1: ring-padded NHWC slice -> T (cg 4)
        b, h, w, n = 2, 64, 64, 64
        x0 = rn(b, h, w, 192)
        pk = P.pack_conv([(rn(n, 128, 1, 1) * 0.1, 0, 64, 0)], rn(n).abs() + 0.5, rn(n), act=L.ACT_RELU)
        ins, tvs = [x0, None], [E.TV(inp("x0", x0, halo=True)), None]
        Y = prog.buf("y", b, h, w, n, cg=4)
    else:                                             # the global contraction: 3x3 taps on x_l + conv2 on u (cg 8)
        b, h, w, n = 2, 64, 64, 128
        x0, x1 = rn(b, h, w, 64), rn(b, h, w, 128)
        pk = P.pack_conv([(rn(n, 64, 3, 3) * 0.1, 0, 0, 1), (rn(n, 128, 1, 1) * 0.1, 1, 0, 0)], rn(n).abs() + 0.5, rn(n),
                         act=L.ACT_RELU)
        ins, tvs = [x0, x1], [E.TV(inp("x0", x0, halo=True)), E.TV(inp("x1", x1, cg=8))]
        Y = prog.buf("y", b, h, w, n)
    prog.ops.append(E.ConvOp(pk, tvs, E.TV(Y)))
    prog.ops.append(E.ToNCHW(E.TV(Y), "y0"))
    prog.outputs = {"y0": (Y.B, pk.n_out, Y.H, Y.W)}
    _finish_borders(prog)
    out = _run_program(prog, feed)
    want = P.apply_packed_reference(pk, ins, (Y.H, Y.W))
    assert _rel_err(out["y0"].permute(0, 2, 3, 1).numpy(), want.numpy()) < 2e-4


def _finish_borders(prog):
    """Hand-built test programs: ToNHWC does not write reflect rings, so add explicit border ops
    (production programs get their rings from the producing kernels' epilogues)."""
    E.insert_border_ops(prog)


# ------------------------------------------------------------------------------------ modules vs goldens
@pytest.mark.parametrize("name,ci,co", [("fu_c8_16x16", 8, 8), ("fu_c4to6_8x32", 4, 6), ("fu_c16_32x32", 16, 16),
                                        ("fu_c4_15x15", 4, 4), ("fu_c4_6x9", 4, 4)])
def test_fourier_unit_golden(name, ci, co, math_mode, monkeypatch):
    a, sd = load_golden(name)
    m = _load(M.FourierUnit(ci, co), sd)
    tol = TOL[math_mode]
    if not m.native_supported():
        # channel count outside the kernels' granularity (multiples of 4): the drop-in must still answer — the
        # documented torch-operator composition on the same device (never the CPU); STRICT would turn it into an error
        monkeypatch.setenv("LAMA_B200_STRICT", "0")
        tol = 1e-3           # torch's own GPU convolution (TF32 by default), as the reference would run it
    with torch.no_grad():
        y = m(torch.from_numpy(a["x"]).to(DEV)).cpu().numpy()
    assert _rel_err(y, a["y"]) < tol


def test_spectral_transform_golden(math_mode):
    a, sd = load_golden("st_16to24_8x8")
    m = _load(M.SpectralTransform(16, 24, enable_lfu=False), sd)
    with torch.no_grad():
        y = m(torch.from_numpy(a["x"]).to(DEV)).cpu().numpy()
    assert _rel_err(y, a["y"]) < TOL[math_mode]


@pytest.mark.parametrize("name,ci,co,stride,lfu", [("st_16to16_s2_16x16", 16, 16, 2, False),
                                                    ("st_32to64_s2_12x20", 32, 64, 2, False),
                                                    ("st_32to32_lfu_8x8", 32, 32, 1, True),
                                                    ("st_32to32_s2_lfu_16x16", 32, 32, 2, True)])
def test_spectral_transform_stride2_and_lfu_golden(name, ci, co, stride, lfu, math_mode):
    """SURVEY.md row f4 on the native path (LAMA_B200_STRICT=1: a torch fallback would fail the test): stride-2
    SpectralTransform (ffc.py:122-125) and LFU (ffc.py:148-157) against goldens from the unmodified reference."""
    a, sd = load_golden(name)
    m = _load(M.SpectralTransform(ci, co, stride=stride, enable_lfu=lfu), sd)
    with torch.no_grad():
        y = m(torch.from_numpy(a["x"]).to(DEV)).cpu().numpy()
    assert _rel_err(y, a["y"]) < TOL[math_mode]


def test_spectral_pos_encoding_golden(math_mode):
    a, sd = load_golden("fu_c8_pos_12x16")
    m = _load(M.FourierUnit(8, 8, spectral_pos_encoding=True), sd)
    with torch.no_grad():
        y = m(torch.from_numpy(a["x"]).to(DEV)).cpu().numpy()
    assert _rel_err(y, a["y"]) < TOL[math_mode]
    a, sd = load_golden("st_16to32_pos_8x8")
    m = _load(M.SpectralTransform(16, 32, enable_lfu=False, spectral_pos_encoding=True), sd)
    with torch.no_grad():
        y = m(torch.from_numpy(a["x"]).to(DEV)).cpu().numpy()
    assert _rel_err(y, a["y"]) < TOL[math_mode]


def test_ffc_bn_act_stride2_global_lfu_and_resblock_lfu_golden(math_mode):
    a, sd = load_golden("ffcbnact_64_s2_lfu_16x16")
    m = _load(M.FFC_BN_ACT(in_channels=64, out_channels=64, kernel_size=3, ratio_gin=0.5, ratio_gout=0.5, stride=2,
                           padding=1, activation_layer=torch.nn.ReLU, enable_lfu=True), sd)
    with torch.no_grad():
        yl, yg = m((torch.from_numpy(a["x_l"]).to(DEV), torch.from_numpy(a["x_g"]).to(DEV)))
    assert _rel_err(yl.cpu().numpy(), a["y_l"]) < TOL[math_mode] and _rel_err(yg.cpu().numpy(), a["y_g"]) < TOL[math_mode]
    a, sd = load_golden("resblock_64_lfu_8x8")
    m = _load(M.FFCResnetBlock(64, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                               activation_layer=torch.nn.ReLU, ratio_gin=0.5, ratio_gout=0.5, enable_lfu=True), sd)
    with torch.no_grad():
        yl, yg = m((torch.from_numpy(a["x_l"]).to(DEV), torch.from_numpy(a["x_g"]).to(DEV)))
    assert _rel_err(yl.cpu().numpy(), a["y_l"]) < TOL[math_mode] and _rel_err(yg.cpu().numpy(), a["y_g"]) < TOL[math_mode]


def test_lfu_on_the_planar_chain_at_the_bottleneck_size(tc_math):
    """LFU inside the channel-group planar chain: 64x64 planes -> 32x32 quadrant planes (both register-transform
    sizes of fft_plane_cg.cu), c = 64; checker: the torch-CPU oracle port."""
    torch.manual_seed(5)
    m = seeded_parameters_(M.SpectralTransform(128, 128, enable_lfu=True).eval(), 5)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(2, 128, 64, 64, generator=torch.Generator().manual_seed(6))
    with torch.no_grad():
        y = m.to(DEV)(x.to(DEV)).cpu()
        ref = otc.spectral_transform(x, sd, enable_lfu=True)
    assert _rel_err(y.numpy(), ref.numpy()) < TOL["bf16x3"]


@pytest.mark.parametrize("name,kw,has_g", [
    ("ffcbnact_32_k3_075", dict(in_channels=32, out_channels=32, kernel_size=3, ratio_gin=0.75, ratio_gout=0.75,
                                padding=1), True),
    ("ffcbnact_4to8_k7_local", dict(in_channels=4, out_channels=8, kernel_size=7, ratio_gin=0, ratio_gout=0,
                                    padding=0), False),
    ("ffcbnact_16to32_s2_to_global", dict(in_channels=16, out_channels=32, kernel_size=3, ratio_gin=0,
                                          ratio_gout=0.75, stride=2, padding=1), False),
])
def test_ffc_bn_act_golden(name, kw, has_g, math_mode):
    a, sd = load_golden(name)
    m = _load(M.FFC_BN_ACT(activation_layer=torch.nn.ReLU, enable_lfu=False, **kw), sd)
    xl = torch.from_numpy(a["x_l"]).to(DEV)
    xg = torch.from_numpy(a["x_g"]).to(DEV) if has_g else 0
    with torch.no_grad():
        yl, yg = m((xl, xg))
    assert _rel_err(yl.cpu().numpy(), a["y_l"]) < TOL[math_mode]
    if "y_g" in a:
        assert _rel_err(yg.cpu().numpy(), a["y_g"]) < TOL[math_mode]
    else:
        assert yg == 0


def test_resnet_block_golden(math_mode):
    a, sd = load_golden("resblock_32_16x16")
    m = _load(M.FFCResnetBlock(32, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                               activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75, enable_lfu=False), sd)
    with torch.no_grad():
        yl, yg = m((torch.from_numpy(a["x_l"]).to(DEV), torch.from_numpy(a["x_g"]).to(DEV)))
    assert _rel_err(yl.cpu().numpy(), a["y_l"]) < TOL[math_mode] and _rel_err(yg.cpu().numpy(), a["y_g"]) < TOL[math_mode]


@pytest.mark.parametrize("name", ["generator_ngf8_b2_64x64", "generator_ngf8_b2_40x72"])
def test_small_generator_golden(name, math_mode):
    a, _ = load_golden(name)
    _, sd = load_golden("generator_ngf8_b2_64x64")
    g = _load(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)), sd)
    with torch.no_grad():
        y = g(torch.from_numpy(a["x"]).to(DEV)).cpu().numpy()
    assert float(np.abs(y - a["y"]).max()) < (5e-6 if math_mode == "fp32" else 1e-4)


def test_generator_with_out_ffc_golden(math_mode):
    a, sd = load_golden("generator_ngf16_outffc_32x32")
    kw = small_lama_kwargs(ngf=16, n_blocks=1, n_downsampling=2)
    kw.update(out_ffc=True, out_ffc_kwargs=dict(ratio_gin=0.5, ratio_gout=0.5, enable_lfu=False))
    g = _load(M.FFCResNetGenerator(**kw), sd)
    with torch.no_grad():
        y = g(torch.from_numpy(a["x"]).to(DEV)).cpu().numpy()
    assert float(np.abs(y - a["y"]).max()) < (5e-6 if math_mode == "fp32" else 1e-4)


def test_generator_with_the_constructor_default_tanh_head(math_mode):
    """add_out_act=True (the constructor default, ffc.py:362) ends the generator with tanh: precise tanhf in the head
    epilogue (the library is built without --use_fast_math), both head implementations."""
    kw = small_lama_kwargs(ngf=8, n_blocks=1)
    kw["add_out_act"] = True
    g = seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 9, gain=1.0)
    sd = {k: v.clone() for k, v in g.state_dict().items()}
    img, mask = synthetic_image_mask(2, 64, 9)
    x = generator_input(img, mask)
    with torch.no_grad():
        y = g.to(DEV)(x.to(DEV)).cpu()
        ref = otc.ffc_resnet_generator(x, sd, **kw)
    assert float(ref.min()) < -0.05, "tanh head should produce negative values on this input"
    assert float((y - ref).abs().max()) < (5e-6 if math_mode == "fp32" else 1e-4)


def test_to_jit_trace_on_cuda_keeps_the_native_kernels(tc_math, tmp_path):
    """bin/to_jit.py:49-72 on a CUDA box: the traced + saved + reloaded model must still run libffc_b200.so — the
    generator is ONE ``lama_b200::ffc_generator`` node (lama_b200/ops.py), its weights travel inside the file."""
    import lama_b200.ops  # noqa: F401  (registers the op; a fresh process loading the file does the same)

    class JITWrapper(torch.nn.Module):            # to_jit.py:14-25 + trainers/default.py:59-71
        def __init__(self, generator):
            super().__init__()
            self.generator = generator

        def forward(self, image, mask):
            masked = torch.cat([image * (1 - mask), mask], dim=1)
            return mask * self.generator(masked) + (1 - mask) * image

    g = seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)).eval(), seed=1).to(DEV)
    w = JITWrapper(g).eval()
    gen = torch.Generator().manual_seed(0)
    image = torch.rand(1, 3, 120, 120, generator=gen).to(DEV)
    mask = (torch.rand(1, 1, 120, 120, generator=gen) > 0.7).float().to(DEV)
    L.get_lib().ffcb_reset_launch_count()
    with torch.no_grad():
        eager = w(image, mask)
        assert L.get_lib().ffcb_launch_count() > 0
        traced = torch.jit.trace(w, (image, mask), strict=False)
    assert "lama_b200::ffc_generator" in str(traced.inlined_graph)
    path = str(tmp_path / "lama.pt")
    traced.save(path)
    loaded = torch.jit.load(path)
    L.get_lib().ffcb_reset_launch_count()
    with torch.no_grad():
        out = loaded(image, mask)
        out2 = loaded(image.flip(-1).contiguous(), mask.flip(-1).contiguous())     # not a baked-in constant
        want2 = w(image.flip(-1).contiguous(), mask.flip(-1).contiguous())
    assert L.get_lib().ffcb_launch_count() > 0, "the reloaded TorchScript did not launch the native kernels"
    assert torch.equal(out, eager) and torch.equal(out2, want2)


@pytest.mark.parametrize("shape", [(2, 128, 384, 32, 32), (1, 128, 384, 64, 64), (1, 32, 96, 12, 20)])
def test_resnet_block_input_gradients_vs_autograd_oracle(shape, math_mode):
    """SURVEY.md row f3 groundwork: dL/dx_l, dL/dx_g through a native FFCResnetBlock (torch.autograd.Function around
    the forward+backward program) vs autograd through the torch-CPU oracle port; 1e-4 (fp32 arm) / 5e-4 (split-bf16
    operands in both directions) of the gradient's range on all but the few elements behind a flipped ReLU mask.  Shapes: the verdict's (2, 128+384, 32, 32) — planar 32x32 chain —, the
    64x64 bottleneck, and a small non-power-of-two plane on the general FFT kernels.  Wider planes (128x128, 96x128,
    256x256, up to engine.BLOCK_GRAD_MAX_PLANE): tests/test_gpu_program_diff.py."""
    b, cl, cg, h, w = shape
    blk = seeded_parameters_(M.FFCResnetBlock(cl + cg, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                              activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                              enable_lfu=False).eval(), 4, gain=1.0)
    sd = {k: v.clone() for k, v in blk.state_dict().items()}
    for p_ in blk.parameters():
        p_.requires_grad_(False)                              # model.freeze() (bin/predict.py:59)
    blk = blk.to(DEV)
    g = torch.Generator().manual_seed(2)
    xl, xg = torch.randn(b, cl, h, w, generator=g), torch.randn(b, cg, h, w, generator=g)
    gl, gg = torch.randn(b, cl, h, w, generator=g), torch.randn(b, cg, h, w, generator=g)
    a_l, a_g = xl.to(DEV).requires_grad_(True), xg.to(DEV).requires_grad_(True)
    L.get_lib().ffcb_reset_launch_count()
    o_l, o_g = blk((a_l, a_g))
    ((o_l * gl.to(DEV)).sum() + (o_g * gg.to(DEV)).sum()).backward()
    assert L.get_lib().ffcb_launch_count() > 10, "the native forward program did not run"   # (the counter is per thread: backward launches from autograd's thread)
    r_l, r_g = xl.clone().requires_grad_(True), xg.clone().requires_grad_(True)
    q_l, q_g = otc.ffc_resnet_block(r_l, r_g, sd, "", ratio_gout=0.75)
    ((q_l * gl).sum() + (q_g * gg).sum()).backward()
    tol = 1e-4 if math_mode == "fp32" else 5e-4
    assert _rel_err(o_l.detach().cpu().numpy(), q_l.detach().numpy()) < TOL[math_mode]
    # ReLU backward multiplies by [y > 0]: an activation within round-off of zero can land on the other side in the two
    # implementations (different summation order), which changes the gradient by O(1) around that element.  Such
    # flips are a handful per million activations, so: the bulk of the elements must agree to `tol`, and the error in
    # the 2-norm must be small.
    for got, want in ((a_l.grad.cpu(), r_l.grad), (a_g.grad.cpu(), r_g.grad)):
        d = (got.double() - want.double()).abs()
        scale = float(want.abs().max())
        # (a flipped mask in the SPECTRUM spreads over its whole plane through the inverse transform: allow a few planes)
        # (measured: 4-8% of the elements beyond tol on the split-bf16 arm at 32x32 / 64x64 — every flipped spectral
        #  mask moves a whole plane of dL/dt and, through conv1's transpose, all of dL/dx_g a little; a wrong
        #  gradient would put ~all elements off and the 2-norm error at O(1))
        assert float((d > tol * scale).double().mean()) < 0.25, "too many elements off"
        # (64x64 planes: ~1.6 M spectral activations per block -> a few flipped spectral masks, each one moving every
        #  element of dL/dx_g by ~5e-5 of its rms; measured median 2.7e-5 of the range on the fp32 arm)
        assert float(d.median()) < tol * scale
        assert float(d.pow(2).sum().sqrt() / want.double().pow(2).sum().sqrt()) < 20 * tol


def test_refinement_with_native_block_gradients_matches_torch_autograd(tc_math, monkeypatch):
    """lama_b200.refine.refine_predict (evaluation/refinement.py:228-314 without kornia) on the GPU: residual blocks run
    the native forward + input-gradient programs; the same loop with the blocks on torch autograd (cuFFT / cuDNN) must
    give the same refined image up to the arithmetic (3 Adam steps at lr 2e-3 amplify 1e-4 gradient differences)."""
    from lama_b200 import refine as R
    g = seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=16, n_blocks=3)).eval(), 2, gain=1.0).to(DEV)
    gen = torch.Generator().manual_seed(0)
    img = torch.rand(1, 3, 136, 200, generator=gen)
    mask = torch.zeros(1, 1, 136, 200); mask[..., 30:90, 50:150] = 1
    kw = dict(modulo=8, n_iters=4, lr=0.002, min_side=64, max_scales=2, px_budget=10 ** 7)
    lib = L.get_lib()
    lib.ffcb_reset_launch_count()
    native = R.refine_predict(img, mask, g, **kw)
    assert lib.ffcb_launch_count() > 100, "native programs did not run inside the refinement loop"
    monkeypatch.setenv("LAMA_B200_NATIVE_GRAD", "0")
    monkeypatch.setenv("LAMA_B200_STRICT", "0")                  # blocks under autograd -> torch composition
    ref = R.refine_predict(img, mask, g, **kw)
    assert torch.isfinite(native).all()
    assert float((native - ref).abs().max()) < 5e-3
    assert float((native - ref).abs().mean()) < 2e-4


def test_stage_by_stage_matches_whole_program():
    """predict_inner_features.py:84 iterates generator.model stage by stage: tuple outputs at every FFC
    stage, each stage on its own native program, same result as the fused whole-generator program."""
    a, sd = load_golden("generator_ngf8_b2_64x64")
    g = _load(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)), sd)
    os.environ["LAMA_B200_STRICT"] = "0"     # ReflectionPad2d / ConvTranspose2d stages are plain torch modules
    try:
        with torch.no_grad():
            h = torch.from_numpy(a["x"]).to(DEV)
            for i, stage in enumerate(g.model):
                h = stage(h)
                if 1 <= i <= 6:
                    assert isinstance(h, tuple)
    finally:
        os.environ["LAMA_B200_STRICT"] = "1"
    assert float(np.abs(h.cpu().numpy() - a["y"]).max()) < 1e-3   # ConvTranspose stages run cuDNN (TF32 allowed)


# ------------------------------------------------------------------------------------ big-lama vs oracle
def _big_lama(seed=0):
    torch.manual_seed(seed)
    g = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), seed)
    sd_cpu = {k: v.clone() for k, v in g.state_dict().items()}
    return g.to(DEV), sd_cpu


@pytest.mark.parametrize("size,batch,seed", [(256, 2, 0), (512, 1, 1), ((384, 640), 1, 2), (1024, 1, 3), (2048, 1, 4)])
def test_big_lama_generator_vs_oracle(size, batch, seed, math_mode):
    """The shipped architecture (configs/training/big-lama.yaml:26-45), seeded weights, vs the torch-CPU
    oracle port (fp32) on identical (image, mask): north_star tolerance 1e-3 max-abs."""
    g, sd = _big_lama(seed)
    # (384, 640): 48 x 80 bottleneck planes -> direct-DFT kernels and partially filled / clipped TMA tiles;
    # 1024: 128 x 128 planes, 128-pixel-wide tiles, stride-2 boxes at the 256-element TMA limit;
    # 2048 (BASELINE config 5 resolution, plain inference): 256 x 256 planes -> 1024-thread FFT CTAs, 128 KB smem
    h, w = (size, size) if isinstance(size, int) else size
    img, mask = synthetic_image_mask(batch, h, seed, width=w)
    x = generator_input(img, mask)
    with torch.no_grad():
        y = g(x.to(DEV)).cpu()
        ref = otc.ffc_resnet_generator(x, sd, **BIG_LAMA_KWARGS)
    err = float((y - ref).abs().max())
    assert ref.std() > 0.05, "degenerate (saturated) reference output"
    assert err < 1e-3, f"north_star tolerance violated: {err:.3e}"
    tight = 5e-5 if math_mode == "fp32" else 3e-4
    assert err < tight, f"{math_mode} arithmetic should be well inside the tolerance: {err:.3e}"


def test_big_lama_bs32_512_batch_independence_and_spot_oracle():
    """BASELINE config 3 (bs32, 512x512): (a) size-independent property — no cross-sample coupling
    (eval BN, per-plane FFT): images of the batch of 32 equal the same images run as a batch of 2,
    bit for bit; (b) eight seeded picks of the batch checked against the oracle (the CPU oracle needs ~0.5 s per
    image; the other 24 are covered by (a) + the per-image independence it proves)."""
    g, sd = _big_lama(0)
    img, mask = synthetic_image_mask(32, 512, 3)
    x = generator_input(img, mask)
    pick = sorted(torch.randperm(32, generator=torch.Generator().manual_seed(11))[:8].tolist())
    with torch.no_grad():
        y32 = g(x.to(DEV)).cpu()
        y2 = torch.cat([g(x[pick[i:i + 2]].contiguous().to(DEV)).cpu() for i in range(0, 8, 2)])
        ref = otc.ffc_resnet_generator(x[pick], sd, **BIG_LAMA_KWARGS)
    assert torch.equal(y32[pick], y2), "batch coupling: results depend on batch composition"
    assert torch.isfinite(y32).all() and float(y32.min()) >= 0.0 and float(y32.max()) <= 1.0
    err = float((y32[pick] - ref).abs().max())
    assert err < 3e-4, f"bs32 512x512 vs oracle on 8 images: {err:.3e}"


def test_inpaint_glue_matches_oracle(math_mode):
    """default.py:59-71 around the generator: mask*pred + (1-mask)*img — known pixels are passed through exactly."""
    a, sd = load_golden("generator_ngf8_b2_64x64")
    g = _load(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)), sd)
    img, mask = torch.from_numpy(a["image"]).to(DEV), torch.from_numpy(a["mask"]).to(DEV)
    with torch.no_grad():
        pred = g(torch.cat([img * (1 - mask), mask], dim=1))
    inp = mask * pred + (1 - mask) * img
    _, want = onp.inpaint_forward(a["image"].astype(np.float64), a["mask"].astype(np.float64),
                                  {k: v.astype(np.float64) for k, v in sd.items()}, **small_lama_kwargs(8, 2))
    assert float(np.abs(inp.cpu().numpy() - want).max()) < (5e-6 if math_mode == "fp32" else 1e-4)
    assert torch.equal(inp[(1 - mask).expand_as(inp).bool()], img[(1 - mask).expand_as(img).bool()])


def test_errors_are_loud():
    lib = L.get_lib()
    d = L.ConvDesc()
    with pytest.raises(ValueError):
        L.check(lib.ffcb_conv(d, None), "ffcb_conv")
    assert b"conv" in lib.ffcb_last_error()
    with pytest.raises(ValueError):   # n_out not a multiple of 4
        t = torch.zeros(1, 4, 4, 8, device=DEV)
        d.inp[0] = L.Tensor(t.data_ptr(), 128, 32, 8, 0, 1, 4, 4, 8, 0, 0, 0, 0)
        d.out = L.Tensor(t.data_ptr(), 128, 32, 8, 0, 1, 4, 4, 6, 0, 0, 0, 0)
        d.n_out, d.nseg, d.stride, d.weight = 6, 1, 1, t.data_ptr()
        L.check(lib.ffcb_conv(d, None), "ffcb_conv")


def test_serving_pipeline_matches_module_call(math_mode):
    """lama_b200.serving.GeneratorPipeline (overlapped H2D / graph replay / D2H) returns exactly what the
    module call returns, for several in-flight batches and slot reuse."""
    from lama_b200.serving import GeneratorPipeline
    a, sd = load_golden("generator_ngf8_b2_64x64")
    g = _load(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)), sd)
    pipe = GeneratorPipeline(g, 2, 64, 64, depth=2)
    xs = [torch.from_numpy(a["x"]).roll(i, dims=0).contiguous().pin_memory() for i in range(5)]
    with torch.no_grad():
        want = [g(x.to(DEV)).cpu() for x in xs]
    tickets = []
    got = []
    for i, x in enumerate(xs):
        tickets.append(pipe.submit(x))
        if i >= 1:
            got.append(pipe.result(tickets[i - 1]).clone())
    got.append(pipe.result(tickets[-1]).clone())
    for w, y in zip(want, got):
        assert torch.equal(w, y)


def test_baseline_config0_single_fourier_unit(math_mode):
    """BASELINE.json configs[0]: single FourierUnit(64, 64) forward on 1x64x256x256 fp32, seeded weights,
    vs the float64 numpy oracle (256x256 planes: 1024-thread two-pass FFT kernels, 128-channel spectral GEMM)."""
    m = seeded_parameters_(M.FourierUnit(64, 64).eval(), 11, gain=1.0)
    sd = {k: v.numpy().astype(np.float64) for k, v in m.state_dict().items() if not k.endswith("num_batches_tracked")}
    x = torch.randn(1, 64, 256, 256, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        y = m.to(DEV)(x.to(DEV)).cpu().numpy()
    want = onp.fourier_unit(x.numpy().astype(np.float64), sd)
    assert _rel_err(y, want) < TOL[math_mode]


def test_baseline_config1_resnet_block_bs8(math_mode):
    """BASELINE.json configs[1]: FFCResnetBlock(512, ratio 0.75/0.75) forward, bs8 at the 512x512 image resolution
    (x_l 8x128x64x64, x_g 8x384x64x64), vs the torch-CPU oracle port."""
    blk = seeded_parameters_(M.FFCResnetBlock(512, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                              activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                              enable_lfu=False).eval(), 12)
    sd = {k: v.clone() for k, v in blk.state_dict().items()}
    g = torch.Generator().manual_seed(1)
    xl, xg = torch.randn(8, 128, 64, 64, generator=g), torch.randn(8, 384, 64, 64, generator=g)
    with torch.no_grad():
        yl, yg = blk.to(DEV)((xl.to(DEV), xg.to(DEV)))
        rl, rg = otc.ffc_resnet_block(xl, xg, sd, "")
    assert _rel_err(yl.cpu().numpy(), rl.numpy()) < TOL[math_mode]
    assert _rel_err(yg.cpu().numpy(), rg.numpy()) < TOL[math_mode]


# ------------------------------------------------------------------- predict path, uint8 I/O (SURVEY.md row f1)


def test_predict_u8_bytes_match_reference_fixture(tc_math):
    """lama_b200.predict.BatchedInpainter (decode-to-bytes fused path) against the bytes the reference pipeline
    produced (tests/golden/predict_ngf8_3x45x52.npz: InpaintingDataset + generator + blend + x255/uint8).
    45x52 images: symmetric padding to 48x56, 6x7 non-power-of-two FFT planes, a full and a partial batch."""
    from lama_b200.predict import BatchedInpainter
    a, _ = load_golden("predict_ngf8_3x45x52")
    _, sd = load_golden("generator_ngf8_b2_64x64")
    g = _load(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)), sd)
    inp = BatchedInpainter(g, max_batch=2)
    outs = np.stack(inp.inpaint(list(zip(a["images"], a["masks"]))))
    hole = a["masks"] > 0
    assert outs.dtype == np.uint8 and outs.shape == a["out"].shape
    assert np.array_equal(outs[~hole], a["out"][~hole])            # bit-exact where the input shows through
    d = np.abs(outs[hole].astype(int) - a["out"][hole].astype(int))
    # prediction error ~3e-5 -> 0.008 grey levels: a truncation boundary is crossed for <~1% of the bytes
    assert d.max() <= 1 and (d != 0).mean() < 0.05, (int(d.max()), float((d != 0).mean()))


@pytest.mark.parametrize("h0,w0,b", [(100, 75, 2), (64, 64, 3)])
def test_predict_u8_equals_float_program_plus_reference_glue(tc_math, h0, w0, b):
    """The fused byte path and the float program share every kernel in between, so the bytes must be IDENTICAL to
    the reference's elementwise glue (oracle/predict_numpy.py) wrapped around the native float generator call."""
    from lama_b200.predict import BatchedInpainter
    from oracle import predict_numpy as opn
    _, sd = load_golden("generator_ngf8_b2_64x64")
    g = _load(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)), sd)
    rng = np.random.default_rng(h0 * 1000 + w0)
    images = rng.integers(0, 256, size=(b, h0, w0, 3), dtype=np.uint8)
    masks = (rng.random((b, h0, w0)) < 0.3).astype(np.uint8) * rng.integers(1, 256, size=(b, h0, w0), dtype=np.uint8)
    masks[:, h0 // 2:, w0 // 2:] = 255                              # a solid hole reaching the padded corner
    x, img, mask = opn.generator_input(images, masks, pad_mod=8)
    with torch.no_grad():
        pred = g(torch.from_numpy(x).to(DEV)).cpu().numpy()
    want = opn.finish(pred, img, mask, h0, w0)
    got = BatchedInpainter(g, max_batch=b)(images, masks)
    assert np.array_equal(got, want)
    # several batches in flight through the same lane (slot and staging-buffer reuse)
    many = [(np.roll(images[i % b], i, axis=1), np.roll(masks[i % b], i, axis=1)) for i in range(4 * b)]
    outs = BatchedInpainter(g, max_batch=b).inpaint(many)
    for i in (0, b + 1, 4 * b - 1):
        xi, ii, mi = opn.generator_input(many[i][0][None], many[i][1][None], pad_mod=8)
        with torch.no_grad():
            pi = g(torch.from_numpy(xi).to(DEV)).cpu().numpy()
        assert np.array_equal(outs[i], opn.finish(pi, ii, mi, h0, w0)[0])


def test_predict_u8_abi_rejects_bad_arguments():
    lib = L.get_lib()
    t = torch.zeros(2, 1, 22, 24, 8, dtype=torch.bfloat16, device=DEV)          # packed view for a 16x16 image
    pk = L.Tensor(t.data_ptr(), 22 * 24 * 8, 24 * 8, 8, 22 * 24 * 8, 1, 22, 24, 8, L.BF16X2, 0, 0, 0)
    img = torch.zeros(1, 7, 16, 3, dtype=torch.uint8, device=DEV)
    msk = torch.zeros(1, 7, 16, dtype=torch.uint8, device=DEV)
    import ctypes as C
    # 7 rows cannot be symmetric-padded to 16 (needs H - H0 <= H0)
    assert lib.ffcb_stem_pack_u8(img.data_ptr(), msk.data_ptr(), 1, 7, 16, C.byref(pk), None) == L.EINVAL
    assert b"symmetric" in lib.ffcb_last_error()
    assert lib.ffcb_stem_pack_u8(None, msk.data_ptr(), 1, 16, 16, C.byref(pk), None) == L.EINVAL
    q = torch.zeros(1, 16, 16, 24, device=DEV)
    qt = L.Tensor(q.data_ptr(), 16 * 16 * 24, 16 * 24, 24, 0, 1, 16, 16, 24, L.F32, 0, 0, 0)
    out = torch.zeros(1, 16, 16, 3, dtype=torch.uint8, device=DEV)
    assert lib.ffcb_head_gather7_blend_u8(C.byref(qt), None, L.ACT_SIGMOID, img.data_ptr(), msk.data_ptr(), 17, 16,
                                          out.data_ptr(), None) == L.EINVAL
