"""GPU tests of rectangular bottleneck planes (H != W, ``pytest -m gpu``): the FFT pair, the generator forward, the
native block gradients and the rear program at planes whose two axes take different plans — 64x128 (two compile-time
radix plans), 96x1024 and 1024x96 (a 32-channel runtime plan on one axis, an 8-channel one on the other), 127x256 (a
single radix-127 pass: primes below 129 never take Bluestein), 1000x1024 (8-channel runtime plans on both axes) and
1x1024 (one row: the column transform is the identity).  Checkers: torch.fft in float64, and float64 autograd through
the oracle composition (oracle/ffc_torch_cpu.py, run on the GPU in float64).

A plane with a 1-point side has no generator or block test: the reflect padding of the 3x3 convolutions needs two
pixels per side, so neither the reference nor the native path takes it (tests/test_rect_planes_cpu.py checks that the
native gates refuse it).  The model is not transposition-equivariant even in the reference (the real FFT halves the
last axis, and the spectral ReLU does not commute with the Hermitian extension), so a W x H input is checked against the
reference at W x H, not against the transposed H x W result."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200.ops import traced_generator_call      # noqa: E402
from lama_b200.predict import BatchedInpainter       # noqa: E402
from lama_b200.serving import GeneratorPipeline      # noqa: E402
from lama_b200.testing import generator_input, seeded_parameters_, small_lama_kwargs, synthetic_image_mask  # noqa: E402
from oracle import ffc_torch_cpu as otc              # noqa: E402
from oracle import predict_numpy as opn              # noqa: E402
from test_gpu_large_planes import _fft_program       # noqa: E402
from test_gpu_refine_large_planes import _bulk_close, _rel2  # noqa: E402

DEV = "cuda:0"
PLANES = [(64, 128), (96, 1024), (1024, 96), (127, 256), (1000, 1024)]
FFT_PLANES = PLANES + [(1, 1024)]


@pytest.fixture(autouse=True)
def _strict_env():
    os.environ["LAMA_B200_STRICT"] = "1"
    yield
    os.environ.pop("LAMA_B200_STRICT", None)


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
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).abs().max()) / (float(ref.abs().max()) or 1.0)


# ------------------------------------------------------------------------------------ FFT pair
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("h,w", FFT_PLANES)
def test_fft_pair_against_torch_fft(h, w, split):
    """ffcb_rfft2 / ffcb_irfft2 vs torch.fft.rfft2 / irfft2 in float64: the forward spectrum, and the inverse of a
    ReLU'd (non-Hermitian) spectrum plus the residual, within the bounds of the square-plane tests (2e-6 of max |ref|
    in fp32, 2e-5 in split bf16).  Two launches per direction: the two-pass kernels, one per axis."""
    b, c = 1, 8
    wf = w // 2 + 1
    g = torch.Generator().manual_seed(h * 1000 + w)
    x = torch.randn(b, c, h, w, generator=g)
    z = torch.relu(torch.randn(b, 2 * c, h, wf, generator=g))
    res = torch.randn(b, c, h, w, generator=g)
    ex = E.CudaExecutor(_fft_program(b, c, h, w, split, 0), torch.device(DEV))
    out = ex.run({"x0": x.to(DEV), "x1": z.to(DEV), "x2": res.to(DEV)})
    spec = torch.fft.rfft2(x.double(), norm="ortho")
    want_s = torch.stack((spec.real, spec.imag), dim=2).reshape(b, 2 * c, h, wf)
    zc = z.double().reshape(b, c, 2, h, wf)
    want_y = torch.fft.irfft2(torch.complex(zc[:, :, 0], zc[:, :, 1]), s=(h, w), norm="ortho") + res.double()
    ef, ei = _rel_err(out["y0"], want_s), _rel_err(out["y1"], want_y)
    print(f"fft {h}x{w} {'split' if split else 'fp32'}: fwd {ef:.2e} inv {ei:.2e}")
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


# ------------------------------------------------------------------------------------ inference
# ngf 32: every channel count a multiple of 8, so the split-bf16 arm runs the tensor-core programs (and the uint8
# predict program exists)
_KW = small_lama_kwargs(ngf=32, n_blocks=1, n_downsampling=1)


def _generator(seed):
    return seeded_parameters_(M.FFCResNetGenerator(**_KW).eval(), seed, gain=1.0)


@pytest.mark.parametrize("h,w", PLANES)
def test_generator_against_the_torch_fft_reference(h, w, math_mode):
    """A generator with one down-sampling stage on a (2h)x(2w) image, so its residual block runs on the h x w plane,
    against the reference's operator sequence (torch.fft, float64) with the bound of the other small-generator tests.
    LAMA_B200_STRICT=1: a fall-back to the torch composition would raise."""
    g = _generator(3)
    sd = {k: v.double().to(DEV) for k, v in g.state_dict().items()}
    img, mask = synthetic_image_mask(1, 2 * h, h + w, width=2 * w)
    x = generator_input(img, mask).to(DEV)
    g = g.to(DEV)
    assert E.generator_supported(g, x)
    L.get_lib().ffcb_reset_launch_count()
    with torch.no_grad():
        y = g(x)
        assert L.get_lib().ffcb_launch_count() > 0, "the native program did not run"
        ref = otc.ffc_resnet_generator(x.double(), sd, **_KW)
    E.invalidate(g)
    err = float((y.double() - ref).abs().max())
    print(f"generator {2 * h}x{2 * w} ({math_mode}): max-abs {err:.2e}")
    assert ref.std() > 0.05 and err < 3e-4, err


@pytest.mark.parametrize("h,w", PLANES)
def test_predict_driver_against_the_reference_glue(h, w):
    """Two (2h)x(2w) uint8 images through BatchedInpainter (the generator_u8 program lama_b200.predict runs; pad_mod 2
    keeps the h x w plane) against the reference predict glue around the oracle generator in float64: exact outside
    the hole, within one grey level inside it, as at 4K-class sizes."""
    os.environ["LAMA_B200_MATH"] = "bf16x3"
    try:
        g = _generator(5)
        sd = {k: v.double().to(DEV) for k, v in g.state_dict().items()}
        g = g.to(DEV)
        h0, w0 = 2 * h, 2 * w
        rng = np.random.default_rng(h + w)
        images = rng.integers(0, 256, size=(2, h0, w0, 3), dtype=np.uint8)
        masks = np.zeros((2, h0, w0), np.uint8)
        masks[0, h0 // 4:h0 // 2 + 1, w0 // 3:w0 // 2 + 1] = 255
        masks[1, h0 // 2:, w0 // 2:] = 17                       # a hole reaching the corner
        got = np.stack(BatchedInpainter(g, max_batch=2, pad_mod=2).inpaint(list(zip(images, masks))))
        E.invalidate(g)
        x, img, mask = opn.generator_input(images, masks, pad_mod=2)
        with torch.no_grad():
            pred = otc.ffc_resnet_generator(torch.from_numpy(x).double().to(DEV), sd, **_KW).float().cpu().numpy()
        want = opn.finish(pred, img, mask, h0, w0)
        hole = masks > 0
        assert np.array_equal(got[~hole], want[~hole])
        d = np.abs(got[hole].astype(int) - want[hole].astype(int))
        print(f"predict {h0}x{w0}: max {int(d.max())}, differing {float((d != 0).mean()):.2e}")
        assert d.max() <= 1 and (d != 0).mean() < 0.05
    finally:
        os.environ.pop("LAMA_B200_MATH", None)


def test_out_of_range_planes_are_refused_naming_both_sides():
    """A 2x2050 image has a 1x1025 bottleneck: refused (as a 1025-wide or a 1-high plane is) by the predict pipeline
    (ValueError) and the traced generator op (RuntimeError), with a message that names the input's sides."""
    g = _generator(3).to(DEV)
    with pytest.raises(ValueError, match="2x2050"):
        GeneratorPipeline(g, 1, 2, 2050)
    with pytest.raises(ValueError, match="2056x96"):
        GeneratorPipeline(g, 1, 2056, 96, u8=True, pad_mod=8)
    with torch.no_grad(), pytest.raises(RuntimeError, match="2x2050"):
        traced_generator_call(g, torch.zeros(1, 4, 2, 2050, device=DEV))


# ------------------------------------------------------------------------------------ refinement
def _block():
    blk = seeded_parameters_(M.FFCResnetBlock(64, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                              activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                              enable_lfu=False).eval(), 4, gain=1.0)
    for p_ in blk.parameters():
        p_.requires_grad_(False)
    return blk


@pytest.mark.parametrize("h,w", PLANES)
def test_block_input_gradients(h, w, math_mode):
    """FFCResnetBlock (16 local + 48 global channels): the native forward + input-gradient program against float64
    autograd through the oracle, with the bounds of the block-gradient tests on large planes."""
    blk = _block()
    sd = {k: v.double().to(DEV) for k, v in blk.state_dict().items()}
    blk = blk.to(DEV)
    gen = torch.Generator().manual_seed(h + w)
    xl, xg, gl, gg = (torch.randn(1, ch, h, w, generator=gen).to(DEV) for ch in (16, 48, 16, 48))
    a_l, a_g = xl.clone().requires_grad_(True), xg.clone().requires_grad_(True)
    L.get_lib().ffcb_reset_launch_count()
    o_l, o_g = blk((a_l, a_g))
    assert L.get_lib().ffcb_launch_count() > 10, "the native forward+backward program did not run"
    ((o_l * gl).sum() + (o_g * gg).sum()).backward()
    r_l, r_g = xl.double().requires_grad_(True), xg.double().requires_grad_(True)
    q_l, q_g = otc.ffc_resnet_block(r_l, r_g, sd, "", ratio_gout=0.75)
    ((q_l * gl.double()).sum() + (q_g * gg.double()).sum()).backward()
    fl, fg = _rel2(o_l.detach(), q_l.detach()), _rel2(o_g.detach(), q_g.detach())
    print(f"\n  {h}x{w} ({math_mode}): forward 2-norm {fl:.2e} / {fg:.2e}")
    assert fl < 5e-5 and fg < 5e-5
    tol = 1e-4 if math_mode == "fp32" else 5e-4
    for got, want in ((a_l.grad, r_l.grad), (a_g.grad, r_g.grad)):
        assert _bulk_close(got, want, tol, 0.5) < 1e-2


@pytest.mark.parametrize("h,w", PLANES)
def test_rear_program(h, w, math_mode):
    """The rear program refinement back-propagates through (residual block, up-sampling stage to 2h x 2w, head) at an
    h x w bottleneck against float64 autograd through the oracle's rear composition."""
    gen = _generator(2)
    for p_ in gen.parameters():
        p_.requires_grad_(False)
    sd = {k: v.double().to(DEV) for k, v in gen.state_dict().items()}
    gen = gen.to(DEV)
    g = torch.Generator().manual_seed(4)
    z1, z2 = torch.randn(1, 16, h, w, generator=g).to(DEV), torch.randn(1, 48, h, w, generator=g).to(DEV)
    g0 = torch.randn(1, 3, 2 * h, 2 * w, generator=g).to(DEV)
    assert E.rear_grad_supported(gen, z1.shape, z2.shape)
    a, b = z1.clone().requires_grad_(True), z2.clone().requires_grad_(True)
    L.get_lib().ffcb_reset_launch_count()
    pred = E.generator_rear_with_input_grad(gen, a, b)
    (pred * g0).sum().backward()
    assert L.get_lib().ffcb_launch_count() > 20
    r1, r2 = z1.double().requires_grad_(True), z2.double().requires_grad_(True)
    y = otc.generator_rear(r1, r2, sd, _KW)
    (y * g0.double()).sum().backward()
    tol = 1e-4 if math_mode == "fp32" else 5e-4
    err = _rel_err(pred.detach(), y.detach())
    print(f"\n  rear {h}x{w} pred ({math_mode}): {err:.2e}")
    assert err < tol
    _bulk_close(a.grad, r1.grad, tol, 0.5)
    _bulk_close(b.grad, r2.grad, tol, 0.5)
