"""GPU tests of the high-resolution path (``pytest -m gpu``): the 8-channel FFT kernels for 448..1024-point axes, the
modules and generators on 4K-class planes, and memory-sized predict batches.  Checkers: numpy float64
(oracle/ffc_numpy.py), the torch-CPU oracle port (oracle/ffc_torch_cpu.py) and the reference predict glue
(oracle/predict_numpy.py).  Tolerances are those of tests/test_gpu_parity.py."""
import gc
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
from oracle import predict_numpy as opn              # noqa: E402

DEV = "cuda:0"
TOL = {"fp32": 2e-5, "bf16x3": 2e-4}


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
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max()) / (float(np.abs(ref).max()) or 1.0)


def _fft_program(b, c, h, w, split, out_c0):
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


# ------------------------------------------------------------------------------------ FFT kernels
@pytest.mark.parametrize("split,out_c0", [(False, 0), (True, 0), (True, 4)])
@pytest.mark.parametrize("b,c,h,w", [(1, 8, 270, 480), (1, 16, 375, 500), (1, 8, 512, 512), (1, 4, 540, 960),
                                     (1, 4, 1024, 1024), (2, 36, 448, 96), (1, 4, 479, 270), (1, 12, 500, 750)])
def test_large_plane_fft_pair_against_numpy(b, c, h, w, split, out_c0):
    """ffcb_rfft2 / ffcb_irfft2 (two launches each) vs numpy float64: the forward spectrum, and the inverse of a
    ReLU'd (non-Hermitian) spectrum plus the residual, in fp32 (2e-6 of max |ref|) and split bf16 (2e-5), the inverse
    also into channels [4, 4 + c) of a wider split-bf16 buffer."""
    rng = np.random.default_rng(h * 1000 + w)
    x = rng.standard_normal((b, c, h, w)).astype(np.float32)
    wf = w // 2 + 1
    z = np.maximum(rng.standard_normal((b, 2 * c, h, wf)), 0).astype(np.float32)
    res = rng.standard_normal((b, c, h, w)).astype(np.float32)
    ex = E.CudaExecutor(_fft_program(b, c, h, w, split, out_c0), torch.device(DEV))
    out = {k: v.cpu() for k, v in ex.run({"x0": torch.from_numpy(x).to(DEV), "x1": torch.from_numpy(z).to(DEV),
                                          "x2": torch.from_numpy(res).to(DEV)}).items()}
    spec = onp.rfft2_ortho(x.astype(np.float64))
    want_s = np.stack((spec.real, spec.imag), axis=2).reshape(b, 2 * c, h, wf)
    zc = z.astype(np.float64).reshape(b, c, 2, h, wf)
    want_y = onp.irfft2_explicit(zc[:, :, 0] + 1j * zc[:, :, 1], h, w) + res
    ef, ei = _rel_err(out["y0"].numpy(), want_s), _rel_err(out["y1"].numpy(), want_y)
    print(f"fft {b}x{c}x{h}x{w} {'split' if split else 'fp32'} c0={out_c0}: fwd {ef:.2e} inv {ei:.2e}")
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


def test_fft_rejects_axes_above_1024():
    ex = E.CudaExecutor(_fft_program(1, 4, 8, 1025, False, 0), torch.device(DEV))
    feed = {"x0": torch.zeros(1, 4, 8, 1025, device=DEV), "x1": torch.zeros(1, 8, 8, 513, device=DEV),
            "x2": torch.zeros(1, 4, 8, 1025, device=DEV)}
    with pytest.raises(ValueError, match="1024-point"):
        ex.run(feed)                                   # ValueError: FFCB_EINVAL


def test_fft_round_trip_and_parseval_at_the_4k_bottleneck():
    """big-lama's spectral planes on a 3840x2160 photo (192 channels, 270x480): irfft2(rfft2(x)) == x and Parseval."""
    b, c, h, w = 1, 192, 270, 480
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
    wgt = torch.full((wf,), 2.0, dtype=torch.float64); wgt[0] = 1.0; wgt[-1] = 1.0
    assert abs(float((p * wgt).sum()) / float((x.double() ** 2).sum()) - 1.0) < 1e-5


# ------------------------------------------------------------------------------------ modules
def test_fourier_unit_and_spectral_transform_at_270x480(math_mode):
    fu = seeded_parameters_(M.FourierUnit(192, 192).eval(), 11, gain=1.0)
    st = seeded_parameters_(M.SpectralTransform(384, 384, enable_lfu=False).eval(), 12, gain=1.0)
    g = torch.Generator().manual_seed(0)
    for m, x in ((fu, torch.randn(1, 192, 270, 480, generator=g)), (st, torch.randn(1, 384, 270, 480, generator=g))):
        sd = {k: v.numpy().astype(np.float64) for k, v in m.state_dict().items()
              if not k.endswith("num_batches_tracked")}
        assert m.native_supported()
        with torch.no_grad():
            y = m.to(DEV)(x.to(DEV)).cpu().numpy()
        ref = (onp.fourier_unit if m is fu else onp.spectral_transform)(x.numpy().astype(np.float64), sd)
        err = _rel_err(y, ref)
        print(f"{type(m).__name__} at 270x480 ({math_mode}): {err:.2e}")
        assert err < TOL[math_mode]


def test_big_lama_resnet_block_at_270x480(math_mode):
    blk = seeded_parameters_(M.FFCResnetBlock(512, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                              activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                              enable_lfu=False).eval(), 12)
    sd = {k: v.clone() for k, v in blk.state_dict().items()}
    g = torch.Generator().manual_seed(1)
    xl, xg = torch.randn(1, 128, 270, 480, generator=g), torch.randn(1, 384, 270, 480, generator=g)
    with torch.no_grad():
        yl, yg = blk.to(DEV)((xl.to(DEV), xg.to(DEV)))
        rl, rg = otc.ffc_resnet_block(xl, xg, sd, "")
    el, eg = _rel_err(yl.cpu().numpy(), rl.numpy()), _rel_err(yg.cpu().numpy(), rg.numpy())
    print(f"FFCResnetBlock(128+384) at 270x480 ({math_mode}): {el:.2e} / {eg:.2e}")
    assert el < TOL[math_mode] and eg < TOL[math_mode]


# ------------------------------------------------------------------------------------ generators
@pytest.mark.parametrize("h,w", [(2160, 3840), (4096, 4096)])
def test_small_generator_at_4k_class_sizes(h, w, math_mode):
    """Bottlenecks of 270x480 and 512x512 against the float64 oracle (torch CPU in double)."""
    kw = small_lama_kwargs(ngf=8, n_blocks=2)
    g = seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 5)
    sd = {k: v.double() for k, v in g.state_dict().items()}
    img, mask = synthetic_image_mask(1, h, 5, width=w)
    x = generator_input(img, mask)
    with torch.no_grad():
        y = g.to(DEV)(x.to(DEV)).cpu()
        ref = otc.ffc_resnet_generator(x.double(), sd, **kw)
    E.invalidate(g)
    err = float((y.double() - ref).abs().max())
    print(f"small generator {h}x{w} ({math_mode}): max-abs {err:.2e}")
    assert err < 3e-4, err


def _big_lama(seed):
    g = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), seed)
    return g, {k: v.clone() for k, v in g.state_dict().items()}


_ORACLE_4K = {}


@pytest.mark.parametrize("seed", [0, 4])
def test_big_lama_at_2160x3840_against_oracle(seed, math_mode):
    """big-lama on a 3840x2160 photo against the CPU fp32 oracle port (the oracle is computed once per seed).  Bounds:
    the fp32 arm 5e-5, as at the smaller sizes; the split-bf16 arm 5e-4, inside the 1e-3 tolerance.  The split-bf16
    arm does not keep below the 3e-4 it keeps up to 2048x2048: against the oracle's sequence run in float64, seed 0 is
    3.2e-4 off on the split-bf16 arm, 1.2e-5 on the fp32 arm, and the CPU fp32 oracle itself 7.3e-6.  So the excess is
    the arm's own rounding (2^-16 per operand), whose largest deviation grows with the 8.3 M output pixels."""
    g, sd = _big_lama(seed)
    img, mask = synthetic_image_mask(1, 2160, seed, width=3840)
    x = generator_input(img, mask)
    with torch.no_grad():
        y = g.to(DEV)(x.to(DEV)).cpu()
    E.invalidate(g)
    del g
    torch.cuda.empty_cache()
    if seed not in _ORACLE_4K:
        with torch.no_grad():
            _ORACLE_4K[seed] = otc.ffc_resnet_generator(x, sd, **BIG_LAMA_KWARGS)
    ref = _ORACLE_4K[seed]
    err = float((y - ref).abs().max())
    print(f"big-lama 2160x3840 seed {seed} ({math_mode}): max-abs {err:.2e}")
    assert ref.std() > 0.05 and err < 1e-3, err
    assert err < (5e-5 if math_mode == "fp32" else 5e-4), err


def test_big_lama_at_2160x3840_batch_independence():
    """Batch 2 equals the two images run at batch 1, bit for bit (the predict driver batches such images)."""
    g, _ = _big_lama(6)
    g = g.to(DEV)
    img, mask = synthetic_image_mask(2, 2160, 6, width=3840)
    x = generator_input(img, mask).to(DEV)
    with torch.no_grad():
        y2 = g(x).cpu()
        E.invalidate(g)
        torch.cuda.empty_cache()
        y1 = torch.cat([g(x[i:i + 1].contiguous()).cpu() for i in range(2)])
    E.invalidate(g)
    assert torch.isfinite(y2).all() and torch.equal(y2, y1)


# ------------------------------------------------------------------------------------ predict driver
def test_batched_inpainter_on_4k_class_images():
    """Two 2157x3838 photos (padded to 2160x3840 inside the program): the bytes of BatchedInpainter equal the
    reference predict glue around the oracle generator (exact outside the hole, within one grey level inside it), and
    a memory budget that forces batches of one gives the same bytes as one batch of two."""
    from lama_b200.predict import BatchedInpainter
    os.environ["LAMA_B200_MATH"] = "bf16x3"
    try:
        kw = small_lama_kwargs(ngf=8, n_blocks=2)
        g = seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 7)
        sd = {k: v.clone() for k, v in g.state_dict().items()}
        g = g.to(DEV)
        h0, w0, b = 2157, 3838, 2
        rng = np.random.default_rng(3)
        images = rng.integers(0, 256, size=(b, h0, w0, 3), dtype=np.uint8)
        masks = np.zeros((b, h0, w0), np.uint8)
        masks[0, 300:900, 1000:2500] = 255
        masks[1, 1500:, 3000:] = 255                          # a hole reaching the padded corner
        masks[1, 100:400, 100:400] = 17
        inp = BatchedInpainter(g, max_batch=b)
        got = np.stack(inp.inpaint(list(zip(images, masks))))
        assert [k[0] for k in inp._pipes] == [b]
        x, img, mask = opn.generator_input(images, masks, pad_mod=8)
        with torch.no_grad():
            pred = otc.ffc_resnet_generator(torch.from_numpy(x), sd, **kw).numpy()
        want = opn.finish(pred, img, mask, h0, w0)
        hole = masks > 0
        assert np.array_equal(got[~hole], want[~hole])
        d = np.abs(got[hole].astype(int) - want[hole].astype(int))
        print(f"4K-class predict bytes vs reference glue: max {int(d.max())}, differing {float((d != 0).mean()):.2e}")
        assert d.max() <= 1 and (d != 0).mean() < 0.05
        one = BatchedInpainter(g, max_batch=b, mem_budget=inp.per_image_bytes(h0, w0) * 3 // 2)
        split = np.stack(one.inpaint(list(zip(images, masks))))
        assert [k[0] for k in one._pipes] == [1]
        assert np.array_equal(split, got)
    finally:
        os.environ.pop("LAMA_B200_MATH", None)


def test_batched_inpainter_frees_a_released_pipeline_before_the_next():
    """Three 2157x3838 photos under a budget of 2.5 images: batches of 2 and 1.  The batch-2 pipeline does not fit
    beside the batch-1 one, so it is released, and its device memory freed, before the batch-1 program allocates: the
    peak stays near two images' worth, not three.  The bytes equal those of one batch of three."""
    from lama_b200.predict import BatchedInpainter
    os.environ["LAMA_B200_MATH"] = "bf16x3"
    try:
        g = seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)).eval(), 8).to(DEV)
        h0, w0 = 2157, 3838
        rng = np.random.default_rng(4)
        images = rng.integers(0, 256, size=(3, h0, w0, 3), dtype=np.uint8)
        masks = np.zeros((3, h0, w0), np.uint8)
        masks[:, 500:1200, 900:2000] = 255
        want = np.stack(BatchedInpainter(g, max_batch=3).inpaint(list(zip(images, masks))))
        E.invalidate(g)
        gc.collect()
        torch.cuda.empty_cache()
        probe = BatchedInpainter(g, max_batch=3)
        per = probe.per_image_bytes(h0, w0)
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        inp = BatchedInpainter(g, max_batch=3, mem_budget=per * 5 // 2)
        got = np.stack(inp.inpaint(list(zip(images, masks))))
        peak = torch.cuda.max_memory_allocated() - base
        print(f"one image {per / 1e9:.2f} GB; peak over the run {peak / 1e9:.2f} GB")
        assert list(inp._pipes) == [(1, h0, w0)]
        assert peak < 2.5 * per, (peak, per)
        assert np.array_equal(got, want)
    finally:
        os.environ.pop("LAMA_B200_MATH", None)
