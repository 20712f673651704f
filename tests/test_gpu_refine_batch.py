"""Batched refinement on the GPU (``pytest -m gpu``, an H100): the refinement-loss gradient kernel against float64
autograd, batch independence bit for bit, graph replay against eager steps bit for bit, the refiner against the
per-image ``refine_predict`` loop, the uint8 entry point, no library kernels in a replayed step, and the fallback."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200 import refine as R                    # noqa: E402
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs, synthetic_image_mask  # noqa: E402
from test_refine_batch_cpu import autograd_loss, counts, loss_case  # noqa: E402

DEV = "cuda:0"
SMALL_KW = dict(modulo=8, n_iters=4, lr=0.002, min_side=64, max_scales=2, px_budget=10 ** 7)


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


@pytest.fixture(params=["fp32", "bf16x3"])
def math_mode(request):
    os.environ["LAMA_B200_MATH"] = request.param
    yield request.param
    os.environ.pop("LAMA_B200_MATH", None)


@pytest.fixture
def f32_taps(monkeypatch):
    orig = R.gaussian_kernel1d
    monkeypatch.setattr(R, "gaussian_kernel1d",
                        lambda ksize=5, sigma=1.0, device=None, dtype=torch.float32:
                        orig(ksize, sigma, device, torch.float32).to(dtype))


def _small_gen(seed=2, **opt):
    kw = small_lama_kwargs(ngf=16, n_blocks=3)
    kw["resnet_conv_kwargs"] = dict(kw["resnet_conv_kwargs"], **opt)
    return seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), seed, gain=1.0).to(DEV)


def _images(n, h=136, w=200, seed=0):
    """Seeded images and masks with different holes (masks as mask / 255 of uint8 bytes: {0, 1})."""
    g = torch.Generator().manual_seed(seed)
    ims, mks = [], []
    for i in range(n):
        ims.append(torch.rand(3, h, w, generator=g))
        m = torch.zeros(1, h, w)
        y, x = 10 + 7 * i, 20 + 13 * i
        m[:, y:y + h // 3, x:x + w // 3] = 1
        m[:, h // 2:h // 2 + 6, 5 + 9 * i:60 + 9 * i] = 1
        mks.append(m)
    return ims, mks


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("b,hp,wp,h0,w0,empty", [(1, 48, 56, 45, 52, ()), (2, 48, 56, 48, 56, ()),
                                                 (3, 48, 56, 45, 52, (1,)), (2, 136, 200, 131, 197, ())])
def test_refine_l1_grad_kernel_matches_autograd(b, hp, wp, h0, w0, empty, f32_taps):
    """ffcb_refine_l1_grad vs float64 autograd of refine.l1_loss o pyrdown: relative error <= 1e-6 on the gradient.
    Every |D pred - ref| and |pred - image| in the selections is exactly 0 or above 1e-4, so float32 rounding cannot
    flip a sign; one image of the B = 3 case has an empty eroded mask (zero gradient from that term, NaN loss)."""
    pred, image, mask, ref, md = loss_case(b, hp, wp, h0, w0, seed=hp + w0 + b, empty=empty)
    g = torch.Generator().manual_seed(b)
    pred = pred.float().double()
    step = (torch.rand(image.shape, generator=g, dtype=torch.float64) * 0.5 + 1e-3) * torch.sign(image - pred)
    image = torch.where(image == pred, pred, pred + step).float().double()     # pred == image kept exactly
    down = R.pyrdown(pred[:, :, :h0, :w0])
    sgn = torch.where(torch.rand(ref.shape, generator=g) > 0.5, 1.0, -1.0).double()
    ref = (down + sgn * (torch.rand(ref.shape, generator=g, dtype=torch.float64) * 0.1 + 1e-3)).float().double()
    inv = counts(mask, md)
    want, want_loss = autograd_loss(pred, image, mask, ref, md, h0, w0)
    t = {k: v.float().contiguous().to(DEV) for k, v in dict(pred=pred, image=image, mask=mask, ref=ref, md=md,
                                                             inv=inv).items()}
    taps = R.gaussian_kernel1d(5, 1.0).to(DEV)
    work = torch.empty(b * 3 * (h0 // 2) * (w0 // 2), device=DEV)
    grad = torch.empty(b, 3, hp, wp, device=DEV)
    loss = torch.empty(b, 2, device=DEV)
    lib = L.get_lib()
    L.check(lib.ffcb_refine_l1_grad(t["pred"].data_ptr(), t["image"].data_ptr(), t["mask"].data_ptr(), b, 3, hp, wp,
                                    h0, w0, t["ref"].data_ptr(), t["md"].data_ptr(), t["inv"].data_ptr(),
                                    taps.data_ptr(), work.data_ptr(), grad.data_ptr(), loss.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream), "ffcb_refine_l1_grad")
    torch.cuda.synchronize()
    err = float((grad.cpu().double() - want).abs().max()) / float(want.abs().max())
    print(f"\n  B={b} {hp}x{wp} crop {h0}x{w0}: gradient rel {err:.2e}")
    assert err <= 1e-6
    assert torch.isfinite(grad).all()
    assert torch.allclose(loss.cpu().double(), want_loss, rtol=1e-5, atol=0, equal_nan=True)


# ------------------------------------------------------------------------------------------------ the refiner
def test_batch_independence_bit_for_bit(math_mode):
    """Four 136x200 images with different holes refined as one batch of 4 equal each refined alone (batch 1)."""
    gen = _small_gen()
    ims, mks = _images(4)
    batched = R.BatchedRefiner(gen, 4, **SMALL_KW).refine(ims, mks)
    alone = R.BatchedRefiner(gen, 1, **SMALL_KW).refine(ims, mks)
    for i, (a, b) in enumerate(zip(batched, alone)):
        assert a.shape == (3, 136, 200)
        assert torch.equal(a, b), (i, float((a - b).abs().max()))


def test_graph_replay_equals_eager_steps(math_mode):
    """The replayed CUDA graph of a step equals the same steps run eagerly, bit for bit; a second batch of the same
    shape (graph reused, Adam state reset) equals a fresh refiner; the executor allocates what program_storage_bytes
    computed."""
    gen = _small_gen()
    ims, mks = _images(4, seed=1)
    graphed = R.BatchedRefiner(gen, 2, **SMALL_KW)
    g_out = graphed.refine(ims, mks)                     # two batches of 2: the second replays the captured graphs
    eager = R.BatchedRefiner(gen, 2, **SMALL_KW)
    eager._graphs = False
    e_out = eager.refine(ims, mks)
    fresh = R.BatchedRefiner(gen, 2, **SMALL_KW).refine(ims[2:], mks[2:])
    for a, b in zip(g_out, e_out):
        assert torch.equal(a, b)
    for a, b in zip(g_out[2:], fresh):
        assert torch.equal(a, b)
    for lane in graphed._lanes.values():
        ex = lane.ex
        alloc = (ex.storage_bytes + ex.ws.numel() + sum(t.numel() * t.element_size() for t in ex.outputs.values())
                 + sum(op.scratch_bytes() for op in ex.prog.ops))
        assert alloc == E.program_storage_bytes(ex.prog)


def _vs_refine_predict(gen, ims, mks, kw):
    ref = R.BatchedRefiner(gen, len(ims), **kw).refine(ims, mks)
    for i, (im, mk) in enumerate(zip(ims, mks)):
        want = R.refine_predict(im[None], mk[None], gen, **kw)[0]
        d = (ref[i] - want).abs()
        print(f"\n  image {i}: max-abs {float(d.max()):.2e}, mean {float(d.mean()):.2e}")
        assert torch.isfinite(ref[i]).all()
        assert float(d.max()) < 5e-3 and float(d.mean()) < 2e-4


def test_against_refine_predict_small(math_mode):
    """BatchedRefiner (batch 3) vs refine_predict per image on the same arithmetic arm: the bounds of
    test_refinement_native_rear_matches_module_path."""
    ims, mks = _images(3, seed=2)
    _vs_refine_predict(_small_gen(), ims, mks, SMALL_KW)


def test_against_refine_predict_big_lama_1024(math_mode):
    """big-lama at 1024x1024 with the reference's refiner settings (two scales, 15 iterations), one image."""
    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to(DEV)
    img, mask = synthetic_image_mask(1, 1024, 3)
    _vs_refine_predict(gen, [img[0]], [mask[0]], dict(modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3,
                                                      px_budget=1800000))


def test_uint8_entry_point_matches_float(math_mode):
    """inpaint's bytes equal clip(float result * 255).astype(uint8) of the float entry point, below and above
    px_budget (the latter refined and returned at the reduced size, as by the reference)."""
    gen = _small_gen()
    kw = dict(SMALL_KW, px_budget=20000)
    rng = np.random.default_rng(0)
    items = []
    for h, w in ((96, 128), (136, 200), (136, 200)):
        m = np.zeros((h, w), np.uint8)
        m[h // 4:h // 2, w // 3:w // 2 + len(items) * 5] = 255
        items.append((rng.integers(0, 256, (h, w, 3), dtype=np.uint8), m))
    ref = R.BatchedRefiner(gen, 4, **kw)
    got = ref.inpaint(items)
    imgs = [torch.from_numpy(im).permute(2, 0, 1).float() / 255 for im, _ in items]
    msks = [torch.from_numpy(mk)[None].float() / 255 for _, mk in items]
    want = [R.to_uint8(x) for x in R.BatchedRefiner(gen, 4, **kw).refine(imgs, msks)]
    assert got[0].shape == (96, 128, 3) and got[1].shape[0] * got[1].shape[1] <= 20000
    for a, b in zip(got, want):
        assert a.dtype == np.uint8 and np.array_equal(a, b)


def test_replayed_step_launches_only_project_kernels():
    """A profiled replay of one step's graph shows the refinement-loss kernels and no cuDNN / cuFFT / cuBLAS kernel."""
    gen = _small_gen()
    ims, mks = _images(2, seed=3)
    ref = R.BatchedRefiner(gen, 2, **SMALL_KW)
    ref.refine(ims, mks)
    lane = next(ln for ln in ref._lanes.values() if ln.graph is not None)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lane.graph.replay()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    banned = [n for n in names if "ffcb" not in n and any(k in n.lower() for k in ("cudnn", "fft", "xmma", "gemm",
                                                                                    "cutlass"))]
    assert not banned, banned
    assert any("refine_full_kernel" in n for n in names) and any("refine_down_kernel" in n for n in names), names


def test_lfu_generator_falls_back_to_refine_predict(monkeypatch):
    """A generator without native step programs (LFU) takes refine_predict per image, and the refiner returns exactly
    what those calls returned.  A second, independent refine_predict run is compared within the bounds of
    test_against_refine_predict_small only: torch's bilinear-interpolation backward on CUDA accumulates with atomics, so
    two runs of that loop are not bit-identical."""
    gen = _small_gen(enable_lfu=True)
    ims, mks = _images(2, h=128, w=128, seed=4)             # LFU takes even square planes only
    ref = R.BatchedRefiner(gen, 2, **SMALL_KW)
    assert not ref.native_ok(128, 128)
    calls = []
    orig = R.refine_predict

    def spy(image, mask, generator, **kw):
        calls.append((image, mask, orig(image, mask, generator, **kw)))
        return calls[-1][2]

    monkeypatch.setattr(R, "refine_predict", spy)
    got = ref.refine(ims, mks)
    monkeypatch.setattr(R, "refine_predict", orig)
    assert len(calls) == 2 and not ref._lanes
    for i in range(2):
        assert torch.equal(calls[i][0][0], ims[i]) and torch.equal(calls[i][1][0], mks[i])
        assert torch.equal(got[i], calls[i][2][0])
        d = (got[i] - R.refine_predict(ims[i][None], mks[i][None], gen, **SMALL_KW)[0]).abs()
        print(f"\n  image {i}: a second refine_predict run differs by max-abs {float(d.max()):.2e}")
        assert float(d.max()) < 5e-3 and float(d.mean()) < 2e-4, (float(d.max()), float(d.mean()))
