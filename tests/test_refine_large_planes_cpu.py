"""Refinement at bottleneck planes above 256 points (images above 2048 px per side, e.g. 21:9 frames refined at about
2072x864, or 4K photos under a raised ``px_budget``), checked on the CPU: the support gates reach every plane the native
FFT pair takes, the interpreted block-gradient program matches float64 autograd through the oracle on wide planes with
Bluestein and 8-channel FFT lengths, big-lama's step programs at these sizes have the storage quoted in DESIGN.md, an
image whose programs exceed the memory budget still runs at batch 1 and a failed allocation is raised, and the
float32-vs-float64 drift of the bilinear source index in the refinement loss stays small at d ~ 2000."""
import numpy as np
import pytest
import torch

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200 import refine as R
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs
from oracle import ffc_torch_cpu as otc
from spec_interp import SpecInterpreter

_BIG = {}


def _big():
    if "g" not in _BIG:
        _BIG["g"] = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    return _BIG["g"]


def _close(got, ref, rel=1e-6):
    scale = float(ref.abs().max()) or 1.0
    err = float((got.double() - ref.double()).abs().max())
    assert err <= rel * scale, f"{err:.3e} > {rel:g}*{scale:.3e}"


# ------------------------------------------------------------------------------------------------ gates
@pytest.mark.parametrize("h,w", [(257, 64), (108, 259), (270, 480), (479, 270), (1024, 128)])
def test_native_gradients_cover_every_native_fft_plane(h, w):
    """Block input gradients, the rear program and the step program take big-lama's bottleneck planes above 256 points:
    Bluestein lengths (257, 259, 479) and the 8-channel lengths (448..1024)."""
    big = _big()
    sl, sg = (1, 128, h, w), (1, 384, h, w)
    assert E.plane_ok(h, w)
    blk = big.model[5]
    assert max(h, w) <= E.BLOCK_GRAD_MAX_PLANE and E.block_grad_supported(blk)
    assert E.ffc_bn_act_shapes_ok(blk.conv1, torch.empty(sl, device="meta"), torch.empty(sg, device="meta"))
    assert E.rear_grad_supported(big, sl, sg)
    assert E.refine_supported(big, sl, sg, (8 * h - 3, 8 * w - 5))


def test_planes_the_fft_rejects_stay_unsupported():
    big = _big()
    assert E.BLOCK_GRAD_MAX_PLANE == E.FFT_MAX_LEN
    for h, w in ((1025, 64), (64, 1025), (1025, 1025)):
        sl, sg = (1, 128, h, w), (1, 384, h, w)
        assert not E.rear_grad_supported(big, sl, sg), (h, w)
        assert not E.refine_supported(big, sl, sg, (8 * h, 8 * w)), (h, w)
        assert not E.ffc_bn_act_shapes_ok(big.model[5].conv1, torch.empty(sl, device="meta"),
                                          torch.empty(sg, device="meta"))


@pytest.mark.parametrize("h,w,px_budget", [(1440, 3440, 1800000), (2160, 3840, 8300000), (864, 2072, 1800000)])
def test_refiner_takes_the_native_path_at_high_resolution(h, w, px_budget):
    """BatchedRefiner plans native step programs for every scale of a 21:9 frame at the default budget and of a 4K photo
    under a raised budget; the largest scale has a bottleneck axis above 256 points."""
    ref = R.BatchedRefiner.__new__(R.BatchedRefiner)
    ref.generator = _big()
    ref.kw = dict(modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3, px_budget=px_budget)
    shapes = ref.scale_shapes(h, w)
    assert max(shapes[-1][0][2:]) > 256
    assert ref.native_ok(h, w)


# ------------------------------------------------------------------------------------------------ the block program
@pytest.mark.parametrize("h,w", [(17, 300), (9, 479)])
def test_block_gradient_program_on_wide_planes_matches_autograd(h, w):
    """The forward+backward program of a small-channel FFCResnetBlock, interpreted in float64, against float64 autograd
    through the oracle on planes whose long axis takes a Bluestein (479) or runtime mixed-radix (300) FFT."""
    blk = seeded_parameters_(M.FFCResnetBlock(64, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                              activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                              enable_lfu=False).eval(), 3, gain=1.0)
    assert E.block_grad_supported(blk)
    b, cl, cg = 1, 16, 48
    g = torch.Generator().manual_seed(h + w)
    xl, xg = torch.randn(b, cl, h, w, generator=g), torch.randn(b, cg, h, w, generator=g)
    gl, gg = torch.randn(b, cl, h, w, generator=g), torch.randn(b, cg, h, w, generator=g)
    with torch.no_grad():
        prog = E.build_module_program(blk, "resnet_block_grad", ((b, cl, h, w), (b, cg, h, w)), L.MATH_FP32)
    out = SpecInterpreter(prog).run(dict(x0=xl, x1=xg, g0=gl, g1=gg))
    sd = {k: v.double() for k, v in blk.state_dict().items()}
    xl64, xg64 = xl.double().requires_grad_(True), xg.double().requires_grad_(True)
    ol, og = otc.ffc_resnet_block(xl64, xg64, sd, "", ratio_gout=0.75)
    ((ol * gl.double()).sum() + (og * gg.double()).sum()).backward()
    _close(out["y0"], ol.detach() - xl.double())
    _close(out["dx0"], xl64.grad)
    _close(out["dx1"], xg64.grad)


# ------------------------------------------------------------------------------------------------ memory
# Device bytes of big-lama's batch-1 step program (kind generator_refine, split-bf16 arm) as program_storage_bytes
# computes them from the buffer shapes: the 3840x2160 scale (270x480 bottleneck) and a 2072x864 scale (259x108).
BIG_LAMA_STEP_BYTES = {(270, 480, 2160, 3840): 29_303_412_744, (108, 259, 864, 2072): 6_360_781_576}


@pytest.mark.parametrize("h,w,h0,w0", list(BIG_LAMA_STEP_BYTES))
def test_big_lama_step_program_storage(h, w, h0, w0):
    with torch.no_grad():
        prog = E.build_module_program(_big(), f"generator_refine:{h0}x{w0}", ((1, 128, h, w), (1, 384, h, w)),
                                      L.MATH_BF16X3)
    got = E.program_storage_bytes(prog)
    print(f"big-lama step program, batch 1, {h0}x{w0} ({h}x{w} bottleneck): {got / 1e9:.2f} GB")
    assert got == BIG_LAMA_STEP_BYTES[(h, w, h0, w0)]


def test_an_image_above_the_budget_runs_alone():
    """Programs of one image larger than the budget: every image still gets a batch of its own."""
    plan = R.BatchedRefiner.plan_batches
    per_image = BIG_LAMA_STEP_BYTES[(270, 480, 2160, 3840)]
    assert plan(list(range(3)), per_image, per_image // 2, 8) == [[0], [1], [2]]
    assert plan([5], per_image, 0, 8) == [[5]]


def test_a_failed_allocation_is_raised_not_replaced(monkeypatch):
    """When the device cannot hold the programs of one image at batch 1, the allocation error reaches the caller: the
    refiner neither falls back to refine_predict nor swallows it."""
    gen = seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval(), 1)
    ref = R.BatchedRefiner.__new__(R.BatchedRefiner)
    ref.generator, ref.device, ref.max_batch, ref.mem_budget = gen, torch.device("cpu"), 4, 1
    ref.kw = dict(modulo=8, n_iters=2, lr=0.002, min_side=32, max_scales=2, px_budget=10 ** 7)
    ref.front, _ = R.split_generator(gen.model)
    ref._lanes, ref._size, ref._graphs = {}, None, True
    built = []

    def no_memory(kind, sl, sg, crop):
        built.append(sl[0])
        raise torch.OutOfMemoryError("CUDA out of memory (test)")

    def no_fallback(*a, **k):
        raise AssertionError("refine_predict must not run")

    monkeypatch.setattr(ref, "_make_lane", no_memory)
    monkeypatch.setattr(R, "refine_predict", no_fallback)
    monkeypatch.delenv("LAMA_B200_STRICT", raising=False)
    assert ref.native_ok(64, 96)
    g = torch.Generator().manual_seed(0)
    ims = [torch.rand(3, 64, 96, generator=g) for _ in range(2)]
    mks = [torch.zeros(1, 64, 96) for _ in range(2)]
    with pytest.raises(torch.OutOfMemoryError):
        ref.refine(ims, mks)
    assert built == [1]                                  # the budget allows one image per batch: batch 1 was tried


# ------------------------------------------------------------------------------------------------ refine_full
def _axis_operator(n_in: int, index_f32: bool) -> np.ndarray:
    """M[d][y] of the refinement loss's 1-D down-scaling operator (bilinear o 5-tap Gaussian, reflect-101), with the
    bilinear source index computed in float64 (ffcb_refine_l1_grad, torch's float64 interpolate) or in float32 (torch's
    float32 interpolate, which the refine_predict loop runs)."""
    taps = R.gaussian_kernel1d(5, 1.0, dtype=torch.float64).numpy()
    n_out = n_in // 2
    d = np.arange(n_out)
    if index_f32:
        sc = np.float32(n_in) / np.float32(n_out)
        src = np.maximum((sc * (d.astype(np.float32) + np.float32(0.5))).astype(np.float32) - np.float32(0.5),
                         np.float32(0)).astype(np.float64)
    else:
        src = np.maximum(n_in / n_out * (d + 0.5) - 0.5, 0.0)
    i0 = src.astype(np.int64)
    i1 = np.where(i0 < n_in - 1, i0 + 1, i0)
    l1 = src - i0
    m = np.zeros((n_out, n_in))
    for i, lam in ((i0, 1.0 - l1), (i1, l1)):
        for a in range(5):
            p = np.abs(i + a - 2)
            p = np.where(p >= n_in, 2 * n_in - 2 - p, p)
            np.add.at(m, (d, p), lam * taps[a])
    return m


@pytest.mark.parametrize("n_in,bound", [(201, 1e-5), (4001, 3e-4), (8191, 5e-4), (4000, 0.0)])
def test_float32_source_index_drift_of_the_loss_adjoint(n_in, bound):
    """refine_full builds D^T from the source index computed in double, as torch's float64 interpolate does; torch's
    float32 interpolate (the per-image loop) computes it in float.  The two differ only for odd crop sides (an even side
    has scale 2, exact in float), by at most 3.5e-4 in the source index at d <= 2000 (7.1e-4 at d <= 4096).  Per axis
    the adjoint applied to a signed residual then moves by at most ``bound`` of its largest entry."""
    a, b = _axis_operator(n_in, False), _axis_operator(n_in, True)
    r = np.random.default_rng(n_in).choice([-1.0, 1.0], size=(n_in // 2, 16))
    ga, gb = a.T @ r, b.T @ r
    err = float(np.abs(ga - gb).max() / np.abs(ga).max())
    print(f"n_in={n_in}: operator max |dM| {np.abs(a - b).max():.2e}, adjoint rel {err:.2e}")
    assert err <= bound
