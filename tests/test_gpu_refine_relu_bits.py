"""GPU tests of the ReLU masks kept as bits (``pytest -m gpu``): ffcb_relu_mask_pack + ffcb_relu_bwd_bits against
ffcb_relu_bwd bit for bit on every view kind, big-lama's bits step program against the values step program bit for bit,
BatchedRefiner with relu_masks="bits" against "values" at 3840x2160, and a 6000x4000 photo refined at full size."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200 import refine as R                    # noqa: E402
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask  # noqa: E402

DEV = "cuda:0"


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


# ------------------------------------------------------------------------------------------------ kernels
def _storage(fmt, shape, gen, zero_frac=0.1):
    """Seeded contents: float32, or split bf16 [2][...] whose lo plane is random too (so hi + lo can change sign)."""
    v = torch.randn((2,) + shape if fmt == L.BF16X2 else shape, generator=gen)
    v[torch.rand(v.shape, generator=gen) < zero_frac] = 0.0
    v[torch.rand(v.shape, generator=gen) < zero_frac / 2] = -0.0
    return v.to(torch.bfloat16 if fmt == L.BF16X2 else torch.float32).to(DEV)


def _view(t, fmt, layout, B, H, W, C, c0=0):
    """ffcb_tensor of storage ``t``: 'ring' = channels-last [B][H+2][W+2][Ctot] with a 1-pixel ring, channels
    [c0, c0+C); 'cg4' / 'cg8' = channel-group planar [C/cg][B][H][W][cg]."""
    es = 2 if fmt == L.BF16X2 else 4
    v = L.Tensor()
    v.B, v.H, v.W, v.C, v.fmt = B, H, W, C, fmt
    if layout == "ring":
        ctot = t.shape[-1]
        v.sx, v.sy, v.sb = ctot, (W + 2) * ctot, (H + 2) * (W + 2) * ctot
        v.lo_off = B * (H + 2) * (W + 2) * ctot if fmt == L.BF16X2 else 0
        v.pad = 1
        v.ptr = t.data_ptr() + ((W + 2 + 1) * ctot + c0) * es
    else:
        cg = int(layout[2:])
        v.cg, v.sx, v.sy, v.sb, v.sg = cg, cg, W * cg, H * W * cg, B * H * W * cg
        v.lo_off = C * B * H * W if fmt == L.BF16X2 else 0
        v.ptr = t.data_ptr()
    return v


def _shape(layout, B, H, W, C):
    return (B, H + 2, W + 2, C + 12) if layout == "ring" else (C // int(layout[2:]), B, H, W, int(layout[2:]))


def _values(t, fmt, layout, B, H, W, C):
    """(B, H, W, C) float32 values of the view as the kernels read them (hi + lo in one float32 addition)."""
    v = t[0].float() + t[1].float() if fmt == L.BF16X2 else t
    if layout == "ring":
        return v[:, 1:H + 1, 1:W + 1, 4:4 + C]
    return v.permute(1, 2, 3, 0, 4).reshape(B, H, W, C)


def _expected_words(y):
    """bits[((b*H + y)*W + x)*nw + c/32] bit c%32 = [y > 0], unused high bits 0 (host restatement)."""
    B, H, W, C = y.shape
    nw = -(-C // 32)
    on = torch.zeros(B, H, W, nw * 32, dtype=torch.int64, device=y.device)
    on[..., :C] = (y > 0).long()
    words = (on.reshape(B, H, W, nw, 32) << torch.arange(32, device=y.device)).sum(-1)
    return words.to(torch.int64).reshape(-1)


@pytest.mark.parametrize("plane", [(128, 1024), (1, 1024)])
@pytest.mark.parametrize("C", [8, 40, 384, 512])
@pytest.mark.parametrize("layout", ["ring", "cg4", "cg8"])
@pytest.mark.parametrize("fmt", [L.F32, L.BF16X2])
def test_pack_then_relu_bwd_bits_equals_relu_bwd(fmt, layout, C, plane):
    """Pack followed by relu_bwd_bits writes exactly the bytes relu_bwd writes (interior and untouched ring alike), and
    the packed words are the documented layout."""
    lib = L.get_lib()
    H, W = plane
    B = 1 if C * H * W > 40 * 128 * 1024 else 2
    g = torch.Generator().manual_seed(C * 7 + H + fmt * 3 + len(layout))
    shape = _shape(layout, B, H, W, C)
    y, dy = _storage(fmt, shape, g), _storage(fmt, shape, g, zero_frac=0.02)
    init = _storage(fmt, shape, g)
    out_ref, out_bits = init.clone(), init.clone()
    c0 = 4 if layout == "ring" else 0
    views = {k: _view(t, fmt, layout, B, H, W, C, c0) for k, t in
             dict(y=y, dy=dy, ref=out_ref, bits=out_bits).items()}
    nw = -(-C // 32)
    words = torch.full((B * H * W * nw,), -1, dtype=torch.int32, device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    L.check(lib.ffcb_relu_bwd(_ref(views["dy"]), _ref(views["y"]), _ref(views["ref"]), s), "relu_bwd")
    L.check(lib.ffcb_relu_mask_pack(_ref(views["y"]), words.data_ptr(), s), "relu_mask_pack")
    L.check(lib.ffcb_relu_bwd_bits(_ref(views["dy"]), words.data_ptr(), _ref(views["bits"]), s), "relu_bwd_bits")
    torch.cuda.synchronize()
    want = _expected_words(_values(y, fmt, layout, B, H, W, C))
    assert torch.equal(words.long() & 0xFFFFFFFF, want & 0xFFFFFFFF)
    a, b = out_ref.view(torch.int16 if fmt == L.BF16X2 else torch.int32), out_bits.view(
        torch.int16 if fmt == L.BF16X2 else torch.int32)
    assert torch.equal(a, b), int((a != b).sum())
    assert not torch.equal(out_ref, init)


def _ref(v):
    return ctypes.byref(v)


# ------------------------------------------------------------------------------------------------ programs
_BIG = {}


def _big():
    if "g" not in _BIG:
        _BIG["g"] = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to(DEV)
        for p in _BIG["g"].parameters():
            p.requires_grad_(False)
    return _BIG["g"]


def _step_inputs(b, H, W, h0, w0, sl, sg, seed):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand(b, 3, H, W, generator=g)
    mask = torch.zeros(b, 1, H, W)
    mask[:, :, H // 4:H // 4 + H // 3, W // 5:W // 5 + W // 2] = 1
    ref = torch.rand(b, 3, h0 // 2, w0 // 2, generator=g)
    md = (torch.rand(b, 1, h0 // 2, w0 // 2, generator=g) > 0.5).float()
    n = torch.stack([3 * (mask < 1e-8).sum((1, 2, 3)), 3 * (md >= 1e-8).sum((1, 2, 3))], 1).double()
    inv = torch.where(n > 0, 1.0 / n.clamp_min(1), torch.zeros_like(n)).float()
    feed = dict(x0=torch.randn(sl, generator=g), x1=torch.randn(sg, generator=g), image=image, mask=mask, ref=ref,
                md=md, inv=inv)
    return {k: v.to(DEV).contiguous() for k, v in feed.items()}


@pytest.mark.parametrize("math", [L.MATH_FP32, L.MATH_BF16X3])
@pytest.mark.parametrize("h0,w0", [(1024, 1024), (864, 2072)])
def test_big_lama_step_program_bits_equals_values(h0, w0, math):
    """One step of big-lama's step program, values and bits, on the same seeded inputs: y0, dy0, dx0, dx1 bit-identical;
    the loss terms, summed with atomics, to 1e-5."""
    gen = _big()
    H, W = h0 + (-h0) % 8, w0 + (-w0) % 8
    sl, sg = (1, 128, H // 8, W // 8), (1, 384, H // 8, W // 8)
    feed = _step_inputs(1, H, W, h0, w0, sl, sg, seed=h0 + w0)
    outs = {}
    for kind in ("generator_refine", "generator_refine_bits"):
        with torch.no_grad():
            prog = E.build_module_program(gen, f"{kind}:{h0}x{w0}", (sl, sg), math)
        assert prog.math == math
        ex = E.CudaExecutor(prog, torch.device(DEV))
        ex.run(feed, part=0)
        ex.run(feed, part=1)
        outs[kind] = {k: ex.outputs[k].clone() for k in ("y0", "loss", "dx0", "dx1", "dy0")}
        n_bits = sum(1 for c in ex.calls if c[0] == "ffcb_relu_bwd_bits")
        print(f"\n  {kind} ({'fp32' if math == L.MATH_FP32 else 'bf16x3'}): {ex.storage_bytes / 1e9:.2f} GB pooled, "
              f"{n_bits} bit-mask backward calls")
        del ex
        torch.cuda.empty_cache()
    for k, want in outs["generator_refine"].items():
        got = outs["generator_refine_bits"][k]
        if k == "loss":
            # the two reported loss terms are sums with float atomics (ffcb_refine_l1_grad), whose order varies from run
            # to run even within one program; the gradient is a fixed-order gather and must match exactly
            assert torch.allclose(got, want, rtol=1e-5, atol=0), (got, want)
            continue
        assert torch.equal(got, want), (k, float((got - want).abs().max()))
    assert float(outs["generator_refine"]["dx1"].abs().max()) > 0


def test_batched_refiner_bits_equals_values_at_4k():
    """big-lama refines a 3840x2160 photo at full size (px_budget 8.3 M, 270x480 bottleneck) with both settings: the
    results are bit-identical."""
    gen = _big()
    h, w = 2160, 3840
    img, mask = synthetic_image_mask(1, h, 5, width=w)
    kw = dict(modulo=8, n_iters=5, lr=0.002, min_side=512, max_scales=3, px_budget=8_300_000)
    res = {}
    for rm in ("values", "bits"):
        ref = R.BatchedRefiner(gen, 1, relu_masks=rm, **kw)
        assert ref.native_ok(h, w) and ref.program_kind(2, (h, w)).startswith(
            "generator_refine_bits:" if rm == "bits" else "generator_refine:")
        torch.cuda.reset_peak_memory_stats()
        res[rm] = ref.refine([img[0]], [mask[0]])[0]
        print(f"\n  {rm}: peak {torch.cuda.max_memory_allocated() / 1e9:.2f} GB")
        del ref
        torch.cuda.empty_cache()
    assert res["bits"].shape == (3, h, w)
    assert torch.equal(res["bits"], res["values"])


def test_24_megapixel_photo_refines_at_full_size():
    """big-lama (seeded) refines a 6000x4000 photo at full size (px_budget 24 M: 500x750 bottleneck at the largest
    scale) on one 80 GB device with relu_masks="bits", twice in one call (two batches of one image, the second after
    the first batch's programs); the values programs of this size would need 107 GB."""
    total = torch.cuda.get_device_properties(0).total_memory
    if total < 79 * 2 ** 30:
        pytest.skip(f"needs an 80 GB device ({total / 2 ** 30:.0f} GiB here)")
    gen = _big()
    h, w = 4000, 6000
    rng = np.random.default_rng(24)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    mask = np.zeros((h, w), np.uint8)
    mask[900:2100, 1500:3300] = 255
    mask[3000:3100, 200:5800] = 255
    image = torch.from_numpy(img).permute(2, 0, 1).float() / 255
    hole = torch.from_numpy(mask)[None].float() / 255
    ref = R.BatchedRefiner(gen, 1, n_iters=4, px_budget=24_000_000, relu_masks="bits")
    assert ref.native_ok(h, w) and ref.scale_shapes(h, w)[-1][2] == (h, w)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    first, second = ref.refine([image, image], [hole, hole])          # two batches of one: the second rebuilds
    peak = torch.cuda.max_memory_allocated()
    print(f"\n  6000x4000 bits: peak {peak / 1e9:.2f} GB of {total / 1e9:.2f} GB, "
          f"programs {ref.per_image_bytes(h, w) / 1e9:.2f} GB")
    out = first
    assert out.shape == (3, h, w) and torch.isfinite(out).all()
    assert torch.equal(first, second)
    keep = (hole[0] == 0).expand(3, -1, -1)
    assert torch.equal(out[keep], image[keep])          # full size: pixels outside the hole come back unchanged
    assert peak < total
