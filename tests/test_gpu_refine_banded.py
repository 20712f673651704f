"""GPU tests of the banded up-sampling tail (``pytest -m gpu``): ffcb_head_bwd7_bits against ffcb_head_bwd7, the row-band
mask pack / ReLU backward against their whole-plane calls and ffcb_head_gather7_rows against ffcb_head_gather7, all bit
for bit; big-lama's banded step program against the bits step program bit for bit; BatchedRefiner with tail="banded"
against "whole" on photos."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import banded as BD                   # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200 import refine as R                    # noqa: E402
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask  # noqa: E402

DEV = "cuda:0"


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


def _plane(fmt, B, H, W, C, gen):
    """Seeded (storage, view of it) of a (B, H, W, C) channels-last plane without ring: float32 or split bf16."""
    shape = (B, H, W, C)
    t = torch.randn((2,) + shape if fmt == L.BF16X2 else shape, generator=gen)
    t[torch.rand(t.shape, generator=gen) < 0.1] = 0.0
    t = t.to(torch.bfloat16 if fmt == L.BF16X2 else torch.float32).to(DEV)
    return t, _view(t, fmt, B, H, W, C)


def _view(t, fmt, B, H, W, C, row0=0, rows=None):
    v = L.Tensor()
    es = 2 if fmt == L.BF16X2 else 4
    v.B, v.H, v.W, v.C, v.fmt = B, H if rows is None else rows, W, C, fmt
    v.sx, v.sy, v.sb = C, W * C, H * W * C
    v.lo_off = B * H * W * C if fmt == L.BF16X2 else 0
    v.ptr = t.data_ptr() + row0 * W * C * es
    return v


def _ref(v):
    return ctypes.byref(v)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bands(H):
    return [(0, H), (0, 5), (3, 9), (H - 11, 11), (H - 1, 1), (17, 8)]


@pytest.mark.parametrize("fmt", [L.F32, L.BF16X2])
@pytest.mark.parametrize("C", [40, 64])
@pytest.mark.parametrize("act", [L.ACT_SIGMOID, L.ACT_NONE])
def test_head_bwd7_bits_equals_head_bwd7(fmt, C, act):
    """Whole plane and row bands (edges included), two images: the bits kernel writes exactly what ffcb_head_bwd7 writes
    with the mask's values."""
    lib, g = L.get_lib(), torch.Generator().manual_seed(C + fmt)
    B, N, H, W = 2, 3, 37, 70
    y = torch.rand(B, N, H, W, generator=g).to(DEV)
    dy = torch.randn(B, N, H, W, generator=g).to(DEV)
    w = torch.randn(N, 49, C, generator=g).to(DEV)
    _m, mv = _plane(fmt, B, H, W, C, g)
    nw = -(-C // 32)
    words = torch.zeros(B * H * W * nw, dtype=torch.int32, device=DEV)
    L.check(lib.ffcb_relu_mask_pack(_ref(mv), words.data_ptr(), _stream()), "relu_mask_pack")
    want = torch.empty(B, H, W, C, device=DEV)
    L.check(lib.ffcb_head_bwd7(y.data_ptr(), dy.data_ptr(), B, N, H, W, w.data_ptr(), act, _ref(mv),
                               _ref(_view(want, L.F32, B, H, W, C)), _stream()), "head_bwd7")
    for row0, rows in _bands(H):
        got = torch.full((B, rows, W, C), float("nan"), device=DEV)
        L.check(lib.ffcb_head_bwd7_bits(y.data_ptr(), dy.data_ptr(), B, N, H, W, w.data_ptr(), act, words.data_ptr(),
                                        row0, _ref(_view(got, L.F32, B, rows, W, C)), _stream()), "head_bwd7_bits")
        torch.cuda.synchronize()
        assert torch.equal(got, want[:, row0:row0 + rows]), (row0, rows)
    assert float(want.abs().max()) > 0


@pytest.mark.parametrize("fmt", [L.F32, L.BF16X2])
@pytest.mark.parametrize("C", [8, 40, 64, 256])
def test_row_band_pack_and_relu_bwd_equal_whole_plane(fmt, C):
    """Packing a plane band by band gives the words of one whole-plane pack (two images, so a band's words are not
    contiguous); ffcb_relu_bwd_bits_rows on a band equals the band of ffcb_relu_bwd_bits."""
    lib, g = L.get_lib(), torch.Generator().manual_seed(C)
    B, H, W = 2, 29, 36
    y, yv = _plane(fmt, B, H, W, C, g)
    dy = torch.randn(B, H, W, C, generator=g).to(DEV)
    nw = -(-C // 32)
    whole = torch.zeros(B * H * W * nw, dtype=torch.int32, device=DEV)
    L.check(lib.ffcb_relu_mask_pack(_ref(yv), whole.data_ptr(), _stream()), "relu_mask_pack")
    banded = torch.full_like(whole, -1)
    for r0 in range(0, H, 6):
        rows = min(6, H - r0)
        L.check(lib.ffcb_relu_mask_pack_rows(_ref(_view(y, fmt, B, H, W, C, r0, rows)), banded.data_ptr(), H, r0,
                                             _stream()), "relu_mask_pack_rows")
    torch.cuda.synchronize()
    assert torch.equal(banded, whole)
    want = torch.empty(B, H, W, C, device=DEV)
    L.check(lib.ffcb_relu_bwd_bits(_ref(_view(dy, L.F32, B, H, W, C)), whole.data_ptr(),
                                   _ref(_view(want, L.F32, B, H, W, C)), _stream()), "relu_bwd_bits")
    for row0, rows in _bands(H):
        got = torch.full((B, rows, W, C), float("nan"), device=DEV)
        L.check(lib.ffcb_relu_bwd_bits_rows(_ref(_view(dy, L.F32, B, H, W, C, row0, rows)), whole.data_ptr(), H, row0,
                                            _ref(_view(got, L.F32, B, rows, W, C)), _stream()), "relu_bwd_bits_rows")
        torch.cuda.synchronize()
        assert torch.equal(got, want[:, row0:row0 + rows]), (row0, rows)


def test_head_gather7_rows_equals_head_gather7():
    lib, g = L.get_lib(), torch.Generator().manual_seed(7)
    B, H, W, N = 2, 23, 150, 3
    q = torch.randn(B, H, W, 24, generator=g).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    want = torch.empty(B, N, H, W, device=DEV)
    L.check(lib.ffcb_head_gather7(_ref(_view(q, L.F32, B, H, W, 24)), bias.data_ptr(), N, L.ACT_SIGMOID,
                                  want.data_ptr(), _stream()), "head_gather7")
    got = torch.full_like(want, float("nan"))
    for r0 in range(0, H, 5):
        rows = min(5, H - r0)
        L.check(lib.ffcb_head_gather7_rows(_ref(_view(q, L.F32, B, H, W, 24, r0, rows)), bias.data_ptr(), N,
                                           L.ACT_SIGMOID, got.data_ptr(), H, r0, _stream()), "head_gather7_rows")
    torch.cuda.synchronize()
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ programs
_BIG = {}


def _big():
    if "g" not in _BIG:
        _BIG["g"] = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 1, gain=1.0).to(DEV)
    return _BIG["g"]


def _step_inputs(b, H, W, h0, w0, sl, sg, seed):
    g = torch.Generator().manual_seed(seed)
    mask = torch.zeros(b, 1, H, W)
    mask[:, :, H // 4:H // 4 + H // 2, W // 3:W // 3 + W // 2] = 1
    md = (torch.rand(b, 1, h0 // 2, w0 // 2, generator=g) > 0.5).float()
    n = torch.stack([3 * (mask < 1e-8).sum((1, 2, 3)), 3 * (md >= 1e-8).sum((1, 2, 3))], 1).double()
    inv = torch.where(n > 0, 1.0 / n.clamp_min(1), torch.zeros_like(n)).float()
    feed = dict(x0=torch.randn(sl, generator=g), x1=torch.randn(sg, generator=g), image=torch.rand(b, 3, H, W,
                generator=g), mask=mask, ref=torch.rand(b, 3, h0 // 2, w0 // 2, generator=g), md=md, inv=inv)
    return {k: v.to(DEV).contiguous() for k, v in feed.items()}


@pytest.mark.parametrize("b,band_px", [(1, 3 * 64 * 128), (2, 5 * 64 * 128), (1, BD.BAND_PX)])
def test_big_lama_banded_step_program_equals_bits(b, band_px, monkeypatch):
    """One step of big-lama's bits and banded step programs at 1024x1024 (a 128x128 bottleneck in bands of 3 and 5 rows,
    and in the default single band) on the same seeded inputs: y0, dy0, dx0, dx1 bit-identical.

    This replaces an op-by-op diff against the float64 interpreter: the bits program is itself checked op by op and
    against float64 autograd (tests/test_gpu_refine_relu_bits.py, tests/test_gpu_refine_rear.py), the banded program
    equals the bits program exactly in the interpreter (tests/test_refine_banded_cpu.py), and every new op's kernel is
    checked above bit for bit against its whole-plane kernel on bands at both plane edges.  Bit equality on the device
    is the stronger check: a tolerance diff could not see a band edge that is off in the last bit."""
    monkeypatch.setattr(BD, "BAND_PX", band_px)
    gen = _big()
    H = W = 1024
    h0, w0 = 1020, 1016
    sl, sg = (b, 128, H // 8, W // 8), (b, 384, H // 8, W // 8)
    feed = _step_inputs(b, H, W, h0, w0, sl, sg, seed=b)
    outs = {}
    for kind in ("generator_refine_bits", "generator_refine_bits_banded"):
        with torch.no_grad():
            prog = E.build_module_program(gen, f"{kind}:{h0}x{w0}", (sl, sg), L.MATH_BF16X3)
        ex = E.CudaExecutor(prog, torch.device(DEV))
        ex.run(feed, part=0)
        ex.run(feed, part=1)
        outs[kind] = {k: ex.outputs[k].clone() for k in ("y0", "dy0", "dx0", "dx1")}
        print(f"\n  {kind} b={b}: {ex.storage_bytes / 1e9:.2f} GB pooled, {len(ex.calls)} calls")
        del ex
        torch.cuda.empty_cache()
    for k, want in outs["generator_refine_bits"].items():
        got = outs["generator_refine_bits_banded"][k]
        assert torch.equal(got, want), (k, float((got - want).abs().max()))
    assert float(outs["generator_refine_bits"]["dx1"].abs().max()) > 0


@pytest.mark.parametrize("h,w,batch,px_budget", [(1024, 1024, 2, 1_800_000), (1440, 3440, 1, 1_800_000),
                                                 (2160, 3840, 1, 8_300_000)])
def test_batched_refiner_banded_equals_whole(h, w, batch, px_budget):
    gen = _big()
    img, mask = synthetic_image_mask(batch, h, 5, width=w)
    kw = dict(modulo=8, n_iters=5, lr=0.002, min_side=512, max_scales=3, px_budget=px_budget)
    res = {}
    for tail in ("whole", "banded"):
        ref = R.BatchedRefiner(gen, batch, relu_masks="bits", tail=tail, **kw)
        assert ref.native_ok(h, w)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        res[tail] = ref.refine(list(img), list(mask))
        print(f"\n  {w}x{h} x{batch} {tail}: peak {torch.cuda.max_memory_allocated() / 1e9:.2f} GB")
        del ref
        torch.cuda.empty_cache()
    for a, b_ in zip(res["banded"], res["whole"]):
        assert torch.equal(a, b_), float((a - b_).abs().max())

