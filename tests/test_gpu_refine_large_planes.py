"""GPU tests of refinement at bottleneck planes above 256 points (``pytest -m gpu``): native block input gradients,
the rear program and the batched step programs at 8-channel (448..1024) and Bluestein FFT lengths, where the torch
composition on the GPU is not a yardstick (DESIGN.md section 9).  Checkers: float64 CPU autograd through the torch-CPU
oracle (blocks, rear) and the refinement loop driven by float64 CPU autograd (BatchedRefiner)."""
import copy
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import modules as M                   # noqa: E402
from lama_b200 import predict as PR                  # noqa: E402
from lama_b200 import refine as R                    # noqa: E402
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs  # noqa: E402
from oracle import ffc_torch_cpu as otc              # noqa: E402
from test_refine_rear_cpu import rear_oracle_grads   # noqa: E402

DEV = "cuda:0"


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


@pytest.fixture(params=["fp32", "bf16x3"])
def math_mode(request):
    os.environ["LAMA_B200_MATH"] = request.param
    yield request.param
    os.environ.pop("LAMA_B200_MATH", None)


def _rel2(got, want):
    got, want = got.double().cpu(), want.double().cpu()
    return float((got - want).pow(2).sum().sqrt() / want.pow(2).sum().sqrt())


def _bulk_close(got, want, tol, frac):
    """Most elements agree to ``tol`` of the range, the median is below it and the 2-norm error is small: activations
    within round-off of zero can fall on the other side of a ReLU in two implementations (DESIGN.md section 9)."""
    got, want = got.double().cpu(), want.double().cpu()
    d = (got - want).abs()
    scale = float(want.abs().max())
    off, med, l2 = float((d > tol * scale).double().mean()), float(d.median()) / scale, _rel2(got, want)
    print(f"  beyond {tol:g}: {off:.3f}, median {med:.2e}, 2-norm {l2:.2e}")
    assert off < frac, "too many elements off"
    assert med < tol
    assert l2 < 20 * tol
    return l2


# ------------------------------------------------------------------------------------------------ block gradients
_BLOCK_ORACLE = {}


@pytest.mark.parametrize("h,w", [(270, 480), (108, 259), (128, 1024)])
def test_big_lama_block_input_gradients(h, w, math_mode):
    """big-lama's FFCResnetBlock (128 + 384 channels) at a 4K photo's bottleneck (270x480: 8-channel rows), a 2072x864
    scale's (108x259: Bluestein rows) and an 8192x1024 image's (128x1024): the native forward + input-gradient program
    against float64 autograd through the torch-CPU oracle.  Relative 2-norm: forward below 5e-5, input gradients below
    1e-2 (DESIGN.md section 9 measures 2.4e-5 and 3-4e-3 on the split-bf16 arm up to 256x256)."""
    cl, cg = 128, 384
    blk = seeded_parameters_(M.FFCResnetBlock(cl + cg, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                              activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                              enable_lfu=False).eval(), 4, gain=1.0)
    sd = {k: v.clone() for k, v in blk.state_dict().items()}
    for p_ in blk.parameters():
        p_.requires_grad_(False)
    blk = blk.to(DEV)
    gen = torch.Generator().manual_seed(h + w)
    xl, xg, gl, gg = (torch.randn(1, ch, h, w, generator=gen) for ch in (cl, cg, cl, cg))
    a_l, a_g = xl.to(DEV).requires_grad_(True), xg.to(DEV).requires_grad_(True)
    L.get_lib().ffcb_reset_launch_count()
    o_l, o_g = blk((a_l, a_g))
    assert L.get_lib().ffcb_launch_count() > 10, "the native forward+backward program did not run"
    ((o_l * gl.to(DEV)).sum() + (o_g * gg.to(DEV)).sum()).backward()
    if (h, w) not in _BLOCK_ORACLE:
        r_l, r_g = xl.double().requires_grad_(True), xg.double().requires_grad_(True)
        q_l, q_g = otc.ffc_resnet_block(r_l, r_g, {k: v.double() for k, v in sd.items()}, "", ratio_gout=0.75)
        ((q_l * gl.double()).sum() + (q_g * gg.double()).sum()).backward()
        _BLOCK_ORACLE.clear()
        _BLOCK_ORACLE[(h, w)] = (q_l.detach(), q_g.detach(), r_l.grad, r_g.grad)
    q_l, q_g, d_l, d_g = _BLOCK_ORACLE[(h, w)]
    fl, fg = _rel2(o_l.detach(), q_l), _rel2(o_g.detach(), q_g)
    print(f"\n  {h}x{w} ({math_mode}): forward 2-norm {fl:.2e} / {fg:.2e}")
    assert fl < 5e-5 and fg < 5e-5
    tol = 1e-4 if math_mode == "fp32" else 5e-4
    for got, want in ((a_l.grad, d_l), (a_g.grad, d_g)):
        assert _bulk_close(got, want, tol, 0.5) < 1e-2


# ------------------------------------------------------------------------------------------------ rear program
def test_rear_program_at_a_259x108_bottleneck(math_mode):
    """The rear program (residual blocks, up-sampling tail to 864x2072, head) of a small generator at a 108x259
    bottleneck (Bluestein rows) against float64 autograd through the oracle's rear composition."""
    kw = small_lama_kwargs(ngf=16, n_blocks=3)
    gen = seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 2, gain=1.0)
    for p_ in gen.parameters():
        p_.requires_grad_(False)
    gen = gen.to(DEV)
    h, w = 108, 259
    g = torch.Generator().manual_seed(4)
    z1, z2 = torch.randn(1, 32, h, w, generator=g), torch.randn(1, 96, h, w, generator=g)
    g0 = torch.randn(1, 3, 8 * h, 8 * w, generator=g)
    assert E.rear_grad_supported(gen, z1.shape, z2.shape)
    a, b = z1.to(DEV).requires_grad_(True), z2.to(DEV).requires_grad_(True)
    L.get_lib().ffcb_reset_launch_count()
    pred = E.generator_rear_with_input_grad(gen, a, b)
    (pred * g0.to(DEV)).sum().backward()
    assert L.get_lib().ffcb_launch_count() > 20
    y, d1, d2 = rear_oracle_grads(gen, z1, z2, g0, kw)
    tol = 1e-4 if math_mode == "fp32" else 5e-4
    err = float((pred.detach().double().cpu() - y).abs().max()) / float(y.abs().max())
    print(f"\n  pred ({math_mode}): {err:.2e}")
    assert err < tol
    _bulk_close(a.grad, d1, tol, 0.5)
    _bulk_close(b.grad, d2, tol, 0.5)


# ------------------------------------------------------------------------------------------------ batched refiner
# 4 iterations, 2 scales: the larger scale has a 108x259 (2072x864) or 270x480 (3840x2160) bottleneck
REFINE_KW = {(864, 2072): dict(modulo=8, n_iters=4, lr=0.002, min_side=512, max_scales=2, px_budget=1800000),
             (2160, 3840): dict(modulo=8, n_iters=4, lr=0.002, min_side=512, max_scales=2, px_budget=8300000)}
_F64_LOOP = {}


def _images(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    ims, mks = [], []
    for i in range(n):
        ims.append(torch.rand(3, h, w, generator=g))
        m = torch.zeros(1, h, w)
        m[:, h // 5 + 11 * i:h // 5 + 11 * i + h // 3, w // 4 + 17 * i:w // 4 + 17 * i + w // 5] = 1
        m[:, h // 2:h // 2 + 9, 40 + 13 * i:w // 2] = 1
        mks.append(m)
    return ims, mks


def _small_gen():
    gen = seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)).eval(), 6, gain=1.0)
    return gen.to(DEV)


@pytest.mark.parametrize("hw", list(REFINE_KW))
def test_batched_refiner_at_high_resolution(hw, math_mode, monkeypatch):
    """Two images through BatchedRefiner: the batch of 2 equals each image alone (batch 1) bit for bit, graph replay
    equals eager steps bit for bit, and image 0 matches the same loop (refine_predict) driven by float64 CPU autograd
    within the bounds of the refiner's tests against refine_predict."""
    h, w = hw
    kw = REFINE_KW[hw]
    gen = _small_gen()
    ims, mks = _images(2, h, w, seed=h)
    ref = R.BatchedRefiner(gen, 2, **kw)
    assert ref.native_ok(h, w)
    assert max(ref.scale_shapes(h, w)[-1][0][2:]) > 256
    batched = ref.refine(ims, mks)
    del ref
    torch.cuda.empty_cache()
    alone = R.BatchedRefiner(gen, 1, **kw).refine(ims, mks)
    torch.cuda.empty_cache()
    eager = R.BatchedRefiner(gen, 1, **kw)
    eager._graphs = False
    e_out = eager.refine(ims[:1], mks[:1])
    del eager
    torch.cuda.empty_cache()
    for i, (a, b) in enumerate(zip(batched, alone)):
        assert a.shape == (3, h, w)
        assert torch.equal(a, b), (i, float((a - b).abs().max()))
    assert torch.equal(alone[0], e_out[0])
    if hw not in _F64_LOOP:
        monkeypatch.delenv("LAMA_B200_STRICT", raising=False)      # the CPU loop runs the torch composition
        g64 = copy.deepcopy(gen).cpu().double()
        _F64_LOOP[hw] = R.refine_predict(ims[0][None].double(), mks[0][None].double(), g64, device="cpu", **kw)[0]
    want = _F64_LOOP[hw]
    d = (batched[0].double() - want).abs()
    print(f"\n  {h}x{w} ({math_mode}): vs float64 loop max-abs {float(d.max()):.2e}, mean {float(d.mean()):.2e}")
    assert torch.isfinite(batched[0]).all()
    assert float(d.max()) < 5e-3 and float(d.mean()) < 2e-4


def test_big_lama_predict_refine_at_3440x1440(tmp_path, monkeypatch):
    """big-lama through the predict driver with ``--refine`` at its defaults on a 21:9 frame (refined at 2073x868, a
    109x260 bottleneck): the run ends, every step program is native, and every byte outside the hole equals the input
    as the refiner resizes it."""
    from PIL import Image
    h, w = 1440, 3440
    rng = np.random.default_rng(7)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    mask = np.zeros((h, w), np.uint8)
    mask[300:700, 1200:2000] = 255
    mask[1000:1040, 100:3000] = 255
    indir = tmp_path / "in"
    indir.mkdir()
    Image.fromarray(img).save(indir / "frame.png")
    Image.fromarray(mask).save(indir / "frame_mask001.png")
    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to(DEV)
    a = PR.build_parser().parse_args(["--model-dir", "unused", "--indir", str(indir), "--outdir", str(tmp_path / "out"),
                                      "--refine"])
    refiner = R.BatchedRefiner(gen, **PR.refiner_kwargs(a))
    assert refiner.native_ok(h, w)
    calls = []
    orig = R.refine_predict
    monkeypatch.setattr(R, "refine_predict", lambda *args, **k: calls.append(1) or orig(*args, **k))
    n = PR.predict_directory(refiner, a.indir, a.outdir)
    assert n == 1 and not calls
    out = np.array(Image.open(tmp_path / "out" / "frame_mask001.png"))
    im_t = torch.from_numpy(img).permute(2, 0, 1).float()[None] / 255
    mk_t = torch.from_numpy(mask)[None, None].float() / 255
    ims, mks = R.image_mask_pyramid(im_t, mk_t, 512, 3, 1800000)
    im_r, mk_r = ims[-1][0], mks[-1][0, 0]
    assert out.shape == (im_r.shape[1], im_r.shape[2], 3) and out.shape[:2] == (868, 2073)
    keep = (mk_r < 1e-8).numpy()
    assert keep.any() and (~keep).any()
    assert np.array_equal(out[keep], R.to_uint8(im_r)[keep])
