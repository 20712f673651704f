"""The batched refinement step on the CPU: the refinement-loss gradient op (RefineLossOp / ffcb_refine_l1_grad) restated
in float64 against autograd of refine.l1_loss o pyrdown, the whole ``generator_refine`` step program interpreted in
float64 against autograd through the oracle rear + loss, the rear program unchanged op for op, batch sizing from
``engine.program_storage_bytes``, and the ``--refine`` command line."""
import json
import os

import numpy as np
import pytest
import torch

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200 import predict as PR
from lama_b200 import refine as R
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs
from oracle import ffc_torch_cpu as otc
from spec_interp import SpecInterpreter, check_liveness, refine_loss_f64, storage_nbytes

GOLDEN_REAR_OPS = os.path.join(os.path.dirname(__file__), "golden", "rear_grad_program_ops.json")


@pytest.fixture
def f32_taps(monkeypatch):
    """refine.gaussian_kernel1d in any dtype returns the float32 taps (what the kernel and the float32 loop use)."""
    orig = R.gaussian_kernel1d
    monkeypatch.setattr(R, "gaussian_kernel1d",
                        lambda ksize=5, sigma=1.0, device=None, dtype=torch.float32:
                        orig(ksize, sigma, device, torch.float32).to(dtype))


def counts(mask, md):
    """(B, 2) inverse element counts of the two selections, 0 where empty."""
    n = torch.stack([3 * (mask < 1e-8).sum((1, 2, 3)), 3 * (md >= 1e-8).sum((1, 2, 3))], 1).double()
    return torch.where(n > 0, 1.0 / n.clamp_min(1), torch.zeros_like(n))


def autograd_loss(pred, image, mask, ref, md, h0, w0):
    """Per image: refine.l1_loss(pred, pyrdown(pred crop), ref, mask3, md3, image) and its gradient (float64)."""
    grads, losses = [], []
    for b in range(pred.shape[0]):
        p = pred[b:b + 1].double().clone().requires_grad_(True)
        m3 = mask[b:b + 1].double().repeat(1, 3, 1, 1)
        d3 = md[b:b + 1].double().repeat(1, 3, 1, 1)
        down = R.pyrdown(p[:, :, :h0, :w0])
        t0 = torch.mean(torch.abs(p[m3 < 1e-8] - image[b:b + 1].double()[m3 < 1e-8]))
        t1 = torch.mean(torch.abs(down[d3 >= 1e-8] - ref[b:b + 1].double()[d3 >= 1e-8]))
        (t0 + t1).backward()
        grads.append(p.grad)
        losses.append(torch.stack([t0.detach(), t1.detach()]))
    return torch.cat(grads), torch.stack(losses)


def loss_case(b, hp, wp, h0, w0, seed, empty=(), equal=True):
    """Seeded pred / image / mask / ref / md; images in ``empty`` get an empty md; with ``equal`` a patch of pixels
    outside the hole has pred == image exactly."""
    g = torch.Generator().manual_seed(seed)
    pred = torch.rand(b, 3, hp, wp, generator=g, dtype=torch.float64)
    image = torch.rand(b, 3, hp, wp, generator=g, dtype=torch.float64)
    mask = torch.zeros(b, 1, hp, wp, dtype=torch.float64)
    for i in range(b):
        y, x = int(torch.randint(0, hp // 2, (1,), generator=g)), int(torch.randint(0, wp // 2, (1,), generator=g))
        mask[i, :, y:y + hp // 2, x:x + wp // 2] = 1
    if equal:
        image[:, :, -3:, :4] = pred[:, :, -3:, :4]
        mask[:, :, -3:, :4] = 0
    ref = torch.rand(b, 3, h0 // 2, w0 // 2, generator=g, dtype=torch.float64)
    md = (torch.rand(b, 1, h0 // 2, w0 // 2, generator=g) > 0.5).double()
    for i in empty:
        md[i] = 0
    return pred, image, mask, ref, md


@pytest.mark.parametrize("b,hp,wp,h0,w0,empty", [(1, 48, 56, 45, 52, ()), (2, 48, 56, 48, 56, ()),
                                                 (3, 48, 56, 45, 52, (1,)), (1, 24, 16, 17, 13, ())])
def test_refine_loss_restatement_matches_autograd(b, hp, wp, h0, w0, empty, f32_taps):
    """The restated op vs float64 autograd of refine.l1_loss o pyrdown: gradient to 1e-12, both loss terms (NaN for an
    empty selection, whose gradient is zero and finite), sign(0) = 0 where pred == image."""
    pred, image, mask, ref, md = loss_case(b, hp, wp, h0, w0, seed=hp * w0 + b, empty=empty)
    assert bool((pred == image).any())
    got, loss = refine_loss_f64(pred, image, mask, ref, md, counts(mask, md), h0, w0, R.gaussian_kernel1d(5, 1.0))
    want, want_loss = autograd_loss(pred, image, mask, ref, md, h0, w0)
    assert torch.isfinite(got).all()
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())
    assert torch.allclose(loss, want_loss, rtol=1e-12, atol=0, equal_nan=True)
    for i in empty:
        assert torch.isnan(loss[i, 1]) and torch.isnan(want_loss[i, 1])


# ------------------------------------------------------------------------------------------- the whole step program
def _gen(**kw):
    kw = dict(small_lama_kwargs(**kw))
    return seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 5, gain=1.0), kw


@pytest.mark.parametrize("math", [L.MATH_FP32, L.MATH_BF16X3])
def test_refine_program_matches_autograd(math, f32_taps):
    """dx0, dx1 (and pred, the loss terms) of the interpreted generator_refine program vs float64 autograd through the
    oracle rear + the refinement loss, to 1e-6 of their range (the rear test's bound); odd crop in a padded plane, two
    images, one of them with an empty eroded mask."""
    gen, kw = _gen(ngf=16, n_blocks=2)
    b, h, w, h0, w0 = 2, 6, 7, 45, 52
    sl, sg = (b, 32, h, w), (b, 96, h, w)
    assert E.refine_supported(gen, sl, sg, (h0, w0))
    with torch.no_grad():
        prog = E.build_module_program(gen, f"generator_refine:{h0}x{w0}", (sl, sg), math)
    assert prog.math == math and sum(isinstance(op, E.RefineLossOp) for op in prog.ops) == 1
    g = torch.Generator().manual_seed(11)
    z1, z2 = torch.randn(sl, generator=g), torch.randn(sg, generator=g)
    _, image, mask, ref, md = loss_case(b, 8 * h, 8 * w, h0, w0, seed=2, empty=(1,), equal=False)
    inv = counts(mask, md)
    out = SpecInterpreter(prog).run(dict(x0=z1, x1=z2, image=image, mask=mask, ref=ref, md=md, inv=inv))
    sd = {k: v.detach().double() for k, v in gen.state_dict().items()}
    a, c = z1.double().requires_grad_(True), z2.double().requires_grad_(True)
    pred = otc.generator_rear(a, c, sd, kw)
    want_g, want_loss = autograd_loss(pred.detach(), image, mask, ref, md, h0, w0)
    pred.backward(want_g)
    for got, want in ((out["y0"], pred.detach()), (out["dx0"], a.grad), (out["dx1"], c.grad), (out["dy0"], want_g)):
        assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max())
    assert torch.allclose(out["loss"], want_loss, rtol=1e-6, atol=0, equal_nan=True)


# ------------------------------------------------------------------------------------------- rear program unchanged
def op_signature(prog):
    """Op kinds, tags and every view's buffer (name, shape, format, ring, layout) and slice, in program order."""
    sig = []
    for op in prog.ops:
        reads, writes = op.views()
        views = [[tv.buf.name, tv.buf.B, tv.buf.H, tv.buf.W, tv.buf.C, tv.buf.pad, tv.buf.fmt, tv.buf.reflect_border,
                  tv.buf.cg, tv.buf.tile, tv.c0, tv.channels, list(tv.phase) if tv.phase else None, tv.window, tv.b0,
                  tv.batch, list(tv.win) if tv.win else None, tv.bcast] for tv in reads + writes]
        names = [getattr(op, k) for k in ("src", "dst", "y", "dy") if isinstance(getattr(op, k, None), str)]
        sig.append([type(op).__name__, getattr(op, "tag", ""), names, views])
    return sig


REAR_CASES = {"small_fp32": (L.MATH_FP32, (2, 16, 6, 10), (2, 48, 6, 10)),
              "small_bf16x3": (L.MATH_BF16X3, (2, 16, 6, 10), (2, 48, 6, 10)),
              "small_bf16x3_odd": (L.MATH_BF16X3, (1, 16, 5, 7), (1, 48, 5, 7))}


def _rear_programs():
    gen = seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)).eval(), 5, gain=1.0)
    with torch.no_grad():
        return {k: E.build_module_program(gen, "generator_rear_grad", (sl, sg), math)
                for k, (math, sl, sg) in REAR_CASES.items()}


def test_rear_grad_program_unchanged():
    """Factoring the rear's forward and backward emission into helpers shared with the refinement step program leaves
    generator_rear_grad the same op for op (kinds, tags, buffers, views) as before (golden written from the previous
    program builder)."""
    with open(GOLDEN_REAR_OPS) as f:
        want = json.load(f)
    got = {k: op_signature(p) for k, p in _rear_programs().items()}
    assert got.keys() == want.keys()
    for k in want:
        assert len(got[k]) == len(want[k]), k
        for i, (a, b) in enumerate(zip(got[k], want[k])):
            assert a == b, (k, i)


def test_refine_program_extends_the_rear():
    """The step program is the rear's forward, the loss op, the rear's backward reading the op's gradient."""
    gen, _ = _gen(ngf=8, n_blocks=2)
    sl, sg = (2, 16, 6, 10), (2, 48, 6, 10)
    with torch.no_grad():
        rear = E.build_module_program(gen, "generator_rear_grad", (sl, sg), L.MATH_BF16X3)
        step = E.build_module_program(gen, "generator_refine:45x77", (sl, sg), L.MATH_BF16X3)
    kinds = lambda p: [type(op).__name__ for op in p.ops]          # noqa: E731
    k = kinds(rear).index("SplitOp")
    assert kinds(step)[:k + 1] == kinds(rear)[:k + 1]
    assert kinds(step)[k + 1] == "RefineLossOp" and kinds(step)[k + 2:] == kinds(rear)[k + 1:]
    hb = next(op for op in step.ops if isinstance(op, E.HeadBwdOp))
    assert hb.dy == "dy0" and "dy0" in step.outputs and "g0" not in step.inputs
    assert set(step.inputs) == {"x0", "x1", "image", "mask", "ref", "md", "inv"}
    assert step.inputs["ref"] == (2, 3, 22, 38) and step.inputs["inv"] == (2, 2)
    assert not E.refine_supported(gen, sl, sg, (49, 80)) and not E.refine_supported(gen, sl, sg, (2, 80))


# ------------------------------------------------------------------------------------------- batch sizing
def test_program_storage_bytes():
    """program_storage_bytes = the pooled buffers (slot by slot, liveness checked) + outputs + FFT workspace + the loss
    op's scratch, computed without a device; it grows with the batch and stays below B x the one-image size plus
    per-buffer rounding.  big-lama's step program at the 1344x1344 scale (168x168 bottleneck) is printed."""
    gen, _ = _gen(ngf=8, n_blocks=2)
    progs = {}
    for b in (1, 3):
        with torch.no_grad():
            progs[b] = E.build_module_program(gen, "generator_refine:45x77", ((b, 16, 6, 10), (b, 48, 6, 10)),
                                              L.MATH_BF16X3)
    p = progs[3]
    want = (check_liveness(p) + sum(4 * int(np.prod(s)) for s in p.outputs.values()) + p.fft_workspace_bytes()
            + 4 * 3 * 3 * 22 * 38)
    assert E.program_storage_bytes(p) == want
    one, three = E.program_storage_bytes(progs[1]), E.program_storage_bytes(progs[3])
    assert 2 * one < three <= 3 * one + len(p.bufs) * 128 * 512 * 4
    big = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    with torch.no_grad():
        bp = E.build_module_program(big, "generator_refine:1344x1344", ((1, 128, 168, 168), (1, 384, 168, 168)),
                                    L.MATH_BF16X3)
    print(f"big-lama step program at 1344x1344: {E.program_storage_bytes(bp) / 1e9:.2f} GB")
    assert E.program_storage_bytes(bp) > storage_nbytes(bp.bufs[0])


def test_plan_batches():
    plan = R.BatchedRefiner.plan_batches
    idx = list(range(10))
    assert plan(idx, 100, 350, 8) == [[0, 1, 2], [3, 4, 5], [6, 7], [8, 9]]          # balanced, never above 3
    assert plan(idx, 100, 10_000, 4) == [[0, 1, 2, 3], [4, 5, 6], [7, 8, 9]]
    assert plan(list(range(20)), 100, 900, 32) == [list(range(0, 7)), list(range(7, 14)), list(range(14, 20))]
    assert plan(idx[:2], 100, 50, 8) == [[0], [1]]                    # one image always runs
    assert plan([], 100, 1000, 8) == []


class _BytesLane:
    """Stand-in lane: the pooled bytes of the program the refiner would build for it."""
    graph = None

    def __init__(self, gen, kind, sl, sg):
        with torch.no_grad():
            self.bytes = E.program_storage_bytes(E.build_module_program(gen, kind, (sl, sg), E.default_math()))


@pytest.mark.parametrize("n,fit", [(7, 3.5), (20, 9.2), (5, 1.0)])
def test_refiner_peak_storage_stays_within_budget(n, fit):
    """A group whose size is not a multiple of the batch: through the refiner's own batch plan and lane policy, the
    programs alive at any time (every scale of the current batch size, sized with program_storage_bytes at that batch)
    pool no more than the budget.  The lowest scale is a forward-only program, smaller than a step program."""
    gen = seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=16, n_blocks=2)).eval(), 1, gain=1.0)
    ref = R.BatchedRefiner.__new__(R.BatchedRefiner)
    ref.generator, ref._lanes, ref._graphs = gen, {}, True
    ref.kw = dict(modulo=8, n_iters=15, lr=0.002, min_side=64, max_scales=3, px_budget=10 ** 7)
    ref._make_lane = lambda kind, sl, sg, crop: _BytesLane(gen, kind, sl, sg)
    h, w = 260, 300
    shapes = ref.scale_shapes(h, w)
    assert len(shapes) == 3
    per_image = ref.per_image_bytes(h, w)
    budget = int(fit * per_image)
    batches = ref.plan_batches(list(range(n)), per_image, budget, 32)
    assert sorted(i for bt in batches for i in bt) == list(range(n))
    assert max(map(len, batches)) - min(map(len, batches)) <= 1
    peak = 0
    for bt in batches:
        for s, (sl, sg, crop) in enumerate(shapes):
            ref._lane(len(bt), s, sl, sg, crop)
            peak = max(peak, sum(ln.bytes for ln in ref._lanes.values()))
    assert len({k[0] for k in ref._lanes}) == 1
    assert peak <= budget, (peak, budget)
    sl, sg, crop = shapes[0]
    fwd = _BytesLane(gen, "generator_rear", sl, sg).bytes
    step = _BytesLane(gen, f"generator_refine:{crop[0]}x{crop[1]}", sl, sg).bytes
    assert fwd < step


def test_scale_shapes_follow_the_pyramid():
    """The per-scale (z1, z2, crop) shapes the refiner plans with are those image_mask_pyramid and the modulo padding
    produce."""
    ref = R.BatchedRefiner.__new__(R.BatchedRefiner)
    ref.generator = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    ref.kw = dict(modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3, px_budget=1800000)
    for h, w in ((1024, 1024), (1344, 1344), (700, 1000), (300, 200), (2000, 1500)):
        ims, _ = R.image_mask_pyramid(torch.zeros(1, 3, h, w), torch.zeros(1, 1, h, w), 512, 3, 1800000)
        shapes = ref.scale_shapes(h, w)
        assert [c for _, _, c in shapes] == [tuple(im.shape[2:]) for im in ims]
        for (sl, sg, (h0, w0)), im in zip(shapes, ims):
            hp, wp = R._pad_to_modulo(im, 8).shape[2:]
            assert sl == (1, 128, hp // 8, wp // 8) and sg == (1, 384, hp // 8, wp // 8)


def test_refiner_needs_cuda():
    g = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        R.BatchedRefiner(g)
    ref = R.BatchedRefiner.__new__(R.BatchedRefiner)
    with pytest.raises(ValueError):
        ref.inpaint([(np.zeros((8, 8, 3), np.float32), np.zeros((8, 8), np.uint8))])


# ------------------------------------------------------------------------------------------- command line
def test_cli_refine_flags_map_to_refiner_kwargs():
    """--refine with no other flag gives configs/prediction/default.yaml's refiner section; modulo is --pad-mod."""
    base = ["--model-dir", "m", "--indir", "i", "--outdir", "o"]
    a = PR.build_parser().parse_args(base + ["--refine"])
    assert a.refine
    assert PR.refiner_kwargs(a) == dict(max_batch=32, modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3,
                                        px_budget=1800000)
    a = PR.build_parser().parse_args(base + ["--refine", "--n-iters", "5", "--lr", "0.01", "--min-side", "256",
                                             "--max-scales", "2", "--px-budget", "1000", "--pad-mod", "16",
                                             "--batch", "4"])
    assert PR.refiner_kwargs(a) == dict(max_batch=4, modulo=16, n_iters=5, lr=0.01, min_side=256, max_scales=2,
                                        px_budget=1000)
    assert not PR.build_parser().parse_args(base).refine
    assert "gpu_ids" in PR.build_parser().format_help().replace("\n", " ").replace("- ", "-")


def test_predict_directory_with_a_refiner_keeps_output_names(tmp_path):
    """predict_directory takes any object with inpaint(items) (the refiner) and writes bin/predict.py's names, at the
    size the inpainter returns."""
    from PIL import Image
    indir = tmp_path / "in"
    (indir / "sub").mkdir(parents=True)
    rng = np.random.default_rng(0)
    for name, (h, w) in (("a", (20, 24)), ("sub/b", (16, 16))):
        Image.fromarray(rng.integers(0, 255, (h, w, 3), dtype=np.uint8)).save(indir / f"{name}.png")
        Image.fromarray((rng.random((h, w)) > 0.5).astype(np.uint8) * 255).save(indir / f"{name}_mask001.png")

    class HalfSize:
        def inpaint(self, items):
            return [im[::2, ::2] for im, _ in items]

    n = PR.predict_directory(HalfSize(), str(indir), str(tmp_path / "out"))
    assert n == 2
    out = sorted(os.path.relpath(os.path.join(d, f), tmp_path / "out") for d, _, fs in os.walk(tmp_path / "out")
                 for f in fs)
    assert out == ["a_mask001.png", "sub/b_mask001.png"]
    assert np.array(Image.open(tmp_path / "out" / "a_mask001.png")).shape == (10, 12, 3)


if __name__ == "__main__":
    # writes the golden of test_rear_grad_program_unchanged from whichever lama_b200 is first on sys.path
    with open(GOLDEN_REAR_OPS, "w") as f:
        json.dump({k: op_signature(p) for k, p in _rear_programs().items()}, f, separators=(",", ":"))
    print("wrote", GOLDEN_REAR_OPS)
