"""The refinement step program with its ReLU masks kept as bits (kind ``generator_refine_bits``, ``relu_masks="bits"``),
checked on the CPU: interpreted in float64 it computes exactly what the default step program computes, its storage
slots never overlap live buffers, the backward reads no full-width forward activation except the head adjoint's mask,
big-lama's storage at 4K / 12 MP / 24 MP bottlenecks is pinned next to the default program's, and the refiner and the
command line select it."""
import pytest
import torch

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200 import predict as PR
from lama_b200 import refine as R
from lama_b200 import relu_bits as RB
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs
from spec_interp import SpecInterpreter, check_liveness
from spec_interp_relu_bits import BitsSpecInterpreter, storage_nbytes_bits

_BIG = {}


def _big():
    if "g" not in _BIG:
        _BIG["g"] = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    return _BIG["g"]


def _small():
    return seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)).eval(), 5, gain=1.0)


def _programs(gen, sl, sg, crop, math):
    with torch.no_grad():
        return tuple(E.build_module_program(gen, f"{k}:{crop[0]}x{crop[1]}", (sl, sg), math)
                     for k in ("generator_refine", "generator_refine_bits"))


def _inputs(b, h, w, h0, w0, sl, sg, seed):
    g = torch.Generator().manual_seed(seed)
    z1, z2 = torch.randn(sl, generator=g), torch.randn(sg, generator=g)
    image = torch.rand(b, 3, h, w, generator=g, dtype=torch.float64)
    mask = torch.zeros(b, 1, h, w, dtype=torch.float64)
    mask[:, :, h // 4:h // 4 + h // 2, w // 3:w // 3 + w // 2] = 1
    ref = torch.rand(b, 3, h0 // 2, w0 // 2, generator=g, dtype=torch.float64)
    md = (torch.rand(b, 1, h0 // 2, w0 // 2, generator=g) > 0.5).double()
    n = torch.stack([3 * (mask < 1e-8).sum((1, 2, 3)), 3 * (md >= 1e-8).sum((1, 2, 3))], 1).double()
    inv = torch.where(n > 0, 1.0 / n.clamp_min(1), torch.zeros_like(n))
    return dict(x0=z1, x1=z2, image=image, mask=mask, ref=ref, md=md, inv=inv)


@pytest.mark.parametrize("math", [L.MATH_FP32, L.MATH_BF16X3])
def test_bits_program_computes_what_the_values_program_computes(math):
    """A seeded ngf-8, 2-block generator on a 32x48 image (4x6 bottleneck), two images: both step programs interpreted
    in float64 on the same inputs give exactly equal y0, loss, dx0 and dx1."""
    gen = _small()
    b, h, w, h0, w0 = 2, 32, 48, 32, 48
    sl, sg = (b, 16, h // 8, w // 8), (b, 48, h // 8, w // 8)
    assert E.refine_supported(gen, sl, sg, (h0, w0))
    values, bits = _programs(gen, sl, sg, (h0, w0), math)
    assert bits.kind == f"generator_refine_bits:{h0}x{w0}" and bits.math == values.math
    feed = _inputs(b, h, w, h0, w0, sl, sg, seed=3)
    want = SpecInterpreter(values).run(feed)
    got = BitsSpecInterpreter(bits).run(feed)
    for k in ("y0", "loss", "dx0", "dx1"):
        assert torch.equal(got[k], want[k]), k
    assert float(want["dx0"].abs().max()) > 0 and float(want["dx1"].abs().max()) > 0


def _forward_written(prog):
    split = next(i for i, op in enumerate(prog.ops) if isinstance(op, E.SplitOp))
    return split, {tv.buf.name for op in prog.ops[:split] for tv in op.views()[1]}


@pytest.mark.parametrize("math", [L.MATH_FP32, L.MATH_BF16X3])
def test_bits_program_structure(math):
    """Liveness holds; every ReluBwdOp of the values backward became a ReluBwdBitsOp and nothing else changed; each mask
    is packed once, right after the last forward write of its activation; after SplitOp the only forward buffers read
    are the bit masks and the last up-sampling output (the head adjoint's mask)."""
    gen = _small()
    sl, sg = (1, 16, 4, 6), (1, 48, 4, 6)
    values, bits = _programs(gen, sl, sg, (32, 48), math)
    check_liveness(bits)
    slots = E.assign_storage_slots(bits)
    pooled = sum(storage_nbytes_bits(next(b for b in bits.bufs if slots[b.name] == s)) for s in set(slots.values()))
    outs = sum(4 * int(torch.Size(v).numel()) for v in bits.outputs.values())
    assert E.program_storage_bytes(bits) == pooled + outs + max(bits.fft_workspace_bytes(), 16) + sum(
        op.scratch_bytes() for op in bits.ops)
    kinds = lambda p: [type(op).__name__ for op in p.ops if not isinstance(op, RB.MaskPackOp)]   # noqa: E731
    assert kinds(bits) == [{"ReluBwdOp": "ReluBwdBitsOp"}.get(k, k) for k in kinds(values)]
    assert not any(isinstance(op, E.ReluBwdOp) for op in bits.ops)
    split, fwd = _forward_written(bits)
    packs = [(i, op) for i, op in enumerate(bits.ops) if isinstance(op, RB.MaskPackOp)]
    assert all(i < split for i, _ in packs)
    assert len({op.y.buf.name for _, op in packs}) == len(packs)
    # per block: Y1, Y2 and T, Z of both FFC_BN_ACTs; one per up-sampling stage but the last
    assert len(packs) == 6 * 2 + 2
    for i, op in packs:
        later = [j for j, o in enumerate(bits.ops[:split]) if j > i and op.y.buf.name in {tv.buf.name for tv in o.views()[1]}
                 and not isinstance(o, E.BorderOp)]
        assert not later, (op.y.buf.name, later)
        assert op.bits.buf.bits and (op.bits.buf.B, op.bits.buf.H, op.bits.buf.W, op.bits.buf.C) == (
            op.y.buf.B, op.y.buf.H, op.y.buf.W, op.y.buf.C)
    head = next(op for op in bits.ops if isinstance(op, E.HeadBwdOp))
    read_after = {tv.buf.name: tv.buf for op in bits.ops[split + 1:] for tv in op.views()[0]}
    fwd_read = {n: b for n, b in read_after.items() if n in fwd}
    assert {n for n, b in fwd_read.items() if not b.bits} == {head.mask.buf.name}
    assert {op.bits.buf.name for _, op in packs} <= set(fwd_read)


def test_default_programs_keep_values():
    """The default step program, the rear programs and the block program contain no bit-mask op or buffer."""
    gen = _small()
    sl, sg = (1, 16, 4, 6), (1, 48, 4, 6)
    with torch.no_grad():
        progs = [E.build_module_program(gen, k, (sl, sg), L.MATH_BF16X3)
                 for k in ("generator_refine:32x48", "generator_rear_grad", "generator_rear")]
        progs.append(E.build_module_program(gen.model[5], "resnet_block_grad", (sl, sg), L.MATH_BF16X3))
    for p in progs:
        assert not any(type(op) in RB.OP_TYPES for op in p.ops) and not any(b.bits for b in p.bufs), p.kind
    assert not set(RB.OP_TYPES) & set(E.OP_TYPES)


def test_bit_mask_op_types_are_declared_bound_and_interpreted():
    for cls in RB.OP_TYPES:
        assert {"reads", "writes", "bind"} <= set(vars(cls)), cls.__name__
        for f in cls.reads + cls.writes + cls.ring_in:
            assert f in cls.__dataclass_fields__, (cls.__name__, f)
        assert callable(getattr(BitsSpecInterpreter, cls.__name__, None)), cls.__name__
    assert {c.__name__ for c in RB.OP_TYPES} == {"MaskPackOp", "ReluBwdBitsOp"}


def test_bit_mask_storage():
    b = E.Buf("m", 2, 5, 7, 40, bits=1)
    assert E.storage_shape(b) == (2, 5, 7, 2)
    assert E.storage_key(b) != E.storage_key(E.Buf("v", 2, 5, 7, 40))


# ------------------------------------------------------------------------------------------------ memory
# program_storage_bytes of big-lama's batch-1 step program (split-bf16 arm), values and bits, at the largest scale of a
# 3840x2160 photo, a 12 MP (4000x3000) and a 24 MP (6000x4000) photo refined at full size
BIG_LAMA_STEP_BYTES_VALUES_BITS = {
    (270, 480, 2160, 3840): (29_303_412_744, 13_665_815_176),
    (375, 500, 3000, 4000): (42_356_902_664, 19_763_256_136),
    (500, 750, 4000, 6000): (84_610_438_664, 39_506_064_136),
}


@pytest.mark.parametrize("h,w,h0,w0", list(BIG_LAMA_STEP_BYTES_VALUES_BITS))
def test_big_lama_bits_step_program_storage(h, w, h0, w0):
    values, bits = _programs(_big(), (1, 128, h, w), (1, 384, h, w), (h0, w0), L.MATH_BF16X3)
    got = (E.program_storage_bytes(values), E.program_storage_bytes(bits))
    print(f"big-lama step program, batch 1, {w0}x{h0}: values {got[0] / 1e9:.2f} GB, bits {got[1] / 1e9:.2f} GB")
    assert got == BIG_LAMA_STEP_BYTES_VALUES_BITS[(h, w, h0, w0)]


def _refiner(relu_masks, px_budget):
    ref = R.BatchedRefiner.__new__(R.BatchedRefiner)
    ref.generator = _big()
    ref.kw = dict(modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3, px_budget=px_budget)
    if relu_masks is not None:
        ref.relu_masks = relu_masks
    return ref


def test_per_image_bytes_of_a_24_megapixel_photo_at_full_size():
    """All three scales of a 6000x4000 photo under px_budget = 24_000_000: the bits programs need 50.5 GB, which an
    80 GB device holds next to the front; the values programs need 106.9 GB, which it does not."""
    h, w = 4000, 6000
    assert [c for _, _, c in _refiner("bits", 24_000_000).scale_shapes(h, w)] == [(1000, 1500), (2000, 3000), (4000, 6000)]
    assert _refiner("bits", 24_000_000).per_image_bytes(h, w) == 50_475_856_592
    assert _refiner("values", 24_000_000).per_image_bytes(h, w) == 106_900_053_648


# ------------------------------------------------------------------------------------------------ interface
def test_program_kind_follows_the_setting():
    crop = (2160, 3840)
    assert _refiner(None, 8_300_000).program_kind(1, crop) == "generator_refine:2160x3840"        # default: values
    assert _refiner("values", 8_300_000).program_kind(2, crop) == "generator_refine:2160x3840"
    assert _refiner("bits", 8_300_000).program_kind(2, crop) == "generator_refine_bits:2160x3840"
    for rm in ("values", "bits"):
        assert _refiner(rm, 8_300_000).program_kind(0, crop) == "generator_rear"


def test_relu_masks_argument_is_checked():
    g = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval()
    with pytest.raises(ValueError, match="relu_masks"):
        R.BatchedRefiner(g, relu_masks="bools")
    with torch.no_grad(), pytest.raises(ValueError, match="relu_masks"):
        E.build_refine_program(E.Program("x", L.MATH_FP32), g, (1, 16, 4, 4), (1, 48, 4, 4), (32, 32),
                               relu_masks="bools")


def test_cli_relu_masks_flag():
    base = ["--model-dir", "m", "--indir", "i", "--outdir", "o", "--refine"]
    a = PR.build_parser().parse_args(base)
    assert a.relu_masks is None and "relu_masks" not in PR.refiner_kwargs(a)
    for v in ("bits", "values"):
        a = PR.build_parser().parse_args(base + ["--relu-masks", v, "--px-budget", "24000000"])
        kw = PR.refiner_kwargs(a)
        assert kw["relu_masks"] == v and kw["px_budget"] == 24_000_000
    with pytest.raises(SystemExit):
        PR.build_parser().parse_args(base + ["--relu-masks", "bools"])
