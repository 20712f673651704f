"""The refinement step program with its up-sampling tail in row bands (kind ``generator_refine_bits_banded``,
``tail="banded"``), checked on the CPU: interpreted in float64 it computes exactly what the bits step program computes
(one and two images, odd bottleneck heights, bands of 1 to 3 bottleneck rows, a last band shorter than the others),
its storage slots never overlap live buffers, big-lama's storage at 24 and 48 MP is pinned next to the bits program's,
and the refiner and the command line select it."""
import pytest
import torch
import torch.nn.functional as F

from lama_b200 import _lib as L
from lama_b200 import banded as BD
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200 import predict as PR
from lama_b200 import refine as R
from lama_b200 import relu_bits as RB
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs
from spec_interp import check_liveness
from spec_interp_relu_bits import BitsSpecInterpreter

_BIG = {}


def _big():
    if "g" not in _BIG:
        _BIG["g"] = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    return _BIG["g"]


def _small():
    return seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)).eval(), 5, gain=1.0)


class BandedSpecInterpreter(BitsSpecInterpreter):
    """Restatements of the four op types of ``lama_b200.banded`` on whole-plane float64 masks (one 0 / 1 per element)."""

    def MaskPackRowsOp(self, op, ext):
        y = self.read(op.y)
        self.mem[op.bits.buf.name][:, op.row0:op.row0 + y.shape[1]] = (y > 0).double()

    def ReluBwdBitsRowsOp(self, op, ext):
        dy = self.read(op.dy)
        self.write(op.out, dy * self.mem[op.bits.buf.name][:, op.row0:op.row0 + dy.shape[1]])

    def HeadGatherRowsOp(self, op, ext):
        if op.dst not in ext:
            ext[op.dst] = torch.full(self.prog.outputs[op.dst], float("nan"), dtype=torch.float64)
        y = self._gather(self.read(op.q), op.bias, op.n_out, op.act)
        ext[op.dst][:, :, op.row0:op.row0 + y.shape[2]] = y

    def HeadBwdBitsOp(self, op, ext):
        whole = E.HeadBwdOp(op.y, op.dy, op.w, op.n_out, op.act, op.bits, op.bits)
        saved = self.mem[op.bits.buf.name].clone()
        self.HeadBwdOp(whole, ext)                      # writes the masked whole-plane gradient over the mask buffer
        g = self.mem[op.bits.buf.name]
        self.write(op.out, g[:, op.row0:op.row0 + op.out.buf.H].clone())
        self.mem[op.bits.buf.name].copy_(saved)


def _programs(gen, sl, sg, crop, band_px, monkeypatch):
    monkeypatch.setattr(BD, "BAND_PX", band_px)
    with torch.no_grad():
        return tuple(E.build_module_program(gen, f"{k}:{crop[0]}x{crop[1]}", (sl, sg), L.MATH_BF16X3)
                     for k in ("generator_refine_bits", "generator_refine_bits_banded"))


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


# (batch, bottleneck h, w, bottleneck rows per band): bands of 1, 2 and 3 rows, odd heights, a short last band, and one
# band covering the plane
CASES = [(1, 5, 6, 1), (2, 5, 6, 2), (1, 7, 5, 3), (2, 4, 6, 3), (1, 3, 4, 3)]


@pytest.mark.parametrize("b,h,w,rows", CASES)
def test_banded_program_computes_what_the_bits_program_computes(b, h, w, rows, monkeypatch):
    gen = _small()
    sl, sg = (b, 16, h, w), (b, 48, h, w)
    H, W = 8 * h, 8 * w
    crop = (H - 3, W - 2)
    assert E.refine_supported(gen, sl, sg, crop)
    bits, banded = _programs(gen, sl, sg, crop, rows * 64 * w, monkeypatch)
    assert BD.band_rows(h, w, 3) == rows
    assert banded.kind == f"generator_refine_bits_banded:{crop[0]}x{crop[1]}"
    n_bands = len(BD.bands(h, rows))
    assert sum(isinstance(op, BD.HeadGatherRowsOp) for op in banded.ops) == n_bands
    assert sum(isinstance(op, BD.HeadBwdBitsOp) for op in banded.ops) == n_bands
    check_liveness(banded)
    feed = _inputs(b, H, W, crop[0], crop[1], sl, sg, seed=11)
    want = BitsSpecInterpreter(bits).run(feed)
    got = BandedSpecInterpreter(banded).run(feed)
    for k in ("y0", "dy0", "loss", "dx0", "dx1"):
        assert torch.equal(got[k], want[k]), k
    assert float(want["dx0"].abs().max()) > 0 and float(want["dx1"].abs().max()) > 0


def test_banded_program_structure(monkeypatch):
    """The blocks part is the bits program's op for op; the tail reads no whole-plane full-resolution buffer but the
    bit masks; no ReluBwdOp or HeadBwdOp is left."""
    gen = _small()
    sl, sg = (1, 16, 5, 6), (1, 48, 5, 6)
    bits, banded = _programs(gen, sl, sg, (40, 48), 2 * 64 * 6, monkeypatch)
    first_tail = lambda p: next(i for i, op in enumerate(p.ops)                            # noqa: E731
                                if isinstance(op, E.ConvOp) and "convT" in op.tag)
    kinds = lambda p, ops: [type(op).__name__ for op in ops]                               # noqa: E731
    assert kinds(bits, bits.ops[:first_tail(bits)]) == kinds(banded, banded.ops[:first_tail(banded)])
    assert not any(isinstance(op, (E.ReluBwdOp, E.HeadBwdOp, E.HeadGatherOp)) for op in banded.ops)
    full = [b for b in banded.bufs if b.H == 40 and not b.bits]
    assert not full, [b.name for b in full]


def test_banded_op_types_are_declared_bound_and_interpreted():
    for cls in BD.OP_TYPES:
        assert {"reads", "writes", "bind"} <= set(vars(cls)), cls.__name__
        for f in cls.reads + cls.writes + cls.ring_in:
            assert f in cls.__dataclass_fields__, (cls.__name__, f)
        assert callable(getattr(BandedSpecInterpreter, cls.__name__, None)), cls.__name__
    assert not set(BD.OP_TYPES) & (set(E.OP_TYPES) | set(RB.OP_TYPES))


def test_band_height_comes_from_the_shape():
    assert BD.band_rows(750, 1000, 3) == 32 and len(BD.bands(750, 32)) == 24
    assert BD.band_rows(500, 750, 3) == 43
    assert BD.band_rows(16, 16, 3) == 16                 # small planes: one band
    assert BD.bands(5, 2) == [(0, 2), (2, 4), (4, 5)]


def test_fp32_arm_is_refused():
    gen = _small()
    with torch.no_grad(), pytest.raises(ValueError, match="tensor-core head"):
        BD.build_refine_banded_program(E.Program("x", L.MATH_FP32), gen, (1, 16, 4, 4), (1, 48, 4, 4), (32, 32))


# ------------------------------------------------------------------------------------------------ memory
# program_storage_bytes of big-lama's batch-1 step programs (split-bf16 arm), bits and banded, at the largest scale of a
# 24 MP (6000x4000) and a 48 MP (8000x6000) photo refined at full size
BIG_LAMA_STEP_BYTES_BITS_BANDED = {
    (500, 750, 4000, 6000): (39_506_064_136, 17_945_139_976),
    (750, 1000, 6000, 8000): (78_982_464_136, 28_763_159_176),
}


@pytest.mark.parametrize("h,w,h0,w0", list(BIG_LAMA_STEP_BYTES_BITS_BANDED))
def test_big_lama_banded_step_program_storage(h, w, h0, w0, monkeypatch):
    bits, banded = _programs(_big(), (1, 128, h, w), (1, 384, h, w), (h0, w0), BD.BAND_PX, monkeypatch)
    got = (E.program_storage_bytes(bits), E.program_storage_bytes(banded))
    print(f"big-lama step program, batch 1, {w0}x{h0}: bits {got[0] / 1e9:.2f} GB, banded {got[1] / 1e9:.2f} GB")
    assert got == BIG_LAMA_STEP_BYTES_BITS_BANDED[(h, w, h0, w0)]


# ------------------------------------------------------------------------------------------------ interface
def _refiner(relu_masks, tail, px_budget=48_000_000):
    ref = R.BatchedRefiner.__new__(R.BatchedRefiner)
    ref.generator = _big()
    ref.kw = dict(modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3, px_budget=px_budget)
    ref.relu_masks = relu_masks
    if tail is not None:
        ref.tail = tail
    return ref


def test_program_kind_follows_the_setting():
    crop = (6000, 8000)
    assert _refiner("bits", None).program_kind(2, crop) == "generator_refine_bits:6000x8000"     # default: whole
    assert _refiner("bits", "whole").program_kind(2, crop) == "generator_refine_bits:6000x8000"
    assert _refiner("bits", "banded").program_kind(2, crop) == "generator_refine_bits_banded:6000x8000"
    assert _refiner("bits", "banded").program_kind(0, crop) == "generator_rear"


def test_tail_argument_is_checked():
    g = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval()
    with pytest.raises(ValueError, match="tail"):
        R.BatchedRefiner(g, relu_masks="bits", tail="bands")
    with pytest.raises(ValueError, match="relu_masks='bits'"):
        R.BatchedRefiner(g, tail="banded")
    with pytest.raises(ValueError, match="relu_masks='bits'"):
        R.BatchedRefiner(g, relu_masks="values", tail="banded")


def test_cli_refine_tail_flag():
    base = ["--model-dir", "m", "--indir", "i", "--outdir", "o", "--refine", "--relu-masks", "bits"]
    a = PR.build_parser().parse_args(base)
    assert a.refine_tail is None and "tail" not in PR.refiner_kwargs(a)
    for v in ("banded", "whole"):
        kw = PR.refiner_kwargs(PR.build_parser().parse_args(base + ["--refine-tail", v, "--px-budget", "48000000"]))
        assert kw["tail"] == v and kw["relu_masks"] == "bits" and kw["px_budget"] == 48_000_000
    with pytest.raises(SystemExit):
        PR.build_parser().parse_args(base + ["--refine-tail", "rows"])


def test_banded_setting_needs_the_tensor_core_head(monkeypatch):
    g = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval()
    assert BD.tail_supported(g, L.MATH_BF16X3) and not BD.tail_supported(g, L.MATH_FP32)
    monkeypatch.setenv("LAMA_B200_HEAD", "simt")
    assert not BD.tail_supported(g, L.MATH_BF16X3)
    with pytest.raises(ValueError, match="tensor-core head"):
        R.BatchedRefiner(g, relu_masks="bits", tail="banded")
