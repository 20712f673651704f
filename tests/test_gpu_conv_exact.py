"""Every instantiation of the tensor-core contraction (conv_tc.cu) checked bit for bit against float64.

Operands come from dyadic grids small enough that every partial sum is exact in float32 (tests/conv_exact.py), so the
kernel's output must equal the float64 reference exactly: a lost low-order product, a stale pipeline stage or a wrong
tile offset shows up as a named element of a named tile, however small.  Each case first asserts the plan it runs
(ffcb_conv_plan: flat / spatial per-tap / rows-resident / column-halo, tile-blocked operands, planar output, N tile),
then runs the tensor-core arm with nonzero weight lo planes; where the fp32 arm accepts the views, both arms also run
with bf16-exact weights and must agree with the reference and with each other.  The last test asserts that the cases
launched every instantiation x N tile that conv_tc() can launch.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from conv_exact import (GRID_BITS, Buf, Case, Layout, Seg, act_ulp_bound, assert_budget, assert_exact,  # noqa: E402
                        budget_check, contraction, dyadic, grid_exp, make_desc, plan, product_grid, reference, rel_err,
                        split_planes, split_rne, weight_planes)

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import packing as P                   # noqa: E402

DEV = torch.device("cuda:0")
FLAT, SPATIAL, ROWS, HALO = L.PLAN_FLAT, L.PLAN_SPATIAL, L.PLAN_ROWS, L.PLAN_HALO
KNOBS = ("FFCB_TC_BN", "FFCB_TC_ROWS", "FFCB_TC_ROWS_TW")
HIT = set()          # (kind, il, po, bn) of every tensor-core launch of this module
RAN = set()          # node ids of the cases of this module that ran in this session


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


@pytest.fixture(autouse=True)
def _no_knobs(monkeypatch, request):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    yield
    RAN.add(request.node.nodeid)


# ------------------------------------------------------------------------------------------------ harness
def _refl(n, p):
    i = (torch.arange(-p, n + p)).abs()
    return torch.where(i >= n, 2 * n - 2 - i, i)


def _padded(v, p):
    """[B, H, W, C] -> its reflection-padded [B, H+2p, W+2p, C]."""
    return v[:, _refl(v.shape[1], p)][:, :, _refl(v.shape[2], p)]


def load_source(lay: Layout, hi, lo) -> Buf:
    """A source buffer: interior planes; a reflected ring is written as the reflection of the interior (what
    ffcb_fill_reflect_border leaves), any other ring stays NaN."""
    b = Buf(lay, DEV)
    if lay.pad and lay.reflect:
        b.write(_padded(hi, lay.pad), _padded(lo, lay.pad), ring=True)
    else:
        b.write(hi, lo)
    return b


def run(case: Case, in_lays, out_lay: Layout, arm: int, *, addend_alias=False, add_lay=None, ins_override=None,
        want_plan=None):
    """One ffcb_conv; on the tensor-core arm its plan is read first and checked against ``want_plan`` before the
    launch.  Returns (output Buf, plan or None)."""
    bufs = ins_override or [load_source(lay, *case.x[s]) if lay is not None else None for s, lay in enumerate(in_lays)]
    w_tc, w_f = weight_planes(case, DEV)
    shift = case.shift.float().to(DEV) if case.shift is not None else None
    out = Buf(out_lay, DEV)
    add_t = None
    if case.addend is not None:
        if addend_alias:                       # the block's in-place residual: addend and out are one view
            out.write(case.addend, torch.zeros_like(case.addend) if out_lay.fmt == L.BF16X2 else None)
            add_t = out.t
        else:
            ab = Buf(add_lay, DEV)
            ab.write(case.addend, torch.zeros_like(case.addend) if add_lay.fmt == L.BF16X2 else None)
            add_t = ab.t
            out._addend = ab                   # keep alive
    w = w_tc if arm == L.MATH_BF16X3 else w_f
    d = make_desc(case, [b.t if b is not None else None for b in bufs], out.t, arm, w.data_ptr(),
                  shift.data_ptr() if shift is not None else None, add_t)
    pl = None
    if arm == L.MATH_BF16X3:
        pl = plan(d)
        HIT.add((pl["kind"], pl["il"], pl["po"], pl["bn"]))
        if want_plan is not None:
            assert {k: pl[k] for k in want_plan} == want_plan, pl
    L.check(L.get_lib().ffcb_conv(ctypes.byref(d), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
            "ffcb_conv")
    torch.cuda.synchronize()
    return out, pl


def check_out(out: Buf, want: torch.Tensor, pl, out_hw, what, ring=False):
    """Exact comparison of an output buffer with the float64 value ``want`` [B, Ho, Wo, N]: float32 storage holds it
    exactly, split-bf16 storage holds its round-to-nearest split (both planes); with ``ring`` the reflected ring too."""
    lay = out.lay
    if lay.fmt == L.F32:
        assert torch.equal(want.float().double(), want), "reference not exact in float32: operand budget broken"
        assert_exact(out.read()[0], want, pl, out_hw, what)
        return
    hi_w, lo_w = split_rne(want)
    hi, lo = out.read()
    assert_exact(hi, hi_w, pl, out_hw, what + " (hi plane)")
    assert_exact(lo, lo_w, pl, out_hw, what + " (lo plane)")
    if ring:
        p = lay.pad
        hi_r, lo_r = out.read(ring=True)
        assert torch.equal(hi_r, _padded(hi_w, p)) and torch.equal(lo_r, _padded(lo_w, p)), \
            what + ": reflected ring of the output differs from the reflection of the reference"


def exact_case(case: Case, in_lays, out_lay: Layout, *, want_plan: dict, fp32=True, ring=False, **kw):
    """The whole protocol of one case: the plan; the tensor-core arm with the case's weights (lo planes nonzero);
    then, when ``fp32``, both arms with the weight lo planes zeroed, equal to the reference and to each other."""
    assert_budget(case, L.MATH_BF16X3, DEV)
    out, pl = run(case, in_lays, out_lay, L.MATH_BF16X3, want_plan=want_plan, **kw)
    check_out(out, reference(case, L.MATH_BF16X3, DEV), pl, case.out_hw, "tensor-core arm", ring=ring)
    if not fp32:
        return pl
    c0 = Case(**{**case.__dict__, "w": (case.w[0], torch.zeros_like(case.w[1]))})
    assert_budget(c0, L.MATH_FP32, DEV)
    want = reference(c0, L.MATH_FP32, DEV)
    assert torch.equal(want, reference(c0, L.MATH_BF16X3, DEV))
    got = {}
    for arm in (L.MATH_BF16X3, L.MATH_FP32):
        o, p = run(c0, in_lays, out_lay, arm, **kw)
        check_out(o, want, p, c0.out_hw, f"{'tensor-core' if arm == L.MATH_BF16X3 else 'fp32'} arm, lo(W) = 0",
                  ring=ring and arm == L.MATH_BF16X3)
        got[arm] = o.read()
    assert all(torch.equal(a, b) for a, b in zip(*got.values()) if a is not None)
    return pl


def make_case(segs, src_shapes, n, out_hw, seed, *, stride=1, border=L.BORDER_REFLECT, act=L.ACT_NONE,
              shift=True, addend=False, addend_post=0, hi=(-2, 2), density=1.0):
    """Random exact operands: sources [B, H, W, C] (None: unused), weights [N, Ktot], shift, addend."""
    g = torch.Generator().manual_seed(seed)
    x = []
    for shp in src_shapes:
        if shp is None:
            x.append(None)
            continue
        h, lo = split_planes(shp, g, hi=hi)
        x.append((h, lo))
    k = sum(s.nch for s in segs)
    wh, wl = split_planes((n, k), g, hi=hi)
    if density < 1.0:
        keep = (torch.rand(n, k, generator=g) < density).double()
        wh, wl = wh * keep, wl * keep
    b = next(s for s in src_shapes if s is not None)[0]
    sh = dyadic((n,), -64, 64, g, GRID_BITS) if shift else None
    ad = dyadic((b, out_hw[0], out_hw[1], n), -8, 8, g, 2) if addend else None
    return Case(segs=segs, x=x, w=(wh, wl), n_out=n, out_hw=out_hw, stride=stride, border=border, act=act,
                shift=sh, addend=ad, addend_post=addend_post)


def g3(src=0, c0=0, nch=64):
    return [Seg(src, dy, dx, c0, nch) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]


def column(dys, c0=0, src=0):
    return [Seg(src, dy, 0, c0, 64) for dy in dys]


def cl(b, h, w, c, pad=0, reflect=1, **kw):
    """Channels-last split-bf16 view (ring of ``pad`` pixels, reflected unless reflect=0)."""
    return Layout(b, h, w, c, pad=pad, reflect=reflect if pad else 0, **kw)


def tiles(b, h, w, tw, th):
    return b * (-(-w // tw)) * (-(-h // th))


# ------------------------------------------------------------------------------------------------ flat
@pytest.mark.parametrize("n", [32, 64, 96, 160, 192, 200, 384])
def test_flat_two_sources(n):
    """B*H*W = 300: three M tiles, the second straddling the two images; N tiles of every width incl. ragged ones."""
    b, h, w = 2, 10, 15
    case = make_case([Seg(0, 0, 0, 0, 64), Seg(1, 0, 0, 32, 128)], [(b, h, w, 64), (b, h, w, 160)], n, (h, w), n)
    bn = {32: 32, 64: 64, 96: 96, 160: 128, 192: 96, 200: 128, 384: 128}[n]
    exact_case(case, [cl(b, h, w, 64), cl(b, h, w, 160, ctot=192, c_off=32)], cl(b, h, w, n),
               want_plan=dict(kind=FLAT, bn=bn, m_tiles=3, n_tiles=-(-n // bn), il=0, po=0))


@pytest.mark.parametrize("cg", [0, 4, 8])
def test_flat_tile_blocked_source(cg):
    """A tile-blocked (FourierUnit) operand next to a channels-last one; the last 128-pixel block is partly outside the
    image (NaN there, never used).  cg > 0: channel-group planar float32 output (the IL + PO instantiation)."""
    b, h, w, n = 2, 10, 15, 64
    case = make_case([Seg(0, 0, 0, 0, 64), Seg(1, 0, 0, 64, 128)], [(b, h, w, 64), (b, h, w, 192)], n, (h, w), 7 + cg)
    out = Layout(b, h, w, n, fmt=L.F32, cg=cg) if cg else cl(b, h, w, n)
    exact_case(case, [cl(b, h, w, 64), Layout(b, h, w, 192, cg=8, tile=128)], out, fp32=False,
               want_plan=dict(kind=FLAT, il=1, po=int(cg > 0)))


@pytest.mark.parametrize("cg", [4, 8])
def test_flat_planar_output(cg):
    b, h, w, n = 1, 16, 24, 96
    case = make_case([Seg(0, 0, 0, 0, 128)], [(b, h, w, 128)], n, (h, w), 20 + cg, act=L.ACT_RELU)
    exact_case(case, [cl(b, h, w, 128)], Layout(b, h, w, n, fmt=L.F32, cg=cg), fp32=False,
               want_plan=dict(kind=FLAT, il=0, po=1, bn=96))


@pytest.mark.parametrize("post", [0, 1])
def test_flat_in_place_addend(post):
    """The addend aliases the output (the residual of the block's second FFC_BN_ACT), before or after the ReLU."""
    b, h, w, n = 2, 9, 13, 128
    case = make_case([Seg(0, 0, 0, 0, 64)], [(b, h, w, 64)], n, (h, w), 30 + post, act=L.ACT_RELU, addend=True,
                     addend_post=post)
    exact_case(case, [cl(b, h, w, 64)], cl(b, h, w, n), addend_alias=True, want_plan=dict(kind=FLAT, bn=128))


def test_flat_float32_addend_view():
    b, h, w, n = 1, 8, 16, 64
    case = make_case([Seg(0, 0, 0, 0, 64)], [(b, h, w, 64)], n, (h, w), 33, act=L.ACT_RELU, addend=True)
    exact_case(case, [cl(b, h, w, 64)], Layout(b, h, w, n, fmt=L.F32), add_lay=Layout(b, h, w, n, fmt=L.F32),
               want_plan=dict(kind=FLAT))


# ------------------------------------------------------------------------------------------------ spatial per-tap
def test_spatial_w20():
    b, h, w, n = 2, 9, 20, 64
    case = make_case(g3(), [(b, h, w, 64)], n, (h, w), 40, act=L.ACT_RELU)
    exact_case(case, [cl(b, h, w, 64, pad=1)], cl(b, h, w, n),
               want_plan=dict(kind=SPATIAL, tw=32, th=4, m_tiles=tiles(b, h, w, 32, 4)))


def test_spatial_stride2_odd():
    b, h, w, n = 2, 17, 21, 128
    ho, wo = 9, 11
    case = make_case(g3(), [(b, h, w, 64)], n, (ho, wo), 41, stride=2)
    exact_case(case, [cl(b, h, w, 64, pad=1)], cl(b, ho, wo, n), want_plan=dict(kind=SPATIAL, tw=16, th=8))


def test_spatial_zero_border_phase_with_nan_ring():
    """The ConvTranspose sub-pixel phase taps (0|1, 0|1) under a zero border: the source's ring is NaN and must never
    be read."""
    b, h, w, n = 1, 8, 64, 64
    segs = [Seg(0, dy, dx, 0, 64) for dy in (0, 1) for dx in (0, 1)]
    case = make_case(segs, [(b, h, w, 64)], n, (h, w), 42, border=L.BORDER_ZERO, act=L.ACT_RELU)
    exact_case(case, [cl(b, h, w, 64, pad=1, reflect=0)], cl(b, h, w, n), want_plan=dict(kind=SPATIAL, tw=64, th=2))


def test_spatial_pad2_ring_read_at_reach1_and_1x1_segment():
    """A reflect ring of 2 pixels read by a 3x3 (reach 1), plus a 1x1 segment over other channels of the source."""
    b, h, w, n = 1, 11, 18, 64
    segs = g3() + [Seg(0, 0, 0, 64, 64)]
    case = make_case(segs, [(b, h, w, 128)], n, (h, w), 43)
    exact_case(case, [cl(b, h, w, 128, pad=2)], cl(b, h, w, n), want_plan=dict(kind=SPATIAL, tw=32, th=4))


@pytest.mark.parametrize("w", [64, 32])
def test_spatial_tile_blocked_source(w):
    """convl2g + st.conv2: a 3x3 group over a ring-padded source plus a 1x1 segment over a tile-blocked one."""
    b, h, n = 1, 256 // w, 128
    case = make_case(g3() + [Seg(1, 0, 0, 0, 64)], [(b, h, w, 64), (b, h, w, 64)], n, (h, w), 44 + w)
    exact_case(case, [cl(b, h, w, 64, pad=1), Layout(b, h, w, 64, cg=8, tile=128)], cl(b, h, w, n), fp32=False,
               want_plan=dict(kind=SPATIAL, il=1, tw=w, th=128 // w))


def test_spatial_w200_stride2_box_limit():
    b, h, w, n = 1, 5, 400, 32
    case = make_case(g3(), [(b, h, w, 64)], n, (3, 200), 46, stride=2)
    exact_case(case, [cl(b, h, w, 64, pad=1)], cl(b, 3, 200, n), want_plan=dict(kind=SPATIAL, tw=128, th=1))


# ------------------------------------------------------------------------------------------------ column halo
@pytest.mark.parametrize("w,h", [(33, 5), (64, 7), (100, 5), (130, 9)])
def test_halo_split_output_with_ring(w, h):
    b, n = 2, 64
    case = make_case(g3(), [(b, h, w, 64)], n, (h, w), 50 + w, act=L.ACT_RELU)
    exact_case(case, [cl(b, h, w, 64, pad=1)], cl(b, h, w, n, pad=1), ring=True,
               want_plan=dict(kind=HALO, tw=64, th=2, ring=1, m_tiles=tiles(b, h, w, 64, 2)))


@pytest.mark.parametrize("groups", [2, 3])
def test_halo_groups_and_trailing_one_tap(groups):
    b, h, w, n = 1, 5, 72, 128
    c = 64 * groups + 64
    segs = [s for i in range(groups) for s in g3(0, 64 * i)] + [Seg(0, 0, 0, 64 * groups, 64)]
    case = make_case(segs, [(b, h, w, c)], n, (h, w), 60 + groups)
    exact_case(case, [cl(b, h, w, c, pad=1)], cl(b, h, w, n), want_plan=dict(kind=HALO, bn=128))


def test_halo_k_tail_nch40():
    """nch = 40: the K block reaches 24 channels past the view (C = 40 in a 64-channel buffer, NaN there): outside
    the view the box is zero-filled."""
    b, h, w, n = 1, 4, 64, 64
    case = make_case(g3(nch=40), [(b, h, w, 40)], n, (h, w), 64)
    exact_case(case, [cl(b, h, w, 40, pad=1, ctot=64)], cl(b, h, w, n), want_plan=dict(kind=HALO))


# ------------------------------------------------------------------------------------------------ rows-resident
@pytest.mark.parametrize("n", [24, 64, 96, 128])
def test_rows_three_taps(n):
    b, h, w = 2, 20, 12
    case = make_case(column((-1, 0, 1)), [(b, h, w, 64)], n, (h, w), 70 + n)
    exact_case(case, [cl(b, h, w, 64, pad=1)], cl(b, h, w, n),
               want_plan=dict(kind=ROWS, tw=8, th=16, m_tiles=tiles(b, h, w, 8, 16)))


@pytest.mark.parametrize("n", [24, 64])
def test_rows_seven_taps(n):
    """The head's row contraction (dy = -3..3 over a 3-pixel reflected ring)."""
    b, h, w = 2, 21, 13
    case = make_case(column(range(-3, 4)), [(b, h, w, 64)], n, (h, w), 80 + n)
    exact_case(case, [cl(b, h, w, 64, pad=3)], cl(b, h, w, n, fmt=L.F32), want_plan=dict(kind=ROWS))


def test_rows_gate_with_planar_output():
    """Three dy-only taps of one 64-channel block into a channel-group planar float32 output: the rows-resident
    instantiation has no planar epilogue, so the plan is per-tap with the PO instantiation."""
    b, h, w, n = 1, 16, 16, 64
    case = make_case(column((-1, 0, 1)), [(b, h, w, 64)], n, (h, w), 90)
    exact_case(case, [cl(b, h, w, 64, pad=1)], Layout(b, h, w, n, fmt=L.F32, cg=4), fp32=False,
               want_plan=dict(kind=SPATIAL, po=1))


def test_rows_seven_taps_n128_falls_back_to_per_tap():
    """Seven resident weight tiles at N = 128 leave no room for two halo stages: per-tap (the launch used to fail)."""
    b, h, w, n = 1, 16, 16, 128
    case = make_case(column(range(-3, 4)), [(b, h, w, 64)], n, (h, w), 91)
    exact_case(case, [cl(b, h, w, 64, pad=3)], cl(b, h, w, n), want_plan=dict(kind=SPATIAL, bn=128))


# ------------------------------------------------------------------------------------------------ persistence
PERSIST = [
    ("flat", [Seg(0, 0, 0, 0, 64)], (2, 128, 128, 64), 384, dict(kind=FLAT, m_tiles=256, n_tiles=3), 0, 0),
    ("spatial", g3(), (4, 300, 20, 64), 200, dict(kind=SPATIAL, m_tiles=300, n_tiles=2), 1, 1),
    ("halo", g3(), (2, 64, 130, 64), 384, dict(kind=HALO, m_tiles=192, n_tiles=3), 1, 1),
    ("rows", column((-1, 0, 1)), (6, 100, 100, 64), 64, dict(kind=ROWS, m_tiles=546, n_tiles=1), 1, 1),
]


@pytest.mark.parametrize("name,segs,shape,n,want,pad,ring", PERSIST, ids=[p[0] for p in PERSIST])
def test_persistence_many_tiles_per_cta(name, segs, shape, n, want, pad, ring):
    """More than 4 x 132 tiles: every CTA wraps its stage ring and barrier phases many times."""
    b, h, w, c = shape
    case = make_case(segs, [shape], n, (h, w), 100 + len(name), act=L.ACT_RELU)
    pl = exact_case(case, [cl(b, h, w, c, pad=pad)], cl(b, h, w, n, pad=ring), fp32=False, ring=bool(ring),
                    want_plan=want)
    assert pl["m_tiles"] * pl["n_tiles"] > 4 * 132


# ------------------------------------------------------------------------------------------------ knobs, coverage
# one descriptor per instantiation (kind, il, po): every N tile must give the same bits, equal to the reference
CONFIGS = {
    "flat": (lambda b, h, w: ([Seg(0, 0, 0, 0, 64)], [cl(b, h, w, 64), None], cl(b, h, w, 128)), FLAT, 0, 0),
    "flat_po": (lambda b, h, w: ([Seg(0, 0, 0, 0, 64)], [cl(b, h, w, 64), None], Layout(b, h, w, 128, fmt=L.F32, cg=8)),
                FLAT, 0, 1),
    "flat_il": (lambda b, h, w: ([Seg(1, 0, 0, 0, 64)], [None, Layout(b, h, w, 64, cg=8, tile=128)], cl(b, h, w, 128)),
                FLAT, 1, 0),
    "flat_il_po": (lambda b, h, w: ([Seg(1, 0, 0, 0, 64)], [None, Layout(b, h, w, 64, cg=8, tile=128)],
                                    Layout(b, h, w, 128, fmt=L.F32, cg=8)), FLAT, 1, 1),
    "spatial": (lambda b, h, w: (g3(), [cl(b, h, w, 64, pad=1), None], cl(b, h, w, 128)), SPATIAL, 0, 0),
    "spatial_po": (lambda b, h, w: (g3(), [cl(b, h, w, 64, pad=1), None], Layout(b, h, w, 128, fmt=L.F32, cg=4)),
                   SPATIAL, 0, 1),
    "spatial_il": (lambda b, h, w: (g3() + [Seg(1, 0, 0, 0, 64)],
                                    [cl(b, h, w, 64, pad=1), Layout(b, h, w, 64, cg=8, tile=128)], cl(b, h, w, 128)),
                   SPATIAL, 1, 0),
    "spatial_il_po": (lambda b, h, w: (g3() + [Seg(1, 0, 0, 0, 64)],
                                       [cl(b, h, w, 64, pad=1), Layout(b, h, w, 64, cg=8, tile=128)],
                                       Layout(b, h, w, 128, fmt=L.F32, cg=8)), SPATIAL, 1, 1),
    "rows": (lambda b, h, w: (column((-1, 0, 1)), [cl(b, h, w, 64, pad=1), None], cl(b, h, w, 128)), ROWS, 0, 0),
    "halo": (lambda b, h, w: (g3(), [cl(b, h, w, 64, pad=1), None], cl(b, h, w, 128, pad=1)), HALO, 0, 0),
}
SHAPES = {"flat": (2, 6, 32), "spatial": (2, 8, 32), "rows": (2, 20, 12), "halo": (1, 5, 64)}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_knob_invariance(name, monkeypatch):
    """FFCB_TC_BN in {32, 64, 96, 128} (and for the rows-resident case FFCB_TC_ROWS in {0, 1}, FFCB_TC_ROWS_TW in
    {8, 16}): the same bits, equal to the reference, whatever the tiling."""
    make, kind, il, po = CONFIGS[name]
    b, h, w = SHAPES[name.split("_")[0]]
    segs, lays, out_lay = make(b, h, w)
    shapes = [(b, h, w, lay.C) if lay is not None else None for lay in lays]
    case = make_case(segs, shapes, 128, (h, w), 200 + len(name), act=L.ACT_RELU)
    assert_budget(case, L.MATH_BF16X3, DEV)
    want = reference(case, L.MATH_BF16X3, DEV)
    bufs = [load_source(lay, *case.x[s]) if lay is not None else None for s, lay in enumerate(lays)]
    settings = [{"FFCB_TC_BN": str(bn)} for bn in (32, 64, 96, 128)]
    if kind == ROWS:
        settings += [{"FFCB_TC_BN": "128", "FFCB_TC_ROWS": "0"}, {"FFCB_TC_ROWS_TW": "16"},
                     {"FFCB_TC_ROWS": "1", "FFCB_TC_ROWS_TW": "8"}]
    first = None
    for env in settings:
        for k in KNOBS:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        out, pl = run(case, lays, out_lay, L.MATH_BF16X3, ins_override=bufs)
        want_kind = kind
        if kind == ROWS and (env.get("FFCB_TC_ROWS") == "0" or pl["n_tiles"] > 1):
            want_kind = SPATIAL          # rows-resident needs one N tile (and the mode enabled)
        assert (pl["kind"], pl["il"], pl["po"]) == (want_kind, il, po), (env, pl)
        if "FFCB_TC_BN" in env:
            assert pl["bn"] == int(env["FFCB_TC_BN"])
        if kind == ROWS and pl["kind"] == ROWS:
            assert pl["tw"] == int(env.get("FFCB_TC_ROWS_TW", "8"))
        check_out(out, want, pl, (h, w), f"{name} under {env}", ring=out_lay.pad == 1)
        bits = out.read()
        if first is None:
            first = bits
        assert all(torch.equal(a, c) for a, c in zip(first, bits) if a is not None), env


# ------------------------------------------------------------------------------------------------ activations
@pytest.mark.parametrize("act", [L.ACT_SIGMOID, L.ACT_TANH])
@pytest.mark.parametrize("kind", ["flat", "halo"])
def test_sigmoid_tanh_epilogue(act, kind):
    """The exact pre-activation through the epilogue's slow_act, against the float64 activation, within the ulp
    bound of conv_exact.act_ulp_bound (derived from the documented errors of __expf, __fdividef and tanhf)."""
    b, h, w, n = 1, 6, 64, 64
    segs = [Seg(0, 0, 0, 0, 64)] if kind == "flat" else g3()
    case = make_case(segs, [(b, h, w, 64)], n, (h, w), 300 + act, act=act, hi=(-1, 1), density=0.08)
    assert_budget(case, L.MATH_BF16X3, DEV)
    out, _ = run(case, [cl(b, h, w, 64, pad=1 if kind == "halo" else 0)], Layout(b, h, w, n, fmt=L.F32),
                 L.MATH_BF16X3, want_plan=dict(kind=FLAT if kind == "flat" else HALO))
    pre = contraction(case, L.MATH_BF16X3, device=DEV) + case.shift.to(DEV)
    assert float(pre.abs().max()) > 2, "pre-activations should span the nonlinear range"
    ref = reference(case, L.MATH_BF16X3, DEV)
    got = out.read()[0]
    err = (got - ref).abs()
    bound = act_ulp_bound(act, pre, ref)
    worst = int((err - bound).argmax())
    assert bool((err <= bound).all()), (f"|err| {float(err.view(-1)[worst]):.3g} > bound {float(bound.view(-1)[worst]):.3g} "
                                        f"at pre-activation {float(pre.view(-1)[worst])}")


# ------------------------------------------------------------------------------------------------ sentinels
def test_channels_beyond_the_view_and_zero_border_ring_are_never_read():
    """NaN in the channels of a wider buffer outside the views (both sources) and in a zero-border source's ring:
    the output is still exact."""
    b, h, w, n = 1, 8, 20, 64
    segs = [Seg(0, dy, dx, 0, 64) for dy in (0, 1) for dx in (0, 1)] + [Seg(1, 0, 0, 0, 32)]
    case = make_case(segs, [(b, h, w, 64), (b, h, w, 32)], n, (h, w), 400, border=L.BORDER_ZERO)
    exact_case(case, [cl(b, h, w, 64, pad=1, reflect=0, ctot=192, c_off=64), cl(b, h, w, 32, ctot=96, c_off=32)],
               cl(b, h, w, n, ctot=128, c_off=64), want_plan=dict(kind=SPATIAL))


def test_uncovered_channels_inside_the_view_are_read():
    """A segment of 40 channels of a 48-channel view: the tensor-core arm multiplies the whole 64-channel block, so
    channels 40..47 are read (times zero weights) — finite values there leave the result exact, a NaN there reaches
    the output (include/ffc_b200.h says so)."""
    b, h, w, n = 1, 4, 64, 64
    case = make_case([Seg(0, 0, 0, 0, 40)], [(b, h, w, 48)], n, (h, w), 401)
    lay = cl(b, h, w, 48)
    exact_case(case, [lay], cl(b, h, w, n), want_plan=dict(kind=FLAT))
    src = load_source(lay, *case.x[0])
    src.store[lay.index(device=DEV)[..., 40:48]] = float("nan")
    out, _ = run(case, [lay], cl(b, h, w, n), L.MATH_BF16X3, ins_override=[src, None])
    assert bool(torch.isnan(out.read()[0]).all())


# ------------------------------------------------------------------------------------------------ sensitivity
def test_exact_check_sees_one_lo_step_the_relative_bound_does_not():
    """A 3x3 over 512 channels (K = 4608) with ONE weight lo element off by one lo-grid step (2^-6): the exact check
    names the output channel it feeds, while max|err| / max|ref| stays under the suite's usual 2e-4."""
    b, h, w, n = 1, 4, 64, 64
    segs = g3(nch=512)
    case = make_case(segs, [(b, h, w, 512)], n, (h, w), 500)
    assert_budget(case, L.MATH_BF16X3, DEV)
    want = reference(case, L.MATH_BF16X3, DEV)
    n0, k0 = 37, 9 * 512 // 2 + 3
    bad = Case(**{**case.__dict__, "w": (case.w[0], case.w[1].clone())})
    bad.w[1][n0, k0] += 2.0 ** -GRID_BITS
    out, pl = run(bad, [cl(b, h, w, 512, pad=1)], Layout(b, h, w, n, fmt=L.F32), L.MATH_BF16X3)
    got = out.read()[0]
    with pytest.raises(AssertionError, match=rf"\(b, y, x, n\) = \(\d+, \d+, \d+, {n0}\)"):
        assert_exact(got, want, pl, (h, w), "perturbed weight")
    assert rel_err(got, want) <= 2e-4
    assert torch.equal(got, reference(bad, L.MATH_BF16X3, DEV))


# ------------------------------------------------------------------------------------------------ the 7x7 shell
# ReflectionPad2d(3) + Conv2d(k7) of the stem (ffc.py:315-317) and the head (ffc.py:360-363), every entry point against
# the float64 convolution.  The tensor-core arm drops lA*lW, so each tensor-core case runs twice: activation lo planes
# with bf16-exact weights, then weight lo planes with bf16-exact activations — both times the three products are the
# whole product.  Values a + c*2^-9 with a = +-1 split into hi = a, lo = c*2^-9 (round to nearest), so a lo plane is
# what ffcb_stem_pack and P.split_bf16 produce themselves.
def conv7_ref(x_nchw, w, bias=None):
    """float64 ReflectionPad2d(3) + conv7 (+ per-channel bias), NCHW."""
    y = torch.nn.functional.conv2d(torch.nn.functional.pad(x_nchw.double(), (3, 3, 3, 3), mode="reflect"), w.double())
    return y if bias is None else y + bias.double().view(1, -1, 1, 1)


def shell_values(shape, g, lo_bits):
    """(value, hi, lo): value = a + c*2^-lo_bits, a in {-1, 1} (lo_bits 9: below half a bf16 ulp of 1, so hi = a and
    lo = c*2^-9) or, with lo_bits None, a in {-1, 0, 1} and no lo part."""
    if lo_bits is None:
        a = dyadic(shape, -1, 1, g)
        return a, a, torch.zeros_like(a)
    a = dyadic(shape, 0, 1, g) * 2 - 1
    c = dyadic(shape, -1, 1, g, lo_bits)
    return a + c, a, c


def shell_budget(xs, ws, shift=None):
    """Budget of a 7x7 contraction of the tensor-core arm: (hi, lo) planes NCHW / [N, C, 7, 7]."""
    g = product_grid(xs[0], xs[1], ws[0], ws[1], L.MATH_BF16X3)
    tot = sum(conv7_ref(a.abs(), w.abs()) for a, w in ((xs[0], ws[0]), (xs[1], ws[0]), (xs[0], ws[1])))
    if shift is not None:
        g = max(g, grid_exp(shift))
        tot = tot + shift.abs().view(1, -1, 1, 1)
    budget_check(tot, g)


def shell_desc(pk, in_t, out_t, w_split, shift):
    case = Case(segs=[Seg(s.src, s.dy, s.dx, s.c0, s.nch) for s in pk.segs], x=[], w=(None, None), n_out=pk.n_out,
                out_hw=(out_t.H, out_t.W), stride=pk.stride, border=pk.border, act=pk.act)
    return make_desc(case, [in_t, None], out_t, L.MATH_BF16X3, w_split.data_ptr(),
                     shift.data_ptr() if shift is not None else None)


def launch_conv(d, want_plan):
    pl = plan(d)
    HIT.add((pl["kind"], pl["il"], pl["po"], pl["bn"]))
    assert {k: pl[k] for k in want_plan} == want_plan, pl
    L.check(L.get_lib().ffcb_conv(ctypes.byref(d), None), "ffcb_conv")
    return pl


@pytest.mark.parametrize("lo_side", ["activations", "weights"])
@pytest.mark.parametrize("cin", [3, 4, 5, 8])
def test_stem_pack_then_windowed_rows_resident_conv(cin, lo_side):
    """ffcb_stem_pack + the windowed rows-resident ffcb_conv (P.pack_stem_windowed: four two-row segments for Cin <= 4,
    seven for Cin 5..8) + shift + ReLU into a split-bf16 output with its reflected ring."""
    b, h, w, n = 2, 21, 37, 64
    g = torch.Generator().manual_seed(600 + cin)
    x, xh, xl = shell_values((b, cin, h, w), g, 9 if lo_side == "activations" else None)
    wt, wh, wl = shell_values((n, cin, 7, 7), g, 9 if lo_side == "weights" else None)
    shift = dyadic((n,), -64, 64, g, GRID_BITS)
    shell_budget((xh, xl), (wh, wl), shift)
    pk = P.pack_stem_windowed(wt.float(), torch.ones(n), shift.float(), device=DEV)
    w_split = pk.split_weights()
    packed = Buf(Layout(b, h + 6, w + 8, 8), DEV)
    x_d = x.float().to(DEV).contiguous()
    L.check(L.get_lib().ffcb_stem_pack(x_d.data_ptr(), b, cin, h, w, ctypes.byref(packed.t), None), "ffcb_stem_pack")
    win = packed.t                       # pixel x exposes the 8 taps x 8 channels starting at packed pixel x
    win.W, win.C, win.window = w, 64, 1
    out = Buf(cl(b, h, w, n, pad=1), DEV)
    pl = launch_conv(shell_desc(pk, win, out.t, w_split, pk.shift), dict(kind=ROWS, bn=64, ring=1))
    torch.cuda.synchronize()
    want = conv7_ref(x, wt, shift).clamp_min(0).permute(0, 2, 3, 1).to(DEV)
    check_out(out, want, pl, (h, w), f"stem Cin={cin}, lo planes in the {lo_side}", ring=True)


@pytest.mark.parametrize("lo_side", ["activations", "weights"])
def test_head_row_contraction_then_gather(lo_side):
    """P.pack_head_rows' rows-resident contraction (dy = -3..3 over a 3-pixel reflected ring) into the float32 partial
    sums q, then ffcb_head_gather7 over the whole plane and ffcb_head_gather7_rows over two row bands: the same output,
    equal to the float64 ReflectionPad2d(3) + conv7 + bias.  W = 131: the gather crosses its 128-column tiles."""
    b, c, h, w, n = 2, 64, 19, 131, 3
    g = torch.Generator().manual_seed(700)
    x, xh, xl = shell_values((b, c, h, w), g, 9 if lo_side == "activations" else None)
    wt, wh, wl = shell_values((n, c, 7, 7), g, 9 if lo_side == "weights" else None)
    bias = dyadic((n,), -64, 64, g, GRID_BITS)
    shell_budget((xh, xl), (wh, wl), bias)
    pk = P.pack_head_rows(wt.float(), device=DEV)
    X = Buf(cl(b, h, w, c, pad=3), DEV)
    X.write(_padded(xh.permute(0, 2, 3, 1), 3), _padded(xl.permute(0, 2, 3, 1), 3), ring=True)
    Q = Buf(Layout(b, h, w, pk.n_out, fmt=L.F32), DEV)
    launch_conv(shell_desc(pk, X.t, Q.t, pk.split_weights(), None), dict(kind=ROWS, bn=32))
    bias_d = bias.float().to(DEV)
    lib = L.get_lib()
    y = torch.full((b, n, h, w), float("nan"), device=DEV)
    L.check(lib.ffcb_head_gather7(ctypes.byref(Q.t), bias_d.data_ptr(), n, L.ACT_NONE, y.data_ptr(), None),
            "ffcb_head_gather7")
    y_rows = torch.full_like(y, float("nan"))
    for r0, r1 in ((0, 8), (8, h)):
        band = Q.t
        band.ptr += r0 * band.sy * 4
        band.H = r1 - r0
        L.check(lib.ffcb_head_gather7_rows(ctypes.byref(band), bias_d.data_ptr(), n, L.ACT_NONE, y_rows.data_ptr(), h,
                                           r0, None), "ffcb_head_gather7_rows")
    torch.cuda.synchronize()
    want = conv7_ref(x, wt, bias).to(DEV)
    assert torch.equal(want.float().double(), want)
    assert_exact(y.double().permute(0, 2, 3, 1), want.permute(0, 2, 3, 1), None, (h, w), "ffcb_head_gather7")
    assert_exact(y_rows.double().permute(0, 2, 3, 1), want.permute(0, 2, 3, 1), None, (h, w),
                 "ffcb_head_gather7_rows")


def fp32_values(shape, g):
    """a + c*2^-4, a, c in {-1, 0, 1}: exact float32 operands of the fp32 shell kernels (products on a 2^-8 grid)."""
    return dyadic(shape, -1, 1, g) + dyadic(shape, -1, 1, g, 4)


@pytest.mark.parametrize("cin", [4, 8])
def test_fp32_stem_conv7(cin):
    b, h, w, n = 2, 21, 37, 64
    g = torch.Generator().manual_seed(800 + cin)
    x, wt = fp32_values((b, cin, h, w), g), fp32_values((n, cin, 7, 7), g)
    shift = dyadic((n,), -64, 64, g, GRID_BITS)
    budget_check(conv7_ref(x.abs(), wt.abs()) + shift.abs().view(1, -1, 1, 1),
                 max(grid_exp(x) + grid_exp(wt), grid_exp(shift)))
    w_kn, sh = P.pack_stem(wt.float(), torch.ones(n), shift.float(), device=DEV)
    out = Buf(Layout(b, h, w, n, fmt=L.F32), DEV)
    x_d = x.float().to(DEV).contiguous()
    L.check(L.get_lib().ffcb_stem_conv7(x_d.data_ptr(), b, cin, h, w, w_kn.data_ptr(), sh.data_ptr(), n,
                                        ctypes.byref(out.t), None), "ffcb_stem_conv7")
    torch.cuda.synchronize()
    want = conv7_ref(x, wt, shift).clamp_min(0).permute(0, 2, 3, 1).to(DEV)
    check_out(out, want, None, (h, w), f"ffcb_stem_conv7 Cin={cin}")


def test_fp32_head_conv7():
    """ffcb_head_conv7 over a split-bf16 channels-last input (hi + lo read as one float32)."""
    b, c, h, w, n = 2, 64, 19, 37, 3
    g = torch.Generator().manual_seed(900)
    xh, xl = dyadic((b, c, h, w), -1, 1, g), dyadic((b, c, h, w), -1, 1, g, 4)
    wt = fp32_values((n, c, 7, 7), g)
    bias = dyadic((n,), -64, 64, g, GRID_BITS)
    budget_check(conv7_ref((xh + xl).abs(), wt.abs()) + bias.abs().view(1, -1, 1, 1),
                 max(grid_exp(xh + xl) + grid_exp(wt), grid_exp(bias)))
    X = Buf(cl(b, h, w, c), DEV)
    X.write(xh.permute(0, 2, 3, 1), xl.permute(0, 2, 3, 1))
    w_d, b_d = P.pack_head(wt.float(), bias.float(), device=DEV)
    y = torch.full((b, n, h, w), float("nan"), device=DEV)
    L.check(L.get_lib().ffcb_head_conv7(ctypes.byref(X.t), w_d.data_ptr(), b_d.data_ptr(), n, L.ACT_NONE,
                                        y.data_ptr(), None), "ffcb_head_conv7")
    torch.cuda.synchronize()
    want = conv7_ref(xh + xl, wt, bias).to(DEV)
    assert torch.equal(want.float().double(), want)
    assert_exact(y.double().permute(0, 2, 3, 1), want.permute(0, 2, 3, 1), None, (h, w), "ffcb_head_conv7")


# ------------------------------------------------------------------------------------------------ coverage
def _launchable():
    """(kind, il, po, bn) that conv_tc()'s launch_bn can start: flat and spatial per-tap with either operand kind and
    either output kind, rows-resident and column-halo with channels-last operands and outputs, each at four N tiles."""
    combos = set()
    for bn in (32, 64, 96, 128):
        for kind in (FLAT, SPATIAL):
            combos |= {(kind, il, po, bn) for il in (0, 1) for po in (0, 1)}
        combos |= {(ROWS, 0, 0, bn), (HALO, 0, 0, bn)}
    return combos


def _n_params(fn) -> int:
    n = 1
    for m in getattr(fn, "pytestmark", []):
        if m.name == "parametrize":
            n *= len(m.args[1])
    return n


def test_every_instantiation_was_launched(request):
    """Runs last: the cases above launched every instantiation x N tile (a gate change that moves a case to another
    path fails the case's plan assertion; one that drops a path altogether fails here).  The launches are collected
    by the cases themselves, so this only judges a session that selected and ran the whole module."""
    mod = request.module
    tests = {name: fn for name, fn in vars(mod).items() if name.startswith("test_") and callable(fn)
             and fn is not test_every_instantiation_was_launched}
    mine = [it for it in request.session.items if it.module is mod and it.originalname in tests]
    selected = {name: sum(it.originalname == name for it in mine) for name in tests}
    if any(selected[name] != _n_params(fn) for name, fn in tests.items()) or not {it.nodeid for it in mine} <= RAN:
        pytest.skip("only part of this module was selected or run: its launches do not cover the instantiations")
    missing = _launchable() - HIT
    assert not missing, f"never launched: {sorted(missing)}"
