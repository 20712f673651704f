"""CPU-only: the dispatch of the tensor-core contraction (ffcb_conv_plan) on every gate boundary of conv_tc() — which
instantiation (flat / spatial per-tap / rows-resident / column-halo, tile-blocked operands, planar output) and which
tiling a descriptor gets.  The plan is the step ffcb_conv itself runs before it launches, so these are the launches.
No device call is made: descriptors carry placeholder pointers."""
import ctypes

import pytest

from conv_exact import FAKE_PTR, Case, Layout, Seg, make_desc, plan

from lama_b200 import _lib as L

FLAT, SPATIAL, ROWS, HALO = L.PLAN_FLAT, L.PLAN_SPATIAL, L.PLAN_ROWS, L.PLAN_HALO


@pytest.fixture(scope="module", autouse=True)
def lib():
    import __graft_entry__ as ge
    ge.build()
    return L.get_lib()


@pytest.fixture(autouse=True)
def _no_knobs(monkeypatch):
    for k in ("FFCB_TC_BN", "FFCB_TC_ROWS", "FFCB_TC_ROWS_TW"):
        monkeypatch.delenv(k, raising=False)


def g3(src=0, c0=0, nch=64):
    """A complete 3x3 group (pad 1)."""
    return [Seg(src, dy, dx, c0, nch) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]


def column(dys, c0=0, src=0, dx=0):
    return [Seg(src, dy, dx, c0, 64) for dy in dys]


def desc(segs, n, out_hw, ins, *, b=1, stride=1, border=L.BORDER_REFLECT, out=None):
    """Descriptor over placeholder pointers; ``ins[s]`` = Layout of source s."""
    case = Case(segs=segs, x=[], w=(None, None), n_out=n, out_hw=out_hw, stride=stride, border=border)
    out = out or Layout(b, out_hw[0], out_hw[1], n, fmt=L.BF16X2)
    return make_desc(case, [lay.tensor(FAKE_PTR) if lay else None for lay in ins], out.tensor(FAKE_PTR << 1),
                     L.MATH_BF16X3, FAKE_PTR << 2)


def ring(b, h, w, c, pad=1):
    return Layout(b, h, w, c, pad=pad, reflect=1)


def tiles(b, h, w, tw, th):
    return b * (-(-w // tw)) * (-(-h // th))


# (id, descriptor factory, expected plan fields)
CASES = [
    # flat: B*H*W = 300 pixels -> 3 M tiles straddling the two images
    ("flat_ragged", lambda: desc([Seg(0, 0, 0, 0, 64)], 64, (10, 15), [Layout(2, 10, 15, 64)], b=2),
     dict(kind=FLAT, bn=64, tw=128, th=1, m_tiles=3, n_tiles=1, il=0, po=0)),
    # W = 32: the 3x3 group stays per-tap (TW 32 x TH 4); W = 33: column-halo (64 x 2)
    ("w32_per_tap", lambda: desc(g3(), 128, (8, 32), [ring(1, 8, 32, 64)]),
     dict(kind=SPATIAL, tw=32, th=4, m_tiles=2, bn=128)),
    ("w33_halo", lambda: desc(g3(), 128, (8, 33), [ring(1, 8, 33, 64)]),
     dict(kind=HALO, tw=64, th=2, m_tiles=4, bn=128, ring=0)),
    ("halo_ring_out", lambda: desc(g3(), 64, (7, 100), [ring(2, 7, 100, 64)], b=2,
                                    out=Layout(2, 7, 100, 64, pad=1, reflect=1)),
     dict(kind=HALO, ring=1, m_tiles=tiles(2, 7, 100, 64, 2))),
    # rows-resident needs three or more dy-only taps of one 64-channel block ...
    ("rows_nseg2", lambda: desc(column((-1, 0)), 64, (16, 16), [ring(1, 16, 16, 64)]), dict(kind=SPATIAL)),
    ("rows_nseg3", lambda: desc(column((-1, 0, 1)), 64, (16, 16), [ring(1, 16, 16, 64)]),
     dict(kind=ROWS, tw=8, th=16, m_tiles=2, bn=64)),
    # ... within a dy span of 8 (zero border: no ring needed for the reach)
    ("rows_span8", lambda: desc(column(range(9)), 32, (16, 16), [Layout(1, 16, 16, 64)], border=L.BORDER_ZERO),
     dict(kind=ROWS, bn=32)),
    ("rows_span9", lambda: desc(column((0, 1, 9)), 32, (16, 16), [Layout(1, 16, 16, 64)], border=L.BORDER_ZERO),
     dict(kind=SPATIAL)),
    # ... and one N tile: N = 128 fits, N = 136 takes two
    ("rows_n128", lambda: desc(column((-1, 0, 1)), 128, (20, 12), [ring(2, 20, 12, 64)], b=2),
     dict(kind=ROWS, bn=128, n_tiles=1, m_tiles=tiles(2, 20, 12, 8, 16))),
    ("rows_n136", lambda: desc(column((-1, 0, 1)), 136, (20, 12), [ring(2, 20, 12, 64)], b=2),
     dict(kind=SPATIAL, bn=128, n_tiles=2)),
    # ... and its resident weights plus two halo stages must fit in shared memory (7 taps: N <= 64)
    ("rows_7tap_n64", lambda: desc(column(range(-3, 4)), 64, (16, 16), [ring(1, 16, 16, 64, pad=3)]),
     dict(kind=ROWS, bn=64, stages=2)),
    ("rows_7tap_n96", lambda: desc(column(range(-3, 4)), 96, (16, 16), [ring(1, 16, 16, 64, pad=3)]),
     dict(kind=SPATIAL, bn=96)),
    ("rows_7tap_n128", lambda: desc(column(range(-3, 4)), 128, (16, 16), [ring(1, 16, 16, 64, pad=3)]),
     dict(kind=SPATIAL, bn=128)),
    # rows-resident has no planar epilogue: a planar output takes the per-tap path with the PO instantiation
    ("rows_planar_out", lambda: desc(column((-1, 0, 1)), 64, (16, 16), [ring(1, 16, 16, 64)],
                                      out=Layout(1, 16, 16, 64, fmt=L.F32, cg=4)),
     dict(kind=SPATIAL, po=1, tw=16, th=8)),
    # N tiles
    ("n192_bn96", lambda: desc([Seg(0, 0, 0, 0, 64)], 192, (8, 16), [Layout(1, 8, 16, 64)]),
     dict(kind=FLAT, bn=96, n_tiles=2)),
    ("n200_bn128", lambda: desc([Seg(0, 0, 0, 0, 64)], 200, (8, 16), [Layout(1, 8, 16, 64)]),
     dict(kind=FLAT, bn=128, n_tiles=2)),
    ("n24_bn32", lambda: desc([Seg(0, 0, 0, 0, 64)], 24, (8, 16), [Layout(1, 8, 16, 64)]),
     dict(kind=FLAT, bn=32, n_tiles=1)),
    ("n384_bn128", lambda: desc([Seg(0, 0, 0, 0, 64)], 384, (8, 16), [Layout(1, 8, 16, 64)]),
     dict(kind=FLAT, bn=128, n_tiles=3)),
    # stride 2 and the zero-border sub-pixel phases stay per-tap, whatever the width
    ("stride2", lambda: desc(g3(), 128, (8, 32), [ring(1, 17, 65, 64)], stride=2),
     dict(kind=SPATIAL, tw=32, th=4)),
    ("stride2_w200", lambda: desc(g3(), 64, (4, 200), [ring(1, 8, 400, 64)], stride=2),
     dict(kind=SPATIAL, tw=128, th=1)),
    ("zero_border_phase", lambda: desc([Seg(0, dy, dx, 0, 64) for dy in (0, 1) for dx in (0, 1)], 64, (8, 64),
                                        [Layout(1, 8, 64, 64)], border=L.BORDER_ZERO),
     dict(kind=SPATIAL, tw=64, th=2)),
    ("w20_per_tap", lambda: desc(g3(), 64, (9, 20), [ring(1, 9, 20, 64)]), dict(kind=SPATIAL, tw=32, th=4)),
    # a 1x1 segment of the same ring-padded source next to a 3x3 group: a one-tap group of the halo mode
    ("halo_1x1_tail", lambda: desc(g3() + [Seg(0, 0, 0, 64, 64)], 64, (8, 64), [ring(1, 8, 64, 128)]),
     dict(kind=HALO)),
    # tile-blocked second source: spatial per-tap with M tiles of whole rows at W = 64 ...
    ("il_spatial_w64", lambda: desc(g3() + [Seg(1, 0, 0, 0, 64)], 128, (64, 64),
                                     [ring(1, 64, 64, 64), Layout(1, 64, 64, 64, cg=8, tile=128)]),
     dict(kind=SPATIAL, il=1, tw=64, th=2)),
    ("il_flat", lambda: desc([Seg(0, 0, 0, 0, 64), Seg(1, 0, 0, 0, 64)], 64, (10, 15),
                             [Layout(2, 10, 15, 64), Layout(2, 10, 15, 64, cg=8, tile=128)], b=2,
                             out=Layout(2, 10, 15, 64, fmt=L.F32, cg=8)),
     dict(kind=FLAT, il=1, po=1)),
]


@pytest.mark.parametrize("name,make,want", CASES, ids=[c[0] for c in CASES])
def test_plan_table(name, make, want):
    got = plan(make())
    assert {k: got[k] for k in want} == want, got


def test_tile_blocked_spatial_source_at_w48_is_refused_like_ffcb_conv():
    """W = 48 gives TW = 64 != W: tile-blocked M tiles would not be whole rows.  The plan refuses with the message
    ffcb_conv gives (ffcb_conv fails in the same planning step, before any device call)."""
    d = desc(g3() + [Seg(1, 0, 0, 0, 64)], 128, (64, 48), [ring(1, 64, 48, 64), Layout(1, 64, 48, 64, cg=8, tile=128)])
    with pytest.raises(ValueError, match="tile-blocked in\\[1\\]") as e:
        plan(d)
    lib = L.get_lib()
    assert lib.ffcb_conv(ctypes.byref(d), None) == L.EINVAL
    assert lib.ffcb_last_error().decode() in str(e.value)


def test_fp32_descriptors_have_no_plan():
    d = desc([Seg(0, 0, 0, 0, 64)], 64, (8, 16), [Layout(1, 8, 16, 64)])
    d.math = L.MATH_FP32
    with pytest.raises(ValueError, match="tensor-core arm"):
        plan(d)


@pytest.mark.parametrize("bn", [32, 64, 96, 128])
def test_knob_n_tile(bn, monkeypatch):
    monkeypatch.setenv("FFCB_TC_BN", str(bn))
    got = plan(desc([Seg(0, 0, 0, 0, 64)], 200, (8, 16), [Layout(1, 8, 16, 64)]))
    assert (got["bn"], got["n_tiles"]) == (bn, -(-200 // bn))
    # an N tile wider than N is cut to N's multiple of 32
    got = plan(desc([Seg(0, 0, 0, 0, 64)], 40, (8, 16), [Layout(1, 8, 16, 64)]))
    assert got["bn"] == (bn if bn < 40 else 64)


def test_knobs_are_read_on_every_call(monkeypatch):
    make = lambda: desc(column((-1, 0, 1)), 64, (16, 16), [ring(1, 16, 16, 64)])  # noqa: E731
    assert (plan(make())["kind"], plan(make())["tw"]) == (ROWS, 8)
    monkeypatch.setenv("FFCB_TC_ROWS_TW", "16")
    assert (plan(make())["kind"], plan(make())["tw"], plan(make())["th"]) == (ROWS, 16, 8)
    monkeypatch.setenv("FFCB_TC_ROWS_TW", "8")
    assert plan(make())["tw"] == 8
    monkeypatch.setenv("FFCB_TC_ROWS", "0")
    assert plan(make())["kind"] == SPATIAL
    monkeypatch.setenv("FFCB_TC_ROWS", "1")
    assert plan(make())["kind"] == ROWS
    monkeypatch.setenv("FFCB_TC_BN", "32")       # two N tiles: not rows-resident any more
    got = plan(make())
    assert (got["kind"], got["bn"], got["n_tiles"]) == (SPATIAL, 32, 2)
