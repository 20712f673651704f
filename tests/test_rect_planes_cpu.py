"""CPU-only checks of rectangular bottleneck planes (H != W):

* each axis of a plane gets its own launch plan: the planner rfft2 / irfft2 launch with (fft_core.cuh:
  make_plane_plans, compiled with g++ by tests/host_emul/fft_plan_emul.cpp) gives the row passes the plan of W and the
  column passes the plan of H;
* the admission gates of inference and refinement take every such plane up to 1024 points per side, and the FFT entry
  points refuse a larger one with a message naming both sides;
* predict batches are sized from the program's real footprint: a 256x1024 image costs what a 512x512 one does, not
  what a 1024x1024 one does.
"""
import ctypes
import os
import subprocess

import pytest
import torch

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200 import predict as PR
from lama_b200.testing import BIG_LAMA_KWARGS, small_lama_kwargs
from test_large_planes_cpu import _inpainter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (H, W) -> {pass: (template length, channels per CTA, Bluestein length, runtime radices)} as csrc/fft.cu's rfft2 and
# irfft2 launch them (fft_core.cuh: make_plane_plans).  Template lengths 4..256: compile-time radix-8/4 passes; 0: the
# runtime Stockham radices (one pass of radix n for a prime; none for a 1-point axis) or Bluestein.  Axes of 448 points
# and more run 8 channels per CTA.  127 is prime but below the 129 points where Bluestein can pay off.
PLANS = {
    (64, 128): {"rows": (128, 32, 0, []), "cols": (64, 32, 0, [])},
    (96, 1024): {"rows": (0, 8, 0, [4, 4, 4, 4, 4]), "cols": (0, 32, 0, [6, 4, 4])},
    (1024, 96): {"rows": (0, 32, 0, [6, 4, 4]), "cols": (0, 8, 0, [4, 4, 4, 4, 4])},
    (127, 256): {"rows": (256, 32, 0, []), "cols": (0, 32, 0, [127])},
    (1000, 1024): {"rows": (0, 8, 0, [4, 4, 4, 4, 4]), "cols": (0, 8, 0, [8, 5, 5, 5])},
    (1, 1024): {"rows": (0, 8, 0, [4, 4, 4, 4, 4]), "cols": (0, 32, 0, [])},
    (479, 256): {"rows": (256, 32, 0, []), "cols": (0, 8, 1024, [])},
}
PLANES = [hw for hw in PLANS if min(hw) >= 2]


@pytest.fixture(scope="module")
def plane_plans(tmp_path_factory):
    exe = tmp_path_factory.mktemp("rect") / "fft_plan_emul"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "host_emul", "fft_plan_emul.cpp"), "-o", str(exe)])
    args = [str(v) for hw in PLANS for v in hw]
    out = subprocess.run([str(exe)] + args, capture_output=True, text=True, check=True).stdout
    got = {}
    for line in out.splitlines():
        head, radices = line.split("|")
        h, w, pass_, n, lanes, m, _np = head.split()
        got.setdefault((int(h), int(w)), {})[pass_] = (int(n), int(lanes), int(m), [int(r) for r in radices.split()])
    return got


@pytest.mark.parametrize("h,w", list(PLANS))
def test_each_axis_gets_its_own_plan(h, w, plane_plans):
    """The row passes run the plan of W and the column passes the plan of H, in both directions."""
    assert plane_plans[(h, w)] == PLANS[(h, w)]


def test_rectangular_planes_pass_the_native_gates():
    """Every plane above, in both orientations (1 x N in one), is native for the FFT pair; as a bottleneck it is native
    for the generator, the block-gradient and rear programs and the refinement step.  A 1-point side is refused by the
    model layers (reflect padding needs two pixels, in the reference too), a side above 1024 by all of them."""
    gen = M.FFCResNetGenerator(**small_lama_kwargs(ngf=16, n_blocks=1, n_downsampling=1)).eval()
    blk = gen.model[3]
    for h, w in PLANES:
        assert E.plane_ok(h, w) and E.plane_ok(w, h), (h, w)
    assert E.plane_ok(1, 1024) and not E.plane_ok(1024, 1)      # the real transform runs along W: W >= 2
    for h, w in PLANES:
        for hh, ww in ((h, w), (w, h)):
            sl, sg = (1, 8, hh, ww), (1, 24, hh, ww)
            assert E.generator_supported(gen, torch.empty(1, 4, 2 * hh, 2 * ww, device="meta")), (hh, ww)
            assert E.ffc_bn_act_shapes_ok(blk.conv1, torch.empty(sl, device="meta"), torch.empty(sg, device="meta"))
            assert E.rear_grad_supported(gen, sl, sg), (hh, ww)
            assert E.refine_supported(gen, sl, sg, (2 * hh - 5, 2 * ww - 3)), (hh, ww)
    assert E.block_grad_supported(blk)
    for h, w in ((1, 1024), (1025, 96), (96, 1025), (1025, 1025)):
        assert not E.generator_supported(gen, torch.empty(1, 4, 2 * h, 2 * w, device="meta")), (h, w)
        assert not E.rear_grad_supported(gen, (1, 8, h, w), (1, 24, h, w)), (h, w)
    assert not E.plane_ok(1025, 96) and not E.plane_ok(96, 1025)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return L.get_lib()


def _desc(b, h, w, c):
    t = L.Tensor()
    t.ptr, t.B, t.H, t.W, t.C = 4096, b, h, w, c          # never dereferenced: the shape checks come first
    t.sx, t.sy, t.sb = c, w * c, h * w * c
    return t


@pytest.mark.parametrize("h,w", [(96, 1025), (1025, 96), (1030, 2000)])
def test_fft_refuses_planes_above_1024_naming_both_sides(lib, h, w):
    x, s, y = _desc(1, h, w, 4), _desc(1, h, w // 2 + 1, 8), _desc(1, h, w, 4)
    assert lib.ffcb_rfft2(ctypes.byref(x), ctypes.byref(s), None, 0, None) == L.EINVAL
    assert f"plane {h}x{w} exceeds the 1024-point FFT limit" in lib.ffcb_last_error().decode()
    assert lib.ffcb_irfft2(ctypes.byref(s), None, ctypes.byref(y), None, 0, None) == L.EINVAL
    assert f"plane {h}x{w} exceeds the 1024-point FFT limit" in lib.ffcb_last_error().decode()


def test_predict_batches_at_256x1024_match_512x512():
    """big-lama's uint8 predict program at 256x1024 (a 32x128 bottleneck) holds what it holds at 512x512 to within
    1 % (the reflect rings grow with the perimeter, the half spectra shrink with H), a quarter of what it holds at
    1024x1024, so under the same budget the two sizes get the same batches."""
    inp = _inpainter({})
    inp.generator = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    rect, square, big = inp.per_image_bytes(256, 1024), inp.per_image_bytes(512, 512), inp.per_image_bytes(1024, 1024)
    print(f"bytes per image: 256x1024 {rect / 1e6:.1f} MB, 512x512 {square / 1e6:.1f} MB, 1024x1024 {big / 1e6:.1f} MB")
    assert abs(rect / square - 1) < 0.01 and rect < 0.3 * big
    idx = list(range(100))
    for k in range(1, 40):
        budget = int((k + 0.5) * square)
        got_r = PR.BatchedInpainter.plan_group(idx, rect, budget, 32)
        got_s = PR.BatchedInpainter.plan_group(idx, square, budget, 32)
        assert [len(p) for p in got_r] == [len(p) for p in got_s], k
