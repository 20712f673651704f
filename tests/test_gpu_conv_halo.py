"""Column-halo mode of the tensor-core contraction (conv_tc.cu, TcParams::seg_taps): stride-1 3x3 reflect contractions
over planes wider than 32 pixels load one (64 ch, 64, 4) box per 64 x 2 tile, channel block and column shift dx, and
read its three dy taps out of it at whole-atom row offsets.  Checked against the torch restatement of ffcb_conv
(packing.apply_packed_reference) and, tap by tap, against the fp32 CUDA-core arm.  Shapes that stay on the per-tap
path are checked too."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import packing as P                   # noqa: E402

DEV = "cuda:0"
TOL = 2e-4           # split-bf16 operands, relative to max|ref| (as test_gpu_parity.test_conv_contract)


@pytest.fixture(autouse=True)
def _strict_env():
    os.environ["LAMA_B200_STRICT"] = "1"
    yield
    os.environ.pop("LAMA_B200_STRICT", None)


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


def _rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max()) / (float(np.abs(ref).max()) or 1.0)


def _run(pk, ins, out_hw, math, planar=(False, False)):
    """One ffcb_conv over NHWC float inputs (None: unused source); planar[s]: source s is tile-blocked (cg 8)."""
    prog = E.Program("conv_halo", math)
    feed, tvs = {}, []
    for i, t in enumerate(ins):
        if t is None:
            tvs.append(None)
            continue
        kw = dict(cg=8) if planar[i] else dict(halo=True)
        bb = prog.buf(f"in{i}", *t.shape, gemm=True, **kw)
        prog.inputs[f"x{i}"] = (t.shape[0], t.shape[3], t.shape[1], t.shape[2])
        prog.ops.append(E.ToNHWC(f"x{i}", E.TV(bb)))
        feed[f"x{i}"] = t.permute(0, 3, 1, 2).contiguous()
        tvs.append(E.TV(bb))
    b = ins[0].shape[0]
    Y = prog.buf("y", b, out_hw[0], out_hw[1], pk.n_out)
    prog.ops.append(E.ConvOp(pk, tvs, E.TV(Y)))
    prog.ops.append(E.ToNCHW(E.TV(Y), "y0"))
    prog.outputs = {"y0": (b, pk.n_out, out_hw[0], out_hw[1])}
    E.insert_border_ops(prog)
    ex = E.CudaExecutor(prog, torch.device(DEV))
    out = ex.run({k: v.to(DEV) for k, v in feed.items()})
    torch.cuda.synchronize()
    return out["y0"].cpu().permute(0, 2, 3, 1)


@pytest.mark.parametrize("ky,kx", [(ky, kx) for ky in range(3) for kx in range(3)])
def test_each_tap_alone_matches_the_fp32_arm(ky, kx):
    """A 3x3 weight that is nonzero at one tap only: every column box (dx) and row offset (dy) for both warpgroups
    (tile rows 0 and 1), on a plane of three tile rows with reflected borders on all four sides."""
    g = torch.Generator().manual_seed(10 * ky + kx)
    b, h, w, cin, n = 2, 6, 64, 64, 128
    wt = torch.zeros(n, cin, 3, 3)
    wt[:, :, ky, kx] = torch.randn(n, cin, generator=g) * 0.1
    pk = P.pack_conv([(wt, 0, 0, 1)], None, torch.randn(n, generator=g), act=L.ACT_NONE)
    x = torch.randn(b, h, w, cin, generator=g)
    got = _run(pk, [x, None], (h, w), L.MATH_BF16X3)
    ref32 = _run(pk, [x, None], (h, w), L.MATH_FP32)
    want = P.apply_packed_reference(pk, [x, None], (h, w))
    assert _rel_err(got.numpy(), ref32.numpy()) < TOL
    assert _rel_err(got.numpy(), want.numpy()) < TOL


@pytest.mark.parametrize("b,h,w,cins,n", [
    (2, 8, 64, (128,), 128),            # 64-wide plane: one tile per two rows
    (1, 6, 128, (384,), 128),           # 128-wide: two column tiles per row pair
    (1, 4, 256, (128,), 384),           # column tiles whose side halo columns belong to the neighbours; 3 N tiles
    (1, 6, 64, (128, 384), 384),        # two 3x3 groups (convl2l + convg2l channel runs of one source)
    (2, 7, 100, (64,), 128),            # ragged: odd H, W not a multiple of 64
])
def test_whole_plane_3x3(b, h, w, cins, n):
    g = torch.Generator().manual_seed(b * 1000 + h * 10 + w + n)
    c = sum(cins)
    parts, c0 = [], 0
    for ci in cins:
        parts.append((torch.randn(n, ci, 3, 3, generator=g) * 0.05, 0, c0, 1))
        c0 += ci
    pk = P.pack_conv(parts, torch.rand(n, generator=g) + 0.5, torch.randn(n, generator=g), act=L.ACT_RELU)
    x = torch.randn(b, h, w, c, generator=g)
    got = _run(pk, [x, None], (h, w), L.MATH_BF16X3)
    want = P.apply_packed_reference(pk, [x, None], (h, w))
    assert _rel_err(got.numpy(), want.numpy()) < TOL


def test_global_contraction_shape():
    """convl2g + st.conv2: a 3x3 group over the local channels plus a 1x1 segment over the tile-blocked FourierUnit
    output, N = 384 (a contraction with a tile-blocked segment keeps the per-tap path)."""
    g = torch.Generator().manual_seed(5)
    b, h, w, n = 2, 64, 64, 384
    x0, x1 = torch.randn(b, h, w, 128, generator=g), torch.randn(b, h, w, 192, generator=g)
    pk = P.pack_conv([(torch.randn(n, 128, 3, 3, generator=g) * 0.05, 0, 0, 1),
                      (torch.randn(n, 192, 1, 1, generator=g) * 0.1, 1, 0, 0)],
                     torch.rand(n, generator=g) + 0.5, torch.randn(n, generator=g), act=L.ACT_RELU)
    got = _run(pk, [x0, x1], (h, w), L.MATH_BF16X3, planar=(False, True))
    want = P.apply_packed_reference(pk, [x0, x1], (h, w))
    assert _rel_err(got.numpy(), want.numpy()) < TOL


def test_one_by_one_segment_of_a_ring_padded_source():
    """A 1x1 segment of a channels-last source next to a 3x3 group: a one-tap group over the same kind of box."""
    g = torch.Generator().manual_seed(6)
    b, h, w, n = 1, 8, 64, 128
    x = torch.randn(b, h, w, 192, generator=g)
    pk = P.pack_conv([(torch.randn(n, 64, 3, 3, generator=g) * 0.05, 0, 0, 1),
                      (torch.randn(n, 128, 1, 1, generator=g) * 0.1, 0, 64, 0)],
                     None, torch.randn(n, generator=g), act=L.ACT_NONE)
    got = _run(pk, [x, None], (h, w), L.MATH_BF16X3)
    want = P.apply_packed_reference(pk, [x, None], (h, w))
    assert _rel_err(got.numpy(), want.numpy()) < TOL


@pytest.mark.parametrize("case", ["w32", "stride2"])
def test_shapes_outside_the_halo_mode(case):
    """32-wide planes and stride-2 3x3 convolutions keep the per-tap path."""
    g = torch.Generator().manual_seed(7)
    if case == "w32":
        b, h, w, cin, n, s = 2, 32, 32, 128, 128, 1
    else:
        b, h, w, cin, n, s = 1, 32, 128, 64, 128, 2
    pk = P.pack_conv([(torch.randn(n, cin, 3, 3, generator=g) * 0.05, 0, 0, 1)], None, torch.randn(n, generator=g),
                     stride=s, act=L.ACT_RELU)
    x = torch.randn(b, h, w, cin, generator=g)
    out_hw = (h // s, w // s)
    got = _run(pk, [x, None], out_hw, L.MATH_BF16X3)
    want = P.apply_packed_reference(pk, [x, None], out_hw)
    assert _rel_err(got.numpy(), want.numpy()) < TOL
