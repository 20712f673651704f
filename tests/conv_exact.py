"""Exact-operand checks of ffcb_conv (include/ffc_b200.h): operands whose float64 contraction is exact in float32.

Every stored operand plane — the bf16 hi and lo planes of the activations and of the weights, the shift and the
addend — is drawn from a small dyadic grid, so every product and every partial sum of the contraction is a multiple of
2^-g (g read off the operands) below 2^(22 - g): exactly representable in float32 whatever the order of accumulation.  The
kernel's output must then equal the float64 reference bit for bit (up to the sign of zero); a split-bf16 output must
equal the round-to-nearest-even split of it, hi plane and lo plane.  ``assert_budget`` checks that premise per case.

The tensor-core arm (FFCB_MATH_BF16X3) multiplies hA*hW + lA*hW + hA*lW and drops lA*lW; the fp32 arm multiplies
(hA + lA) * W.  The references below model exactly that.  The lo planes are not the round-to-nearest split of hi + lo,
so they are written into storage directly (``Buf.write``), not through a conversion kernel: the kernels only read the
two planes.

Storage is addressed as include/ffc_b200.h defines it (the addressing ``Decoder`` of test_gpu_program_diff.py uses):
  channels-last     (b, y, x, c) at ptr + b*sb + y*sy + x*sx + c, y, x in [-pad, H+pad) (the ring), inside a buffer of
                    ``ctot`` channels at channel ``c_off``
  channel groups    (b, y, x, c) at ptr + (c/cg)*sg + ((b*H + y)*W + x)*cg + c%cg
  tile-blocked      (m, c) at ptr + (m/128)*sg + (c/8)*1024 + (m%128)*8 + c%8,  m = (b*H + y)*W + x
Split bf16: the lo plane ``lo_off`` elements after the hi plane.  Everything outside the view is NaN.
"""
import ctypes
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import torch

from lama_b200 import _lib as L

GRID_BITS = 6               # operand grids: hi in integers, lo in multiples of 2^-GRID_BITS
BUDGET_BITS = 22            # sum_k |terms| * 2^g below 2^22: two bits under float32's 24-bit significand
BM = 128


# ------------------------------------------------------------------------------------------------ layouts
@dataclass
class Layout:
    """Geometry of one ffcb_tensor view and of the allocation behind it (elements of the storage type)."""
    B: int
    H: int
    W: int
    C: int
    fmt: int = L.BF16X2
    pad: int = 0
    reflect: int = 0
    ctot: Optional[int] = None       # channels-last: channels per pixel of the buffer (a wider buffer: view = a slice)
    c_off: int = 0
    cg: int = 0
    tile: int = 0

    def __post_init__(self):
        if self.ctot is None:
            self.ctot = self.C
        B, H, W, p = self.B, self.H, self.W, self.pad
        if self.tile:
            assert self.cg == 8 and self.tile == 128 and p == 0
            self.sg = self.C // 8 * 1024
            self.plane = -(-(B * H * W) // BM) * self.sg
            self.sx, self.sy, self.sb = 8, W * 8, H * W * 8      # ignored by the kernels, checked as for cg == 8
            self.base = 0
        elif self.cg:
            assert p == 0
            self.sx, self.sy, self.sb = self.cg, W * self.cg, H * W * self.cg
            self.sg = B * H * W * self.cg
            self.plane = self.C // self.cg * self.sg
            self.base = 0
        else:
            self.sx = self.ctot
            self.sy = (W + 2 * p) * self.sx
            self.sb = (H + 2 * p) * self.sy
            self.sg = 0
            self.plane = B * self.sb
            self.base = p * self.sy + p * self.sx + self.c_off
        self.plane = -(-self.plane // 64) * 64         # lo plane 128-byte aligned

    @property
    def esz(self) -> int:
        return 4 if self.fmt == L.F32 else 2

    def index(self, ring: bool = False, device=None) -> torch.Tensor:
        """Element offsets (from the start of the hi plane) of (b, y, x, c): [B, H, W, C], or with ``ring`` the
        padded extent [B, H+2p, W+2p, C]."""
        p = self.pad if ring else 0
        ar = lambda n, d, o=0: (torch.arange(n, device=device) - o).view([-1 if i == d else 1 for i in range(4)])  # noqa: E731,E501
        b, y, x, c = ar(self.B, 0), ar(self.H + 2 * p, 1, p), ar(self.W + 2 * p, 2, p), ar(self.C, 3)
        if self.tile:
            m = (b * self.H + y) * self.W + x
            return (m // BM) * self.sg + (c // 8) * 1024 + (m % BM) * 8 + c % 8
        if self.cg:
            return (c // self.cg) * self.sg + ((b * self.H + y) * self.W + x) * self.cg + c % self.cg
        return self.base + b * self.sb + y * self.sy + x * self.sx + c

    def tensor(self, ptr: int) -> "L.Tensor":
        """The ffcb_tensor of this view over an allocation starting at ``ptr``."""
        t = L.Tensor()
        t.ptr = ptr + self.base * self.esz
        t.sb, t.sy, t.sx = self.sb, self.sy, self.sx
        t.lo_off = self.plane if self.fmt == L.BF16X2 else 0
        t.B, t.H, t.W, t.C = self.B, self.H, self.W, self.C
        t.fmt, t.pad, t.reflect_border = self.fmt, self.pad, self.reflect
        t.cg, t.tile, t.sg = self.cg, self.tile, self.sg
        return t


FAKE_PTR = 1 << 32      # plan queries never dereference pointers


class Buf:
    """One device allocation holding a view; every element outside what ``write`` sets is NaN."""

    def __init__(self, lay: Layout, device):
        self.lay = lay
        dt = torch.float32 if lay.fmt == L.F32 else torch.bfloat16
        n = lay.plane * (2 if lay.fmt == L.BF16X2 else 1)
        self.store = torch.full((n,), float("nan"), dtype=dt, device=device)
        self.device = device

    @property
    def t(self) -> "L.Tensor":
        return self.lay.tensor(self.store.data_ptr())

    def write(self, hi: torch.Tensor, lo: Optional[torch.Tensor] = None, ring: bool = False):
        """Store planes [B, H(+2p), W(+2p), C] (values representable in the storage type, checked)."""
        idx = self.lay.index(ring, self.device)
        dt = self.store.dtype
        for plane, v in ((0, hi), (1, lo)):
            if v is None:
                continue
            v = v.to(self.device)
            s = v.to(dt)
            assert torch.equal(s.double(), v.double()), "operand not representable in the storage type"
            self.store[idx + plane * self.lay.plane] = s

    def read(self, ring: bool = False):
        """(hi, lo) float64 planes [B, H(+2p), W(+2p), C]; lo is None for float32 storage."""
        idx = self.lay.index(ring, self.device)
        hi = self.store[idx].double()
        lo = self.store[idx + self.lay.plane].double() if self.lay.fmt == L.BF16X2 else None
        return hi, lo


# ------------------------------------------------------------------------------------------------ operands
def dyadic(shape, lo: int, hi: int, gen: torch.Generator, scale_bits: int = 0, density: float = 1.0):
    """Integers in [lo, hi] times 2^-scale_bits, float64; ``density`` < 1 zeroes the rest."""
    v = torch.randint(lo, hi + 1, tuple(shape), generator=gen).double() * 2.0 ** -scale_bits
    if density < 1.0:
        v = v * (torch.rand(tuple(shape), generator=gen) < density)
    return v


def split_planes(shape, gen, hi=(-2, 2), lo=(-1, 1)):
    """(hi, lo): hi integers in ``hi``, lo multiples of 2^-GRID_BITS in ``lo``."""
    return dyadic(shape, *hi, gen), dyadic(shape, *lo, gen, GRID_BITS)


@dataclass
class Seg:
    src: int
    dy: int
    dx: int
    c0: int
    nch: int


@dataclass
class Case:
    """One contraction with exact operands.  ``x[s]`` = (hi, lo) of source s over its interior [B, H, W, C] (the ring
    is derived: reflected, or left NaN under a zero border); ``w`` = (hi, lo) [N, Ktot] (K = the segments' channels in
    order); shift [N]; addend [B, Ho, Wo, N] (value)."""
    segs: List[Seg]
    x: list
    w: tuple
    n_out: int
    out_hw: tuple
    stride: int = 1
    border: int = L.BORDER_REFLECT
    act: int = L.ACT_NONE
    shift: Optional[torch.Tensor] = None
    addend: Optional[torch.Tensor] = None
    addend_post: int = 0
    meta: dict = field(default_factory=dict)

    @property
    def k_total(self) -> int:
        return sum(s.nch for s in self.segs)


def _gather(case: Case, src_val: torch.Tensor, s: Seg) -> torch.Tensor:
    """[B, Ho, Wo, nch] of source values sampled by segment s (reflect or zero border), float64."""
    ho, wo = case.out_hw
    h, w = src_val.shape[1], src_val.shape[2]
    dev = src_val.device
    yi = torch.arange(ho, device=dev) * case.stride + s.dy
    xi = torch.arange(wo, device=dev) * case.stride + s.dx
    if case.border == L.BORDER_REFLECT:
        yi = yi.abs(); yi = torch.where(yi >= h, 2 * h - 2 - yi, yi)
        xi = xi.abs(); xi = torch.where(xi >= w, 2 * w - 2 - xi, xi)
        return src_val[:, yi][:, :, xi][..., s.c0:s.c0 + s.nch]
    my, mx = (yi >= 0) & (yi < h), (xi >= 0) & (xi < w)
    g = src_val[:, yi.clamp(0, h - 1)][:, :, xi.clamp(0, w - 1)][..., s.c0:s.c0 + s.nch]
    return g * (my[:, None] & mx[None, :])[None, :, :, None]


def contraction(case: Case, arm: int, absolute: bool = False, device=None) -> torch.Tensor:
    """Pre-activation sum without shift / addend, float64 [B, Ho, Wo, N]: the tensor-core arm's
    sum hA*hW + lA*hW + hA*lW, or the fp32 arm's sum (hA + lA) * (hW + lW).  ``absolute``: sum of |terms|."""
    f = (lambda v: v.abs()) if absolute else (lambda v: v)
    b = case.x[case.segs[0].src][0].shape[0]
    ho, wo = case.out_hw
    acc = torch.zeros(b, ho, wo, case.n_out, dtype=torch.float64, device=device)
    whi, wlo = (f(v.to(device)) for v in case.w)
    k0 = 0
    for s in case.segs:
        hi, lo = (f(v.to(device)) for v in case.x[s.src])
        gh, gl = _gather(case, hi, s), _gather(case, lo, s)
        wh, wl = whi[:, k0:k0 + s.nch].t(), wlo[:, k0:k0 + s.nch].t()
        if arm == L.MATH_BF16X3:
            acc += gh @ wh + gl @ wh + gh @ wl
        else:
            acc += (gh @ wh + gl @ wh + gh @ wl + gl @ wl) if absolute else (gh + gl) @ (wh + wl)
        k0 += s.nch
    return acc


def epilogue(case: Case, v: torch.Tensor, act_ref: bool = True) -> torch.Tensor:
    """shift, addend (before or after the activation), activation — float64."""
    if case.shift is not None:
        v = v + case.shift.to(v.device)
    add = case.addend.to(v.device) if case.addend is not None else None
    if add is not None and not case.addend_post:
        v = v + add
    if case.act == L.ACT_RELU:
        v = v.clamp_min(0)
    elif case.act == L.ACT_SIGMOID and act_ref:
        v = torch.sigmoid(v)
    elif case.act == L.ACT_TANH and act_ref:
        v = torch.tanh(v)
    if add is not None and case.addend_post:
        v = v + add
    return v


def reference(case: Case, arm: int, device=None) -> torch.Tensor:
    return epilogue(case, contraction(case, arm, device=device))


def grid_exp(v: torch.Tensor) -> int:
    """Smallest e with every element of ``v`` a multiple of 2^-e."""
    for e in range(64):
        if torch.equal(torch.round(v * 2.0 ** e), v * 2.0 ** e):
            return e
    raise AssertionError("operand is not dyadic")


def budget_check(total_abs: torch.Tensor, g: int):
    """Every term and partial sum is a multiple of 2^-g; with sum |terms| below 2^(BUDGET_BITS - g) all of them are
    exact in float32 (24-bit significand), whatever the order of accumulation."""
    units = float(total_abs.max()) * 2.0 ** g
    assert units < 2.0 ** BUDGET_BITS, f"operand budget exceeded: {units:.3g} units of 2^-{g} >= 2^{BUDGET_BITS}"


def product_grid(a_hi, a_lo, w_hi, w_lo, arm: int) -> int:
    """Grid exponent of the arm's products: hA*hW, lA*hW, hA*lW (tensor cores) or (hA + lA) * (hW + lW) (fp32)."""
    if arm == L.MATH_BF16X3:
        return max(grid_exp(a_hi) + grid_exp(w_hi), grid_exp(a_lo) + grid_exp(w_hi), grid_exp(a_hi) + grid_exp(w_lo))
    return grid_exp(a_hi + a_lo) + grid_exp(w_hi + w_lo)


def assert_budget(case: Case, arm: int, device=None):
    """Every partial sum of every output is a multiple of 2^-g (g: the finest grid of the arm's products, the shift
    and the addend, read off the operands) of magnitude below 2^(BUDGET_BITS - g): exact in float32."""
    g = max(product_grid(*case.x[s.src], *case.w, arm) for s in case.segs)
    for t in (case.shift, case.addend):
        if t is not None:
            g = max(g, grid_exp(t))
    tot = contraction(case, arm, absolute=True, device=device)
    if case.shift is not None:
        tot = tot + case.shift.abs().to(tot.device)
    if case.addend is not None:
        tot = tot + case.addend.abs().to(tot.device)
    budget_check(tot, g)


def split_rne(v: torch.Tensor):
    """The split-bf16 store of float32 ``v`` (common.cuh split_pair): hi = bf16_rn(v), lo = bf16_rn(v - hi)."""
    f = v.float()
    hi = f.bfloat16()
    lo = (f - hi.float()).bfloat16()
    return hi.double(), lo.double()


# ------------------------------------------------------------------------------------------------ descriptors
def weight_planes(case: Case, device):
    """bf16 [2][N][Kpad] (tensor-core arm: every segment zero-padded to whole 64-channel blocks) and float32
    [Ktot][N] (fp32 arm: hW + lW)."""
    cols_h, cols_l, k0 = [], [], 0
    for s in case.segs:
        pad = (-s.nch) % 64
        for src, dst in ((case.w[0], cols_h), (case.w[1], cols_l)):
            blk = src[:, k0:k0 + s.nch]
            dst.append(torch.cat([blk, blk.new_zeros(blk.shape[0], pad)], 1) if pad else blk)
        k0 += s.nch
    w_tc = torch.stack([torch.cat(cols_h, 1), torch.cat(cols_l, 1)]).to(torch.bfloat16)
    assert torch.equal(w_tc[0].double(), torch.cat(cols_h, 1)) and torch.equal(w_tc[1].double(), torch.cat(cols_l, 1))
    w_f = (case.w[0] + case.w[1]).t().contiguous().float()
    assert torch.equal(w_f.double(), (case.w[0] + case.w[1]).t())
    return w_tc.contiguous().to(device), w_f.to(device)


def make_desc(case: Case, ins: Sequence[Optional["L.Tensor"]], out: "L.Tensor", math: int, weight_ptr: int,
              shift_ptr: Optional[int] = None, addend: Optional["L.Tensor"] = None) -> "L.ConvDesc":
    d = L.ConvDesc()
    for i, t in enumerate(ins):
        if t is not None:
            d.inp[i] = t
    d.out = out
    if addend is not None:
        d.addend = addend
    d.weight = weight_ptr
    d.shift = shift_ptr
    d.n_out, d.stride, d.border, d.act = case.n_out, case.stride, case.border, case.act
    d.nseg, d.math, d.addend_post = len(case.segs), math, case.addend_post
    for i, s in enumerate(case.segs):
        d.seg[i] = L.KSeg(s.src, s.dy, s.dx, s.c0, s.nch)
    return d


def plan(desc: "L.ConvDesc") -> dict:
    """ffcb_conv_plan as a dict (raises ValueError with the library's message on FFCB_EINVAL)."""
    info = L.ConvPlanInfo()
    L.check(L.get_lib().ffcb_conv_plan(ctypes.byref(desc), ctypes.byref(info)), "ffcb_conv_plan")
    return {k: getattr(info, k) for k, _ in L.ConvPlanInfo._fields_ if k != "_reserved"}


KIND_NAMES = {L.PLAN_FLAT: "flat", L.PLAN_SPATIAL: "spatial", L.PLAN_ROWS: "rows", L.PLAN_HALO: "halo"}


def tile_of(pl: dict, out_hw, b: int, y: int, x: int, n: int):
    """(M tile, N tile) holding output element (b, y, x, n) under plan ``pl``."""
    H, W = out_hw
    if pl["kind"] == L.PLAN_FLAT:
        m = ((b * H + y) * W + x) // BM
    else:
        tx, ty = -(-W // pl["tw"]), -(-H // pl["th"])
        m = (b * ty + y // pl["th"]) * tx + x // pl["tw"]
    return m, n // pl["bn"]


def first_mismatch(got: torch.Tensor, want: torch.Tensor):
    """(b, y, x, n) of the first element that differs (NaN differs from everything), or None."""
    bad = ~(got == want)
    if not bool(bad.any()):
        return None
    return tuple(int(i) for i in bad.nonzero()[0])


def assert_exact(got: torch.Tensor, want: torch.Tensor, pl: Optional[dict], out_hw, what: str):
    """Bit for bit (up to the sign of zero); the message names the first bad element with its M and N tile."""
    assert got.shape == want.shape, (got.shape, want.shape)
    pos = first_mismatch(got, want)
    if pos is None:
        return
    nbad = int((~(got == want)).sum())
    where = ""
    if pl is not None:
        m, nt = tile_of(pl, out_hw, *pos)
        where = f" (M tile {m}, N tile {nt} of {KIND_NAMES[pl['kind']]} BN={pl['bn']})"
    raise AssertionError(f"{what}: {nbad} elements differ; first at (b, y, x, n) = {pos}{where}: got "
                         f"{float(got[pos])!r}, want {float(want[pos])!r}")


# ------------------------------------------------------------------------------------------------ activations
def act_ulp_bound(act: int, pre: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    """Largest |got - ref| the tensor-core epilogue may show for an exact pre-activation (float64 ``pre``):
    sigmoid = __fdividef(1, 1 + __expf(-v)): __expf within 2 + floor(|1.173 v|) ulp (CUDA programming guide, intrinsic
    functions), the rounding of 1 + e half an ulp, __fdividef within 2 ulp — relative errors of 2^-23 per ulp that add
    up in the quotient; tanh = tanhf within 2 ulp of its result; the float32 result spacing below |ref|."""
    if act == L.ACT_SIGMOID:
        ulps = 2 + torch.floor((1.173 * pre).abs()) + 0.5 + 2
        return ulps * 2.0 ** -23 * ref.abs()
    assert act == L.ACT_TANH
    # 2 ulp of the float32 result: ulp(r) <= 2^-23 |r| for normal r, 2^-149 below
    return 2 * torch.maximum(ref.abs() * 2.0 ** -23, torch.full_like(ref, 2.0 ** -149))


def rel_err(got: torch.Tensor, ref: torch.Tensor) -> float:
    """The suite's usual criterion: max |got - ref| / max |ref|."""
    return float((got - ref).abs().max()) / (float(ref.abs().max()) or 1.0)

