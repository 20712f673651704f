"""Host-side weight preparation: fold eval-mode BatchNorm into the preceding convolution and
lay weights out the way ``ffcb_conv`` consumes them (include/ffc_b200.h).

Pure torch tensor algebra (runs on CPU or GPU, done once per weight version, never on the
per-image path), so it is unit-tested on the CPU box against an einsum restatement
(tests/test_packing.py).

K-segment convention shared with the kernels: a convolution is a list of segments
``(src, dy, dx, c0, nch)``; the packed weight's K axis is the concatenation of the segments'
channel ranges in list order.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib as L


def bn_scale_shift(bn: torch.nn.BatchNorm2d, conv_bias: Optional[torch.Tensor] = None
                   ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Eval-mode BN as ``y = scale * x + shift`` (float64).  ffc.py:60,131,243-244,353.
    ``conv_bias``: the bias of the convolution BN follows (pix2pixhd.py convs carry one), folded into the shift:
    BN(conv(x) + bias) = scale * conv(x) + (shift + scale * bias)."""
    var = bn.running_var.detach().double()
    mean = bn.running_mean.detach().double()
    gamma = bn.weight.detach().double() if bn.weight is not None else torch.ones_like(var)
    beta = bn.bias.detach().double() if bn.bias is not None else torch.zeros_like(var)
    scale = gamma / torch.sqrt(var + bn.eps)
    shift = beta - mean * scale
    if conv_bias is not None:
        shift = shift + scale * conv_bias.detach().double().to(shift.device)
    return scale, shift


@dataclass
class Seg:
    src: int
    dy: int
    dx: int
    c0: int
    nch: int


@dataclass
class PackedConv:
    """Everything ``ffcb_conv`` needs besides the activation views."""
    segs: List[Seg]
    n_out: int
    w_kn: torch.Tensor                  # float32 [Ktot][N]   (FFCB_MATH_FP32)
    shift: Optional[torch.Tensor]       # float32 [N]
    stride: int = 1
    border: int = L.BORDER_REFLECT
    act: int = L.ACT_NONE
    w_split: Optional[torch.Tensor] = None   # bf16 [2][N][Ktot] (FFCB_MATH_BF16X3), built on demand
    meta: dict = field(default_factory=dict)

    @property
    def k_total(self) -> int:
        return sum(s.nch for s in self.segs)

    def split_weights(self) -> torch.Tensor:
        """bf16 [2][N][Kpad]: K-major, every segment zero-padded to a multiple of 64 channels (one
        128-byte swizzle row per K block of the wgmma arm)."""
        if self.w_split is None:
            w_nk = self.w_kn.t()
            cols, k0 = [], 0
            for s in self.segs:
                blk = w_nk[:, k0:k0 + s.nch]
                padk = (-s.nch) % 64
                if padk:
                    blk = torch.cat([blk, blk.new_zeros(blk.shape[0], padk)], dim=1)
                cols.append(blk)
                k0 += s.nch
            self.w_split = split_bf16(torch.cat(cols, dim=1).contiguous())
        return self.w_split


def split_bf16(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> stacked (hi, lo) bfloat16 planes with hi + lo ~= x (|err| <= 2^-17 |x|)."""
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return torch.stack((hi, lo), dim=0).contiguous()


def taps(k: int, pad: int) -> List[Tuple[int, int, int, int]]:
    """(ky, kx, dy, dx) of a k x k correlation with ``pad`` pixels of padding."""
    return [(ky, kx, ky - pad, kx - pad) for ky in range(k) for kx in range(k)]


def pack_conv(parts: Sequence[Tuple[torch.Tensor, int, int, int]], scale: Optional[torch.Tensor],
              shift: Optional[torch.Tensor], *, stride: int = 1, border: int = L.BORDER_REFLECT,
              act: int = L.ACT_NONE, device=None) -> PackedConv:
    """Pack one fused convolution.

    ``parts``: sequence of ``(weight [N, C, kh, kw], src, c0, pad)`` — each part is an
    ``nn.Conv2d`` weight applied to channels ``[c0, c0+C)`` of input tensor ``src`` with
    ``pad`` pixels of padding; parts are summed (e.g. convl2l(x_l) + convg2l(x_g), or
    convl2g(x_l) + conv2(u)).  ``scale``/``shift``: folded BN (+bias) per output channel.
    """
    segs: List[Seg] = []
    cols = []
    n_out = parts[0][0].shape[0]
    for w, src, c0, pad in parts:
        w = w.detach().double()
        n, c, kh, kw = w.shape
        assert n == n_out and kh == kw
        for ky, kx, dy, dx in taps(kh, pad):
            segs.append(Seg(src, dy, dx, c0, c))
            cols.append(w[:, :, ky, kx])                      # [N, C]
    w_nk = torch.cat(cols, dim=1)                             # [N, Ktot]
    if scale is not None:
        w_nk = w_nk * scale.double()[:, None]
    w_kn = w_nk.t().contiguous().float()
    sh = shift.float().contiguous() if shift is not None else None
    if device is not None:
        w_kn = w_kn.to(device)
        sh = sh.to(device) if sh is not None else None
    assert len(segs) <= L.MAX_KSEG, f"{len(segs)} K-segments exceed FFCB_MAX_KSEG"
    if all(pad == 0 for _w, _s, _c, pad in parts):
        border = L.BORDER_ZERO      # no tap ever leaves the interior; the border mode is moot
    return PackedConv(segs=segs, n_out=n_out, w_kn=w_kn, shift=sh, stride=stride, border=border, act=act)


def pack_conv_transpose_phases(weight: torch.Tensor, bias: Optional[torch.Tensor], scale: torch.Tensor,
                               shift: torch.Tensor, *, act: int, device=None) -> List[Tuple[int, int, PackedConv]]:
    """``nn.ConvTranspose2d(k=3, stride=2, padding=1, output_padding=1)`` (ffc.py:350-352) as four
    sub-pixel phases.  weight: [Cin, Cout, 3, 3].  Output pixel (2i+a, 2j+b) only sees taps whose
    parity matches: out[o] += in[i'] * w[ky] with o = 2 i' - 1 + ky, so
        a == 0: (ky=1, di=0)            a == 1: (ky=2, di=0), (ky=0, di=+1)
    and the same along x.  Inputs beyond the last row/column are zero (FFCB_BORDER_ZERO).
    Returns [(a, b, PackedConv)] with folded BN: scale*(conv + bias) + shift.
    """
    wt = weight.detach().double()          # [Cin, Cout, 3, 3]
    cin, cout = wt.shape[0], wt.shape[1]
    full_shift = shift.double() + (scale.double() * bias.detach().double() if bias is not None else 0.0)
    sel = {0: [(1, 0)], 1: [(2, 0), (0, 1)]}
    out = []
    for a in (0, 1):
        for b in (0, 1):
            segs, cols = [], []
            for ky, di in sel[a]:
                for kx, dj in sel[b]:
                    segs.append(Seg(0, di, dj, 0, cin))
                    cols.append(wt[:, :, ky, kx].t())         # [Cout, Cin]
            w_nk = torch.cat(cols, dim=1) * scale.double()[:, None]
            w_kn = w_nk.t().contiguous().float()
            sh = full_shift.float().contiguous()
            if device is not None:
                w_kn, sh = w_kn.to(device), sh.to(device)
            out.append((a, b, PackedConv(segs=segs, n_out=cout, w_kn=w_kn, shift=sh, stride=1,
                                         border=L.BORDER_ZERO, act=act)))
    return out


def pack_stem(weight: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, device=None):
    """7x7 stem (ffc.py:316): [N, Cin, 7, 7] -> float [(ky*7+kx)*Cin + c][N], BN folded."""
    w = weight.detach().double() * scale.double()[:, None, None, None]
    w = w.permute(2, 3, 1, 0).reshape(-1, w.shape[0]).contiguous().float()
    sh = shift.float().contiguous()
    if device is not None:
        w, sh = w.to(device), sh.to(device)
    return w, sh


def pack_stem_windowed(weight: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, device=None) -> PackedConv:
    """7x7 stem (ffc.py:316) for the tensor-core arm over the packed NHWC8 image of ffcb_stem_pack.
    Cin <= 4 (two-row packing: channels 4..7 of a packed pixel are the pixel one row below): FOUR K-segments
    (dy = 0, 2, 4, 6) of 64 = 8 taps x (kernel row dy | kernel row dy+1) x 4 channels; K index inside a segment =
    kx*8 + r*4 + c; kernel row 7, tap 7 and channels >= Cin carry zero weights.
    Cin in 5..8: seven K-segments (one per kernel row), K index = kx*8 + c."""
    w = weight.detach().double() * scale.double()[:, None, None, None]           # [N, Cin, 7, 7]
    n, cin = w.shape[0], w.shape[1]
    assert cin <= 8 and w.shape[2] == 7 and w.shape[3] == 7
    sh = shift.float().contiguous()
    if cin <= 4:
        full = torch.zeros(n, 4, 8, 2, 4, dtype=torch.float64, device=w.device)  # [N, ky pair, kx, row in pair, c]
        for ky in range(7):
            full[:, ky // 2, :7, ky % 2, :cin] = w[:, :, ky, :].permute(0, 2, 1)
        w_kn = full.reshape(n, 4 * 64).t().contiguous().float()
        segs = [Seg(0, 2 * j, 0, 0, 64) for j in range(4)]
    else:
        full = torch.zeros(n, 7, 8, 8, dtype=torch.float64, device=w.device)     # [N, ky, kx, c]
        full[:, :, :7, :cin] = w.permute(0, 2, 3, 1)
        w_kn = full.reshape(n, 7 * 64).t().contiguous().float()
        segs = [Seg(0, ky, 0, 0, 64) for ky in range(7)]
    if device is not None:
        w_kn, sh = w_kn.to(device), sh.to(device)
    return PackedConv(segs=segs, n_out=n, w_kn=w_kn, shift=sh, stride=1, border=L.BORDER_ZERO, act=L.ACT_RELU)


def pack_head_rows(weight: torch.Tensor, device=None) -> PackedConv:
    """7x7 head (ffc.py:361) for the tensor-core arm, kernel-ROW part: output channel n*7+kx of the contraction is
    sum_ky sum_c in[y+ky-3, x', c] * w[n, c, ky, kx]; seven K-segments (dy = ky-3, dx = 0).  N*7 is padded to a
    multiple of 8 with zero rows.  Bias and activation are applied by ffcb_head_gather7."""
    w = weight.detach().double()                                   # [N, C, 7, 7]
    n, c = w.shape[0], w.shape[1]
    nq = (7 * n + 7) // 8 * 8
    rows = torch.zeros(nq, 7, c, dtype=torch.float64, device=w.device)          # [(n,kx), ky, c]
    rows[: 7 * n] = w.permute(0, 3, 2, 1).reshape(7 * n, 7, c)
    w_kn = rows.reshape(nq, 7 * c).t().contiguous().float()
    if device is not None:
        w_kn = w_kn.to(device)
    segs = [Seg(0, ky - 3, 0, 0, c) for ky in range(7)]
    return PackedConv(segs=segs, n_out=nq, w_kn=w_kn, shift=None, stride=1, border=L.BORDER_REFLECT, act=L.ACT_NONE)


def pack_head(weight: torch.Tensor, bias: Optional[torch.Tensor], device=None):
    """7x7 head (ffc.py:361): [N, C, 7, 7] -> float [N][49][C]; bias [N]."""
    w = weight.detach().float().permute(0, 2, 3, 1).reshape(weight.shape[0], 49, weight.shape[1]).contiguous()
    b = bias.detach().float().contiguous() if bias is not None else torch.zeros(weight.shape[0])
    if device is not None:
        w, b = w.to(device), b.to(device)
    return w, b


# ----------------------------------------------------------------------------- einsum restatement
def apply_packed_reference(p: PackedConv, inputs: Sequence[torch.Tensor], out_hw: Tuple[int, int],
                           addend: Optional[torch.Tensor] = None, addend_post: bool = False) -> torch.Tensor:
    """Slow torch restatement of the ffcb_conv contract on NHWC float64 tensors — the spec the
    CUDA kernels are tested against and the CPU test of this module's packing.
    inputs[src]: [B, H, W, C]; returns [B, Ho, Wo, N]."""
    ho, wo = out_hw
    b = inputs[0].shape[0]
    acc = torch.zeros(b, ho, wo, p.n_out, dtype=torch.float64, device=inputs[0].device)
    k0 = 0
    w = p.w_kn.double().to(acc.device)          # packed on the module's device, checked wherever the data is
    ys = torch.arange(ho, device=acc.device) * p.stride
    xs = torch.arange(wo, device=acc.device) * p.stride
    for s in p.segs:
        x = inputs[s.src].double()
        h, wd = x.shape[1], x.shape[2]
        yi, xi = ys + s.dy, xs + s.dx
        if p.border == L.BORDER_REFLECT:
            yi = yi.abs(); yi = torch.where(yi >= h, 2 * h - 2 - yi, yi)
            xi = xi.abs(); xi = torch.where(xi >= wd, 2 * wd - 2 - xi, xi)
            my = torch.ones_like(yi, dtype=torch.bool); mx = torch.ones_like(xi, dtype=torch.bool)
        else:
            my = (yi >= 0) & (yi < h); mx = (xi >= 0) & (xi < wd)
            yi = yi.clamp(0, h - 1); xi = xi.clamp(0, wd - 1)
        g = x[:, yi][:, :, xi][..., s.c0:s.c0 + s.nch]                     # [B, Ho, Wo, nch]
        g = g * (my[:, None] & mx[None, :])[None, :, :, None]
        acc += g @ w[k0:k0 + s.nch]
        k0 += s.nch
    if p.shift is not None:
        acc += p.shift.double().to(acc.device)
    if addend is not None and not addend_post:
        acc += addend.double()
    if p.act == L.ACT_RELU:
        acc = acc.clamp_min(0)
    elif p.act == L.ACT_SIGMOID:
        acc = torch.sigmoid(acc)
    elif p.act == L.ACT_TANH:
        acc = torch.tanh(acc)
    if addend is not None and addend_post:
        acc += addend.double()
    return acc
