"""The refinement step program with its up-sampling tail run in row bands (kind
``generator_refine_bits_banded:<H0>x<W0>``, ``BatchedRefiner(..., relu_masks="bits", tail="banded")``).

At 24 to 50 megapixels most of the bits step program's storage is the full-resolution tail: the three
ConvTranspose(3, s2) + BN + ReLU outputs, the head's row sums and, in the backward, the gradients of the same maps.  The
tail is local, and its backward needs nothing from the forward but ReLU masks, so this program runs it band by band
over bottleneck rows [r0, r1); its band buffers then pool across bands (``engine.assign_storage_slots``) and hold one
band's worth.  The residual blocks are those of the bits program (``relu_bits.pack_relu_masks``).

Forward, per band, top to bottom: the up-sampling stages read bottleneck rows [r0 - 1, r1 + 2) (clipped to the plane;
for big-lama's three stages) and each writes a band buffer that is its own small image: its own reflected ring and zero
border stand where the plane's neighbour rows would be.  That is wrong only within the halo.  A transposed conv's even
output rows read input row i and its odd rows rows i and i + 1, so each stage spoils one more row at the band's bottom
(7 full-resolution rows after three stages) and none at its top; the head's 7x7 reflection spoils 3 rows at either end.
One bottleneck row above and two below (8 and 16 full-resolution rows) leave every row the head's interior
[8 r0, 8 r1) reads exact, and where a band buffer ends at the plane's own edge its ring and border are the plane's.
Each stage packs its interior rows into a whole-plane bit mask (ffcb_relu_mask_pack_rows) and the head writes its
interior rows of ``pred`` (ffcb_head_gather7_rows).

Backward, per band, bottom to top: ffcb_head_bwd7_bits writes full-resolution gradient rows [8 (r0 - 1), 8 r1) from the
whole ``dpred`` (it folds the reflection only at the plane's edges, so every row it writes is exact), then each stage
adjoint (a stride-2 zero-border contraction) and ffcb_relu_bwd_bits_rows.  A band's first row at every level reads a
zero row above it, so the bottleneck gradient rows [r0 - 1, r1) it writes are exact except row r0 - 1, which the band
above, run next, writes again.

Every output pixel of every op gets the operands of the whole-plane op, in the same order, so the program computes bit
for bit what the bits program computes.  It needs the tensor-core head (split-bf16 arithmetic).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Tuple

import torch

from . import _lib as L
from . import engine as E
from . import packing as P
from .relu_bits import _words, pack_relu_masks

OP_TYPES: List[type] = []

# Full-resolution pixels per band: about 0.4 GB of split-bf16 band buffers per 64-channel map (a band's buffers pool
# across bands, so the tail holds a few GB at any photo size, against about 57 GB for the whole 8000x6000 tail).
BAND_PX = 1 << 21


@dataclass
class MaskPackRowsOp(E.Op, registry=OP_TYPES):
    """bits rows [row0, row0 + y.H) = [y > 0] (ffcb_relu_mask_pack_rows); ``bits`` is a whole-plane bit mask."""
    reads, writes = ("y",), ("bits",)
    y: E.TV
    bits: E.TV
    row0: int

    def bind(self, ex):
        return "ffcb_relu_mask_pack_rows", ex.lib.ffcb_relu_mask_pack_rows, [
            ex.ref(self.y), _words(ex, self.bits), self.bits.buf.H, self.row0]


@dataclass
class ReluBwdBitsRowsOp(E.Op, registry=OP_TYPES):
    """out = dy * bit, the bits of rows [row0, row0 + out.H) of a whole-plane mask (ffcb_relu_bwd_bits_rows)."""
    reads, writes = ("dy", "bits"), ("out",)
    dy: E.TV
    bits: E.TV
    row0: int
    out: E.TV

    def bind(self, ex):
        return "ffcb_relu_bwd_bits_rows", ex.lib.ffcb_relu_bwd_bits_rows, [
            ex.ref(self.dy), _words(ex, self.bits), self.bits.buf.H, self.row0, ex.ref(self.out)]


@dataclass
class HeadGatherRowsOp(E.Op, registry=OP_TYPES):
    """Rows [row0, row0 + q.H) of the external NCHW output ``dst`` (ffcb_head_gather7_rows)."""
    reads, writes = ("q",), ()
    q: E.TV
    bias: torch.Tensor
    n_out: int
    act: int
    dst: str
    row0: int

    def bind(self, ex):
        return "ffcb_head_gather7_rows", ex.lib.ffcb_head_gather7_rows, [
            ex.ref(self.q), ex.keep(self.bias), self.n_out, self.act, E.Ext(self.dst), ex.prog.outputs[self.dst][2],
            self.row0]


@dataclass
class HeadBwdBitsOp(E.Op, registry=OP_TYPES):
    """Rows [row0, row0 + out.H) of the head adjoint ``E.HeadBwdOp``, masked by the whole-plane bits of the last
    up-sampling output (ffcb_head_bwd7_bits)."""
    reads, writes = ("bits",), ("out",)
    y: str
    dy: str
    w: torch.Tensor
    n_out: int
    act: int
    bits: E.TV
    row0: int
    out: E.TV

    def bind(self, ex):
        return "ffcb_head_bwd7_bits", ex.lib.ffcb_head_bwd7_bits, [
            E.Ext(self.y), E.Ext(self.dy), *ex.prog.outputs[self.y], ex.keep(self.w), self.act, _words(ex, self.bits),
            self.row0, ex.ref(self.out)]


def tail_supported(gen, math: int) -> bool:
    """The banded tail exists for this generator under arithmetic ``math``: the tensor-core head applies
    (``engine._tc_head``, for planes wider than 3).  Shapes are checked by ``engine.refine_supported``."""
    lay = E._generator_layout(gen)
    return lay is not None and E._tc_head(E.Program("banded", math), lay[5], 4, 4)


def band_rows(h: int, w: int, n_ups: int) -> int:
    """Bottleneck rows per band of an h x w bottleneck whose tail up-samples by 2 ** n_ups."""
    return max(1, min(h, BAND_PX // (4 ** n_ups * w)))


def bands(h: int, rows: int) -> List[Tuple[int, int]]:
    return [(r0, min(r0 + rows, h)) for r0 in range(0, h, rows)]


def build_refine_banded_program(prog: E.Program, gen, sl: Tuple[int, ...], sg: Tuple[int, ...],
                                crop: Tuple[int, int]):
    """``engine.build_refine_program(..., relu_masks="bits")`` with the up-sampling tail and head run in row bands
    (module docstring): the same inputs, outputs and results."""
    from .refine import gaussian_kernel1d
    _stem, _downs, _blocks, ups, _out_blk, head, out_act = E._generator_layout(gen)
    b, _cl, h, w = sl
    f = 2 ** len(ups)
    H, W = h * f, w * f
    if not E._tc_head(prog, head, H, W):
        raise ValueError("the banded up-sampling tail needs the tensor-core head (split-bf16 arithmetic)")
    dev = head.weight.device
    n = head.out_channels
    X, saved = E.emit_rear_blocks(prog, gen, sl, sg)
    prog.outputs["y0"] = (b, n, H, W)
    masks = [E.Buf(f"relu_bits.up{k}#{len(prog.bufs) + k}", b, h * 2 ** (k + 1), w * 2 ** (k + 1), ct.out_channels,
                   bits=1) for k, (ct, _bn) in enumerate(ups)]
    prog.bufs.extend(masks)
    rows = bands(h, band_rows(h, w, len(ups)))
    above, below = -(-3 // f), 1 + -(-2 // f)        # bottleneck halo rows of a forward band (module docstring)

    # forward, top to bottom
    pkh = P.pack_head_rows(head.weight, device=dev)
    bias = (head.bias.detach().float().contiguous() if head.bias is not None else torch.zeros(n)).to(dev)
    ups_packed = [P.pack_conv_transpose_phases(ct.weight, ct.bias, *P.bn_scale_shift(bn), act=L.ACT_RELU,
                                               device=ct.weight.device) for ct, bn in ups]
    for r0, r1 in rows:
        s0, e0 = max(r0 - above, 0), min(r1 + below, h)
        src = E.TV(X, win=(s0, 0, e0 - s0, w))
        for k, (ct, _bn) in enumerate(ups):
            g, last = 2 ** (k + 1), k == len(ups) - 1
            U = prog.buf("band.up", b, g * (e0 - s0), g * w, ct.out_channels, gemm=True, halo=True,
                         halo_px=3 if last else 1)
            for a, bb, pk in ups_packed[k]:
                prog.ops.append(E.ConvOp(pk, [src, None], E.TV(U, phase=(a, bb)),
                                         tag=f"band convT phase {a}{bb}+bn+relu"))
            interior = E.TV(U, win=(g * (r0 - s0), 0, g * (r1 - r0), g * w))
            prog.ops.append(MaskPackRowsOp(interior, E.TV(masks[k]), g * r0))
            src = E.TV(U)
        Q = prog.buf("band.head.q", b, src.buf.H, W, pkh.n_out)
        prog.ops.append(E.ConvOp(pkh, [src, None], E.TV(Q), tag="band head 7x7 rows"))
        prog.ops.append(HeadGatherRowsOp(E.TV(Q, win=(f * (r0 - s0), 0, f * (r1 - r0), W)), bias, n, out_act, "y0",
                                         f * r0))

    prog.ops.append(E.SplitOp())
    h0, w0 = crop
    prog.inputs.update(image=(b, n, H, W), mask=(b, 1, H, W), ref=(b, n, h0 // 2, w0 // 2),
                       md=(b, 1, h0 // 2, w0 // 2), inv=(b, 2))
    prog.outputs.update(dy0=(b, n, H, W), loss=(b, 2))
    prog.ops.append(E.RefineLossOp("y0", "image", "mask", "ref", "md", "inv", h0, w0, gaussian_kernel1d(5, 1.0),
                                   "dy0", "loss", b * n * (h0 // 2) * (w0 // 2)))

    # backward, bottom to top
    wh, _ = P.pack_head(head.weight, head.bias, device=dev)
    adj = [E.pack_up_adjoint(ct, bn, dev) for ct, bn in ups]
    DX = prog.buf("grad.dx", b, h, w, ups[0][0].in_channels)
    for r0, r1 in reversed(rows):
        s0 = max(r0 - 1, 0)
        D = prog.buf("band.grad.dup", b, f * (r1 - s0), W, head.in_channels, gemm=True)
        prog.ops.append(HeadBwdBitsOp("y0", "dy0", wh, n, out_act, E.TV(masks[-1]), f * s0, E.TV(D)))
        for k in reversed(range(len(ups))):
            ct = ups[k][0]
            hi, wi = D.H // 2, D.W // 2
            if k > 0:
                E_ = prog.buf("band.grad.up_in", b, hi, wi, ct.in_channels)
                prog.ops.append(E.ConvOp(adj[k], [E.TV(D), None], E.TV(E_), tag=f"band grad: convT{k}^T (stride 2)"))
                D = prog.buf("band.grad.dup", b, hi, wi, ct.in_channels, gemm=True)
                prog.ops.append(ReluBwdBitsRowsOp(E.TV(E_), E.TV(masks[k - 1]), 2 ** k * s0, E.TV(D)))
            else:
                prog.ops.append(E.ConvOp(adj[0], [E.TV(D), None], E.TV(DX, win=(s0, 0, r1 - s0, w)),
                                         tag="band grad: convT0^T (stride 2)"))
    E.emit_rear_blocks_backward(prog, saved, DX, sl, sg)
    pack_relu_masks(prog)
