"""Bit-packed ReLU masks for the refinement step program (kind ``generator_refine_bits:<H0>x<W0>``).

The backward of the generator's rear reads most forward activations only as ReLU masks ``[y > 0]``: per residual block
the outputs Y1 and Y2 of its two FFC_BN_ACTs and, for both of them, the SpectralTransform's conv1 output T and the
FourierUnit's post-GEMM spectrum Z; then every up-sampling output but the last (the head adjoint's mask).
``pack_relu_masks`` rewrites a built step program so that a ``MaskPackOp`` (ffcb_relu_mask_pack) stores each of them as
one bit per element right after the op that last writes it in the forward, and the backward reads the bits
(``ReluBwdBitsOp``, ffcb_relu_bwd_bits) where it read the values.  The full-width buffers then die at their last
forward read and ``engine.assign_storage_slots`` gives their storage to later buffers.  Nothing is recomputed and the
bits are ``[y > 0]`` of the stored values, so the program computes bit for bit what the default program computes.

The two op types register in ``OP_TYPES`` of this module, apart from ``engine.OP_TYPES``: the default programs never
contain them.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List

from . import engine as E

OP_TYPES: List[type] = []


@dataclass
class MaskPackOp(E.Op, registry=OP_TYPES):
    """bits = [y > 0], one bit per element of the interior of ``y`` (ffcb_relu_mask_pack)."""
    reads, writes = ("y",), ("bits",)
    y: E.TV
    bits: E.TV        # a whole bit-mask buffer (Buf.bits) of y's shape

    def bind(self, ex):
        return "ffcb_relu_mask_pack", ex.lib.ffcb_relu_mask_pack, [ex.ref(self.y), _words(ex, self.bits)]


@dataclass
class ReluBwdBitsOp(E.Op, registry=OP_TYPES):
    """out = dy * bit (ffcb_relu_bwd_bits): ReLU backward with the forward activation's packed mask."""
    reads, writes = ("dy", "bits"), ("out",)
    dy: E.TV
    bits: E.TV
    out: E.TV

    def bind(self, ex):
        return "ffcb_relu_bwd_bits", ex.lib.ffcb_relu_bwd_bits, [ex.ref(self.dy), _words(ex, self.bits),
                                                                 ex.ref(self.out)]


def _words(ex, tv: E.TV) -> int:
    """Device pointer of a whole bit-mask buffer (the kernels take its words dense, sized by the activation's view)."""
    assert tv.buf.bits and _whole(tv)
    return ex.storage[tv.buf.name].data_ptr()


def _whole(tv: E.TV) -> bool:
    return (tv.c0 == 0 and tv.C is None and tv.phase is None and not tv.window and tv.b0 == 0 and tv.nb is None
            and tv.win is None and not tv.bcast)


def pack_relu_masks(prog: E.Program) -> None:
    """Replace every ReluBwdOp of the backward part whose activation the forward part writes by a ReluBwdBitsOp, and
    pack that activation's mask once, right after its last forward write."""
    split = next(i for i, op in enumerate(prog.ops) if isinstance(op, E.SplitOp))
    last_write: Dict[str, int] = {}
    for i, op in enumerate(prog.ops[:split]):
        for tv in op.views()[1]:
            last_write[tv.buf.name] = i
    masks: Dict[str, E.Buf] = {}
    packs: Dict[int, list] = {}           # forward op index -> MaskPackOps that follow it
    ops = list(prog.ops)
    for j in range(split + 1, len(ops)):
        op = ops[j]
        if not (isinstance(op, E.ReluBwdOp) and op.y.buf.name in last_write):
            continue
        y = op.y.buf
        assert _whole(op.y), "a ReLU mask is packed for a whole activation buffer"
        m = masks.get(y.name)
        if m is None:
            m = E.Buf(f"relu_bits.{y.name}#{len(prog.bufs)}", y.B, y.H, y.W, y.C, bits=1)
            prog.bufs.append(m)
            masks[y.name] = m
            packs.setdefault(last_write[y.name], []).append(MaskPackOp(E.TV(y), E.TV(m)))
        ops[j] = ReluBwdBitsOp(op.dy, E.TV(m), op.out)
    prog.ops = [x for i, op in enumerate(ops) for x in [op] + packs.get(i, [])]
