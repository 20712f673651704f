"""Input gradients through the whole generator (kind ``generator_grad``, ``engine.generator_with_input_grad``).

Code that trains or optimises something upstream of a frozen inpainter (mask predictors, object-removal pipelines,
robustness studies) differentiates the generator's output w.r.t. its 4-channel input.  This program is the whole
generator's forward and its input gradient, in two parts like ``generator_rear_grad``:

  part 0   the generator program's front (stem, stride-2 downs; their outputs stay allocated for their ReLU masks),
           the residual blocks with every activation the backward reads kept (``engine.emit_block_chain``: the first
           identity add writes a new buffer, so the last down's output survives), the up-sampling tail and the head:
           input x0 (B, Cin, H, W) -> output y0
  part 1   the rear's backward from g0 = dL/dy0 (``engine.emit_tail_backward`` / ``emit_block_chain_backward``), then per
           down in reverse its ReLU backward and the adjoint of its 3x3 stride-2 contraction (BN scale folded), then the
           stem's ReLU backward and ``ffcb_stem_bwd7``: output dx0 (B, Cin, H, W)

The adjoint of a stride-2 contraction is four sub-pixel phase contractions of the output gradient
(``packing.pack_down_adjoint_phases``).  A reflect-padded FFC down writes them onto the (H+2) x (W+2) padded plane,
ring included, and ``ffcb_fold_reflect_border`` folds the ring back; a zero-padded LaMa-Regular down writes the
interior phases directly (the ring's gradient has nowhere to go).  The last FFC down emits (l, g) through convl2l and
convl2g from one input, so its adjoint is one contraction over all its gradient channels.

The LaMa-Regular blocks (``ResnetBlock``: X + bn2(conv2(pad(relu(bn1(conv1(pad(X))))))) run backward as two
transposed-weight 3x3 contractions (flipped taps, zero border, onto the padded plane) with a fold each; the second fold
adds the identity path's gradient.  Their gradient buffers are contraction operands (split bf16 on the tensor-core arm).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List

import torch
import torch.nn as nn

from . import _lib as L
from . import engine as E
from . import packing as P

OP_TYPES: List[type] = []

HEAD_ACTS = (L.ACT_NONE, L.ACT_SIGMOID, L.ACT_TANH)       # head activations ffcb_head_bwd7 differentiates


@dataclass
class StemBwdOp(E.Op, registry=OP_TYPES):
    """dst = Fold3(Conv7^T(g)): the adjoint of ReflectionPad2d(3) + the 7x7 stem conv w.r.t. the program's NCHW input
    (ffcb_stem_bwd7); ``g`` is the stem pre-activation's gradient (ReLU mask applied), the BN scale is in ``w``."""
    reads, writes = ("g",), ()
    g: E.TV
    w: torch.Tensor   # [N][49][Cin] (packing.pack_stem_adjoint)
    cin: int
    dst: str          # external NCHW output

    def bind(self, ex):
        return "ffcb_stem_bwd7", ex.lib.ffcb_stem_bwd7, [ex.ref(self.g), ex.keep(self.w), self.cin, E.Ext(self.dst)]


# ------------------------------------------------------------------------------------------------ gate
def _ffc_down_ok(d) -> bool:
    """An FFC down with an adjoint here: local input only, a 3x3 stride-2 reflect-padded convl2l (and convl2g, fused
    into one contraction by ``engine.emit_ffc_bn_act``), ReLU on every output half."""
    f = d.ffc
    c = f.convl2l
    if not (f.global_in_num == 0 and type(c) is nn.Conv2d and c.kernel_size == (3, 3) and c.stride == (2, 2)
            and c.padding == (1, 1) and c.dilation == (1, 1) and c.groups == 1 and c.padding_mode == "reflect"
            and c.bias is None and E._act_code(d.act_l) == L.ACT_RELU):
        return False
    g = f.convl2g
    if isinstance(g, nn.Identity):
        return True
    return (type(g) is nn.Conv2d and g.kernel_size == c.kernel_size and g.stride == c.stride and g.padding == c.padding
            and g.dilation == (1, 1) and g.groups == 1 and g.padding_mode == "reflect" and g.bias is None
            and E._act_code(d.act_g) == L.ACT_RELU)


def generator_grad_supported(gen, shape) -> bool:
    """The ``generator_grad`` program exists for input ``shape`` (B, Cin, H, W): the generator is in eval mode with
    every parameter frozen, and
      * FFCResNetGenerator: the no-grad generator program exists (``engine.generator_supported``), every down passes
        ``_ffc_down_ok``, and the rear from the bottleneck has its program (``engine.rear_grad_supported``: block
        gradients, no LFU / gated / out_ffc, a none / sigmoid / tanh head with N <= 4, plane sizes);
      * GlobalGenerator: the no-grad program exists (``engine.global_supported``), at least one up-sampling stage and a
        none / sigmoid / tanh head with N <= 4."""
    if gen.training or any(p.requires_grad for p in gen.parameters()):
        return False
    if shape is None or len(shape) != 4 or shape[0] < 1:
        return False
    x = torch.empty(tuple(shape), device="meta")
    glob = E._global_layout(gen)
    if glob is not None:
        _stem, _bn, _downs, _blocks, ups, head, out_act = glob
        return E.global_supported(glob, x) and bool(ups) and out_act in HEAD_ACTS and head.out_channels <= 4
    lay = E._generator_layout(gen)
    if lay is None or not E.generator_supported(gen, x):
        return False
    _stem, downs, _blocks, _ups, _out_blk, _head, _act = lay
    if not downs or not all(_ffc_down_ok(d) for d in downs):
        return False
    b, _c, h, w = shape
    f = 2 ** len(downs)
    last = downs[-1].ffc
    cl = last.convl2l.out_channels
    cg = 0 if isinstance(last.convl2g, nn.Identity) else last.convl2g.out_channels
    return E.rear_grad_supported(gen, (b, cl, h // f, w // f), (b, cg, h // f, w // f))


# ------------------------------------------------------------------------------------------------ builders
def build_generator_grad_program(prog: E.Program, gen, shape):
    """inputs x0 (forward), g0 (backward part); outputs y0 (as the generator's forward), dx0 = d<y0, g0>/dx0."""
    glob = E._global_layout(gen)
    if glob is not None:
        return _build_global(prog, glob, shape)
    stem, downs, blocks, ups, _out_blk, head, out_act = E._generator_layout(gen)
    b = shape[0]
    s0, sh0 = P.bn_scale_shift(stem.bn_l)
    X = E.emit_stem(prog, stem.ffc.convl2l.weight, s0, sh0, shape, None)
    E.keep_relu_output(prog, stem.bn_l, E.TV(X))
    front = [X]
    cl, cg = X.C, 0
    for d in downs:
        X, cl, cg = E.emit_ffc_bn_act(prog, d, X, cl, cg)
        front.append(X)
    out = prog.buf("in", b, X.H, X.W, X.C, gemm=True, halo=True)
    saved = E.emit_block_chain(prog, blocks, X, out, cl, cg)
    ups_out = E.emit_rear_tail(prog, ups, head, out_act, out)
    prog.ops.append(E.SplitOp())
    prog.inputs["g0"] = prog.outputs["y0"]
    D = E.emit_tail_backward(prog, ups, head, out_act, ups_out, "g0")
    D = E.emit_block_chain_backward(prog, saved, D, cl, cg)
    for k in reversed(range(len(downs))):
        m = downs[k]
        f = m.ffc
        dev = f.convl2l.weight.device
        ws = [f.convl2l.weight]
        scales = [E._fold(m.bn_l, f.convl2l.out_channels, dev)[0]]
        if not isinstance(f.convl2g, nn.Identity):
            ws.append(f.convl2g.weight)
            scales.append(E._fold(m.bn_g, f.convl2g.out_channels, dev)[0])
        D = emit_down_adjoint(prog, front[k + 1], D, torch.cat(ws, 0), torch.cat(scales), front[k], padded=True)
    emit_stem_adjoint(prog, front[0], D, stem.ffc.convl2l.weight, s0, shape)


def _build_global(prog: E.Program, lay, shape):
    """``build_global_program``'s forward with every block's ReLU output kept and the first identity add into a new
    buffer, then its backward (module docstring)."""
    stem, stem_bn, downs, blocks, ups, head, out_act = lay
    b = shape[0]
    dev = head.weight.device
    s0, sh0 = P.bn_scale_shift(stem_bn, stem.bias)
    X = E.emit_stem(prog, stem.weight, s0, sh0, shape, None)
    E.keep_relu_output(prog, stem_bn, E.TV(X))
    front = [X]
    for conv, bn in downs:
        Y = prog.buf("down", b, X.H // 2, X.W // 2, conv.out_channels, gemm=True, halo=True)
        pk = P.pack_conv([(conv.weight, 0, 0, 1)], *P.bn_scale_shift(bn, conv.bias), stride=2, border=L.BORDER_ZERO,
                         act=L.ACT_RELU, device=dev)
        prog.ops.append(E.ConvOp(pk, [E.TV(X), None], E.TV(Y), tag="down 3x3 s2 (zero border)+bn+relu"))
        E.keep_relu_output(prog, bn, E.TV(Y))
        X = Y
        front.append(X)
    out = prog.buf("in", b, X.H, X.W, X.C, gemm=True, halo=True) if blocks else X
    saved = []
    for c1, bn1, c2, bn2 in blocks:
        Y = prog.buf("block.y", b, X.H, X.W, X.C, gemm=True, halo=True)
        pk1 = P.pack_conv([(c1.weight, 0, 0, 1)], *P.bn_scale_shift(bn1, c1.bias), act=L.ACT_RELU, device=dev)
        prog.ops.append(E.ConvOp(pk1, [E.TV(X), None], E.TV(Y), tag="block conv1+bn1+relu"))
        E.keep_relu_output(prog, bn1, E.TV(Y))
        pk2 = P.pack_conv([(c2.weight, 0, 0, 1)], *P.bn_scale_shift(bn2, c2.bias), device=dev)
        prog.ops.append(E.ConvOp(pk2, [E.TV(Y), None], E.TV(out), addend=E.TV(X), addend_post=True,
                                 tag="block conv2+bn2 + x"))
        saved.append((c1, bn1, c2, bn2, Y))
        X = out
    ups_out = E.emit_rear_tail(prog, ups, head, out_act, out)
    prog.ops.append(E.SplitOp())
    prog.inputs["g0"] = prog.outputs["y0"]
    D = E.emit_tail_backward(prog, ups, head, out_act, ups_out, "g0", gemm=True)
    for c1, bn1, c2, bn2, Y in reversed(saved):
        h, w, c = Y.H, Y.W, Y.C
        s1, _ = P.bn_scale_shift(bn1, c1.bias)
        s2, _ = P.bn_scale_shift(bn2, c2.bias)
        GP = prog.buf("grad.gpad", b, h + 2, w + 2, c)
        pk = P.pack_conv([(E._flip_t(c2.weight.detach().double() * s2.double()[:, None, None, None]), 0, 0, 2)],
                         None, None, border=L.BORDER_ZERO, device=dev)
        prog.ops.append(E.ConvOp(pk, [E.TV(D), None], E.TV(GP), tag="grad: block conv2^T"))
        DY = prog.buf("grad.dy", b, h, w, c)
        prog.ops.append(E.FoldOp(E.TV(GP), [], E.TV(DY)))
        DP = prog.buf("grad.dp", b, h, w, c, gemm=True)
        prog.ops.append(E.ReluBwdOp(E.TV(DY), E.TV(Y), E.TV(DP)))
        GP = prog.buf("grad.gpad", b, h + 2, w + 2, c)
        pk = P.pack_conv([(E._flip_t(c1.weight.detach().double() * s1.double()[:, None, None, None]), 0, 0, 2)],
                         None, None, border=L.BORDER_ZERO, device=dev)
        prog.ops.append(E.ConvOp(pk, [E.TV(DP), None], E.TV(GP), tag="grad: block conv1^T"))
        DN = prog.buf("grad.dblock", b, h, w, c, gemm=True)
        prog.ops.append(E.FoldOp(E.TV(GP), [(E.TV(D), 0)], E.TV(DN)))
        D = DN
    for k in reversed(range(len(downs))):
        conv, bn = downs[k]
        D = emit_down_adjoint(prog, front[k + 1], D, conv.weight, P.bn_scale_shift(bn, conv.bias)[0], front[k],
                              padded=False)
    emit_stem_adjoint(prog, front[0], D, stem.weight, s0, shape)


def emit_down_adjoint(prog: E.Program, Y: E.Buf, D: E.Buf, weight: torch.Tensor, scale: torch.Tensor, X: E.Buf,
                      padded: bool) -> E.Buf:
    """Gradient w.r.t. the input ``X`` of Y = relu(scale * conv3x3_s2(pad(X)) + shift), given D = dL/dY: ReLU backward,
    then the four phase contractions onto the padded plane and the reflection's fold (``padded``), or onto the
    interior (zero padding)."""
    b = Y.B
    dev = weight.device
    DP = prog.buf("grad.ddown", b, Y.H, Y.W, Y.C, gemm=True)
    prog.ops.append(E.ReluBwdOp(E.TV(D), E.TV(Y), E.TV(DP)))
    phases = P.pack_down_adjoint_phases(weight, scale, padded=padded, device=dev)
    DX = prog.buf("grad.dx", b, X.H, X.W, X.C)
    if padded:
        GP = prog.buf("grad.gpad", b, X.H + 2, X.W + 2, X.C)
        for a, bb, pk in phases:
            prog.ops.append(E.ConvOp(pk, [E.TV(DP), None], E.TV(GP, phase=(a, bb)),
                                     tag=f"grad: down^T phase {a}{bb} (padded plane)"))
        prog.ops.append(E.FoldOp(E.TV(GP), [], E.TV(DX)))
    else:
        for a, bb, pk in phases:
            prog.ops.append(E.ConvOp(pk, [E.TV(DP), None], E.TV(DX, phase=(a, bb)), tag=f"grad: down^T phase {a}{bb}"))
    return DX


def emit_stem_adjoint(prog: E.Program, S: E.Buf, D: E.Buf, weight: torch.Tensor, scale: torch.Tensor, shape):
    """dx0 from D = dL/dS, S = relu(scale * conv7(reflect_pad3(x0)) + shift): ReLU backward, then ffcb_stem_bwd7."""
    DS = prog.buf("grad.dstem", S.B, S.H, S.W, S.C)
    prog.ops.append(E.ReluBwdOp(E.TV(D), E.TV(S), E.TV(DS)))
    prog.ops.append(StemBwdOp(E.TV(DS), P.pack_stem_adjoint(weight, scale, device=weight.device), shape[1], "dx0"))
    prog.outputs["dx0"] = tuple(shape)
