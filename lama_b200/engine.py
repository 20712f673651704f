"""Program builder + CUDA executor behind the drop-in modules.

A *program* is a straight-line list of op records over named channels-last activation buffers
(``Buf``), built once per (module, input shape, device, math mode) from the module's parameters:
BatchNorm folded, weights packed (``lama_b200.packing``), K-segment lists laid out, buffers
wired so that the local|global halves of an FFC feature map share one allocation (split / concat
are free) and residual adds, bias, BN and activations live in GEMM epilogues.

The executor binds every op to one C-ABI call of ``libffc_b200.so`` with pre-built ctypes
descriptors; replaying a program is a loop of foreign calls on the current CUDA stream (no
allocation, no synchronisation) and is therefore CUDA-graph capturable (``GraphedProgram``).

The op records are plain data so that ``tests/spec_interp.py`` can interpret the very same
program with slow torch/numpy restatements on the CPU box — that is test infrastructure; the
product path below only ever executes through the CUDA library.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import _lib as L
from . import packing as P

PROGRAM_CACHE_SIZE = 3          # executors (programs + their buffers) kept per module, LRU
MATH_ENV = "LAMA_B200_MATH"     # "bf16x3" (default: wgmma arm) | "fp32" (CUDA-core arm)


def default_math() -> int:
    return {"fp32": L.MATH_FP32, "bf16x3": L.MATH_BF16X3}[os.environ.get(MATH_ENV, "bf16x3").lower()]


# ------------------------------------------------------------------------------------------- IR
@dataclass
class Buf:
    """Channels-last activation buffer [B][H+2p][W+2p][C] (fp32) or [2][B][H+2p][W+2p][C] (split bf16)."""
    name: str
    B: int
    H: int
    W: int
    C: int
    pad: int = 0
    fmt: int = L.F32
    reflect_border: int = 0
    cg: int = 0        # > 0: channel-group planar storage [C/cg][B][H][W][cg] (FourierUnit chain, include/ffc_b200.h)
    tile: int = 0      # 128 (with cg == 8, split bf16): tile-blocked [pixel block of 128][C/8][128][8] — wgmma operand tiles
    bits: int = 0      # 1: a ReLU mask, one bit per element — uint32 words [B][H][W][ceil(C/32)] (lama_b200.relu_bits)


@dataclass
class TV:
    """View of a Buf: channel slice [c0, c0+C) and, for transposed-conv outputs, a sub-pixel phase."""
    buf: Buf
    c0: int = 0
    C: Optional[int] = None
    phase: Optional[Tuple[int, int]] = None   # (a, b): pixels (2i+a, 2j+b) of the buffer
    window: int = 0                           # sliding-window view: pixel x exposes pixels x..x+window-1 (C*window channels)
    b0: int = 0                               # batch slice [b0, b0+nb)
    nb: Optional[int] = None
    win: Optional[Tuple[int, int, int, int]] = None   # spatial sub-rectangle (y0, x0, h, w) of the buffer (LFU quadrants)
    bcast: int = 0                            # > 0: a one-image buffer read as a batch of `bcast` images (stride 0)

    @property
    def channels(self) -> int:
        if self.window:
            return self.buf.C * self.window
        return self.buf.C - self.c0 if self.C is None else self.C

    @property
    def batch(self) -> int:
        if self.bcast:
            return self.bcast
        return self.buf.B - self.b0 if self.nb is None else self.nb

    def bslice(self, b0: int, nb: int) -> "TV":
        if self.bcast:
            return TV(self.buf, self.c0, self.C, self.phase, self.window, 0, None, self.win, nb)
        return TV(self.buf, self.c0, self.C, self.phase, self.window, self.b0 + b0, nb, self.win)

    @property
    def hw(self) -> Tuple[int, int]:
        if self.window:
            return (self.buf.H, self.buf.W - self.window)
        if self.win is not None:
            return (self.win[2], self.win[3])
        return (self.buf.H // 2, self.buf.W // 2) if self.phase else (self.buf.H, self.buf.W)


@dataclass(frozen=True)
class Ext:
    """A program input or output named in a call's argument list.  The executor turns an output into its tensor's
    pointer when it binds the call, and an input into a slot that ``CudaExecutor.bind_inputs`` patches."""
    name: str


OP_TYPES: List[type] = []       # every op record type of the default programs (tests check that each one is fully declared)

# What an op does to the reflected ring of a buffer it writes:
STALE = "stale"          # the interior changes, the ring does not: insert_border_ops refreshes it before a ring read
REWRITES = "rewrites"    # the op writes the ring from the new interior itself
KEEPS = "keeps"          # the op sums reflected rings, so the output ring stays a reflection (ffcb_add)


class Op:
    """Base of the op records.  Each type declares, in one place, the fields holding the views it reads and writes
    (``reads`` / ``writes``; a field may hold a view, None, or a list of views or of (view, int) pairs), its ring
    effect on the buffers it writes and the reads that need a valid ring (``ring_in``), its FFT workspace and scratch,
    and ``bind(ex)``: its one C-ABI call on executor ``ex`` as (call name, library function, argument list without the
    trailing stream), or None.  A subclass joins ``OP_TYPES``, or the list given as its ``registry`` class argument
    (the op types of an opt-in program variant defined in another module)."""
    reads: Tuple[str, ...]          # every op type sets both
    writes: Tuple[str, ...]
    ring_in: Tuple[str, ...] = ()
    ring = STALE

    def __init_subclass__(cls, registry: Optional[List[type]] = None, **kw):
        super().__init_subclass__(**kw)
        (OP_TYPES if registry is None else registry).append(cls)

    def _tvs(self, names) -> List[TV]:
        flat = [x for v in (getattr(self, n) for n in names) for x in (v if isinstance(v, list) else [v])]
        return [x[0] if isinstance(x, tuple) else x for x in flat if x is not None]     # (view, int) pairs: FoldOp

    def views(self) -> Tuple[List[TV], List[TV]]:
        """(views read, views written) — the basis of the buffer liveness analysis."""
        return self._tvs(self.reads), self._tvs(self.writes)

    def ring_reads(self) -> List[TV]:
        return self._tvs(self.ring_in)

    def ring_effect(self, prog) -> str:
        return self.ring

    def workspace_bytes(self) -> int:
        return 0

    def scratch_bytes(self) -> int:
        """Device scratch the op's binding allocates besides the program's buffers."""
        return 0


@dataclass
class ToNHWC(Op):
    reads, writes = (), ("out",)
    src: str          # name of an external NCHW float tensor
    out: TV

    def bind(self, ex):
        return "ffcb_nchw_to_nhwc", ex.lib.ffcb_nchw_to_nhwc, [Ext(self.src), *ex.prog.inputs[self.src], ex.ref(self.out)]


@dataclass
class ToNCHW(Op):
    reads, writes = ("inp",), ()
    inp: TV
    dst: str          # name of an external NCHW float output

    def bind(self, ex):
        return "ffcb_nhwc_to_nchw", ex.lib.ffcb_nhwc_to_nchw, [ex.ref(self.inp), Ext(self.dst)]


@dataclass
class StemOp(Op):
    reads, writes = (), ("out",)
    src: str          # external NCHW input
    cin: int
    w: torch.Tensor   # [(ky*7+kx)*Cin + c][N]
    shift: torch.Tensor
    out: TV

    def bind(self, ex):
        return "ffcb_stem_conv7", ex.lib.ffcb_stem_conv7, [Ext(self.src), *ex.prog.inputs[self.src], ex.keep(self.w),
                                                           ex.keep(self.shift), self.w.shape[1], ex.ref(self.out)]


@dataclass
class StemPackOp(Op):
    """NCHW float input -> reflect-padded NHWC8 image for the tensor-core stem (ffcb_stem_pack)."""
    reads, writes = (), ("out",)
    src: str
    cin: int
    out: TV           # Buf (B, H+6, W+8, 8)

    def bind(self, ex):
        return "ffcb_stem_pack", ex.lib.ffcb_stem_pack, [Ext(self.src), *ex.prog.inputs[self.src], ex.ref(self.out)]


@dataclass
class HeadOp(Op):
    reads, writes = ("inp",), ()
    inp: TV
    w: torch.Tensor   # [N][49][C]
    bias: torch.Tensor
    n_out: int
    act: int
    dst: str

    def bind(self, ex):
        return "ffcb_head_conv7", ex.lib.ffcb_head_conv7, [ex.ref(self.inp), ex.keep(self.w), ex.keep(self.bias),
                                                           self.n_out, self.act, Ext(self.dst)]


@dataclass
class HeadGatherOp(Op):
    """y = act(bias + sum_kx q[.., reflect(x+kx-3), n*7+kx]) -> external NCHW output (ffcb_head_gather7)."""
    reads, writes = ("q",), ()
    q: TV
    bias: torch.Tensor
    n_out: int
    act: int
    dst: str

    def bind(self, ex):
        return "ffcb_head_gather7", ex.lib.ffcb_head_gather7, [ex.ref(self.q), ex.keep(self.bias), self.n_out, self.act,
                                                               Ext(self.dst)]


@dataclass
class StemPackU8Op(Op):
    """Decoded RGB bytes + mask bytes -> packed stem image (ffcb_stem_pack_u8): /255, symmetric pad to the
    modulo size, mask > 0, img * (1 - mask), cat(mask), ReflectionPad2d(3)."""
    reads, writes = (), ("out",)
    img: str          # external uint8 (B, H0, W0, 3)
    mask: str         # external uint8 (B, H0, W0)
    h0: int
    w0: int
    out: TV           # Buf (B, H+6, W+8, 8)

    def bind(self, ex):
        return "ffcb_stem_pack_u8", ex.lib.ffcb_stem_pack_u8, [Ext(self.img), Ext(self.mask), ex.prog.inputs[self.img][0],
                                                               self.h0, self.w0, ex.ref(self.out)]


@dataclass
class HeadGatherU8Op(Op):
    """ffcb_head_gather7_blend_u8: head gather + activation + blend with the input + crop + x255/clip/truncate."""
    reads, writes = ("q",), ()
    q: TV
    bias: torch.Tensor
    act: int
    img: str
    mask: str
    h0: int
    w0: int
    dst: str          # external uint8 (B, H0, W0, 3)

    def bind(self, ex):
        return "ffcb_head_gather7_blend_u8", ex.lib.ffcb_head_gather7_blend_u8, [
            ex.ref(self.q), ex.keep(self.bias), self.act, Ext(self.img), Ext(self.mask), self.h0, self.w0, Ext(self.dst)]


@dataclass
class ConvOp(Op):
    reads, writes, ring_in = ("ins", "addend"), ("out",), ("ins",)
    packed: P.PackedConv
    ins: List[Optional[TV]]
    out: TV
    addend: Optional[TV] = None
    addend_post: bool = False
    tag: str = ""

    def ring_effect(self, prog):
        return REWRITES if conv_writes_ring(prog, self) else STALE

    def bind(self, ex):
        d = L.ConvDesc()
        pk = self.packed
        d.inp[0] = ex.tensor(self.ins[0])
        if self.ins[1] is not None:
            d.inp[1] = ex.tensor(self.ins[1])
        d.out = ex.tensor(self.out)
        if self.addend is not None:
            d.addend = ex.tensor(self.addend)
        d.weight = ex.keep(pk.split_weights() if ex.prog.math == L.MATH_BF16X3 else pk.w_kn)
        if pk.shift is not None:
            d.shift = ex.keep(pk.shift)
        d.n_out, d.stride, d.border, d.act = pk.n_out, pk.stride, pk.border, pk.act
        d.nseg, d.math, d.addend_post = len(pk.segs), ex.prog.math, int(self.addend_post)
        for i, s in enumerate(pk.segs):
            d.seg[i] = L.KSeg(s.src, s.dy, s.dx, s.c0, s.nch)
        return "ffcb_conv:" + self.tag, ex.lib.ffcb_conv, [ex.ref(d)]


@dataclass
class RfftOp(Op):
    reads, writes = ("inp",), ("spec",)
    inp: TV
    spec: TV

    def workspace_bytes(self):
        return 8 * self.inp.batch * self.inp.hw[0] * (self.inp.hw[1] // 2 + 1) * self.inp.channels

    def bind(self, ex):
        return "ffcb_rfft2", ex.lib.ffcb_rfft2, [ex.ref(self.inp), ex.ref(self.spec), ex.ws.data_ptr(), ex.ws_bytes]


@dataclass
class IrfftOp(Op):
    reads, writes = ("spec", "residual"), ("out",)
    spec: TV
    residual: Optional[TV]
    out: TV

    def workspace_bytes(self):
        return 8 * self.out.batch * self.out.hw[0] * (self.out.hw[1] // 2 + 1) * self.out.channels

    def bind(self, ex):
        return "ffcb_irfft2", ex.lib.ffcb_irfft2, [ex.ref(self.spec), ex.ref(self.residual), ex.ref(self.out),
                                                   ex.ws.data_ptr(), ex.ws_bytes]


@dataclass
class BorderOp(Op):
    """(Re)build the reflected ring of a padded buffer after a producer that does not write it."""
    reads, writes, ring = ("view",), ("view",), REWRITES
    view: TV

    def bind(self, ex):
        return "ffcb_fill_reflect_border", ex.lib.ffcb_fill_reflect_border, [ex.ref(self.view)]


@dataclass
class ReluBwdOp(Op):
    """out = dy * [y > 0] (ffcb_relu_bwd): ReLU backward with the forward activation."""
    reads, writes = ("dy", "y"), ("out",)
    dy: TV
    y: TV
    out: TV

    def bind(self, ex):
        return "ffcb_relu_bwd", ex.lib.ffcb_relu_bwd, [ex.ref(self.dy), ex.ref(self.y), ex.ref(self.out)]


@dataclass
class FoldOp(Op):
    """Adjoint of the 1-pixel reflect padding (ffcb_fold_reflect_border): gradient w.r.t. the padded plane ``gpad``
    (B,H+2,W+2,C) folded onto the interior, plus optional addends written as (view, first output channel)."""
    reads, writes = ("gpad", "addends"), ("out",)
    gpad: TV
    addends: List[Tuple[TV, int]]
    out: TV

    def bind(self, ex):
        adds = [(ex.ref(tv), c0) for tv, c0 in self.addends] + [(None, 0)] * 2
        return "ffcb_fold_reflect_border", ex.lib.ffcb_fold_reflect_border, [
            ex.ref(self.gpad), adds[0][0], adds[0][1], adds[1][0], adds[1][1], ex.ref(self.out)]


@dataclass
class AddOp(Op):
    """out = a + b over the whole padded extent of three views of one geometry (ffcb_add); ``out`` may be ``a``."""
    reads, writes, ring_in, ring = ("a", "b"), ("out",), ("a", "b"), KEEPS
    a: TV
    b: TV
    out: TV

    def bind(self, ex):
        return "ffcb_add", ex.lib.ffcb_add, [ex.ref(self.a), ex.ref(self.b), ex.ref(self.out)]


@dataclass
class HeadBwdOp(Op):
    """Adjoint of ReflectionPad2d(3) + 7x7 head + act, masked by the last up-sampling ReLU (ffcb_head_bwd7):
    out = [mask > 0] * Fold3(Conv7^T(act'(y) * dy)), with y / dy the external NCHW output and its gradient."""
    reads, writes = ("mask",), ("out",)
    y: str            # external output of the forward part (the head's)
    dy: str           # external NCHW gradient: an input of the backward part, or an output an earlier op writes
    w: torch.Tensor   # [N][49][C] (pack_head)
    n_out: int
    act: int
    mask: TV
    out: TV

    def bind(self, ex):
        return "ffcb_head_bwd7", ex.lib.ffcb_head_bwd7, [Ext(self.y), Ext(self.dy), *ex.prog.outputs[self.y],
                                                         ex.keep(self.w), self.act, ex.ref(self.mask), ex.ref(self.out)]


@dataclass
class RefineLossOp(Op):
    """Gradient of the refinement loss w.r.t. the prediction, and its two terms (ffcb_refine_l1_grad): every operand
    is an external NCHW tensor of the program — ``pred`` and the outputs ``grad`` / ``loss`` are program outputs, the
    rest per-scale inputs (image, mask, ref, md, inv = 1 / n per image and term)."""
    pred: str
    image: str
    mask: str
    ref: str
    md: str
    inv: str
    h0: int
    w0: int
    taps: torch.Tensor    # the 5 float32 Gaussian taps (refine.gaussian_kernel1d)
    grad: str
    loss: str
    ref_numel: int        # B * C * (H0/2) * (W0/2): the kernel's low-resolution scratch
    reads, writes = (), ()    # external tensors only

    def scratch_bytes(self):
        return 4 * self.ref_numel

    def bind(self, ex):
        work = ex.keep(torch.empty(self.ref_numel, dtype=torch.float32))
        return "ffcb_refine_l1_grad", ex.lib.ffcb_refine_l1_grad, [
            Ext(self.pred), Ext(self.image), Ext(self.mask), *ex.prog.outputs[self.pred], self.h0, self.w0,
            Ext(self.ref), Ext(self.md), Ext(self.inv), ex.keep(self.taps.float()), work, Ext(self.grad), Ext(self.loss)]


@dataclass
class SplitOp(Op):
    """Boundary between the forward and the backward part of a forward+backward program (no kernel)."""
    reads, writes = (), ()

    def bind(self, ex):
        ex.split = len(ex.calls)
        return None


@dataclass
class Program:
    kind: str
    math: int
    bufs: List[Buf] = field(default_factory=list)
    ops: list = field(default_factory=list)
    inputs: Dict[str, Tuple[int, ...]] = field(default_factory=dict)    # name -> NCHW shape
    outputs: Dict[str, Tuple[int, ...]] = field(default_factory=dict)
    dtypes: Dict[str, torch.dtype] = field(default_factory=dict)       # inputs / outputs that are not float32
    meta: Dict[tuple, dict] = field(default_factory=dict)              # buffers a backward program needs (per module)
    consts: Dict[str, torch.Tensor] = field(default_factory=dict)      # buffer name -> initial contents [B,H,W,C] float

    def buf(self, name, B, H, W, C, gemm=False, halo=False, halo_px=1, cg=0) -> Buf:
        """``gemm``: the buffer is an operand of a contraction; ``halo``: that contraction has spatial taps.
        FFCB_MATH_BF16X3 stores gemm operands as split bf16, and gives halo buffers a reflected border
        ring so that the TMA box of tap (dy,dx) is the tile shifted by (dx,dy); everything else (FFT
        inputs, spectra leaving the GEMM, the head's input) stays float32 without padding."""
        tc = self.math == L.MATH_BF16X3 and gemm
        ring = halo_px if (tc and halo) else 0
        assert not (cg and ring) and (cg == 0 or C % cg == 0)
        # channel-group planar contraction operands are tile-blocked: one contiguous 16 KB run per (M tile, K block, plane)
        tile = 128 if (cg == 8 and tc) else 0
        b = Buf(f"{name}#{len(self.bufs)}", B, H, W, C, pad=ring, fmt=L.BF16X2 if tc else L.F32,
                reflect_border=1 if ring else 0, cg=cg, tile=tile)
        self.bufs.append(b)
        return b

    def fft_workspace_bytes(self) -> int:
        return max((op.workspace_bytes() for op in self.ops), default=0)


# ------------------------------------------------------------------------------- support predicates
def _act_code(m: nn.Module) -> Optional[int]:
    if isinstance(m, nn.ReLU):
        return L.ACT_RELU
    if isinstance(m, nn.Identity):
        return L.ACT_NONE
    if isinstance(m, nn.Sigmoid):
        return L.ACT_SIGMOID
    if isinstance(m, nn.Tanh):
        return L.ACT_TANH
    return None


def bn_foldable(bn) -> bool:
    """Eval-mode BatchNorm that can be folded into the preceding weights: it must carry running statistics
    (track_running_stats=False uses batch statistics even in eval mode — the torch composition handles that)."""
    if isinstance(bn, nn.Identity):
        return True
    return (isinstance(bn, nn.BatchNorm2d) and bn.track_running_stats and bn.running_var is not None
            and bn.running_mean is not None)


def _plain_conv(conv, k_ok=(1, 3, 7)) -> bool:
    return (isinstance(conv, nn.Conv2d) and conv.groups == 1 and conv.dilation == (1, 1) and conv.bias is None
            and conv.kernel_size[0] == conv.kernel_size[1] and conv.kernel_size[0] in k_ok
            and conv.stride[0] == conv.stride[1] and conv.stride[0] in (1, 2)
            and conv.padding[0] == conv.padding[1] and isinstance(conv.padding[0], int)
            and (conv.padding_mode == 'reflect' or conv.padding[0] == 0)
            and conv.padding[0] <= 1          # activation buffers carry a 1-pixel reflected ring
            and conv.in_channels % 4 == 0 and conv.out_channels % 4 == 0)


FFT_MAX_LEN = 1024


def fft_len_ok(n: int) -> bool:
    """Lengths the shared-memory FFT kernels take (csrc/fft.cu: make_plan, check_fft_shapes): every length 1 .. 1024.
    Lengths up to 447 run 32 channels per CTA, 448 .. 1024 (the bottlenecks of 4K-class photos) 8 channels per CTA."""
    return 1 <= n <= FFT_MAX_LEN


def plane_ok(h: int, w: int) -> bool:
    """Plane sizes the native FFT pair accepts (others take the torch composition)."""
    return w >= 2 and fft_len_ok(h) and fft_len_ok(w)


def ffc_bn_act_supported(m) -> bool:
    f = m.ffc
    if m.training or f.gated:
        return False
    convs = [c for c in (f.convl2l, f.convl2g, f.convg2l) if not isinstance(c, nn.Identity)]
    if not convs or not all(_plain_conv(c) for c in convs):
        return False
    c0 = convs[0]
    if any((c.kernel_size, c.stride, c.padding) != (c0.kernel_size, c0.stride, c0.padding) for c in convs):
        return False
    if c0.kernel_size[0] ** 2 + 1 > L.MAX_KSEG:
        return False
    if not isinstance(f.convg2g, nn.Identity):
        if not f.convg2g.native_supported():
            return False
        if isinstance(f.convl2g, nn.Identity):      # global-only input is never produced by the generator
            return False
    for bn in (m.bn_l, m.bn_g):
        if not bn_foldable(bn):
            return False
    return _act_code(m.act_l) is not None and _act_code(m.act_g) is not None


def ffc_bn_act_shapes_ok(m, x_l, x_g) -> bool:
    f = m.ffc
    if not torch.is_tensor(x_l) or x_l.dim() != 4:
        return False
    in_cg = f.global_in_num
    if (in_cg > 0) != torch.is_tensor(x_g):
        return False
    if torch.is_tensor(x_g) and (x_g.shape[0] != x_l.shape[0] or x_g.shape[2:] != x_l.shape[2:]):
        return False
    c = next(c for c in (f.convl2l, f.convl2g, f.convg2l) if not isinstance(c, nn.Identity))
    k, p = c.kernel_size[0], c.padding[0]
    h, w = x_l.shape[2], x_l.shape[3]
    if p > 0 and (h <= p or w <= p):     # reflect padding needs pad < size
        return False
    if h + 2 * p < k or w + 2 * p < k:
        return False
    if not isinstance(f.convg2g, nn.Identity):
        st = f.convg2g
        if not plane_ok(*st_out_hw(st, h, w)) or not st.native_supported((h, w)):   # LFU needs even square planes
            return False
        if st.stride == 2 and (c.stride[0] != 2 or ((h + 2 * p - k) // 2 + 1, (w + 2 * p - k) // 2 + 1) != (h // 2, w // 2)):
            return False
    return True


def _generator_layout(gen):
    """Parse ``gen.model`` into (stem, downs, blocks, ups, head_conv, out_act) or None."""
    from .modules import FFC_BN_ACT, FFCResnetBlock, ConcatTupleLayer
    mods = list(gen.model)
    i = 0
    try:
        if not (isinstance(mods[0], nn.ReflectionPad2d) and tuple(mods[0].padding) == (3, 3, 3, 3)):
            return None
        stem = mods[1]
        if not (isinstance(stem, FFC_BN_ACT) and isinstance(stem.ffc.convl2l, nn.Conv2d)
                and stem.ffc.convl2l.kernel_size == (7, 7) and stem.ffc.convl2l.padding == (0, 0)
                and stem.ffc.convl2l.stride == (1, 1) and isinstance(stem.ffc.convl2g, nn.Identity)
                and stem.ffc.global_in_num == 0 and isinstance(stem.bn_l, nn.BatchNorm2d) and bn_foldable(stem.bn_l)
                and isinstance(stem.act_l, nn.ReLU) and stem.ffc.convl2l.bias is None
                and stem.ffc.convl2l.groups == 1 and stem.ffc.convl2l.in_channels <= 16
                and stem.ffc.convl2l.out_channels % 4 == 0 and not stem.ffc.gated):
            return None
        i = 2
        downs = []
        while isinstance(mods[i], FFC_BN_ACT):
            if not mods[i].native_supported():
                return None
            downs.append(mods[i]); i += 1
        blocks = []
        while isinstance(mods[i], FFCResnetBlock):
            if mods[i].inline or not mods[i].native_supported():
                return None
            blocks.append(mods[i]); i += 1
        if not isinstance(mods[i], ConcatTupleLayer):
            return None
        i += 1
        ups, i = _up_stages(mods, i)
        if ups is None:
            return None
        out_blk = None
        if isinstance(mods[i], FFCResnetBlock):          # out_ffc=True (ffc.py:356-358): an inline block at full resolution
            if not (mods[i].inline and mods[i].native_supported()):
                return None
            out_blk = mods[i]; i += 1
        head, out_act = _head_stage(mods, i)
        if head is None:
            return None
        return stem, downs, blocks, ups, out_blk, head, out_act
    except IndexError:
        return None


def _up_stages(mods, i):
    """ConvTranspose2d(k3, s2, p1, op1) + BN + ReLU stages from ``mods[i]`` on (ffc.py:350-354, pix2pixhd.py:424-429):
    ([(ct, bn)], index after them), or (None, i) when one of them is off the native path."""
    ups = []
    while isinstance(mods[i], nn.ConvTranspose2d):
        ct, bn, act = mods[i], mods[i + 1], mods[i + 2]
        if not (ct.kernel_size == (3, 3) and ct.stride == (2, 2) and ct.padding == (1, 1)
                and ct.output_padding == (1, 1) and ct.groups == 1 and ct.dilation == (1, 1)
                and isinstance(bn, nn.BatchNorm2d) and bn_foldable(bn) and isinstance(act, nn.ReLU)
                and ct.in_channels % 4 == 0 and ct.out_channels % 4 == 0):
            return None, i
        ups.append((ct, bn)); i += 3
    return ups, i


def _head_stage(mods, i):
    """ReflectionPad2d(3) + Conv2d 7x7 [+ activation] ending ``mods`` at ``mods[i]`` (ffc.py:360-363,
    pix2pixhd.py:430-433): (head conv, activation code), or (None, None)."""
    if not (isinstance(mods[i], nn.ReflectionPad2d) and tuple(mods[i].padding) == (3, 3, 3, 3)):
        return None, None
    head = mods[i + 1]
    if not (isinstance(head, nn.Conv2d) and head.kernel_size == (7, 7) and head.padding == (0, 0)
            and head.stride == (1, 1) and head.groups == 1 and head.out_channels <= 4
            and head.in_channels % 4 == 0):
        return None, None
    i += 2
    out_act = L.ACT_NONE
    if i < len(mods):
        out_act = _act_code(mods[i])
        if out_act is None:
            return None, None
        i += 1
    return (head, out_act) if i == len(mods) else (None, None)


def _affine_bn(bn) -> bool:
    return isinstance(bn, nn.BatchNorm2d) and bn.affine and bn_foldable(bn)


def _biased_conv(conv, k: int, stride: int, padding: int, padding_mode: str) -> bool:
    return (type(conv) is nn.Conv2d and conv.kernel_size == (k, k) and conv.stride == (stride, stride)
            and conv.padding == (padding, padding) and conv.dilation == (1, 1) and conv.groups == 1
            and conv.padding_mode == padding_mode and conv.in_channels % 4 == 0 and conv.out_channels % 4 == 0)


def _global_layout(gen):
    """Parse the ``model`` of a LaMa-Regular generator (``lama_b200.pix2pixhd.GlobalGenerator``,
    pix2pixhd.py:341-436) into (stem conv, stem bn, downs [(conv, bn)], blocks [(conv1, bn1, conv2, bn2)], ups
    [(ct, bn)], head conv, out act), or None when a stage is off the native path: every conv plain (groups 1,
    dilation 1), every norm an eval BatchNorm with affine parameters, every activation ReLU, the blocks reflect-padded
    ``ResnetBlock``s without an input conv or dropout."""
    from .pix2pixhd import GlobalGenerator, ResnetBlock
    if not isinstance(gen, GlobalGenerator):
        return None
    mods = list(gen.model)
    try:
        if not (isinstance(mods[0], nn.ReflectionPad2d) and tuple(mods[0].padding) == (3, 3, 3, 3)):
            return None
        stem, stem_bn = mods[1], mods[2]
        if not (type(stem) is nn.Conv2d and stem.kernel_size == (7, 7) and stem.padding == (0, 0)
                and stem.stride == (1, 1) and stem.groups == 1 and stem.in_channels <= 16
                and stem.out_channels % 4 == 0 and _affine_bn(stem_bn) and isinstance(mods[3], nn.ReLU)):
            return None
        i = 4
        downs = []
        while type(mods[i]) is nn.Conv2d:
            conv, bn, act = mods[i], mods[i + 1], mods[i + 2]
            if not (_biased_conv(conv, 3, 2, 1, 'zeros') and _affine_bn(bn) and isinstance(act, nn.ReLU)):
                return None
            downs.append((conv, bn)); i += 3
        blocks = []
        while isinstance(mods[i], ResnetBlock):
            blk = mods[i]
            cb = list(blk.conv_block)
            if blk.in_dim is not None or len(cb) != 7:
                return None
            pad1, c1, bn1, act, pad2, c2, bn2 = cb
            if not (all(isinstance(p, nn.ReflectionPad2d) and tuple(p.padding) == (1, 1, 1, 1) for p in (pad1, pad2))
                    and all(_biased_conv(c, 3, 1, 0, 'zeros') and c.in_channels == c.out_channels for c in (c1, c2))
                    and _affine_bn(bn1) and _affine_bn(bn2) and isinstance(act, nn.ReLU)):
                return None
            blocks.append((c1, bn1, c2, bn2)); i += 1
        ups, i = _up_stages(mods, i)
        if ups is None:
            return None
        head, out_act = _head_stage(mods, i)
        if head is None:
            return None
        return stem, stem_bn, downs, blocks, ups, head, out_act
    except IndexError:
        return None


def generator_in_channels(gen) -> int:
    """Input channels of a drop-in generator (image + mask: 4 for the shipped models)."""
    from .pix2pixhd import GlobalGenerator
    return gen.model[1].in_channels if isinstance(gen, GlobalGenerator) else gen.model[1].ffc.convl2l.in_channels


def generator_supported(gen, x) -> bool:
    glob = _global_layout(gen)
    if glob is not None:
        return global_supported(glob, x)
    lay = _generator_layout(gen)
    if lay is None or x.dim() != 4:
        return False
    stem, downs, _blocks, _ups, out_blk, _head, _ = lay
    b, c, h, w = x.shape
    if out_blk is not None:        # its FourierUnit transforms full-resolution planes
        f0 = out_blk.conv1.ffc
        if not ffc_bn_act_shapes_ok(out_blk.conv1, torch.empty(1, f0.convl2l.in_channels, h, w, device="meta"),
                                    torch.empty(1, f0.global_in_num, h, w, device="meta")):
            return False
    if c != stem.ffc.convl2l.in_channels or h < 4 or w < 4:
        return False
    f = 2 ** len(downs)
    if h % f or w % f:                      # ConvTranspose doubles sizes: only exact multiples round-trip
        return False
    if blocks_use_fft(gen) and not plane_ok(h // f, w // f):     # e.g. 1025-wide planes (images above 8192 px)
        return False
    return h // f >= 2 and w // f >= 2      # reflect pad 1 at the bottleneck


def global_supported(lay, x) -> bool:
    """A GlobalGenerator program exists for input ``x``: 4 x H x W with H and W multiples of 2^n_down and at least
    2 pixels per bottleneck axis (the blocks' reflect padding of 1).  No FFT runs, so no plane-size limit applies."""
    stem, _bn, downs, _blocks, _ups, _head, _act = lay
    if x.dim() != 4:
        return False
    _b, c, h, w = x.shape
    f = 2 ** len(downs)
    return (c == stem.in_channels and h >= 4 and w >= 4 and h % f == 0 and w % f == 0
            and h // f >= 2 and w // f >= 2)


def blocks_use_fft(gen) -> bool:
    lay = _generator_layout(gen)
    return lay is not None and any(not isinstance(b.conv1.ffc.convg2g, nn.Identity) for b in lay[2])


# -------------------------------------------------------------------------------------- builders
def _fold(bn, n, device):
    if isinstance(bn, nn.BatchNorm2d):
        return P.bn_scale_shift(bn)
    return torch.ones(n, dtype=torch.float64, device=device), torch.zeros(n, dtype=torch.float64, device=device)


def fu_batch_chunk(batch: int, h: int, w: int, c: int) -> int:
    """Images per pass of the rfft2 -> GEMM -> irfft2 chain.  Running the chain over slices of the batch keeps
    its intermediates inside the 50 MB L2 at the cost of extra launches and partial waves.  Default: whole batch;
    LAMA_B200_FU_CHUNK=n slices."""
    n = int(os.environ.get("LAMA_B200_FU_CHUNK", "0"))
    return batch if n <= 0 else min(batch, n)


def fu_planar_ok(prog: Program, st, h: int, w: int) -> bool:
    """Channel-group planar storage for the SpectralTransform chain (conv1 -> rfft2 -> spectral conv -> irfft2 ->
    conv2): every (image, 4-channel group) plane set is one dense block for the second-generation plane FFT kernels
    (csrc/fft_plane_cg.cu) and the GEMMs read [K/8][pixel][8] operand tiles.  Needs the tensor-core arm, 64x64 or 32x32
    planes (the 512x512 / 256x256 bottleneck) and whole 64-channel K blocks on every contraction of the chain.
    LAMA_B200_FU_LAYOUT=nhwc keeps the round-1 channels-last chain (A/B measurements)."""
    if prog.math != L.MATH_BF16X3 or os.environ.get("LAMA_B200_FU_LAYOUT", "planar") != "planar":
        return False
    dev = st.conv2.weight.device
    if dev.type == "cuda" and not planar_selftest(dev):
        return False
    c = st.conv1[0].out_channels
    fu = st.fu
    if st.enable_lfu and not ((h, w) == (64, 64) and c % 32 == 0):      # LFU quadrants: 32x32 planes, c/4 % 8 == 0
        return False
    return ((h, w) in ((64, 64), (32, 32)) and c % 64 == 0 and fu.conv_layer.in_channels == 2 * c + (2 if fu.spectral_pos_encoding else 0)
            and fu.conv_layer.out_channels == 2 * c)


_PLANAR_OK: Dict[int, bool] = {}


def planar_selftest(device: torch.device) -> bool:
    """Once per process and device: run the planar chain's three kernels (plane FFT pair, interleaved-operand GEMM with
    a planar output) on a small random problem and compare with torch on the same device.  The chain depends on
    details no compile-time check covers (wgmma no-swizzle descriptor fields, bulk-copy tile layout); if the check
    fails the process keeps the channels-last chain of round 1 (still the native kernels) and says so loudly —
    LAMA_B200_FU_LAYOUT=planar! skips the check and forces the planar chain, =nhwc forces the other."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if os.environ.get("LAMA_B200_FU_LAYOUT") == "planar!":
        return True
    if idx in _PLANAR_OK:
        return _PLANAR_OK[idx]
    ok, why = True, ""
    try:
        with torch.no_grad():
            b, c, h = 2, 64, 64
            wf = h // 2 + 1
            g = torch.Generator().manual_seed(1234)
            prog = Program("planar_selftest", L.MATH_BF16X3)
            X = prog.buf("x", b, h, h, c, cg=4)
            S = prog.buf("s", b, h, wf, 2 * c, gemm=True, cg=8)
            Z = prog.buf("z", b, h, wf, 2 * c, cg=8)
            U = prog.buf("u", b, h, h, c, gemm=True, cg=8)
            wgt = torch.randn(2 * c, 2 * c, 1, 1, generator=g) * 0.1
            pk = P.pack_conv([(wgt, 0, 0, 0)], None, None, act=L.ACT_RELU)
            prog.inputs = {"x0": (b, c, h, h)}
            prog.ops += [ToNHWC("x0", TV(X)), RfftOp(TV(X), TV(S)), ConvOp(pk, [TV(S), None], TV(Z)),
                         IrfftOp(TV(Z), TV(X), TV(U)), ToNCHW(TV(U), "y0")]
            prog.outputs = {"y0": (b, c, h, h)}
            x = torch.randn(b, c, h, h, generator=g).to(device)
            y = CudaExecutor(prog, device).run({"x0": x})["y0"]
            f = torch.fft.rfftn(x.double(), dim=(-2, -1), norm="ortho")
            f = torch.stack((f.real, f.imag), dim=2).reshape(b, 2 * c, h, wf)
            f = torch.relu(torch.einsum("nk,bkyx->bnyx", wgt[:, :, 0, 0].double().to(device), f))
            f = f.reshape(b, c, 2, h, wf)
            want = x.double() + torch.fft.irfftn(torch.complex(f[:, :, 0], f[:, :, 1]), s=(h, h), dim=(-2, -1), norm="ortho")
            err = float((y.double() - want).abs().max()) / float(want.abs().max())
            ok, why = err < 1e-3, f"relative error {err:.2e}"
    except Exception as e:  # noqa: BLE001  (a launch failure is an answer too)
        ok, why = False, f"{type(e).__name__}: {e}"
    _PLANAR_OK[idx] = ok
    if not ok:
        import warnings
        msg = (f"lama_b200: the channel-group planar FourierUnit chain failed its start-up check on cuda:{idx} ({why}); "
               f"using the channels-last chain (native round-1 kernels) instead")
        warnings.warn(msg, RuntimeWarning)
        print(msg, file=__import__("sys").stderr, flush=True)
    return ok


def emit_fourier_unit(prog: Program, fu, t: TV, out: TV, residual: Optional[TV]):
    """FourierUnit (ffc.py:76-113): rfft2 -> [1x1 conv + BN + ReLU] on the interleaved spectrum -> irfft2,
    optionally with the SpectralTransform residual fused into the inverse (out = residual + fu(t))."""
    b = t.batch
    h, w = t.hw
    wf = w // 2 + 1
    cout2 = fu.conv_layer.out_channels
    cin2 = fu.conv_layer.in_channels - (2 if fu.spectral_pos_encoding else 0)       # spectrum channels (ffc.py:57)
    planar = t.buf.cg == 4      # FourierUnit chain in channel-group planar storage (emit_spectral_transform decides)
    S = prog.buf("spectrum", b, h, wf, cin2, gemm=True, cg=8 if planar else 0)
    Z = prog.buf("spectrum_out", b, h, wf, cout2, cg=8 if planar else 0)
    prog.meta[("fu", id(fu))] = dict(S=S, Z=Z)
    scale, shift = P.bn_scale_shift(fu.bn)
    wconv, pos = fu.conv_layer.weight, None
    if fu.spectral_pos_encoding:
        # ffc.py:91-95 prepends two coordinate channels (linspace over H and over W/2+1) to the spectrum.  They do not
        # depend on the data: their contribution W[:, :2] . (v, h) is a per-position addend of the spectral GEMM
        # (BN scale folded), broadcast over the batch.
        wpos = wconv.detach().double()[:, :2, 0, 0] * scale.double()[:, None]                     # [2co, 2]
        wconv = wconv[:, 2:]
        vert = torch.linspace(0, 1, h, dtype=torch.float64, device=wpos.device)
        hor = torch.linspace(0, 1, wf, dtype=torch.float64, device=wpos.device)
        PE = prog.buf("fu.pos_addend", 1, h, wf, cout2)
        prog.consts[PE.name] = (vert[:, None, None] * wpos[:, 0] + hor[None, :, None] * wpos[:, 1])[None].float()
        pos = TV(PE, bcast=b)
    cin2 = wconv.shape[1]
    pk = P.pack_conv([(wconv, 0, 0, 0)], scale, shift, act=L.ACT_RELU, device=fu.conv_layer.weight.device)
    chunk = fu_batch_chunk(b, h, w, cin2 // 2) if prog.math == L.MATH_BF16X3 else b
    if planar and ((chunk * h * wf) % 128 or (chunk * h * w) % 128):
        chunk = b          # tile-blocked buffers can only be sliced on 128-pixel blocks
    for b0 in range(0, b, chunk):
        nb = min(chunk, b - b0)
        prog.ops.append(RfftOp(t.bslice(b0, nb), TV(S).bslice(b0, nb)))
        prog.ops.append(ConvOp(pk, [TV(S).bslice(b0, nb), None], TV(Z).bslice(b0, nb),
                               addend=pos.bslice(b0, nb) if pos is not None else None, tag="fu.conv_layer+bn+relu"))
        prog.ops.append(IrfftOp(TV(Z).bslice(b0, nb), residual.bslice(b0, nb) if residual is not None else None,
                                out.bslice(b0, nb)))


def st_out_hw(st, h: int, w: int) -> Tuple[int, int]:
    """Spatial size SpectralTransform works at: AvgPool2d(2, 2) first when stride == 2 (ffc.py:122-125)."""
    return (h // 2, w // 2) if st.stride == 2 else (h, w)


def lfu_supported(st, h: int, w: int) -> bool:
    """LFU (ffc.py:148-157) natively: the first c/4 channels, cut into 2x2 quadrants stacked as channels — the
    reference splits rows AND columns by h // 2, which only type-checks for even square planes; quadrant views carry
    c/4 channels and every view needs a multiple of 4."""
    c = st.conv1[0].out_channels
    return h == w and h % 2 == 0 and h >= 4 and c % 16 == 0 and st.lfu.native_supported()


def emit_spectral_transform(prog: Program, st, x: TV, u_consumer=None) -> Tuple[TV, P.PackedConv]:
    """SpectralTransform (ffc.py:142-163) up to, but not including, conv2: returns the view holding
    ``x1 + fu(x1) [+ tile(lfu(quadrants(x1)))]`` and lets the caller fuse conv2 into its own contraction.
    stride 2: AvgPool2d(2,2) + the 1x1 conv1 are ONE 2x2 stride-2 contraction (four taps with conv1.weight / 4)."""
    b = x.buf.B
    h, w = st_out_hw(st, *x.hw)
    c = st.conv1[0].out_channels
    dev = st.conv2.weight.device
    planar = fu_planar_ok(prog, st, h, w)
    T = prog.buf("st.t", b, h, w, c, cg=4 if planar else 0)
    U = prog.buf("st.u", b, h, w, c, gemm=True, cg=8 if planar else 0)
    s1, b1 = P.bn_scale_shift(st.conv1[1])
    if st.stride == 2:
        w1 = st.conv1[0].weight.detach().repeat(1, 1, 2, 2) / 4.0
        pk1 = P.pack_conv([(w1, 0, x.c0, 0)], s1, b1, stride=2, act=L.ACT_RELU, device=dev)
        tag = "st.avgpool2x2+conv1+bn+relu"
    else:
        pk1 = P.pack_conv([(st.conv1[0].weight, 0, x.c0, 0)], s1, b1, act=L.ACT_RELU, device=dev)
        tag = "st.conv1+bn+relu"
    prog.ops.append(ConvOp(pk1, [TV(x.buf), None], TV(T), tag=tag))
    prog.meta[("st", id(st))] = dict(T=T, U=U)
    residual = TV(T)
    if st.enable_lfu:
        # xs = lfu(quadrants of the first c/4 channels) tiled 2x2; XS = T + tile(xs) becomes the residual of the main
        # inverse transform, so  U = T + fu(T) + tile(xs)  (ffc.py:161) costs no extra pass over U
        lfu, c4, s = st.lfu, c // 4, h // 2
        sf = s // 2 + 1
        XS = prog.buf("st.xs", b, h, w, c, cg=4 if planar else 0)
        LS = prog.buf("lfu.spectrum", b, s, sf, 2 * c, gemm=True, cg=8 if planar else 0)
        LZ = prog.buf("lfu.spectrum_out", b, s, sf, 2 * c, cg=8 if planar else 0)
        # channel order of the two torch.cat calls (ffc.py:152-155): top-left, bottom-left, top-right, bottom-right
        for q, (qy, qx) in enumerate([(0, 0), (1, 0), (0, 1), (1, 1)]):
            prog.ops.append(RfftOp(TV(T, 0, c4, win=(qy * s, qx * s, s, s)), TV(LS, q * 2 * c4, 2 * c4)))
        sc, sh = P.bn_scale_shift(lfu.bn)
        pkl = P.pack_conv([(lfu.conv_layer.weight, 0, 0, 0)], sc, sh, act=L.ACT_RELU, device=dev)
        prog.ops.append(ConvOp(pkl, [TV(LS), None], TV(LZ), tag="lfu.conv_layer+bn+relu"))
        for ty in (0, 1):
            for tx in (0, 1):          # .repeat(1, 1, 2, 2) (ffc.py:157): the same s x s result in all four quadrants
                wq = (ty * s, tx * s, s, s)
                prog.ops.append(IrfftOp(TV(LZ), TV(T, win=wq), TV(XS, win=wq)))
        residual = TV(XS)
    emit_fourier_unit(prog, st.fu, TV(T), TV(U), residual=residual)
    return TV(U)


def emit_ffc_bn_act(prog: Program, m, X: Buf, in_cl: int, in_cg: int, residual: Optional[Buf] = None,
                    Y: Optional[Buf] = None) -> Tuple[Buf, int, int]:
    """FFC + BN + activation (ffc.py:205-225, 251-255) reading [x_l | x_g] from ``X`` and writing
    [y_l | y_g] into ``Y`` (allocated here unless given).  With ``residual`` the block identity
    (ffc.py:288) is added after the activation in the same epilogues.
    Returns (Y, out_cl, out_cg)."""
    f = m.ffc
    dev = next(m.parameters()).device
    conv0 = next(c for c in (f.convl2l, f.convl2g, f.convg2l) if not isinstance(c, nn.Identity))
    k, s, p = conv0.kernel_size[0], conv0.stride[0], conv0.padding[0]
    out_cl = f.convl2l.out_channels if not isinstance(f.convl2l, nn.Identity) else (
        f.convg2l.out_channels if not isinstance(f.convg2l, nn.Identity) else 0)
    out_cg = f.convl2g.out_channels if not isinstance(f.convl2g, nn.Identity) else 0
    ho, wo = (X.H + 2 * p - k) // s + 1, (X.W + 2 * p - k) // s + 1
    if Y is None:
        Y = prog.buf("ffc.out", X.B, ho, wo, out_cl + out_cg, gemm=True, halo=True)
    act_l, act_g = _act_code(m.act_l), _act_code(m.act_g)
    sl, bl = _fold(m.bn_l, out_cl, dev)
    sg, bg = _fold(m.bn_g, out_cg, dev)
    has_spectral = not isinstance(f.convg2g, nn.Identity)
    res_l = TV(residual, 0, out_cl) if residual is not None else None
    res_g = TV(residual, out_cl, out_cg) if residual is not None else None

    if in_cg == 0 and out_cl > 0 and out_cg > 0 and act_l == act_g:
        # local input only (stem-like / downsample-to-global): convl2l and convl2g read the same
        # pixels, so they are ONE contraction with N = out_cl + out_cg.
        wcat = torch.cat([f.convl2l.weight, f.convl2g.weight], dim=0)
        pk = P.pack_conv([(wcat, 0, 0, p)], torch.cat([sl, sg]), torch.cat([bl, bg]), stride=s, act=act_l, device=dev)
        prog.ops.append(ConvOp(pk, [TV(X, 0, in_cl), None], TV(Y), addend=TV(residual) if residual else None,
                               addend_post=True, tag="convl2l|convl2g+bn+act"))
        return Y, out_cl, out_cg

    if out_cl > 0:
        # y_l = act(bn_l(convl2l(x_l) + convg2l(x_g))): x_l|x_g are adjacent channels of X, so the
        # two convolutions are one contraction over C = in_cl + in_cg.
        ws = [f.convl2l.weight] + ([f.convg2l.weight] if in_cg > 0 else [])
        pk = P.pack_conv([(torch.cat(ws, dim=1), 0, 0, p)], sl, bl, stride=s, act=act_l, device=dev)
        prog.ops.append(ConvOp(pk, [TV(X), None], TV(Y, 0, out_cl), addend=res_l, addend_post=True,
                               tag="convl2l+convg2l+bn_l+act"))
    if out_cg > 0:
        parts = [(f.convl2g.weight, 0, 0, p)]     # ffc_bn_act_supported() guarantees convl2g exists
        ins = [TV(X), None]
        pre = None
        if has_spectral:
            U = emit_spectral_transform(prog, f.convg2g, TV(X, in_cl, in_cg))
            if s == 1:
                parts.append((f.convg2g.conv2.weight, 1, 0, 0))
                ins[1] = U
            else:
                # stride-2 FFC (ffc.py:122-125, 221-224): convl2g samples X with stride 2 while conv2 reads the already
                # pooled u with stride 1 — one ffcb_conv has one stride, so conv2 (with bn_g's scale folded, no shift)
                # runs first and joins the 3x3 contraction as its pre-activation addend.  Never a residual layer.
                assert residual is None
                A = prog.buf("st.conv2.out", X.B, ho, wo, out_cg)
                pk2 = P.pack_conv([(f.convg2g.conv2.weight, 0, 0, 0)], sg, None, device=dev)
                prog.ops.append(ConvOp(pk2, [U, None], TV(A), tag="st.conv2 (x bn_g scale)"))
                pre = TV(A)
        # y_g = act(bn_g(convl2g(x_l) + conv2(x1 + fu(x1)))): conv2 rides as one more K-segment.
        pk = P.pack_conv(parts, sg, bg, stride=s, act=act_g, device=dev)
        prog.ops.append(ConvOp(pk, ins, TV(Y, out_cl, out_cg), addend=pre if pre is not None else res_g,
                               addend_post=pre is None, tag="convl2g+st.conv2+bn_g+act"))
    return Y, out_cl, out_cg


def emit_resnet_block(prog: Program, blk, X: Buf, cl: int, cg: int, in_place: bool) -> Buf:
    """FFCResnetBlock (ffc.py:277-292): X <- X + conv2(conv1(X)).  With ``in_place`` the second
    FFC_BN_ACT writes its result over X (each output pixel only reads its own residual pixel)."""
    Y, ycl, ycg = emit_ffc_bn_act(prog, blk.conv1, X, cl, cg)
    out = X if in_place else prog.buf("block.out", X.B, X.H, X.W, X.C, gemm=True, halo=True)
    emit_ffc_bn_act(prog, blk.conv2, Y, ycl, ycg, residual=X, Y=out)
    return out


# Largest plane side the forward+backward block program (and the rear / refinement step programs built on it) is used
# for: every plane the native FFT pair takes.  Its input gradients are tested against float64 autograd through the
# oracle from 12x20 up to 256x256 (tests/test_gpu_parity.py, tests/test_gpu_program_diff.py), at 211x251 (Bluestein,
# tests/test_gpu_fft_bluestein.py) and at 270x480, 259x108 and 128x1024 (8-channel and Bluestein FFT lengths,
# tests/test_gpu_refine_large_planes.py).  Wider planes are rejected by the FFT kernels and take torch autograd.
BLOCK_GRAD_MAX_PLANE = FFT_MAX_LEN


def block_grad_supported(blk) -> bool:
    """Input gradients (SURVEY.md row f3) exist for the residual-block flavour of the shipped generators: two
    FFC_BN_ACT with local and global halves on both sides, 3x3 reflect convs, stride 1, ReLU, no LFU / gating."""
    if blk.inline or not blk.native_supported():
        return False
    for m in (blk.conv1, blk.conv2):
        f = m.ffc
        if any(isinstance(c, nn.Identity) for c in (f.convl2l, f.convl2g, f.convg2l, f.convg2g)):
            return False
        st = f.convg2g
        if (f.convl2l.kernel_size != (3, 3) or f.convl2l.stride != (1, 1) or f.convl2l.padding != (1, 1)
                or st.enable_lfu or st.stride != 1 or _act_code(m.act_l) != L.ACT_RELU or _act_code(m.act_g) != L.ACT_RELU):
            return False
    return True


def _flip_t(w: torch.Tensor) -> torch.Tensor:
    """[N, C, k, k] forward conv weight -> [C, N, k, k] weight of the gradient convolution (taps flipped)."""
    return w.detach().double().flip(-1, -2).transpose(0, 1).contiguous()


def emit_ffc_bn_act_backward(prog: Program, m, Y: Buf, DO: TV, in_cl: int, in_cg: int,
                             extra: Optional[TV] = None) -> Buf:
    """Gradient of one FFC_BN_ACT (ffc.py:205-225, 251-255; eval-mode BN) w.r.t. its input [x_l | x_g], given the
    gradient ``DO`` w.r.t. its output and the forward activations kept in ``prog`` (Y, t, z).  Every step is one of
    the forward's own operations with transposed weights:
      dP   = dO * [Y > 0]
      d[x_l|x_g]_pad = 3x3 gradient convolutions of dP (flipped taps, zero border) -> folded back (reflect adjoint)
      du   = W2^T (s_g dP_g);  dz = rfft2(du) * [z > 0];  ds = Wf^T (s_f dz);  dt = du + irfft2(ds)
             (the half-spectrum weights 2 and 1/2 of the two adjoint transforms cancel around the per-position GEMM)
      dx_g += W1^T (s_1 (dt * [t > 0]))
    ``extra``: one more gradient added into the result (the block's identity path)."""
    f = m.ffc
    st = f.convg2g
    dev = f.convl2l.weight.device
    b, h, w = Y.B, Y.H, Y.W
    out_cl, out_cg = f.convl2l.out_channels, f.convl2g.out_channels
    sl, _ = _fold(m.bn_l, out_cl, dev)
    sg, _ = _fold(m.bn_g, out_cg, dev)
    s1, _ = P.bn_scale_shift(st.conv1[1])
    sf, _ = P.bn_scale_shift(st.fu.bn)
    saved_st, saved_fu = prog.meta[("st", id(st))], prog.meta[("fu", id(st.fu))]
    T, Z = saved_st["T"], saved_fu["Z"]
    planar = T.cg == 4
    c = st.conv1[0].out_channels
    wf_ = w // 2 + 1
    k4 = lambda t: t[:, :, None, None]      # noqa: E731
    col = lambda v: v.double()[:, None, None, None]   # noqa: E731

    DP = prog.buf("grad.dP", b, h, w, out_cl + out_cg, gemm=True)
    prog.ops.append(ReluBwdOp(DO, TV(Y), TV(DP)))
    GP = prog.buf("grad.gpad", b, h + 2, w + 2, in_cl + in_cg)
    w_to_l = torch.cat([f.convl2l.weight.detach().double() * col(sl), f.convl2g.weight.detach().double() * col(sg)], dim=0)
    pk_a = P.pack_conv([(_flip_t(w_to_l), 0, 0, 2)], None, None, border=L.BORDER_ZERO, device=dev)
    prog.ops.append(ConvOp(pk_a, [TV(DP), None], TV(GP, 0, in_cl), tag="grad: d x_l (3x3^T of dP_l|dP_g)"))
    pk_b = P.pack_conv([(_flip_t(f.convg2l.weight.detach().double() * col(sl)), 0, 0, 2)], None, None,
                       border=L.BORDER_ZERO, device=dev)
    prog.ops.append(ConvOp(pk_b, [TV(DP), None], TV(GP, in_cl, in_cg), tag="grad: d x_g (3x3^T of dP_l)"))

    DU = prog.buf("grad.du", b, h, w, c, cg=4 if planar else 0)
    w2 = st.conv2.weight.detach().double()[:, :, 0, 0] * sg.double()[:, None]            # [out_cg, c]
    pk2 = P.pack_conv([(k4(w2.t().contiguous()), 0, out_cl, 0)], None, None, device=dev)
    prog.ops.append(ConvOp(pk2, [TV(DP), None], TV(DU), tag="grad: du = conv2^T"))
    DZ = prog.buf("grad.dz", b, h, wf_, 2 * c, gemm=True, cg=8 if planar else 0)
    prog.ops.append(RfftOp(TV(DU), TV(DZ)))
    DPZ = prog.buf("grad.dpz", b, h, wf_, 2 * c, gemm=True, cg=8 if planar else 0)
    prog.ops.append(ReluBwdOp(TV(DZ), TV(Z), TV(DPZ)))
    DS = prog.buf("grad.ds", b, h, wf_, 2 * c, cg=8 if planar else 0)
    wfu = st.fu.conv_layer.weight.detach().double()[:, :, 0, 0] * sf.double()[:, None]  # [2c out, 2c in]
    pkf = P.pack_conv([(k4(wfu.t().contiguous()), 0, 0, 0)], None, None, device=dev)
    prog.ops.append(ConvOp(pkf, [TV(DPZ), None], TV(DS), tag="grad: ds = fu.conv_layer^T"))
    DT = prog.buf("grad.dt", b, h, w, c, cg=4 if planar else 0)
    prog.ops.append(IrfftOp(TV(DS), TV(DU), TV(DT)))
    DPT = prog.buf("grad.dpt", b, h, w, c, gemm=True, cg=8 if planar else 0)
    prog.ops.append(ReluBwdOp(TV(DT), TV(T), TV(DPT)))
    DG = prog.buf("grad.dg", b, h, w, in_cg)
    w1 = st.conv1[0].weight.detach().double()[:, :, 0, 0] * s1.double()[:, None]        # [c, in_cg]
    pk1 = P.pack_conv([(k4(w1.t().contiguous()), 0, 0, 0)], None, None, device=dev)
    prog.ops.append(ConvOp(pk1, [TV(DPT), None], TV(DG), tag="grad: d x_g += conv1^T"))
    DX = prog.buf("grad.dx", b, h, w, in_cl + in_cg)
    prog.ops.append(FoldOp(TV(GP), [(TV(DG), in_cl)] + ([(extra, 0)] if extra is not None else []), TV(DX)))
    return DX


def build_block_grad_program(prog: Program, blk, sl: Tuple[int, ...], sg: Tuple[int, ...]):
    """Forward of FFCResnetBlock WITHOUT the identity add (all activations kept) | SplitOp | input-gradient program.
    inputs  x0, x1 (forward), g0, g1 (gradient w.r.t. the block outputs);
    outputs y0, y1 = conv2(conv1(x)) halves, dx0, dx1 = gradients w.r.t. x_l, x_g (identity path included)."""
    b, cl, h, w = sl
    cg = sg[1]
    prog.inputs.update(x0=tuple(sl), x1=tuple(sg), g0=tuple(sl), g1=tuple(sg))
    X = prog.buf("in", b, h, w, cl + cg, gemm=True, halo=True)
    prog.ops.append(ToNHWC("x0", TV(X, 0, cl)))
    prog.ops.append(ToNHWC("x1", TV(X, cl, cg)))
    Y1, _, _ = emit_ffc_bn_act(prog, blk.conv1, X, cl, cg)
    Y2, _, _ = emit_ffc_bn_act(prog, blk.conv2, Y1, cl, cg)
    prog.ops.append(ToNCHW(TV(Y2, 0, cl), "y0")); prog.outputs["y0"] = tuple(sl)
    prog.ops.append(ToNCHW(TV(Y2, cl, cg), "y1")); prog.outputs["y1"] = tuple(sg)
    prog.ops.append(SplitOp())
    DO = prog.buf("grad.dout", b, h, w, cl + cg)
    prog.ops.append(ToNHWC("g0", TV(DO, 0, cl)))
    prog.ops.append(ToNHWC("g1", TV(DO, cl, cg)))
    D1 = emit_ffc_bn_act_backward(prog, blk.conv2, Y2, TV(DO), cl, cg)
    D0 = emit_ffc_bn_act_backward(prog, blk.conv1, Y1, TV(D1), cl, cg, extra=TV(DO))
    prog.ops.append(ToNCHW(TV(D0, 0, cl), "dx0")); prog.outputs["dx0"] = tuple(sl)
    prog.ops.append(ToNCHW(TV(D0, cl, cg), "dx1")); prog.outputs["dx1"] = tuple(sg)


def build_module_program(module, kind: str, shapes: Sequence[Optional[Tuple[int, ...]]], math: int) -> Program:
    """Programs for stand-alone module calls: NCHW float in -> channels-last inside -> NCHW float out."""
    prog = Program(kind=kind, math=math)
    if kind == "fourier_unit":
        b, c, h, w = shapes[0]
        prog.inputs["x0"] = shapes[0]
        X = prog.buf("in", b, h, w, c)
        prog.ops.append(ToNHWC("x0", TV(X)))
        co = module.conv_layer.out_channels // 2
        O = prog.buf("out", b, h, w, co)
        emit_fourier_unit(prog, module, TV(X), TV(O), residual=None)
        prog.ops.append(ToNCHW(TV(O), "y0")); prog.outputs["y0"] = (b, co, h, w)
    elif kind == "spectral_transform":
        b, c, h, w = shapes[0]
        prog.inputs["x0"] = shapes[0]
        X = prog.buf("in", b, h, w, c, gemm=True, halo=module.stride == 2)
        prog.ops.append(ToNHWC("x0", TV(X)))
        U = emit_spectral_transform(prog, module, TV(X))
        co = module.conv2.out_channels
        h, w = st_out_hw(module, h, w)
        O = prog.buf("out", b, h, w, co)
        pk = P.pack_conv([(module.conv2.weight, 0, 0, 0)], None, None, device=module.conv2.weight.device)
        prog.ops.append(ConvOp(pk, [U, None], TV(O), tag="st.conv2"))
        prog.ops.append(ToNCHW(TV(O), "y0")); prog.outputs["y0"] = (b, co, h, w)
    elif kind in ("ffc_bn_act", "resnet_block"):
        sl, sg = shapes
        b, cl, h, w = sl
        cg = sg[1] if sg is not None else 0
        prog.inputs["x0"] = sl
        X = prog.buf("in", b, h, w, cl + cg, gemm=True, halo=True)
        prog.ops.append(ToNHWC("x0", TV(X, 0, cl)))
        if cg:
            prog.inputs["x1"] = sg
            prog.ops.append(ToNHWC("x1", TV(X, cl, cg)))
        if kind == "ffc_bn_act":
            Y, ocl, ocg = emit_ffc_bn_act(prog, module, X, cl, cg)
        else:
            Y = emit_resnet_block(prog, module, X, cl, cg, in_place=False)
            ocl, ocg = cl, cg
        if ocl:
            prog.ops.append(ToNCHW(TV(Y, 0, ocl), "y0")); prog.outputs["y0"] = (b, ocl, Y.H, Y.W)
        if ocg:
            prog.ops.append(ToNCHW(TV(Y, ocl, ocg), "y1")); prog.outputs["y1"] = (b, ocg, Y.H, Y.W)
    elif kind == "resnet_block_grad":
        build_block_grad_program(prog, module, shapes[0], shapes[1])
    elif kind == "generator":
        build_generator_program(prog, module, shapes[0])
    elif kind == "generator_rear_grad":
        build_rear_grad_program(prog, module, shapes[0], shapes[1])
    elif kind == "generator_rear":                       # the rear's forward alone (lowest refinement scale)
        emit_rear_forward(prog, module, shapes[0], shapes[1])
    elif kind.startswith("generator_refine:"):          # "generator_refine:<H0>x<W0>" (crop of the prediction)
        h0, w0 = (int(v) for v in kind.split(":")[1].split("x"))
        build_refine_program(prog, module, shapes[0], shapes[1], (h0, w0))
    elif kind.startswith("generator_refine_bits:"):     # the same step, ReLU masks kept as bits (relu_masks="bits")
        h0, w0 = (int(v) for v in kind.split(":")[1].split("x"))
        build_refine_program(prog, module, shapes[0], shapes[1], (h0, w0), relu_masks="bits")
    elif kind.startswith("generator_u8"):            # "generator_u8:<pad modulo>", shapes = (img, mask)
        mod = int(kind.split(":")[1]) if ":" in kind else 8
        b, h0, w0, _ = shapes[0]
        h, w = -(-h0 // mod) * mod, -(-w0 // mod) * mod
        build_generator_program(prog, module, (b, 4, h, w), u8_size=(h0, w0))
    else:
        raise ValueError(kind)
    if math == L.MATH_BF16X3 and not tc_compatible(prog):
        if kind.startswith("generator_u8"):
            raise ValueError("the uint8 predict path needs channel counts in multiples of 8 (tensor-core arm)")
        return build_module_program(module, kind, shapes, L.MATH_FP32)
    insert_border_ops(prog)
    return prog


def build_generator_program(prog: Program, gen, shape, u8_size: Optional[Tuple[int, int]] = None):
    """FFCResNetGenerator (ffc.py:306-367) as one program: stem -> stride-2 convs -> residual blocks
    (in place on one 512-channel buffer) -> sub-pixel transposed convs -> head.

    ``u8_size=(H0, W0)``: the predict-path variant (SURVEY.md row f1).  Inputs are the decoded bytes "img"
    (B,H0,W0,3) and "mask" (B,H0,W0); ``shape`` is the modulo-padded generator input (B,4,H,W); the output "y0" is
    the inpainted RGB bytes (B,H0,W0,3).  Pre/post-processing lives in the pack and gather kernels."""
    glob = _global_layout(gen)
    if glob is not None:
        return build_global_program(prog, glob, shape, u8_size)
    stem, downs, blocks, ups, out_blk, head, out_act = _generator_layout(gen)
    b, cin, h, w = shape
    s0, b0 = P.bn_scale_shift(stem.bn_l)
    X = emit_stem(prog, stem.ffc.convl2l.weight, s0, b0, shape, u8_size)
    cl, cg = X.C, 0
    for d in downs:
        X, cl, cg = emit_ffc_bn_act(prog, d, X, cl, cg)
    for blk in blocks:
        X = emit_resnet_block(prog, blk, X, cl, cg, in_place=True)
    # ConcatTupleLayer (ffc.py:295-302) is free: x_l | x_g already share X.
    tc_head = _tc_head(prog, head, h, w)
    ups_out = emit_up_tail(prog, ups, X, tc_head)
    X = ups_out[-1] if ups_out else X
    if out_blk is not None:
        # out_ffc: FFCResnetBlock(inline=True) splits its input as x[:, :-g] | x[:, -g:] (ffc.py:278-280) — exactly the
        # [local | global] channel order of the buffer, so it runs in place like the bottleneck blocks
        ocg = out_blk.conv1.ffc.global_in_num
        X = emit_resnet_block(prog, out_blk, X, X.C - ocg, ocg, in_place=True)
    emit_generator_head(prog, head, out_act, X, tc_head, bool(ups), shape, u8_size)


def emit_stem(prog: Program, weight: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, shape,
              u8_size: Optional[Tuple[int, int]]) -> Buf:
    """The generator's inputs and its ReflectionPad2d(3) + 7x7 conv + BN + ReLU stem (ffc.py:314-317,
    pix2pixhd.py:365-368; a conv bias is folded into ``shift``); returns the stem's output buffer."""
    b, cin, h, w = shape
    dev = weight.device
    if u8_size is None:
        prog.inputs["x0"] = tuple(shape)
    else:
        h0, w0 = u8_size
        prog.inputs["img"], prog.inputs["mask"] = (b, h0, w0, 3), (b, h0, w0)
        prog.dtypes.update(img=torch.uint8, mask=torch.uint8, y0=torch.uint8)
    n0 = weight.shape[0]
    wst, shst = P.pack_stem(weight, scale, shift, device=dev)
    X = prog.buf("stem", b, h, w, n0, gemm=True, halo=True)
    tc_stem = (prog.math == L.MATH_BF16X3 and cin <= 8 and n0 % 8 == 0
               and os.environ.get("LAMA_B200_STEM", "tc") == "tc")
    if u8_size is not None and not (tc_stem and cin == 4):
        raise ValueError("the uint8 predict path needs the tensor-core stem (bf16x3 arithmetic, 4 input channels)")
    if tc_stem:
        # tensor-core stem: the 7x7 window of the packed image is 7 contiguous 128-byte K blocks per pixel
        Pk = prog.buf("stem.packed", b, h + 6, w + 8, 8, gemm=True)
        if u8_size is None:
            prog.ops.append(StemPackOp("x0", cin, TV(Pk)))
        else:
            prog.ops.append(StemPackU8Op("img", "mask", h0, w0, TV(Pk)))
        pk = P.pack_stem_windowed(weight, scale, shift, device=dev)
        prog.ops.append(ConvOp(pk, [TV(Pk, window=8), None], TV(X), tag="stem 7x7 (windowed)+bn+relu"))
    else:
        prog.ops.append(StemOp("x0", cin, wst, shst, TV(X)))
    return X


def emit_generator_head(prog: Program, head, out_act: int, X: Buf, tc_head: bool, has_ups: bool, shape,
                        u8_size: Optional[Tuple[int, int]]):
    """The head (``emit_head``) and the program output "y0" of a generator program."""
    b, _cin, h, w = shape
    if u8_size is not None and not (tc_head and has_ups and head.out_channels == 3):
        raise ValueError("the uint8 predict path needs the tensor-core head with 3 output channels")
    emit_head(prog, head, out_act, X, tc_head and has_ups, u8_size)
    prog.outputs["y0"] = (b, head.out_channels, h, w) if u8_size is None else (b, u8_size[0], u8_size[1], 3)


def build_global_program(prog: Program, lay, shape, u8_size: Optional[Tuple[int, int]] = None):
    """LaMa-Regular ``GlobalGenerator`` (pix2pixhd.py:341-436; layout from ``_global_layout``) as one program: the
    FFC generator's stem, up-sampling tail and head around
      * 3x3 stride-2 convs with ZERO padding + BN + ReLU (pix2pixhd.py:375-379), conv biases folded into the shifts;
      * ``ResnetBlock``s in place on one bottleneck buffer X (pix2pixhd.py:47-90):
            Y = relu(bn1(conv1(reflect_pad(X))))          epilogue writes Y's reflected ring
            X = X + bn2(conv2(reflect_pad(Y)))            no activation; the residual is the epilogue's addend, and
                                                          each output pixel reads only its own residual pixel
    ``u8_size``: the predict-path variant, as in ``build_generator_program``."""
    stem, stem_bn, downs, blocks, ups, head, out_act = lay
    b, cin, h, w = shape
    dev = head.weight.device
    X = emit_stem(prog, stem.weight, *P.bn_scale_shift(stem_bn, stem.bias), shape, u8_size)
    for conv, bn in downs:
        sc, sh = P.bn_scale_shift(bn, conv.bias)
        Y = prog.buf("down", b, X.H // 2, X.W // 2, conv.out_channels, gemm=True, halo=True)
        pk = P.pack_conv([(conv.weight, 0, 0, 1)], sc, sh, stride=2, border=L.BORDER_ZERO, act=L.ACT_RELU, device=dev)
        prog.ops.append(ConvOp(pk, [TV(X), None], TV(Y), tag="down 3x3 s2 (zero border)+bn+relu"))
        X = Y
    for c1, bn1, c2, bn2 in blocks:
        Y = prog.buf("block.y", b, X.H, X.W, X.C, gemm=True, halo=True)
        pk1 = P.pack_conv([(c1.weight, 0, 0, 1)], *P.bn_scale_shift(bn1, c1.bias), act=L.ACT_RELU, device=dev)
        prog.ops.append(ConvOp(pk1, [TV(X), None], TV(Y), tag="block conv1+bn1+relu"))
        pk2 = P.pack_conv([(c2.weight, 0, 0, 1)], *P.bn_scale_shift(bn2, c2.bias), device=dev)
        prog.ops.append(ConvOp(pk2, [TV(Y), None], TV(X), addend=TV(X), addend_post=True, tag="block conv2+bn2 + x"))
    tc_head = _tc_head(prog, head, h, w)
    ups_out = emit_up_tail(prog, ups, X, tc_head)
    emit_generator_head(prog, head, out_act, ups_out[-1] if ups_out else X, tc_head, bool(ups), shape, u8_size)


def _tc_head(prog: Program, head, h: int, w: int) -> bool:
    """The tensor-core head (row contraction + gather) applies: split-bf16 arithmetic, N <= 3, planes wider than 3."""
    return (prog.math == L.MATH_BF16X3 and head.in_channels % 8 == 0 and head.out_channels <= 3
            and min(h, w) > 3 and os.environ.get("LAMA_B200_HEAD", "tc") == "tc")


def emit_up_tail(prog: Program, ups, X: Buf, tc_head: bool) -> List[Buf]:
    """ConvTranspose2d(k3, s2, p1, op1) + BN + ReLU stages (ffc.py:350-354) as sub-pixel phases; returns the ReLU
    output of every stage.  The last one feeds the head: with the tensor-core head its row contraction reads 3 pixels
    up and down -> split bf16 with a ring of 3; with the CUDA-core head float32."""
    outs = []
    for iu, (ct, bn) in enumerate(ups):
        sc, sh = P.bn_scale_shift(bn)
        last = iu == len(ups) - 1
        Yb = prog.buf("up", X.B, X.H * 2, X.W * 2, ct.out_channels, gemm=(not last) or tc_head,
                      halo=(not last) or tc_head, halo_px=3 if last else 1)
        for a, bb, pk in P.pack_conv_transpose_phases(ct.weight, ct.bias, sc, sh, act=L.ACT_RELU,
                                                      device=ct.weight.device):
            prog.ops.append(ConvOp(pk, [TV(X), None], TV(Yb, phase=(a, bb)), tag=f"convT phase {a}{bb}+bn+relu"))
        X = Yb
        outs.append(Yb)
    return outs


def emit_head(prog: Program, head, out_act: int, X: Buf, tc_head: bool, u8_size: Optional[Tuple[int, int]] = None):
    """ReflectionPad2d(3) + Conv2d 7x7 + act (ffc.py:360-363) of ``X`` into the external output "y0"; ``u8_size``: the
    predict path's blend / crop / uint8 variant of the tensor-core head."""
    dev = head.weight.device
    if tc_head:
        pkh = P.pack_head_rows(head.weight, device=dev)
        Q = prog.buf("head.q", X.B, X.H, X.W, pkh.n_out)
        prog.ops.append(ConvOp(pkh, [TV(X), None], TV(Q), tag="head 7x7 rows"))
        bias = head.bias.detach().float().contiguous() if head.bias is not None else torch.zeros(head.out_channels)
        if u8_size is None:
            prog.ops.append(HeadGatherOp(TV(Q), bias.to(dev), head.out_channels, out_act, "y0"))
        else:
            h0, w0 = u8_size
            prog.ops.append(HeadGatherU8Op(TV(Q), bias.to(dev), out_act, "img", "mask", h0, w0, "y0"))
    else:
        wh, bh = P.pack_head(head.weight, head.bias, device=dev)
        prog.ops.append(HeadOp(TV(X), wh, bh, head.out_channels, out_act, "y0"))


def rear_grad_supported(gen, shape_l, shape_g) -> bool:
    """The generator's rear — residual blocks, up-sampling tail, head (``generator.model[first_block:]``) — has a
    native forward + input-gradient program for inputs (z1, z2) of these shapes: every block has block gradients
    (``block_grad_supported``), no out_ffc block, at least one up-sampling stage, a none / sigmoid / tanh head with
    N <= 4, bottleneck planes the native FFT takes (``plane_ok``, axes up to BLOCK_GRAD_MAX_PLANE = FFT_MAX_LEN)."""
    lay = _generator_layout(gen)
    if lay is None or shape_l is None or shape_g is None or len(shape_l) != 4 or len(shape_g) != 4:
        return False
    _stem, _downs, blocks, ups, out_blk, head, out_act = lay
    if out_blk is not None or not blocks or not ups or out_act not in (L.ACT_NONE, L.ACT_SIGMOID, L.ACT_TANH):
        return False
    if head.out_channels > 4 or not all(block_grad_supported(b) for b in blocks):
        return False
    b, cl, h, w = shape_l
    f = blocks[0].conv1.ffc
    if (b < 1 or shape_g[0] != b or tuple(shape_g[2:]) != (h, w) or cl != f.convl2l.in_channels
            or shape_g[1] != f.global_in_num or ups[0][0].in_channels != cl + shape_g[1]):
        return False
    if max(h, w) > BLOCK_GRAD_MAX_PLANE:
        return False
    return ffc_bn_act_shapes_ok(blocks[0].conv1, torch.empty(shape_l, device="meta"),
                                torch.empty(shape_g, device="meta"))


def build_rear_grad_program(prog: Program, gen, sl: Tuple[int, ...], sg: Tuple[int, ...]):
    """``generator.model[first_block:]`` (ffc.py:345-363) forward | SplitOp | input gradients, for refinement
    (evaluation/refinement.py:137-167 optimises z1, z2 through exactly this part).
    inputs  x0, x1 (z1, z2: local / global halves at the bottleneck), g0 (dL/dpred, backward part);
    outputs y0 (pred, as ``rear((z1, z2))``), dx0, dx1 (dL/dz1, dL/dz2).
    Forward: ``emit_rear_forward``; backward: ``emit_rear_backward``."""
    fwd = emit_rear_forward(prog, gen, sl, sg)
    prog.ops.append(SplitOp())
    prog.inputs["g0"] = prog.outputs["y0"]
    emit_rear_backward(prog, gen, fwd, "g0")


def emit_rear_forward(prog: Program, gen, sl: Tuple[int, ...], sg: Tuple[int, ...]) -> dict:
    """Forward part of the rear programs: inputs x0, x1 (z1, z2) -> output y0 (pred).  Per block conv1 -> Y1, conv2 ->
    its own Y2 (kept: its ReLU mask is read by the backward, which the fused residual epilogue's X + Y2 would not give
    back), X <- X + Y2 (ffcb_add); then the generator program's tail.  Returns what the backward reads."""
    _stem, _downs, blocks, ups, _out_blk, head, out_act = _generator_layout(gen)
    b, cl, h, w = sl
    cg = sg[1]
    prog.inputs.update(x0=tuple(sl), x1=tuple(sg))
    X = prog.buf("in", b, h, w, cl + cg, gemm=True, halo=True)
    prog.ops.append(ToNHWC("x0", TV(X, 0, cl)))
    prog.ops.append(ToNHWC("x1", TV(X, cl, cg)))
    saved = []
    for blk in blocks:
        Y1, _, _ = emit_ffc_bn_act(prog, blk.conv1, X, cl, cg)
        Y2, _, _ = emit_ffc_bn_act(prog, blk.conv2, Y1, cl, cg)
        prog.ops.append(AddOp(TV(X), TV(Y2), TV(X)))
        saved.append((blk, Y1, Y2))
    H, W = X.H * 2 ** len(ups), X.W * 2 ** len(ups)
    ups_out = emit_up_tail(prog, ups, X, _tc_head(prog, head, H, W))
    emit_head(prog, head, out_act, ups_out[-1], _tc_head(prog, head, H, W))
    prog.outputs["y0"] = (b, head.out_channels, H, W)
    return dict(sl=tuple(sl), sg=tuple(sg), saved=saved, ups_out=ups_out)


def emit_rear_backward(prog: Program, gen, fwd: dict, dy: str):
    """Input-gradient part of the rear programs, from ``dy`` (the NCHW gradient w.r.t. y0: an external input or an
    output another op of the program writes) to the outputs dx0, dx1: ffcb_head_bwd7 -> for every up stage in reverse
    the adjoint of ConvTranspose2d(k3, s2, p1, op1): a stride-2, zero-border 3x3 ffcb_conv with the transposed conv's
    own weight [Cin, Cout, 3, 3] (no flip) and the BN scale folded along its input axis, then the ReLU mask of the stage
    below -> the blocks in reverse, each as two FFC_BN_ACT backwards with the identity path added by the second."""
    _stem, _downs, _blocks, ups, _out_blk, head, out_act = _generator_layout(gen)
    sl, sg, saved, ups_out = fwd["sl"], fwd["sg"], fwd["saved"], fwd["ups_out"]
    b, cl, cg = sl[0], sl[1], sg[1]
    H, W = ups_out[-1].H, ups_out[-1].W
    dev = head.weight.device
    n = head.out_channels
    wh, _ = P.pack_head(head.weight, head.bias, device=dev)
    D = prog.buf("grad.dup", b, H, W, head.in_channels, gemm=True)
    prog.ops.append(HeadBwdOp("y0", dy, wh, n, out_act, TV(ups_out[-1]), TV(D)))
    for k in reversed(range(len(ups))):
        ct, bn = ups[k]
        sc, _ = P.bn_scale_shift(bn)
        wadj = ct.weight.detach().double() * sc.double()[None, :, None, None]       # [Cin_ct, Cout_ct, 3, 3]
        pk = P.pack_conv([(wadj, 0, 0, 1)], None, None, stride=2, border=L.BORDER_ZERO, device=dev)
        hi, wi = ups_out[k].H // 2, ups_out[k].W // 2
        if k > 0:
            E_ = prog.buf("grad.up_in", b, hi, wi, ct.in_channels)
            prog.ops.append(ConvOp(pk, [TV(D), None], TV(E_), tag=f"grad: convT{k}^T (stride 2)"))
            D = prog.buf("grad.dup", b, hi, wi, ct.in_channels, gemm=True)
            prog.ops.append(ReluBwdOp(TV(E_), TV(ups_out[k - 1]), TV(D)))
        else:
            DX = prog.buf("grad.dx", b, hi, wi, ct.in_channels)
            prog.ops.append(ConvOp(pk, [TV(D), None], TV(DX), tag=f"grad: convT{k}^T (stride 2)"))
    for blk, Y1, Y2 in reversed(saved):
        D1 = emit_ffc_bn_act_backward(prog, blk.conv2, Y2, TV(DX), cl, cg)
        DX = emit_ffc_bn_act_backward(prog, blk.conv1, Y1, TV(D1), cl, cg, extra=TV(DX))
    prog.ops.append(ToNCHW(TV(DX, 0, cl), "dx0")); prog.outputs["dx0"] = tuple(sl)
    prog.ops.append(ToNCHW(TV(DX, cl, cg), "dx1")); prog.outputs["dx1"] = tuple(sg)


def refine_supported(gen, shape_l, shape_g, crop: Tuple[int, int]) -> bool:
    """The refinement step program (``build_refine_program``) exists: the rear program does
    (``rear_grad_supported``), the head writes 3 channels (the image's), and the crop (H0, W0) lies inside the
    prediction and is at least 3x3 (the Gaussian's reflect padding of 2)."""
    if not rear_grad_supported(gen, shape_l, shape_g):
        return False
    lay = _generator_layout(gen)
    H, W = shape_l[2] * 2 ** len(lay[3]), shape_l[3] * 2 ** len(lay[3])
    return lay[5].out_channels == 3 and 3 <= crop[0] <= H and 3 <= crop[1] <= W


def build_refine_program(prog: Program, gen, sl: Tuple[int, ...], sg: Tuple[int, ...], crop: Tuple[int, int],
                         relu_masks: str = "values"):
    """One Adam step of the refinement loop (evaluation/refinement.py:137-167) without the optimiser:
    rear forward | SplitOp | RefineLossOp | rear backward.
    inputs  x0, x1 (z1, z2), and the per-scale constants image (B,3,H,W), mask (B,1,H,W) in {0,1}, ref (B,3,H0/2,W0/2),
            md (B,1,H0/2,W0/2) (the eroded down-scaled mask), inv (B,2) (1 / n_out, 1 / n_down, 0 for an empty term);
    outputs y0 (pred), dy0 (dL/dpred, written by RefineLossOp and read by the head adjoint), loss (B,2), dx0, dx1.
    ``run(part=0)`` alone is the forward-only rear (the last forward of a scale, and the lowest scale).
    ``relu_masks="bits"``: the backward's ReLU masks of forward activations are kept as bits
    (``relu_bits.pack_relu_masks``): the same results in less than half the storage at large planes."""
    from .refine import gaussian_kernel1d
    if relu_masks not in ("values", "bits"):
        raise ValueError(f"relu_masks must be 'values' or 'bits', not {relu_masks!r}")
    h0, w0 = crop
    fwd = emit_rear_forward(prog, gen, sl, sg)
    b, n, H, W = prog.outputs["y0"]
    prog.ops.append(SplitOp())
    prog.inputs.update(image=(b, n, H, W), mask=(b, 1, H, W), ref=(b, n, h0 // 2, w0 // 2),
                       md=(b, 1, h0 // 2, w0 // 2), inv=(b, 2))
    prog.outputs.update(dy0=(b, n, H, W), loss=(b, 2))
    prog.ops.append(RefineLossOp("y0", "image", "mask", "ref", "md", "inv", h0, w0, gaussian_kernel1d(5, 1.0),
                                 "dy0", "loss", b * n * (h0 // 2) * (w0 // 2)))
    emit_rear_backward(prog, gen, fwd, "dy0")
    if relu_masks == "bits":
        from .relu_bits import pack_relu_masks
        pack_relu_masks(prog)


def tc_compatible(prog: Program) -> bool:
    """The tensor-core arm needs 16-byte aligned bf16 pixels/slices: channel counts and slice starts in
    multiples of 8.  Programs that do not qualify run the fp32 CUDA-core arm (still native)."""
    for op in prog.ops:
        if isinstance(op, ConvOp):
            for tv in op.ins:
                if tv is not None and (tv.buf.C % 8 or tv.c0 % 8):
                    return False
            if any(sg.c0 % 8 for sg in op.packed.segs):
                return False
            if op.out.buf.fmt == L.BF16X2 and (op.out.buf.C % 8 or op.out.c0 % 8):
                return False
    return True


def insert_border_ops(prog: Program):
    """Producers never write the reflected ring of a padded buffer (the tensor-core epilogue stores through a
    tensor map of the interior; layout conversions, the stem and the FFT kernels write pixels only).  Insert
    a BorderOp lazily: right before the first contraction that reads a buffer whose interior changed since
    its ring was last rebuilt.  For the in-place residual blocks that is one ring refresh per FFC_BN_ACT."""
    out, dirty = [], set()
    for op in prog.ops:
        for tv in op.ring_reads():
            if tv.buf.reflect_border and id(tv.buf) in dirty:
                out.append(BorderOp(TV(tv.buf)))
                dirty.discard(id(tv.buf))
        out.append(op)
        if op.ring_effect(prog) == STALE:
            dirty.update(id(tv.buf) for tv in op.views()[1] if tv.buf.reflect_border)
    prog.ops = out


def conv_writes_ring(prog: Program, op) -> bool:
    """The tensor-core contraction writes the mirrored copies of rows 1 / H-2 and columns 1 / W-2 into a 1-pixel reflected
    ring of its output itself (conv_tc.cu, TcParams::ring) — whole-plane outputs only (a sub-pixel phase or a window
    does not own the ring)."""
    if os.environ.get("LAMA_B200_RING_KERNEL", "0") == "1":        # A/B: always refresh rings with the ring kernel
        return False
    return (prog.math == L.MATH_BF16X3 and isinstance(op, ConvOp) and op.out.phase is None and op.out.win is None
            and not op.out.window and op.out.buf.pad == 1 and op.out.buf.fmt == L.BF16X2 and op.out.buf.H >= 4
            and op.out.buf.W >= 4)


# ------------------------------------------------------------------------------------- executor
def op_views(op) -> Tuple[List[TV], List[TV]]:
    """(views read, views written) by one op of a program: ``op.views()``."""
    return op.views()


def op_scratch_bytes(op) -> int:
    return op.scratch_bytes()


def storage_key(b: Buf) -> tuple:
    """Buffers with equal keys have byte-identical storage (dtype, shape, ring, layout)."""
    return (b.fmt, b.B, b.H, b.W, b.C, b.pad, b.reflect_border, b.cg, b.tile, b.bits)


def storage_shape(b: Buf) -> Tuple[int, ...]:
    """Shape of a buffer's storage tensor: float32, or bfloat16 with a leading 2 (hi / lo halves) for split bf16, or
    int32 words of 32 mask bits for a bit mask."""
    if b.bits:
        return (b.B, b.H, b.W, -(-b.C // 32))
    if b.tile:
        return (-(-(b.B * b.H * b.W) // 128), b.C // 8, 128, 8)      # zero-initialised: the tail block stays finite
    if b.cg:
        return (b.C // b.cg, b.B, b.H, b.W, b.cg)
    return (b.B, b.H + 2 * b.pad, b.W + 2 * b.pad, b.C)


def program_storage_bytes(prog: Program) -> int:
    """Device bytes a ``CudaExecutor`` of ``prog`` allocates for activations, computed from the buffer shapes and
    storage slots before anything is allocated: the pooled buffers, the FFT workspace, the program's outputs and op
    scratch (packed weights, a few MB, are not counted).  Used to size refinement batches."""
    slots = assign_storage_slots(prog)
    seen, total = set(), 0
    for b in prog.bufs:
        if slots[b.name] not in seen:
            seen.add(slots[b.name])
            total += 4 * math.prod(storage_shape(b))           # float32, two bfloat16 halves, or int32 mask words
    for name, shape in prog.outputs.items():
        total += math.prod(shape) * (1 if prog.dtypes.get(name, torch.float32) == torch.uint8 else 4)
    return total + max(prog.fft_workspace_bytes(), 16) + sum(op.scratch_bytes() for op in prog.ops)


def assign_storage_slots(prog: Program) -> Dict[str, int]:
    """Buffer name -> storage slot.  A program is a straight-line op list on one stream, so a buffer is dead after
    the last op that touches it and its storage can back a later buffer.  Only buffers with IDENTICAL storage
    (``storage_key``) share a slot: whatever a kernel leaves unwritten (zero-initialised pixel / channel padding, the
    reflected ring before its producer ran) then holds what the same kind of buffer held there before, never foreign
    bits.  For big-lama this folds the 18 residual blocks' ~150 buffers onto two blocks' worth: 28 GB -> 10 GB at bs32
    512x512, and bs64 1024x1024 (BASELINE config 4's global batch) pools to about 64 GB.  Constant buffers
    (``prog.consts``) keep their own storage; ``LAMA_B200_POOL=0`` gives every buffer its own."""
    first: Dict[str, int] = {}
    last: Dict[str, int] = {}
    for i, op in enumerate(prog.ops):
        reads, writes = op.views()
        for tv in reads + writes:
            first.setdefault(tv.buf.name, i)
            last[tv.buf.name] = i
    pooling = os.environ.get("LAMA_B200_POOL", "1") != "0"
    slots: Dict[str, int] = {}
    free_at: List[Tuple[tuple, int]] = []          # per slot: (storage key, index of the last op that touches it)
    for b in sorted(prog.bufs, key=lambda bb: first.get(bb.name, -1)):
        key = storage_key(b)
        reuse = None
        if pooling and b.name in first and b.name not in prog.consts:
            for si, (k, until) in enumerate(free_at):
                if k == key and until is not None and until < first[b.name]:
                    reuse = si
                    break
        if reuse is None:
            reuse = len(free_at)
            free_at.append((key, None))
        # constants and never-touched buffers hold their slot for good
        free_at[reuse] = (key, last[b.name] if (b.name in last and b.name not in prog.consts) else None)
        slots[b.name] = reuse
    return slots


class CudaExecutor:
    """Binds a Program to device buffers and pre-built C-ABI calls."""

    def __init__(self, prog: Program, device: torch.device):
        self.prog = prog
        self.device = device
        self.lib = L.get_lib()
        self.dev_index = device.index if device.index is not None else torch.cuda.current_device()
        L.check(self.lib.ffcb_check_device(self.dev_index), "ffcb_check_device")
        self.storage: Dict[str, torch.Tensor] = {}
        self.slots = assign_storage_slots(prog)          # buffers whose lifetimes do not overlap share storage
        slot_tensor: Dict[int, torch.Tensor] = {}
        for b in prog.bufs:
            si = self.slots[b.name]
            if si in slot_tensor:
                self.storage[b.name] = slot_tensor[si]
                continue
            shape = storage_shape(b)
            if b.bits:
                slot_tensor[si] = torch.zeros(shape, dtype=torch.int32, device=device)
            elif b.fmt == L.F32:
                slot_tensor[si] = torch.empty(shape, dtype=torch.float32, device=device)
            else:
                slot_tensor[si] = torch.zeros((2,) + shape, dtype=torch.bfloat16, device=device)
            self.storage[b.name] = slot_tensor[si]
        self.storage_bytes = sum(t.numel() * t.element_size() for t in slot_tensor.values())
        for name, val in prog.consts.items():
            assert self.storage[name].dtype == torch.float32 and tuple(self.storage[name].shape) == tuple(val.shape)
            self.storage[name].copy_(val.to(device=device, dtype=torch.float32))
        ws_bytes = prog.fft_workspace_bytes()
        self.ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=device)
        self.ws_bytes = ws_bytes
        self.outputs = {k: torch.empty(v, dtype=prog.dtypes.get(k, torch.float32), device=device)
                        for k, v in prog.outputs.items()}
        self._launches = None
        self._keep = []          # ctypes objects / tensors that must outlive the calls
        self.calls = []          # (name, fn, args) with a trailing stream argument appended at run time
        self.input_slots: Dict[str, List[Tuple[int, int]]] = {}   # input name -> [(call idx, arg idx)]
        self.split = None        # forward+backward programs: index of the first backward call (SplitOp)
        self.generation = 0      # bumped by every forward part: a stale backward must not read newer activations
        assert not prog.inputs.keys() & prog.outputs.keys(), "a name is both a program input and a program output"
        for op in prog.ops:
            call = op.bind(self)
            if call is None:
                continue
            name, fn, args = call
            for ai, a in enumerate(args):
                if isinstance(a, Ext):
                    if a.name in self.outputs:
                        args[ai] = self.outputs[a.name].data_ptr()
                    else:
                        assert a.name in prog.inputs, f"{name} reads {a.name!r}, neither an input nor an output"
                        self.input_slots.setdefault(a.name, []).append((len(self.calls), ai))
                        args[ai] = None
            self.calls.append((name, fn, args))
        # part -> (first call, end, inputs its calls read); parts 0 / 1 exist for forward+backward programs
        n = len(self.calls)
        spans = {None: (0, n)} if self.split is None else {None: (0, n), 0: (0, self.split), 1: (self.split, n)}
        self._parts = {p: (lo, hi, {n for n, sl in self.input_slots.items() if any(lo <= ci < hi for ci, _ in sl)})
                       for p, (lo, hi) in spans.items()}
        self._bound = set()      # inputs bound at least once

    # -- view construction
    def tensor(self, tv: TV) -> L.Tensor:
        b = tv.buf
        st = self.storage[b.name]
        es = 4 if b.fmt == L.F32 else 2
        if b.tile:
            assert (tv.phase is None and not tv.window and tv.win is None and b.pad == 0 and tv.c0 % 8 == 0
                    and tv.channels % 8 == 0)
            m0 = tv.b0 * b.H * b.W
            if m0 % 128:
                raise ValueError("a batch slice of a tile-blocked buffer must start on a 128-pixel block")
            t = L.Tensor()
            nblk, groups = -(-(b.B * b.H * b.W) // 128), b.C // 8
            t.cg, t.tile, t.sg = 8, 128, groups * 1024
            t.sx, t.sy, t.sb = 8, b.W * 8, b.H * b.W * 8
            t.lo_off = nblk * groups * 1024
            t.ptr = st.data_ptr() + ((tv.c0 // 8) * 1024 + (m0 // 128) * t.sg) * es
            t.B, t.H, t.W, t.C = tv.batch, b.H, b.W, tv.channels
            t.fmt, t.pad, t.reflect_border = b.fmt, 0, 0
            return t
        if b.cg:
            assert tv.phase is None and not tv.window and b.pad == 0 and tv.c0 % b.cg == 0 and tv.channels % b.cg == 0
            t = L.Tensor()
            t.sx, t.sy, t.sb = b.cg, b.W * b.cg, b.H * b.W * b.cg
            t.sg, t.cg = b.B * b.H * b.W * b.cg, b.cg
            t.lo_off = b.C * b.B * b.H * b.W if b.fmt == L.BF16X2 else 0
            off = (tv.c0 // b.cg) * t.sg + tv.b0 * t.sb
            h, w = b.H, b.W
            if tv.win is not None:
                y0, x0, h, w = tv.win
                off += y0 * t.sy + x0 * t.sx
            t.ptr = st.data_ptr() + off * es
            t.B, t.H, t.W, t.C = tv.batch, h, w, tv.channels
            t.fmt, t.pad, t.reflect_border = b.fmt, 0, 0
            return t
        wp, hp = b.W + 2 * b.pad, b.H + 2 * b.pad
        sx, sy, sb = b.C, wp * b.C, hp * wp * b.C
        off = (b.pad * wp + b.pad) * b.C + tv.c0
        h, w = b.H, b.W
        if tv.phase is not None:
            a, bb = tv.phase
            off += a * sy + bb * sx
            sy, sx, h, w = 2 * sy, 2 * sx, b.H // 2, b.W // 2
        if tv.win is not None:
            assert tv.phase is None and not tv.window
            y0, x0, h, w = tv.win
            off += y0 * sy + x0 * sx
        t = L.Tensor()
        t.ptr = 0  # set below (after the batch-slice offset)
        t.sb, t.sy, t.sx = sb, sy, sx
        t.lo_off = b.B * hp * wp * b.C if b.fmt == L.BF16X2 else 0
        off += tv.b0 * sb
        t.ptr = st.data_ptr() + off * es
        t.B, t.H, t.W, t.C = tv.batch, h, w, tv.channels
        if tv.bcast:
            t.sb = 0                 # every image of the batch reads the same plane (position-dependent addends)
        t.fmt, t.pad, t.reflect_border = b.fmt, b.pad, b.reflect_border
        if tv.phase is not None or tv.win is not None:     # not a whole image: no ring semantics
            t.pad, t.reflect_border = 0, 0
        if tv.window:                # pixel x exposes the buf.C * window contiguous elements starting at x * sx
            t.W, t.C, t.window = b.W - tv.window, b.C * tv.window, 1
        return t

    def ref(self, x):
        """``byref`` of a ctypes structure, or of the descriptor of a view, kept alive with the executor (None: None)."""
        if x is None:
            return None
        self._keep.append(self.tensor(x) if isinstance(x, TV) else x)
        return C.byref(self._keep[-1])

    def keep(self, t: torch.Tensor) -> int:
        """Pointer of a packed parameter (or scratch) copied to the executor's device, kept alive with the executor."""
        self._keep.append(t.to(self.device).contiguous())
        return self._keep[-1].data_ptr()

    def bind_inputs(self, inputs: Dict[str, torch.Tensor]) -> None:
        """Check each given input (on the executor's device type, declared dtype and shape, contiguous) and patch its
        pointer into the calls that read it.  Inputs stay bound until rebound; the caller keeps them alive."""
        for name, t in inputs.items():
            shape, dt = tuple(self.prog.inputs[name]), self.prog.dtypes.get(name, torch.float32)
            if not (t.device.type == self.device.type and t.dtype == dt and t.is_contiguous() and tuple(t.shape) == shape):
                raise ValueError(f"input {name}: expected a contiguous {dt} {shape} on {self.device.type}, got "
                                 f"{t.dtype} {tuple(t.shape)} on {t.device}")
            for ci, ai in self.input_slots.get(name, ()):
                self.calls[ci][2][ai] = t.data_ptr()
            self._bound.add(name)

    def run(self, inputs: Dict[str, torch.Tensor], stream: Optional[int] = None,
            part: Optional[int] = None) -> Dict[str, torch.Tensor]:
        """Bind ``inputs`` and issue every call on ``stream`` (default: torch's current stream).  Outputs are the
        executor's own tensors (overwritten by the next run).  ``part``: 0 / 1 run only the forward / backward half
        of a forward+backward program; inputs bound by an earlier run may be left out."""
        if torch.cuda.current_device() != self.dev_index:
            # the module lives on another GPU than the caller's current device (one process driving several GPUs):
            # kernels must be launched with that device current, as torch's own ops do through their device guards
            with torch.cuda.device(self.dev_index):
                return self.run(inputs, stream, part)
        if part not in self._parts:
            raise ValueError(f"part={part}: not a forward+backward program")
        lo, hi, needs = self._parts[part]
        self.bind_inputs(inputs)
        if not needs <= self._bound:
            raise ValueError(f"inputs never bound: {sorted(needs - self._bound)}")
        if stream is None:
            stream = torch.cuda.current_stream(self.device).cuda_stream
        first = part is None and self._launches is None
        if first:
            self.lib.ffcb_reset_launch_count()
        for name, fn, args in self.calls[lo:hi]:
            rc = fn(*args, stream)
            if rc != 0:
                L.check(rc, name)
        if first:
            self._launches = int(self.lib.ffcb_launch_count())
        if part == 0:
            self.generation += 1
        return self.outputs

    @property
    def launches_per_run(self) -> int:
        """Kernel launches of one replay, counted by the library itself during the first run."""
        assert self._launches is not None, "run the executor once first"
        return self._launches


class GraphedProgram:
    """CUDA-graph replay of an executor with static input tensors (bench / serving path)."""

    def __init__(self, ex: CudaExecutor, warmup: int = 2):
        self.ex = ex
        self.static_in = {k: torch.empty(v, dtype=ex.prog.dtypes.get(k, torch.float32), device=ex.device)
                          for k, v in ex.prog.inputs.items()}
        side = torch.cuda.Stream(device=ex.device)
        side.wait_stream(torch.cuda.current_stream(ex.device))
        with torch.cuda.stream(side):
            for _ in range(warmup):
                ex.run(self.static_in)
        torch.cuda.current_stream(ex.device).wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            ex.run(self.static_in)

    def __call__(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        for k, t in inputs.items():
            self.static_in[k].copy_(t, non_blocking=True)
        self.graph.replay()
        return self.ex.outputs


# ---------------------------------------------------------------------------- module entry point
# Executor caches live OUTSIDE the module (weak keys): they hold ctypes pointers / byref objects, which must never
# end up in `module.__dict__` — the reference deep-copies the generator for its EMA copy (trainers/base.py:168) and
# `torch.save(module)` / pickling / DataParallel replication walk `__dict__`.
import weakref

_PROGRAMS: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()      # module -> {key: (signature, executor)}
_TENSORS: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()       # module -> [flat tensor list, calls since walk]
_REWALK_EVERY = 8
_SMALL_MODULE = 64       # modules with fewer tensors are re-walked on every call (the walk is cheap there)


def invalidate(module) -> None:
    """Drop every cached program / packed weight of ``module`` (call after editing weights in a way the automatic
    checks cannot see; load_state_dict, .to(), in-place ops and ``.data`` edits ARE seen)."""
    _PROGRAMS.pop(module, None)
    _TENSORS.pop(module, None)


def drop_executor(ex: "CudaExecutor") -> None:
    """Remove ``ex`` from every module's executor cache, so that its buffers are freed once the caller lets go of it
    (a pipeline that releases its program to make room for another)."""
    for cache in list(_PROGRAMS.values()):
        for k in [k for k, v in cache.items() if v[1] is ex]:
            del cache[k]


def _content_checksum(tensors) -> float:
    """One number per weight version: the sum of all tensors' L2 norms (a handful of fused multi-tensor kernels and
    one scalar read).  Catches what (data_ptr, _version) cannot: edits through ``.data`` — the reference's EMA update
    (trainers/base.py:40) and the common ``weight.data.copy_()`` loading idiom leave ``_version`` unchanged."""
    fl = [t for t in tensors if t.is_floating_point() and t.numel()]
    if not fl:
        return 0.0
    groups = {}
    for t in fl:
        groups.setdefault((t.device, t.dtype), []).append(t.detach())
    total = 0.0
    for ts in groups.values():
        total += float(torch.stack(torch._foreach_norm(ts)).double().sum())
    return total


def _weights_signature(module, content: bool = True) -> Tuple:
    """(data_ptr, version) of every parameter / buffer — changes on load_state_dict, .to(), in-place edits — plus,
    with ``content``, a checksum of the values (``.data`` edits).  Walking the module tree costs ~1.5 ms for big-lama
    (989 tensors), so the flat tensor list is cached and re-walked every few calls (every call for small modules);
    a replaced Parameter object whose storage was freed changes data_ptr and is seen at once in practice.
    LAMA_B200_TRUST_WEIGHTS=1 skips the checksum (serving loops that never touch the weights)."""
    st = _TENSORS.get(module)
    if st is None or st[1] >= _REWALK_EVERY or len(st[0]) <= _SMALL_MODULE:
        st = [list(module.parameters()) + list(module.buffers()), 0]
        _TENSORS[module] = st
    st[1] += 1
    sig = tuple((t.data_ptr(), t._version) for t in st[0])
    if content and os.environ.get("LAMA_B200_TRUST_WEIGHTS", "0") != "1":
        sig = sig + (_content_checksum(st[0]),)
    return sig


def get_executor(module, kind: str, tensors, math: Optional[int] = None,
                 device: Optional[torch.device] = None) -> CudaExecutor:
    """``tensors`` only contribute their shapes (meta tensors are fine when ``device`` is given)."""
    math = default_math() if math is None else math
    shapes = tuple(tuple(t.shape) if torch.is_tensor(t) else None for t in tensors)
    dev = device if device is not None else next(t for t in tensors if torch.is_tensor(t)).device
    key = (kind, shapes, str(dev), math)
    cache = _PROGRAMS.setdefault(module, {})
    sig = _weights_signature(module)
    hit = cache.get(key)
    if hit is not None and hit[0] == sig:
        cache[key] = cache.pop(key)          # LRU: most recently used last
        return hit[1]
    with torch.no_grad():
        prog = build_module_program(module, kind, shapes, math)
    ex = CudaExecutor(prog, dev)
    cache.pop(key, None)                      # stale weights
    # every executor owns its activation buffers (~0.3 GB per 512x512 image for big-lama): keep only the few most
    # recently used shapes per module so that a stream of differently sized images cannot exhaust HBM
    while len(cache) >= PROGRAM_CACHE_SIZE:
        cache.pop(next(iter(cache)))
    cache[key] = (sig, ex)
    return ex


class _SplitProgramFn(torch.autograd.Function):
    """Native forward AND native input gradients through a forward+backward program, weights frozen — what the
    reference's refinement loop (evaluation/refinement.py:137-167) needs: ``resnet_block_grad`` for one FFCResnetBlock
    (SURVEY.md row f3), ``generator_rear_grad`` for the whole rear (residual blocks, up-sampling tail, head).
    Forward runs part 0 on inputs x0, x1 and returns the program outputs ``ys`` (plus x0 / x1 with ``residual``: the block
    program leaves the identity add to the caller); backward runs part 1 on one gradient g<i> per output.  The forward's
    activations stay in the executor's buffers, one executor per (module, shape): a second forward before the backward
    of the first would overwrite them, which raises instead of returning wrong gradients."""

    @staticmethod
    def forward(ctx, module, kind, ys, residual, what, x0, x1):
        ex = get_executor(module, kind, (x0, x1))
        xs = (x0.detach().contiguous(), x1.detach().contiguous())
        outs = ex.run({"x0": xs[0], "x1": xs[1]}, part=0)
        ctx.ex, ctx.generation, ctx.what = ex, ex.generation, what
        res = tuple(x + outs[y] if residual else outs[y].clone() for y, x in zip(ys, xs))
        return res if len(res) > 1 else res[0]

    @staticmethod
    def backward(ctx, *grads):
        ex = ctx.ex
        if ex.generation != ctx.generation:
            raise RuntimeError(f"lama_b200: {ctx.what} ran forward again (same shape) before this backward; "
                               "its saved activations were overwritten")
        outs = ex.run({f"g{i}": g.contiguous() for i, g in enumerate(grads)}, part=1)
        return None, None, None, None, None, outs["dx0"].clone(), outs["dx1"].clone()


def block_with_input_grad(module, x_l, x_g):
    """(out_l, out_g) of an FFCResnetBlock, differentiable w.r.t. x_l / x_g on the native path."""
    return _SplitProgramFn.apply(module, "resnet_block_grad", ("y0", "y1"), True, "the same FFCResnetBlock", x_l, x_g)


def generator_rear_with_input_grad(gen, z1, z2):
    """pred = ``gen.model[first_block:]((z1, z2))`` on the native path, differentiable w.r.t. z1 / z2 (the weights are
    frozen).  Callers check ``rear_grad_supported(gen, z1.shape, z2.shape)`` first."""
    return _SplitProgramFn.apply(gen, "generator_rear_grad", ("y0",), False, "the generator's rear", z1, z2)


def run_module(module, kind: str, tensors):
    """Execute ``module`` natively on NCHW float CUDA tensors; returns fresh tensors (or the int 0
    for an empty FFC side)."""
    first = next(t for t in tensors if torch.is_tensor(t))
    if first.shape[0] == 0:
        # empty batch (the reference returns empty tensors of the right shape): nothing to launch; the output
        # shapes come from the program of a one-image batch
        shapes = tuple((1,) + tuple(t.shape[1:]) if torch.is_tensor(t) else None for t in tensors)
        with torch.no_grad():
            prog = build_module_program(module, kind, shapes, L.MATH_FP32)
        outs = {k: torch.empty((0,) + tuple(v[1:]), dtype=prog.dtypes.get(k, torch.float32), device=first.device)
                for k, v in prog.outputs.items()}
        y0 = outs.get("y0", 0)
        if kind in ("ffc_bn_act", "resnet_block"):
            return y0, outs.get("y1", 0)
        return (y0,)
    ex = get_executor(module, kind, tensors)
    feed = {}
    i = 0
    for t in tensors:
        if torch.is_tensor(t):
            feed[f"x{i}"] = t.contiguous()
            i += 1
    outs = ex.run(feed)
    y0 = outs["y0"].clone() if "y0" in outs else 0
    if kind in ("ffc_bn_act", "resnet_block"):
        return y0, (outs["y1"].clone() if "y1" in outs else 0)
    return (y0,)
