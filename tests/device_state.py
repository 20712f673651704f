"""TEST INFRASTRUCTURE: issue an ``engine.Program`` on the GPU one C-ABI call at a time and read its device state back.

- ``Decoder``: the device storage of a ``Buf`` as float64, whatever its layout and format.
- ``DeviceRun``: a program bound to a ``CudaExecutor`` whose calls run one by one, with hooks before and after each.
- ``diff_program``: every op judged against ``tests/spec_interp.py`` on the device state it saw.
- ``relu_sites`` / ``MaskCapture``: the ReLU outputs a program keeps (``engine.keep_relu_output``), named by the oracle's
  sites (the BN state-dict prefixes of ``oracle/ffc_torch_cpu.py``), and the masks its backward read from them.

Importing this module needs no GPU; running a program does.
"""
import torch

from lama_b200 import _lib as L
from lama_b200 import engine as E
from spec_interp import SpecInterpreter

DEV = "cuda:0"


# ------------------------------------------------------------------------------------------- decoding
class Decoder:
    """Device storage of a ``Buf`` -> float64 [B, H, W, C] on the CPU, addressed as include/ffc_b200.h defines it
    (independent of the shape the executor allocated the storage with):
      plain             (b, y, x, c) at ((b*Hp + y+p)*Wp + x+p)*C + c      (Hp, Wp: with the ring of p pixels)
      channel groups    (b, y, x, c) at (c/cg)*B*H*W*cg + ((b*H + y)*W + x)*cg + c%cg
      tile-blocked      (m, c) at (m/128)*sg + (c/8)*1024 + (m%128)*8 + c%8,  m = (b*H + y)*W + x, sg = C/8*1024
    Split bf16 is hi + lo with the lo plane ``lo_off`` elements after the hi plane."""

    def __init__(self, ex):
        self.ex = ex
        self._idx = {}

    def _index(self, b):
        if b.name not in self._idx:
            p = b.pad
            B, H, W, C = b.B, b.H + 2 * p, b.W + 2 * p, b.C
            ar = lambda n, d: torch.arange(n, device=DEV).view([-1 if i == d else 1 for i in range(4)])  # noqa: E731
            bi, y, x, c = ar(B, 0), ar(H, 1), ar(W, 2), ar(C, 3)
            if b.tile:
                assert b.cg == 8 and b.tile == 128 and p == 0
                m = (bi * H + y) * W + x
                idx = (m // 128) * (C // 8 * 1024) + (c // 8) * 1024 + (m % 128) * 8 + c % 8
                lo_off = -(-(B * H * W) // 128) * (C // 8) * 1024
            elif b.cg:
                assert p == 0
                idx = (c // b.cg) * (B * H * W * b.cg) + ((bi * H + y) * W + x) * b.cg + c % b.cg
                lo_off = B * H * W * C
            else:
                idx = ((bi * H + y) * W + x) * C + c
                lo_off = B * H * W * C
            self._idx[b.name] = (idx, lo_off)
        return self._idx[b.name]

    def __call__(self, b, ring=False):
        """Interior [B, H, W, C]; with ``ring`` the whole padded plane [B, H+2p, W+2p, C]."""
        idx, lo_off = self._index(b)
        flat = self.ex.storage[b.name].reshape(-1)
        if b.fmt == L.F32:
            v = flat[idx].double()
        else:
            v = flat[idx].double() + flat[idx + lo_off].double()
        if b.pad and not ring:
            p = b.pad
            v = v[:, p:p + b.H, p:p + b.W]
        return v.cpu()


def split_bf16(v: torch.Tensor) -> torch.Tensor:
    """The value a split-bf16 store keeps of ``v``: hi = bf16(v), lo = bf16(v - hi), in float32 (csrc/common.cuh)."""
    f = v.float()
    hi = f.bfloat16().float()
    return hi.double() + (f - hi).bfloat16().double()


def ring_is_reflection(full: torch.Tensor, p: int) -> bool:
    """[B, H+2p, W+2p, C]: does every ring pixel hold the reflection (no edge repeat) of the interior?"""
    h, w = full.shape[1] - 2 * p, full.shape[2] - 2 * p

    def refl(n):
        i = (torch.arange(-p, n + p)).abs()
        return torch.where(i >= n, 2 * n - 2 - i, i)
    want = full[:, p:p + h, p:p + w][:, refl(h)][:, :, refl(w)]
    return torch.equal(full, want)


# ------------------------------------------------------------------------------------------- call at a time
class DeviceRun:
    """``prog`` bound to a ``CudaExecutor`` on ``DEV`` with ``inputs``; ``run`` issues its calls one at a time."""

    def __init__(self, prog: E.Program, inputs):
        self.prog = prog
        self.ex = E.CudaExecutor(prog, torch.device(DEV))
        assert len(self.ex.calls) == sum(not isinstance(op, E.SplitOp) for op in prog.ops)
        self.feed = {k: v.to(DEV).contiguous() for k, v in inputs.items()}    # bind_inputs keeps pointers only
        self.ex.bind_inputs(self.feed)
        self.dec = Decoder(self.ex)

    def run(self, before=None, after=None):
        """Issue every call on the current stream.  ``before(i, op)`` runs before the call of op i, ``after(i, op)``
        once it has completed (the device is synchronised)."""
        stream = torch.cuda.current_stream().cuda_stream
        calls = iter(self.ex.calls)
        torch.cuda.synchronize()
        for i, op in enumerate(self.prog.ops):
            if isinstance(op, E.SplitOp):
                continue
            if before is not None:
                before(i, op)
            name, fn, args = next(calls)
            L.check(fn(*args, stream), name)
            torch.cuda.synchronize()
            if after is not None:
                after(i, op)

    def outputs(self):
        return {k: v.cpu() for k, v in self.ex.outputs.items()}


# ------------------------------------------------------------------------------------------- per-op check
def op_label(i, op) -> str:
    s = f"op {i} {type(op).__name__}"
    if isinstance(op, E.ConvOp):
        s += f" [{op.tag}]"
    _, writes = op.views()
    return s + "".join(f" -> {tv.buf.name}" for tv in writes)


def op_tol(op, math: int, out_fmt: int):
    """(limit on max-abs / max|ref|, compare against the split-bf16 rounding of the reference?)"""
    if isinstance(op, (E.ConvOp, E.StemOp, E.HeadOp, E.HeadGatherOp, E.HeadBwdOp)):           # contractions
        return (2e-4 if math == L.MATH_BF16X3 else 2e-5), False
    if isinstance(op, (E.RfftOp, E.IrfftOp)):
        return (2e-5 if out_fmt == L.BF16X2 else 2e-6), False
    return 1e-6, out_fmt == L.BF16X2           # layout, ring, ReLU backward, fold, add, loss: exact up to the storage format


def max_rel(got, ref) -> float:
    """max |got - ref| / max |ref| (0 for empty tensors)."""
    scale = float(ref.abs().max()) if ref.numel() else 0.0
    return float((got - ref).abs().max()) / (scale or 1.0) if ref.numel() else 0.0


def diff_program(prog: E.Program, inputs, after_call=None):
    """Run ``prog`` on the GPU one call at a time and judge every op against the interpreter, fed with the device
    state the kernel saw.  ``after_call(i, op, ex)`` runs right after the call of op i (the harness self-test uses it).
    Returns [(op index, label, error, limit)] of the ops that disagree, and raises on a bad reflected ring."""
    run = DeviceRun(prog, inputs)
    ex, dec = run.ex, run.dec
    host_in = {k: v.cpu() for k, v in inputs.items()}
    interp = SpecInterpreter(prog)
    bad = []

    def before(i, op):
        reads, writes = op.views()
        touched = {tv.buf.name: tv.buf for tv in reads + writes}
        for name, b in touched.items():
            interp.mem[name] = dec(b)
        if isinstance(op, E.ConvOp) and op.packed.border == L.BORDER_REFLECT:
            for s, tv in enumerate(op.ins):
                if tv is not None and tv.buf.pad and any(g.src == s and (g.dy or g.dx) for g in op.packed.segs):
                    assert ring_is_reflection(dec(tv.buf, ring=True), tv.buf.pad), \
                        f"{op_label(i, op)}: the ring of input {tv.buf.name} is not the reflection of its interior"

    def after(i, op):
        if after_call is not None:
            after_call(i, op, ex)
            torch.cuda.synchronize()
        _, writes = op.views()
        out = {k: v.cpu() for k, v in ex.outputs.items()}     # the device's outputs as they stand before the call
        before_ = dict(out)
        interp.step(op, host_in, out)
        worst = None
        for tv in writes:
            ref = interp.read(tv)
            want = interp.mem[tv.buf.name]
            interp.mem[tv.buf.name] = dec(tv.buf)
            got = interp.read(tv)
            interp.mem[tv.buf.name] = want
            tol, rounded = op_tol(op, prog.math, tv.buf.fmt)
            err = max_rel(got, split_bf16(ref) if rounded else ref)
            if not err <= tol:
                worst = (i, op_label(i, op), err, tol)
        for dst in prog.outputs:
            if out[dst] is before_[dst]:
                continue                                # not written by this op
            tol, _ = op_tol(op, prog.math, L.F32)
            err = max_rel(ex.outputs[dst].cpu().double(), out[dst].double())
            if not err <= tol:
                worst = (i, op_label(i, op) + f" -> {dst}", err, tol)
        if worst is not None:
            bad.append(worst)

    run.run(before, after)
    return bad


# ------------------------------------------------------------------------------------------- ReLU masks
def relu_sites(prog: E.Program, module, prefix: str = "") -> dict:
    """{oracle site: view} of the ReLU outputs ``prog`` keeps: each BN module recorded by ``engine.keep_relu_output``
    named through ``module.named_modules()``, as ``prefix + name + "."`` (the state-dict prefix the oracle uses)."""
    names = {id(m): name for name, m in module.named_modules()}
    return {prefix + names[key[1]] + ".": rec["out"] for key, rec in prog.meta.items() if key[0] == "relu"}


def mask_view(op):
    """The view whose ReLU mask a backward op reads, or None."""
    if isinstance(op, E.ReluBwdOp):
        return op.y
    if isinstance(op, E.HeadBwdOp):
        return op.mask
    return None


def covers(outer: E.TV, inner: E.TV) -> bool:
    """Does view ``outer`` include the channels of view ``inner`` (both whole-plane views)?"""
    return (outer.buf.name == inner.buf.name
            and outer.c0 <= inner.c0 and inner.c0 + inner.channels <= outer.c0 + outer.channels)


class MaskCapture:
    """The ReLU masks a program's backward reads, per oracle site (NCHW bool).  Call ``before(op, read)`` before each
    op runs, with ``read(buf)`` -> the buffer's interior as [B, H, W, C] (``Decoder`` on the device, the interpreter's
    memory on the CPU): right before the ReLU backward that reads a kept output, that output is read — pooled storage
    is reused afterwards.  Each kept output must be read by exactly one backward op (``assert_complete``)."""

    def __init__(self, prog: E.Program, module, prefix: str = ""):
        self.sites = relu_sites(prog, module, prefix)
        self.masks = {}

    def before(self, op, read):
        tv = mask_view(op)
        if tv is None:
            return
        for site, v in self.sites.items():
            if covers(tv, v):
                assert site not in self.masks, f"the ReLU output of {site} is read by two backward ops"
                val = read(v.buf)[..., v.c0:v.c0 + v.channels]
                self.masks[site] = (val > 0).permute(0, 3, 1, 2).contiguous()

    def assert_complete(self):
        missing = sorted(set(self.sites) - set(self.masks))
        assert not missing, f"kept ReLU outputs no backward op reads: {missing}"
