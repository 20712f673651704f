"""TEST INFRASTRUCTURE: interpret a ``lama_b200.engine.Program`` on the CPU with slow torch
restatements of each op's contract (include/ffc_b200.h).  This checks the *host logic* of the
product — BN folding, weight packing, K-segment lists, buffer wiring, residual placement,
sub-pixel phases — against the goldens on the GPU-less build box.  It is not a fallback: the
product only executes programs through libffc_b200.so (lama_b200.engine.CudaExecutor).
"""
from collections import ChainMap

import torch
import torch.nn.functional as F

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200.packing import apply_packed_reference


class SpecInterpreter:
    def __init__(self, prog: E.Program):
        self.prog = prog
        # buffers share storage exactly as in the product's executor (engine.assign_storage_slots): a buffer whose
        # slot is reused too early would be read back corrupted here too, on the CPU
        slots = E.assign_storage_slots(prog)
        by_slot = {}
        self.mem = {}
        for b in prog.bufs:
            if slots[b.name] not in by_slot:
                by_slot[slots[b.name]] = torch.full((b.B, b.H, b.W, b.C), float("nan"), dtype=torch.float64)
            self.mem[b.name] = by_slot[slots[b.name]]
            assert tuple(self.mem[b.name].shape) == (b.B, b.H, b.W, b.C)
        self.n_slots = len(by_slot)
        for name, val in prog.consts.items():
            self.mem[name] = val.double().clone()

    def read(self, tv: E.TV) -> torch.Tensor:
        t = self.mem[tv.buf.name][tv.b0:tv.b0 + tv.batch]
        if tv.bcast:
            t = self.mem[tv.buf.name].expand(tv.bcast, -1, -1, -1)
        if tv.window:      # sliding-window view: pixel x exposes pixels x .. x+window-1, channel index = j*C + c
            w_out = tv.buf.W - tv.window
            return torch.cat([t[:, :, j:j + w_out] for j in range(tv.window)], dim=-1)
        if tv.phase is not None:
            a, b = tv.phase
            t = t[:, a::2, b::2]
        if tv.win is not None:
            y0, x0, h, w = tv.win
            t = t[:, y0:y0 + h, x0:x0 + w]
        return t[..., tv.c0:tv.c0 + tv.channels]

    def write(self, tv: E.TV, val: torch.Tensor):
        t = self.mem[tv.buf.name][tv.b0:tv.b0 + tv.batch]
        if tv.phase is not None:
            a, b = tv.phase
            t[:, a::2, b::2, tv.c0:tv.c0 + tv.channels] = val
        elif tv.win is not None:
            y0, x0, h, w = tv.win
            t[:, y0:y0 + h, x0:x0 + w, tv.c0:tv.c0 + tv.channels] = val
        else:
            t[..., tv.c0:tv.c0 + tv.channels] = val

    @staticmethod
    def _gather(q, bias, n_out, act):
        """ffcb_head_gather7: q [B,H,W,>=7N] -> act(bias + sum_kx q[.., reflect(x+kx-3), n*7+kx]) as NCHW."""
        w = q.shape[2]
        xi = torch.arange(w)[:, None] + torch.arange(7)[None, :] - 3           # [W,7]
        xi = xi.abs(); xi = torch.where(xi >= w, 2 * w - 2 - xi, xi)
        ys = []
        for n in range(n_out):
            g = q[:, :, :, n * 7:n * 7 + 7]                  # [B,H,W,7]
            ys.append(sum(g[:, :, xi[:, kx], kx] for kx in range(7)) + float(bias[n]))
        return _ACT[act](torch.stack(ys, dim=1))

    @staticmethod
    def _two_rows(p, cin):
        """ffcb_stem_pack's two-row packing (Cin <= 4): channels 4..7 of a packed pixel = channels 0..3 one row below."""
        if cin > 4:
            return p
        p = p.clone()
        p[:, :-1, :, 4:4 + cin] = p[:, 1:, :, :cin]
        return p

    @staticmethod
    def _u8_front(img, mask, h, w):
        """ffcb_stem_pack_u8 up to the reflection ring: (B,H0,W0,3) u8 + (B,H0,W0) u8 -> (B,4,H,W) float32."""
        h0, w0 = mask.shape[1:]
        ys = torch.arange(h); ys = torch.where(ys < h0, ys, 2 * h0 - 1 - ys)
        xs = torch.arange(w); xs = torch.where(xs < w0, xs, 2 * w0 - 1 - xs)
        x = (img.float() / 255)[:, ys][:, :, xs].permute(0, 3, 1, 2)
        m = (mask > 0).float()[:, ys][:, :, xs][:, None]
        return torch.cat([x * (1 - m), m], dim=1)

    def run(self, inputs):
        out = {}
        for op in self.prog.ops:
            self.step(op, inputs, out)
        return out

    def step(self, op, inputs, out):
        """Interpret one op: read its views from ``self.mem``, write its views there.  Its external tensors resolve
        from one namespace, as in the executor: the program's inputs (``inputs``) and the outputs written so far
        (``out``); the outputs it writes go to ``out``."""
        getattr(self, type(op).__name__)(op, ChainMap(out, inputs))

    def ToNHWC(self, op, ext):
        self.write(op.out, ext[op.src].double().permute(0, 2, 3, 1))

    def ToNCHW(self, op, ext):
        ext[op.dst] = self.read(op.inp).permute(0, 3, 1, 2).contiguous()

    def StemPackOp(self, op, ext):
        x = F.pad(ext[op.src].double(), (3, 3, 3, 3), mode="reflect")
        x = F.pad(x, (0, 2, 0, 0, 0, 8 - op.cin))          # W+6 -> W+8, Cin -> 8 (zeros)
        self.write(op.out, self._two_rows(x.permute(0, 2, 3, 1), op.cin))

    def StemPackU8Op(self, op, ext):
        x = self._u8_front(ext[op.img], ext[op.mask], op.out.buf.H - 6, op.out.buf.W - 8)
        x = F.pad(x.double(), (3, 3, 3, 3), mode="reflect")
        x = F.pad(x, (0, 2, 0, 0, 0, 4))
        self.write(op.out, self._two_rows(x.permute(0, 2, 3, 1), 4))

    def HeadGatherU8Op(self, op, ext):
        pred = self._gather(self.read(op.q), op.bias, 3, op.act).float()[:, :, :op.h0, :op.w0]
        img = ext[op.img].permute(0, 3, 1, 2).float() / 255
        hole = (ext[op.mask] > 0)[:, None]
        res = torch.where(hole, pred, img)                      # mask*pred + (1-mask)*img, mask in {0,1}
        ext[op.dst] = (res * 255).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()

    def StemOp(self, op, ext):
        x = F.pad(ext[op.src].double(), (3, 3, 3, 3), mode="reflect")
        cin = op.cin
        w = op.w.double().to(x.device).reshape(7, 7, cin, -1).permute(3, 2, 0, 1)       # [N, Cin, 7, 7]
        y = F.conv2d(x, w) + op.shift.double().to(x.device)[None, :, None, None]
        self.write(op.out, y.clamp_min(0).permute(0, 2, 3, 1))

    def HeadOp(self, op, ext):
        x = self.read(op.inp).permute(0, 3, 1, 2)
        x = F.pad(x, (3, 3, 3, 3), mode="reflect")
        w = op.w.double().to(x.device).reshape(op.n_out, 7, 7, -1).permute(0, 3, 1, 2)
        ext[op.dst] = _ACT[op.act](F.conv2d(x, w, op.bias.double().to(x.device)))

    def HeadGatherOp(self, op, ext):
        ext[op.dst] = self._gather(self.read(op.q), op.bias, op.n_out, op.act)

    def ConvOp(self, op, ext):
        ins = [self.read(tv) if tv is not None else None for tv in op.ins]
        assert all(not torch.isnan(t).any() for t in ins if t is not None), f"{op.tag}: reads unwritten data"
        add = self.read(op.addend).clone() if op.addend is not None else None
        y = apply_packed_reference(op.packed, ins, op.out.hw, addend=add, addend_post=op.addend_post)
        self.write(op.out, y)

    def BorderOp(self, op, ext):
        pass        # the interpreter's buffers have no physical ring (taps use index math)

    def SplitOp(self, op, ext):
        pass

    def ReluBwdOp(self, op, ext):
        self.write(op.out, self.read(op.dy) * (self.read(op.y) > 0))

    def FoldOp(self, op, ext):
        g = self.read(op.gpad)                                  # [B, H+2, W+2, C]
        h, w = g.shape[1] - 2, g.shape[2] - 2
        acc = torch.zeros(g.shape[0], h, w, g.shape[3], dtype=g.dtype)
        for yp in range(h + 2):
            y = abs(yp - 1); y = 2 * h - 2 - y if y >= h else y
            for xp in range(w + 2):
                x = abs(xp - 1); x = 2 * w - 2 - x if x >= w else x
                acc[:, y, x] += g[:, yp, xp]
        for tv, c0 in op.addends:
            a = self.read(tv)
            acc[..., c0:c0 + a.shape[-1]] += a
        self.write(op.out, acc)

    def AddOp(self, op, ext):
        self.write(op.out, self.read(op.a) + self.read(op.b))

    def HeadBwdOp(self, op, ext):
        y, dy = ext[op.y].double().cpu(), ext[op.dy].double().cpu()
        d = {L.ACT_NONE: dy, L.ACT_SIGMOID: dy * y * (1 - y), L.ACT_TANH: dy * (1 - y * y)}[op.act]
        w = op.w.double().cpu().reshape(op.n_out, 7, 7, -1).permute(0, 3, 1, 2)              # [N, C, 7, 7]
        gp = F.conv_transpose2d(d, w)                                                     # [B, C, H+6, W+6]
        h, wd = gp.shape[2] - 6, gp.shape[3] - 6
        # Fold3: padded row / column p came from interior reflect(p - 3)
        ry = (torch.arange(h + 6) - 3).abs(); ry = torch.where(ry >= h, 2 * h - 2 - ry, ry)
        rx = (torch.arange(wd + 6) - 3).abs(); rx = torch.where(rx >= wd, 2 * wd - 2 - rx, rx)
        g = torch.zeros(gp.shape[0], gp.shape[1], h, wd + 6, dtype=gp.dtype).index_add_(2, ry, gp)
        g = torch.zeros(gp.shape[0], gp.shape[1], h, wd, dtype=gp.dtype).index_add_(3, rx, g)
        m = self.read(op.mask)
        self.write(op.out, g.permute(0, 2, 3, 1) * (m > 0))

    def RefineLossOp(self, op, ext):
        f = {k: ext[getattr(op, k)].double().cpu() for k in ("pred", "image", "mask", "ref", "md", "inv")}
        ext[op.grad], ext[op.loss] = refine_loss_f64(f["pred"], f["image"], f["mask"], f["ref"], f["md"], f["inv"],
                                                     op.h0, op.w0, op.taps)

    def RfftOp(self, op, ext):
        x = self.read(op.inp)                                            # [B,H,W,C]
        f = torch.fft.rfftn(x, dim=(1, 2), norm="ortho")                 # [B,H,Wf,C]
        self.write(op.spec, torch.view_as_real(f).reshape(*f.shape[:3], -1))   # channel 2c=Re, 2c+1=Im

    def IrfftOp(self, op, ext):
        z = self.read(op.spec)
        zc = torch.view_as_complex(z.reshape(*z.shape[:3], -1, 2).contiguous())
        h, w = op.out.hw
        y = torch.fft.irfftn(zc, s=(h, w), dim=(1, 2), norm="ortho")
        if op.residual is not None:
            y = y + self.read(op.residual)
        self.write(op.out, y)


def storage_nbytes(b):
    if b.tile:
        return -(-(b.B * b.H * b.W) // 128) * 128 * b.C * 4
    if b.cg:
        return b.B * b.H * b.W * b.C * 4
    return b.B * (b.H + 2 * b.pad) * (b.W + 2 * b.pad) * b.C * 4


def check_liveness(prog):
    """No two buffers of one storage slot are live at once (a forward write must survive to its backward read); returns
    the pooled storage in bytes."""
    slots = E.assign_storage_slots(prog)
    first, last = {}, {}
    for i, op in enumerate(prog.ops):
        r, w = op.views()
        for tv in r + w:
            first.setdefault(tv.buf.name, i)
            last[tv.buf.name] = i
    by_slot = {}
    for b in prog.bufs:
        by_slot.setdefault(slots[b.name], []).append(b)
    for members in by_slot.values():
        assert len({E.storage_key(b) for b in members}) == 1
        members = sorted(members, key=lambda b: first.get(b.name, -1))
        for a, b in zip(members, members[1:]):
            assert last[a.name] < first[b.name], (a.name, b.name)
    return sum(storage_nbytes(m[0]) for m in by_slot.values())


_ACT = {L.ACT_NONE: lambda y: y, L.ACT_RELU: lambda y: y.clamp_min(0), L.ACT_SIGMOID: torch.sigmoid,
        L.ACT_TANH: torch.tanh}


def _axis_matrix(n_in: int, taps) -> torch.Tensor:
    """1-D operator of D along one axis, [n_in // 2, n_in]: bilinear (align_corners=False) rows of the 5-tap Gaussian
    with reflect-101 padding (include/ffc_b200.h: ffcb_refine_l1_grad)."""
    n_out = n_in // 2
    scale = n_in / n_out
    m = torch.zeros(n_out, n_in, dtype=torch.float64)
    for d in range(n_out):
        src = max(scale * (d + 0.5) - 0.5, 0.0)
        i0 = int(src)
        i1 = i0 + (1 if i0 < n_in - 1 else 0)
        l1 = src - i0
        for i, lam in ((i0, 1.0 - l1), (i1, l1)):
            for a in range(5):
                p = abs(i + a - 2)
                p = 2 * n_in - 2 - p if p >= n_in else p
                m[d, p] += lam * float(taps[a])
    return m


def refine_loss_f64(pred, image, mask, ref, md, inv, h0, w0, taps):
    """(grad, loss (B,2)) of ffcb_refine_l1_grad in float64."""
    inv = inv.double()
    sel = (mask < 1e-8).double()
    d = pred - image
    grad = torch.sign(d) * sel * inv[:, 0, None, None, None]
    my, mx = _axis_matrix(h0, taps), _axis_matrix(w0, taps)
    e = torch.einsum("iy,bcyx,jx->bcij", my, pred[:, :, :h0, :w0], mx) - ref
    seld = (md >= 1e-8).double()
    r = torch.sign(e) * seld * inv[:, 1, None, None, None]
    grad[:, :, :h0, :w0] += torch.einsum("iy,bcij,jx->bcyx", my, r, mx)
    nan = torch.tensor(float("nan"), dtype=torch.float64)
    l0 = torch.where(inv[:, 0] > 0, (d.abs() * sel).sum((1, 2, 3)) * inv[:, 0], nan)
    l1 = torch.where(inv[:, 1] > 0, (e.abs() * seld).sum((1, 2, 3)) * inv[:, 1], nan)
    return grad, torch.stack([l0, l1], 1)
