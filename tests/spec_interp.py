"""TEST INFRASTRUCTURE: interpret a ``lama_b200.engine.Program`` on the CPU with slow torch
restatements of each op's contract (include/ffc_b200.h).  This checks the *host logic* of the
product — BN folding, weight packing, K-segment lists, buffer wiring, residual placement,
sub-pixel phases — against the goldens on the GPU-less build box.  It is not a fallback: the
product only executes programs through libffc_b200.so (lama_b200.engine.CudaExecutor).
"""
import torch

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
        y = torch.stack(ys, dim=1)
        return {L.ACT_NONE: y, L.ACT_RELU: y.clamp_min(0), L.ACT_SIGMOID: torch.sigmoid(y),
                L.ACT_TANH: torch.tanh(y)}[act]

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
        """Interpret one op: read its views from ``self.mem``, write its views there, and put external outputs
        (ToNCHW, the heads) into ``out``.  ``inputs`` holds the program's external NCHW (or uint8) inputs."""
        if isinstance(op, E.ToNHWC):
            self.write(op.out, inputs[op.src].double().permute(0, 2, 3, 1))
        elif isinstance(op, E.ToNCHW):
            out[op.dst] = self.read(op.inp).permute(0, 3, 1, 2).contiguous()
        elif isinstance(op, E.StemPackOp):
            x = torch.nn.functional.pad(inputs[op.src].double(), (3, 3, 3, 3), mode="reflect")
            x = torch.nn.functional.pad(x, (0, 2, 0, 0, 0, 8 - op.cin))          # W+6 -> W+8, Cin -> 8 (zeros)
            self.write(op.out, self._two_rows(x.permute(0, 2, 3, 1), op.cin))
        elif isinstance(op, E.StemPackU8Op):
            x = self._u8_front(inputs[op.img], inputs[op.mask], op.out.buf.H - 6, op.out.buf.W - 8)
            x = torch.nn.functional.pad(x.double(), (3, 3, 3, 3), mode="reflect")
            x = torch.nn.functional.pad(x, (0, 2, 0, 0, 0, 4))
            self.write(op.out, self._two_rows(x.permute(0, 2, 3, 1), 4))
        elif isinstance(op, E.HeadGatherU8Op):
            pred = self._gather(self.read(op.q), op.bias, 3, op.act).float()[:, :, :op.h0, :op.w0]
            img = inputs[op.img].permute(0, 3, 1, 2).float() / 255
            hole = (inputs[op.mask] > 0)[:, None]
            res = torch.where(hole, pred, img)                      # mask*pred + (1-mask)*img, mask in {0,1}
            out[op.dst] = (res * 255).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
        elif isinstance(op, E.StemOp):
            x = torch.nn.functional.pad(inputs[op.src].double(), (3, 3, 3, 3), mode="reflect")
            cin = op.cin
            w = op.w.double().to(x.device).reshape(7, 7, cin, -1).permute(3, 2, 0, 1)       # [N, Cin, 7, 7]
            y = torch.nn.functional.conv2d(x, w) + op.shift.double().to(x.device)[None, :, None, None]
            self.write(op.out, y.clamp_min(0).permute(0, 2, 3, 1))
        elif isinstance(op, E.HeadOp):
            x = self.read(op.inp).permute(0, 3, 1, 2)
            x = torch.nn.functional.pad(x, (3, 3, 3, 3), mode="reflect")
            w = op.w.double().to(x.device).reshape(op.n_out, 7, 7, -1).permute(0, 3, 1, 2)
            y = torch.nn.functional.conv2d(x, w, op.bias.double().to(x.device))
            y = {L.ACT_NONE: y, L.ACT_RELU: y.clamp_min(0), L.ACT_SIGMOID: torch.sigmoid(y),
                 L.ACT_TANH: torch.tanh(y)}[op.act]
            out[op.dst] = y
        elif isinstance(op, E.HeadGatherOp):
            out[op.dst] = self._gather(self.read(op.q), op.bias, op.n_out, op.act)
        elif isinstance(op, E.ConvOp):
            ins = [self.read(tv) if tv is not None else None for tv in op.ins]
            assert all(not torch.isnan(t).any() for t in ins if t is not None), f"{op.tag}: reads unwritten data"
            add = self.read(op.addend).clone() if op.addend is not None else None
            y = apply_packed_reference(op.packed, ins, op.out.hw, addend=add, addend_post=op.addend_post)
            self.write(op.out, y)
        elif isinstance(op, E.BorderOp) or isinstance(op, E.SplitOp):
            pass        # the interpreter's buffers have no physical ring (taps use index math)
        elif isinstance(op, E.ReluBwdOp):
            self.write(op.out, self.read(op.dy) * (self.read(op.y) > 0))
        elif isinstance(op, E.FoldOp):
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
        elif isinstance(op, E.RfftOp):
            x = self.read(op.inp)                                            # [B,H,W,C]
            f = torch.fft.rfftn(x, dim=(1, 2), norm="ortho")                 # [B,H,Wf,C]
            self.write(op.spec, torch.view_as_real(f).reshape(*f.shape[:3], -1))   # channel 2c=Re, 2c+1=Im
        elif isinstance(op, E.IrfftOp):
            z = self.read(op.spec)
            zc = torch.view_as_complex(z.reshape(*z.shape[:3], -1, 2).contiguous())
            h, w = op.out.hw
            y = torch.fft.irfftn(zc, s=(h, w), dim=(1, 2), norm="ortho")
            if op.residual is not None:
                y = y + self.read(op.residual)
            self.write(op.out, y)
        else:
            raise TypeError(op)
