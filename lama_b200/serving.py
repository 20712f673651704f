"""Throughput-oriented public entry point: a copy/compute pipeline around the generator program.

``bin/predict.py`` feeds one image at a time from host memory (predict.py:67-94).  For batched serving the
host<->device copies of one batch (134 MB in, 100 MB out at bs32 512x512) would add ~10% to every step if they
ran serially with the kernels, so :class:`GeneratorPipeline` keeps ``depth`` batches in flight on three CUDA
streams: H2D of batch i+1 and D2H of batch i-1 overlap the CUDA-graph replay of batch i.

    pipe = GeneratorPipeline(generator, batch=32, height=512, width=512)
    t = pipe.submit(x_pinned)        # (B,4,H,W) float32, pinned host memory; returns immediately
    y = pipe.result(t)               # (B,3,H,W) float32 pinned host tensor (valid until the slot is reused)

``u8=True`` selects the predict-path program (SURVEY.md row f1): the pipeline then takes the decoded bytes
(images (B,H0,W0,3) uint8, masks (B,H0,W0) uint8 — 1 byte per sample instead of 4 over PCIe) and returns the
inpainted RGB bytes (B,H0,W0,3); /255, symmetric modulo padding, mask multiply / concat, blend, crop and x255 run
inside the first and last kernels of the program (lama_b200.predict builds on this).
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import engine as E


class GeneratorPipeline:
    def __init__(self, generator, batch: int, height: int, width: int, device: Optional[torch.device] = None,
                 depth: int = 2, math: Optional[int] = None, u8: bool = False, pad_mod: int = 8):
        dev = device if device is not None else next(generator.parameters()).device
        assert dev.type == "cuda", "GeneratorPipeline needs the generator on a CUDA device"
        self.device, self.depth = dev, depth
        cin = E.generator_in_channels(generator)
        hp, wp = (-(-height // pad_mod) * pad_mod, -(-width // pad_mod) * pad_mod) if u8 else (height, width)
        probe = torch.empty(batch, cin, hp, wp, device=dev)
        if not E.generator_supported(generator, probe):
            raise ValueError(f"generator / {hp}x{wp} input is outside the native path")
        del probe
        if u8:
            metas = (torch.empty(batch, height, width, 3, dtype=torch.uint8, device="meta"),
                     torch.empty(batch, height, width, dtype=torch.uint8, device="meta"))
            self.ex = E.get_executor(generator, f"generator_u8:{pad_mod}", metas, math=math, device=dev)
        else:
            self.ex = E.get_executor(generator, "generator", (torch.empty(batch, cin, height, width, device="meta"),),
                                     math=math, device=dev)
        self.graph = E.GraphedProgram(self.ex)
        prog = self.ex.prog
        self.in_names = list(prog.inputs)
        self.in_shapes = [tuple(prog.inputs[k]) for k in self.in_names]
        self.in_dtypes = [prog.dtypes.get(k, torch.float32) for k in self.in_names]
        self.in_shape = self.in_shapes[0]
        self.out_shape = tuple(prog.outputs["y0"])
        self.out_dtype = prog.dtypes.get("y0", torch.float32)
        self.s_in, self.s_run, self.s_out = (torch.cuda.Stream(dev) for _ in range(3))
        self.dev_in = [[torch.empty(sh, dtype=dt, device=dev) for sh, dt in zip(self.in_shapes, self.in_dtypes)]
                       for _ in range(depth)]
        self.dev_out = [torch.empty(self.out_shape, dtype=self.out_dtype, device=dev) for _ in range(depth)]
        self.host_out = [torch.empty(self.out_shape, dtype=self.out_dtype).pin_memory() for _ in range(depth)]
        ev = lambda: [torch.cuda.Event() for _ in range(depth)]  # noqa: E731
        self.ev_in, self.ev_run, self.ev_out, self.ev_free = ev(), ev(), ev(), ev()
        self._n = 0
        self._pending: List[int] = []

    def submit(self, *hosts: torch.Tensor) -> int:
        """Enqueue one batch (pinned host tensors: (B,4,H,W) float32, or images + masks bytes for ``u8``);
        returns a ticket for :meth:`result`."""
        assert len(hosts) == len(self.in_names), f"expected {self.in_names}"
        for t, sh, dt in zip(hosts, self.in_shapes, self.in_dtypes):
            assert tuple(t.shape) == sh and t.dtype == dt, f"expected {dt} {sh}, got {t.dtype} {tuple(t.shape)}"
        n, slot = self._n, self._n % self.depth
        if n >= self.depth:
            self.ev_out[slot].synchronize()          # the host buffer of this slot must have been drained
        with torch.cuda.stream(self.s_in):
            if n >= self.depth:
                self.s_in.wait_event(self.ev_free[slot])     # its device input must have been consumed
            for d, t in zip(self.dev_in[slot], hosts):
                d.copy_(t, non_blocking=True)
            self.ev_in[slot].record(self.s_in)
        with torch.cuda.stream(self.s_run):
            self.s_run.wait_event(self.ev_in[slot])
            if n >= self.depth:
                self.s_run.wait_event(self.ev_out[slot])     # D2H of the previous occupant has read dev_out[slot]
            for k, d in zip(self.in_names, self.dev_in[slot]):
                self.graph.static_in[k].copy_(d, non_blocking=True)
            self.ev_free[slot].record(self.s_run)
            self.graph.graph.replay()
            self.dev_out[slot].copy_(self.ex.outputs["y0"], non_blocking=True)
            self.ev_run[slot].record(self.s_run)
        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(self.ev_run[slot])
            self.host_out[slot].copy_(self.dev_out[slot], non_blocking=True)
            self.ev_out[slot].record(self.s_out)
        self._n += 1
        return n

    def result(self, ticket: int) -> torch.Tensor:
        """Block until batch ``ticket`` is on the host; the tensor is reused ``depth`` submissions later."""
        assert self._n - self.depth <= ticket < self._n, "result no longer (or not yet) available"
        slot = ticket % self.depth
        self.ev_out[slot].synchronize()
        return self.host_out[slot]

    def drain(self):
        for s in (self.s_in, self.s_run, self.s_out):
            s.synchronize()

    @property
    def launches_per_batch(self) -> int:
        return self.ex.launches_per_run
