#!/usr/bin/env python
"""Forward + input gradient through a whole frozen generator: the native ``generator_grad`` program against the
torch path the drop-in took before it (``LAMA_B200_NATIVE_GRAD=0``: the residual blocks as per-block native programs
for the FFC generator, everything else torch autograd on cuDNN with its default TF32).

    python tools/generator_grad_bench.py [--steps 10] [--warmup 2] [--out DIR]

Per case and arm: ms per ``y = gen(x); torch.autograd.grad(y, x, g)`` (CUDA events over ``--steps`` after ``--warmup``
untimed passes, mean) and the peak of ``torch.cuda.max_memory_allocated`` over the timed passes.  Cases: big-lama at
512x512 bs8 and 1024x1024 bs1, lama-regular at 512x512 bs8, and big-lama at 2160x3840 bs1 on the native arm alone (its
torch arm does not fit in 80 GB).  Seeded weights, random inputs.  The card's name, power limit and maximum SM clock are
read in the same run.  One JSON line per measurement on stdout; with ``--out`` the lines also go to
DIR/generator_grad_bench.jsonl.  Nothing else is written.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [("big-lama", 8, 512, 512, True), ("big-lama", 1, 1024, 1024, True), ("lama-regular", 8, 512, 512, True),
         ("big-lama", 1, 2160, 3840, False)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def make(model):
    from lama_b200 import modules as M
    from lama_b200 import pix2pixhd as PX
    from lama_b200.testing import BIG_LAMA_KWARGS, LAMA_REGULAR_KWARGS, seeded_parameters_
    gen = M.FFCResNetGenerator(**BIG_LAMA_KWARGS) if model == "big-lama" else PX.GlobalGenerator(**LAMA_REGULAR_KWARGS)
    return seeded_parameters_(gen.eval(), 0, gain=1.0).requires_grad_(False).cuda()


def measure(gen, b, h, w, steps, warmup):
    import torch
    gx = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(b, 4, h, w, device="cuda", generator=gx).requires_grad_(True)
    g = torch.rand(b, 3, h, w, device="cuda", generator=gx)

    def step():
        y = gen(x)
        return torch.autograd.grad(y, x, g)[0]

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        dx = step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated() / 1e9, dx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from lama_b200 import engine as E
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    lines = [dict(card=card(), torch=torch.__version__)]
    print(json.dumps(lines[-1]), flush=True)
    for model, b, h, w, torch_arm in CASES:
        gen = make(model)
        assert E.generator_grad_supported(gen, (b, 4, h, w))
        dx = {}
        for arm in (("native", "torch") if torch_arm else ("native",)):
            os.environ["LAMA_B200_NATIVE_GRAD"] = "1" if arm == "native" else "0"
            ms, gb, dx[arm] = measure(gen, b, h, w, a.steps, a.warmup)
            E.invalidate(gen)
            rec = dict(model=model, batch=b, h=h, w=w, arm=arm, ms_per_fwd_bwd=round(ms, 2), peak_gb=round(gb, 2))
            lines.append(rec)
            print(json.dumps(rec), flush=True)
            torch.cuda.empty_cache()
        if torch_arm:
            rel = float((dx["native"] - dx["torch"]).abs().max() / dx["torch"].abs().max())
            lines.append(dict(model=model, batch=b, h=h, w=w, dx_native_vs_torch_max_rel=rel))
            print(json.dumps(lines[-1]), flush=True)
        del gen, dx
        torch.cuda.empty_cache()
    os.environ.pop("LAMA_B200_NATIVE_GRAD", None)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "generator_grad_bench.jsonl"), "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
