#!/usr/bin/env python
"""FFT pair per axis length: the Bluestein mode against the runtime plans it replaces, and against cuFFT.

    python tools/fft_lengths_bench.py [--lo 100] [--hi 1024] [--lengths 479,502,...] [--rounds 3] [--out DIR]

Times ffcb_rfft2 + ffcb_irfft2 (+ residual) on big-lama's spectral shape: batch 1, 192 channels, an n x n plane, in the
generator program's formats (float32 planes, split-bf16 forward spectrum and inverse output).  Lengths: every n in
[lo, hi] the planner routes to Bluestein, and the neighbours n - 1, n + 1 that keep their runtime plan.  Three arms,
alternated within each round on the same inputs:
  * default      — the shipped plans (Bluestein where fft_core.cuh's make_bluestein_plan picks it);
  * bluestein0   — FFCB_FFT_BLUESTEIN=0: the runtime mixed-radix plans (a direct DFT for primes);
  * torch        — torch.fft.rfftn / irfftn (cuFFT, float32 NCHW) of the same plane, plus the residual.
Each sample is CUDA events around enough pairs to fill ~20 ms; the median of ``--rounds`` samples is reported.  The
planner's choices and modelled costs come from tests/host_emul/fft_bluestein_emul.cpp, compiled with g++ into a
temporary directory.  The card's name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def planner():
    """{n: (m, lanes, modelled Bluestein cost, modelled runtime-plan cost, radices)} for n = 2..1024 (m = 0: the
    runtime plan of n)."""
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "fft_bluestein_emul")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I/usr/local/cuda/include",
                               os.path.join(ROOT, "tests", "host_emul", "fft_bluestein_emul.cpp"), "-o", exe])
        out = subprocess.run([exe, "plans"], capture_output=True, text=True, check=True).stdout
    plans = {}
    for line in out.splitlines():
        head, radices = line.split("|")
        n, m, lanes, cost, direct = head.split()
        plans[int(n)] = (int(m), int(lanes), float(cost), int(direct), [int(r) for r in radices.split()])
    return plans


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lo", type=int, default=100)
    ap.add_argument("--hi", type=int, default=1024)
    ap.add_argument("--lengths", default=None, help="comma-separated lengths instead of the sweep")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    from lama_b200 import _lib as L
    from lama_b200 import engine as E

    assert torch.cuda.is_available(), "fft_lengths_bench.py needs a GPU"
    dev = torch.device("cuda:0")
    plans = planner()
    if a.lengths:
        lengths = sorted({int(s) for s in a.lengths.split(",")})
    else:
        bs = [n for n in range(a.lo, a.hi + 1) if plans[n][0] > 0]
        lengths = sorted(set(bs) | {k for n in bs for k in (n - 1, n + 1) if a.lo <= k <= a.hi and plans[k][0] == 0})
    info = {"card": card(), "torch": torch.__version__, "B": 1, "C": 192, "lengths": []}
    print("card (name, power limit, max SM clock):", info["card"], flush=True)
    b, c = 1, 192
    stream = torch.cuda.current_stream().cuda_stream
    for n in lengths:
        h = w = n
        wf = w // 2 + 1
        prog = E.Program("fft_len_bench", L.MATH_BF16X3)
        X = prog.buf("x", b, h, w, c); S = prog.buf("s", b, h, wf, 2 * c, gemm=True)
        Z = prog.buf("z", b, h, wf, 2 * c); O = prog.buf("o", b, h, w, c, gemm=True)
        prog.ops += [E.RfftOp(E.TV(X), E.TV(S)), E.IrfftOp(E.TV(Z), E.TV(X), E.TV(O))]
        ex = E.CudaExecutor(prog, dev)
        ex.storage[X.name].normal_()
        ex.storage[Z.name].normal_()
        xt = torch.randn(b, c, h, w, device=dev)

        def native():
            for name, fn, args in ex.calls:
                L.check(fn(*args, stream), name)

        def cufft():
            s = torch.fft.rfftn(xt, dim=(-2, -1), norm="ortho")
            return torch.fft.irfftn(s, s=(h, w), dim=(-2, -1), norm="ortho") + xt

        arms = {"default": ({}, native), "bluestein0": ({"FFCB_FFT_BLUESTEIN": "0"}, native), "torch": ({}, cufft)}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps, samples = {}, {k: [] for k in arms}
        for k, (env, fn) in arms.items():              # warm-up, and the pairs per sample
            os.environ.pop("FFCB_FFT_BLUESTEIN", None)
            os.environ.update(env)
            fn()
            torch.cuda.synchronize()
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            reps[k] = max(1, min(200, int(20.0 / max(e0.elapsed_time(e1), 1e-3))))
        for _ in range(a.rounds):
            for k, (env, fn) in arms.items():
                os.environ.pop("FFCB_FFT_BLUESTEIN", None)
                os.environ.update(env)
                e0.record()
                for _ in range(reps[k]):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                samples[k].append(e0.elapsed_time(e1) / reps[k])
        os.environ.pop("FFCB_FFT_BLUESTEIN", None)
        m, lanes, cost, direct, radices = plans[n]
        r = {"n": n, "m": m, "lanes": lanes, "plan": radices, "model_ratio": round(cost / direct, 3) if cost else None}
        for k, v in samples.items():
            r[f"{k}_ms"] = round(sorted(v)[len(v) // 2], 4)
        r["speedup_vs_bluestein0"] = round(r["bluestein0_ms"] / r["default_ms"], 3)
        r["vs_torch"] = round(r["torch_ms"] / r["default_ms"], 3)
        info["lengths"].append(r)
        print(json.dumps(r), flush=True)
        del ex, prog, xt
        torch.cuda.empty_cache()
    sel = [r for r in info["lengths"] if r["m"] > 0]
    if sel:
        worst = min(sel, key=lambda r: r["speedup_vs_bluestein0"])
        print(f"{len(sel)} Bluestein lengths; smallest speed-up over FFCB_FFT_BLUESTEIN=0: "
              f"{worst['speedup_vs_bluestein0']}x at n = {worst['n']}", flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fft_lengths_bench.json"), "w") as fh:
            json.dump(info, fh, indent=1)


if __name__ == "__main__":
    main()
