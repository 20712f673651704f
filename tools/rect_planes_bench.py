#!/usr/bin/env python
"""Rectangular bottleneck planes against the square plane with the same pixel count.

    python tools/rect_planes_bench.py [--rounds 5] [--steps 10] [--out DIR]

Two workloads per plane, each group of planes with equal pixel counts alternated within every round (same inputs):
  * fft_ms — ffcb_rfft2 + ffcb_irfft2 (+ residual) on big-lama's spectral shape: batch 1, 192 channels, the generator
             program's formats (float32 planes, split-bf16 forward spectrum and inverse output); CUDA events around
             enough pairs to fill ~20 ms.  A 64x64 plane takes the fused whole-plane kernels, every other plane the
             two-pass kernels (one launch per axis and direction).
  * gen_ms — big-lama's generator program at batch 1 on an image 8x the plane (CUDA-graph replays, CUDA events over
             ``--steps`` replays), for the groups whose images have at most 2048x2048 pixels.
The median of ``--rounds`` samples is reported with its ratio to the group's square plane (1024x96 and 96x1024 have no
square of equal area: they are compared with each other).  The card's name and power limit are read in the same run
and printed with the numbers.  Nothing is written outside ``--out``.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GROUPS = [[(64, 64), (32, 128), (128, 32)],
          [(128, 128), (64, 256), (256, 64)],
          [(256, 256), (128, 512), (512, 128)],
          [(512, 512), (256, 1024), (1024, 256)],
          [(96, 1024), (1024, 96)]]
GEN_MAX_PIXELS = 2048 * 2048


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    os.environ["LAMA_B200_STRICT"] = "1"
    from lama_b200 import _lib as L
    from lama_b200 import engine as E
    from lama_b200 import modules as M
    from lama_b200.testing import BIG_LAMA_KWARGS, generator_input, seeded_parameters_, synthetic_image_mask

    assert torch.cuda.is_available(), "rect_planes_bench.py needs a GPU"
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    info = {"card": card(), "torch": torch.__version__, "math": "bf16x3", "B": 1, "C": 192, "groups": []}
    print("card (name, power limit, max SM clock):", info["card"], flush=True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to(dev)

    def timed(fn, reps):
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    def alternate(arms, reps):
        """{plane: median ms} over ``--rounds`` rounds, the arms alternated within each round."""
        samples = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                samples[k].append(timed(fn, reps[k]))
        return {k: sorted(v)[len(v) // 2] for k, v in samples.items()}

    for group in GROUPS:
        # ---- FFT pair
        b, c = 1, 192
        arms, keep = {}, []
        for h, w in group:
            wf = w // 2 + 1
            prog = E.Program("rect_fft_bench", L.MATH_BF16X3)
            X = prog.buf("x", b, h, w, c); S = prog.buf("s", b, h, wf, 2 * c, gemm=True)
            Z = prog.buf("z", b, h, wf, 2 * c); O = prog.buf("o", b, h, w, c, gemm=True)
            prog.ops += [E.RfftOp(E.TV(X), E.TV(S)), E.IrfftOp(E.TV(Z), E.TV(X), E.TV(O))]
            ex = E.CudaExecutor(prog, dev)
            ex.storage[X.name].normal_()
            ex.storage[Z.name].normal_()
            keep.append(ex)
            arms[(h, w)] = (lambda ex=ex: [L.check(fn(*args, stream), name) for name, fn, args in ex.calls])
        reps = {}
        for k, fn in arms.items():                      # warm-up, and the pairs per sample
            fn()
            torch.cuda.synchronize()
            reps[k] = max(1, min(500, int(20.0 / max(timed(fn, 1), 1e-3))))
        fft = alternate(arms, reps)
        del keep, arms
        torch.cuda.empty_cache()
        # ---- generator program
        gms = {}
        if 64 * group[0][0] * group[0][1] <= GEN_MAX_PIXELS:
            arms, keep = {}, []
            for i, (h, w) in enumerate(group):
                img, mask = synthetic_image_mask(1, 8 * h, i, width=8 * w)
                x = generator_input(img, mask).to(dev)
                ex = E.get_executor(gen, "generator", (x,))
                gp = E.GraphedProgram(ex)
                gp({"x0": x})
                keep.append((ex, gp))
                arms[(h, w)] = gp.graph.replay
            torch.cuda.synchronize()
            gms = alternate(arms, {k: a.steps for k in arms})
            del keep, arms
            E.invalidate(gen)
            torch.cuda.empty_cache()
        base = group[0]
        rows = []
        for h, w in group:
            r = {"plane": f"{h}x{w}", "pixels": h * w, "fft_ms": round(fft[(h, w)], 4),
                 "fft_vs_first": round(fft[(h, w)] / fft[base], 3)}
            if gms:
                r.update(image=f"{8 * h}x{8 * w}", gen_ms=round(gms[(h, w)], 3),
                         gen_vs_first=round(gms[(h, w)] / gms[base], 3))
            rows.append(r)
            print(json.dumps(r), flush=True)
        info["groups"].append(rows)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "rect_planes_bench.json"), "w") as fh:
            json.dump(info, fh, indent=1)


if __name__ == "__main__":
    main()
