#!/usr/bin/env python
"""Refinement with the backward's ReLU masks kept as values (default) or as bits (``relu_masks="bits"``): big-lama
(seeded weights), the reference's refiner settings (15 iterations, min_side 512, max_scales 3), one seeded image with a
hole per case, BatchedRefiner(max_batch=1).  Per case and arm:
  step_ms     one replayed step graph (rear forward, loss gradient, rear backward, Adam) of the largest scale, CUDA
              events, mean of 10 replays;
  s_per_image wall time of one refine() after a warm-up run that builds the programs and captures the graphs;
  peak_gb     torch.cuda.max_memory_allocated over that run;
  step_gb     program_storage_bytes of the largest scale's step program.
The arms of a case alternate (values, bits, values, bits, ... for --reps rounds); cases listed with --bits-only run
bits alone (their values programs do not fit an 80 GB device).  Also the card's name, power limit and SM clocks read
in the same run, and whether the two arms' results are bit-identical.  One JSON line per case, then all.

    python tools/refine_relu_bits_bench.py [--cases 1024x1024@1800000 3440x1440@1800000 3840x2160@8300000]
                                           [--bits-only 4000x3000@12000000 6000x4000@24000000] [--reps 1]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({type(e).__name__})"


def step_ms(lane, n=10):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    lane.graph.replay()
    ev[0].record()
    for _ in range(n):
        lane.graph.replay()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / n


def run_arm(gen, relu_masks, kw, ims, mks, h, w):
    from lama_b200 import engine as E
    from lama_b200 import refine as R
    ref = R.BatchedRefiner(gen, 1, relu_masks=relu_masks, **kw)
    sl, sg, crop = ref.scale_shapes(h, w)[-1]
    with torch.no_grad():
        step = E.build_module_program(gen, ref.program_kind(len(ref.scale_shapes(h, w)) - 1, crop), (sl, sg),
                                      E.default_math())
    rec = {"step_gb": round(E.program_storage_bytes(step) / 1e9, 2),
           "per_image_gb_all_scales": round(ref.per_image_bytes(h, w) / 1e9, 2)}
    del step
    ref.refine(ims, mks)                                             # warm-up: programs, graphs
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = ref.refine(ims, mks)
    torch.cuda.synchronize()
    rec["s_per_image"] = round(time.perf_counter() - t0, 3)
    rec["peak_gb"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    top = max(ref._lanes.items(), key=lambda kv: kv[0][3][0] * kv[0][3][1])[1]
    rec["step_ms"] = round(step_ms(top), 2) if top.graph is not None else None
    del ref, top
    torch.cuda.empty_cache()
    return rec, out[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="*", default=["1024x1024@1800000", "3440x1440@1800000", "3840x2160@8300000"])
    ap.add_argument("--bits-only", nargs="*", default=["4000x3000@12000000", "6000x4000@24000000"])
    ap.add_argument("--reps", type=int, default=1)
    a = ap.parse_args()
    from lama_b200 import modules as M
    from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask
    assert torch.cuda.is_available(), "needs a CUDA device"
    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to("cuda:0")
    report = {"card": card(), "reps": a.reps, "cases": {}}
    for case in a.cases + a.bits_only:
        size, px = case.split("@")
        w, h = map(int, size.split("x"))
        kw = dict(modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3, px_budget=int(float(px)))
        img, mask = synthetic_image_mask(1, h, 11, width=w)
        ims, mks = [img[0]], [mask[0]]
        arms = ["bits"] if case in a.bits_only else ["values", "bits"]
        rec = {"settings": kw, "runs": {arm: [] for arm in arms}}
        outs = {}
        for _ in range(a.reps):
            for arm in arms:
                r, outs[arm] = run_arm(gen, arm, kw, ims, mks, h, w)
                rec["runs"][arm].append(r)
        rec["result_shape"] = list(outs["bits"].shape)
        rec["finite"] = bool(torch.isfinite(outs["bits"]).all())
        if "values" in outs:
            rec["bit_identical"] = bool(torch.equal(outs["values"], outs["bits"]))
        report["cases"][case] = rec
        print(json.dumps({case: rec}), flush=True)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
