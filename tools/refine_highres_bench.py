#!/usr/bin/env python
"""High-resolution refinement timing: big-lama (seeded weights) with the reference's refiner settings (15 iterations,
min_side 512, max_scales 3) on the two cases where a bottleneck axis exceeds 256 points:
  3440x1440 at the default px_budget (1.8 M: refined at 2073x868, 109x260 bottleneck),
  3840x2160 at px_budget 8.3 M (refined at full size, 270x480 bottleneck).
Arms, per size, one seeded image with a hole, in one process:
  native_b1   BatchedRefiner(max_batch=1): a step program per scale, graph-replayed (after one warm-up run that builds
              the programs and captures the graphs);
  fallback    LAMA_B200_NATIVE_GRAD=0: refine_predict with torch autograd through the blocks and the tail, the path
              these sizes took before the native programs covered them (an out-of-memory error is reported as such);
  step        ms per replayed step graph (rear forward, loss gradient, rear backward, Adam) of the largest scale.
Also: the output difference between the two arms, the pooled bytes of the native programs, the peak device memory
of each arm, and the card's name, power limit and SM clocks read in the same run.  One JSON line per size, then all.

    python tools/refine_highres_bench.py [--cases 3440x1440@1800000 3840x2160@8300000] [--reps 2]
                                         [--skip-fallback]"""
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


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out, torch.cuda.max_memory_allocated()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=["3440x1440@1800000", "3840x2160@8300000"])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--skip-fallback", action="store_true")
    a = ap.parse_args()
    from lama_b200 import modules as M
    from lama_b200 import refine as R
    from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask
    assert torch.cuda.is_available(), "needs a CUDA device"
    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to("cuda:0")
    report = {"card": card(), "cases": {}}
    for case in a.cases:
        size, px = case.split("@")
        w, h = map(int, size.split("x"))
        kw = dict(modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3, px_budget=int(float(px)))
        img, mask = synthetic_image_mask(1, h, 11, width=w)
        ims, mks = [img[0]], [mask[0]]
        ref = R.BatchedRefiner(gen, 1, **kw)
        rec = {"settings": kw, "scales": [list(c) for _, _, c in ref.scale_shapes(h, w)],
               "bottleneck": list(ref.scale_shapes(h, w)[-1][0][2:]), "native": ref.native_ok(h, w),
               "bytes_per_image_all_scales": ref.per_image_bytes(h, w)}
        timed(lambda: ref.refine(ims, mks))                         # warm-up: programs, graphs
        runs = [timed(lambda: ref.refine(ims, mks)) for _ in range(a.reps)]
        rec["native_b1_s"] = [round(t, 3) for t, _, _ in runs]
        rec["native_b1_peak_gb"] = round(runs[-1][2] / 1e9, 2)
        native_out = runs[-1][1][0]
        top = max(ref._lanes.items(), key=lambda kv: kv[0][3][0] * kv[0][3][1])[1]
        rec["step_ms_largest_scale"] = round(step_ms(top), 2) if top.graph is not None else None
        del ref, top, runs
        torch.cuda.empty_cache()
        if not a.skip_fallback:
            os.environ["LAMA_B200_NATIVE_GRAD"] = "0"
            try:
                dt, out, peak = timed(lambda: R.BatchedRefiner(gen, 1, **kw).refine(ims, mks))
                rec["fallback_s"] = round(dt, 3)
                rec["fallback_peak_gb"] = round(peak / 1e9, 2)
                d = (out[0] - native_out).abs()
                rec["native_vs_fallback"] = {"max_abs": float(d.max()), "mean_abs": float(d.mean())}
            except torch.OutOfMemoryError as e:
                rec["fallback_s"] = f"out of memory: {str(e).splitlines()[0][:160]}"
            finally:
                os.environ.pop("LAMA_B200_NATIVE_GRAD", None)
                torch.cuda.empty_cache()
        report["cases"][case] = rec
        print(json.dumps({case: rec}), flush=True)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
