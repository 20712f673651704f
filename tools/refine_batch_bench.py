#!/usr/bin/env python
"""Batched refinement timing: lama_b200.refine.BatchedRefiner against refine_predict (evaluation/refinement.py:228-314)
with the big-lama generator (seeded weights) and the reference's refiner settings (configs/prediction/default.yaml:
15 iterations, min_side 512, max_scales 3, px_budget 1.8 M).  8 seeded images with different holes per size (1024^2
and 1344^2; the latter is above px_budget and refined at 1341^2).  Arms, alternated in one process after one warm-up
pass each:
  refine_predict   the shipped loop, one image at a time;
  batched_b1       BatchedRefiner(max_batch=1);
  batched_b4/_b8   BatchedRefiner(max_batch=4 / 8), where the step programs fit the free device memory.
Reports images/s per arm, ms per replayed step (CUDA events over the captured step graph) per scale, the max / mean
output differences of every batched arm against refine_predict, and the card name and power limit.  One JSON line.

    python tools/refine_batch_bench.py [--sizes 1024 1344] [--images 8] [--reps 2]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from refine_bench import card  # noqa: E402


def step_ms(lane, n=10):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    lane.graph.replay()
    ev[0].record()
    for _ in range(n):
        lane.graph.replay()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1024, 1344])
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    from lama_b200 import modules as M
    from lama_b200 import refine as R
    from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = "cuda:0"
    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to(dev)
    kw = dict(modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3, px_budget=1800000)
    report = {"card": card(), "settings": kw, "images": a.images, "sizes": {}}
    for size in a.sizes:
        img, mask = synthetic_image_mask(a.images, size, 7)
        ims, mks = list(img), list(mask)
        refiners = {"batched_b1": R.BatchedRefiner(gen, 1, **kw)}
        per_image = refiners["batched_b1"].per_image_bytes(size, size)
        for b in (4, 8):
            if b * per_image <= 0.7 * torch.cuda.mem_get_info()[0]:
                refiners[f"batched_b{b}"] = R.BatchedRefiner(gen, b, **kw)

        def run(arm):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if arm == "refine_predict":
                out = [R.refine_predict(im[None], mk[None], gen, **kw)[0] for im, mk in zip(ims, mks)]
            else:
                out = refiners[arm].refine(ims, mks)
            torch.cuda.synchronize()
            return time.perf_counter() - t0, out

        # refine_predict and batched_b1 alternate with their programs and graphs kept (the steady state of a
        # directory run); each larger batch then runs on its own, its step programs dropped before the next one
        rec = report["sizes"].setdefault(str(size), {"ms_per_step": {}})
        outs, times = {}, {}
        groups = [["refine_predict", "batched_b1"]] + [[arm] for arm in refiners if arm != "batched_b1"]
        for group in groups:
            for arm in group:
                _, outs[arm] = run(arm)                   # warm-up: programs, graphs, library start-up
            for _ in range(a.reps):
                for arm in group:
                    dt, outs[arm] = run(arm)
                    times.setdefault(arm, []).append(dt)
            for arm in group:
                if arm != "refine_predict":
                    rec["ms_per_step"][arm] = {
                        f"{c[0]}x{c[1]}": round(step_ms(lane), 2)
                        for (_b, _sl, _sg, c), lane in sorted(refiners[arm]._lanes.items(), key=lambda kv: kv[0][3])
                        if lane.graph is not None}
                    refiners[arm]._lanes.clear()
                    refiners[arm]._size = None
                    torch.cuda.empty_cache()
        rec = report["sizes"].setdefault(str(size), {})
        rec["bytes_per_image_all_scales"] = per_image
        rec["images_per_s"] = {arm: [round(a.images / t, 3) for t in ts] for arm, ts in times.items()}
        rec["diff_vs_refine_predict"] = {}
        for arm in refiners:
            d = torch.stack([(x - y).abs().max() for x, y in zip(outs[arm], outs["refine_predict"])])
            m = torch.stack([(x - y).abs().mean() for x, y in zip(outs[arm], outs["refine_predict"])])
            rec["diff_vs_refine_predict"][arm] = {"max_abs": float(d.max()), "mean_abs": float(m.mean())}
        rec["batched_b1_vs_b4_equal"] = (all(torch.equal(x, y) for x, y in zip(outs["batched_b1"], outs["batched_b4"]))
                                         if "batched_b4" in outs else None)
        print(json.dumps({str(size): rec}), flush=True)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
