#!/usr/bin/env python
"""Refinement with the up-sampling tail over the whole image (``tail="whole"``) or in row bands (``tail="banded"``),
both with ``relu_masks="bits"``: big-lama (seeded weights), the reference's refiner settings (15 iterations, min_side
512, max_scales 3), one seeded image with a hole per case, BatchedRefiner(max_batch=1).  Per case and arm the records
of tools/refine_relu_bits_bench.py (step_ms, s_per_image, peak_gb, step_gb, per_image_gb_all_scales); the arms of a
case alternate (whole, banded, ... for --reps rounds); cases listed with --banded-only run banded alone (their whole-tail
step programs do not fit an 80 GB device, so the tool never builds them).  Also the card's name, power limit and SM
clocks read in the same run, and whether the two arms' results are bit-identical.  One JSON line per case, then all.

    python tools/refine_banded_bench.py [--cases 6000x4000@24000000] [--banded-only 8000x6000@48000000] [--reps 1]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402
from refine_relu_bits_bench import card, step_ms  # noqa: E402


def run_arm(gen, tail, kw, ims, mks, h, w):
    import time
    from lama_b200 import engine as E
    from lama_b200 import refine as R
    ref = R.BatchedRefiner(gen, 1, relu_masks="bits", tail=tail, **kw)
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
    rec["device_gb"] = round(torch.cuda.get_device_properties(0).total_memory / 1e9, 2)
    top = max(ref._lanes.items(), key=lambda kv: kv[0][3][0] * kv[0][3][1])[1]
    rec["step_ms"] = round(step_ms(top), 2) if top.graph is not None else None
    del ref, top
    torch.cuda.empty_cache()
    return rec, out[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="*", default=["6000x4000@24000000"])
    ap.add_argument("--banded-only", nargs="*", default=["8000x6000@48000000"])
    ap.add_argument("--reps", type=int, default=1)
    a = ap.parse_args()
    from lama_b200 import modules as M
    from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask
    assert torch.cuda.is_available(), "needs a CUDA device"
    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to("cuda:0")
    report = {"card": card(), "reps": a.reps, "cases": {}}
    for case in a.cases + a.banded_only:
        size, px = case.split("@")
        w, h = map(int, size.split("x"))
        kw = dict(modulo=8, n_iters=15, lr=0.002, min_side=512, max_scales=3, px_budget=int(float(px)))
        img, mask = synthetic_image_mask(1, h, 11, width=w)
        arms = ["banded"] if case in a.banded_only else ["whole", "banded"]
        rec = {"settings": kw, "runs": {arm: [] for arm in arms}}
        outs = {}
        for _ in range(a.reps):
            for arm in arms:
                r, outs[arm] = run_arm(gen, arm, kw, [img[0]], [mask[0]], h, w)
                rec["runs"][arm].append(r)
        rec["result_shape"] = list(outs["banded"].shape)
        rec["finite"] = bool(torch.isfinite(outs["banded"]).all())
        if "whole" in outs:
            rec["bit_identical"] = bool(torch.equal(outs["whole"], outs["banded"]))
        report["cases"][case] = rec
        print(json.dumps({case: rec}), flush=True)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
