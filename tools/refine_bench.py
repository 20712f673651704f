#!/usr/bin/env python
"""Row f3 timing: lama_b200.refine.refine_predict (evaluation/refinement.py:228-314) on one image with the big-lama
generator.  Three arms, alternated in one process:
  native_rear   refine_predict as shipped: the generator's rear (blocks + tail + head) as one native forward +
                input-gradient program per scale;
  per_module    image_mask_pyramid + infer_scale driven by the module slice generator.model[first_block:] — native
                per-block gradients, the up-sampling tail and head on torch autograd (cuDNN, TF32 as torch defaults);
  torch         LAMA_B200_NATIVE_GRAD=0: torch autograd throughout (TF32 as torch defaults).
Also times one rear forward + backward per scale shape (native rear vs module slice) with CUDA events, and prints the
card name and power limit beside the numbers.  Prints one JSON line.

    python tools/refine_bench.py [--size 1024] [--iters 15] [--reps 2]"""
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({type(e).__name__})"
    return q


def refine_with_modules(R, img, mask, gen, *, modulo, n_iters, lr, min_side, max_scales, px_budget):
    """refine_predict's scale loop with rear = the module slice (no native rear program)."""
    dev = next(gen.parameters()).device
    for p in gen.parameters():
        p.requires_grad_(False)
    front, rear = R.split_generator(gen.model)
    images, masks = R.image_mask_pyramid(img, mask, min_side, max_scales, px_budget)
    result = None
    for im, mk in zip(images, masks):
        orig = tuple(im.shape[2:])
        im_p, mk_p = R._pad_to_modulo(im, modulo).to(dev), R._pad_to_modulo(mk, modulo).to(dev)
        mk_p = (mk_p >= 1e-8).to(mk_p.dtype)
        result = R.infer_scale(im_p, mk_p, front, rear, result, orig, n_iters, lr)[:, :, :orig[0], :orig[1]]
    return result.cpu()


def scale_shapes(R, img, mask, gen, kw):
    """(z1, z2) of every pyramid scale (front under no_grad on the padded masked image)."""
    dev = next(gen.parameters()).device
    front, _ = R.split_generator(gen.model)
    images, masks = R.image_mask_pyramid(img, mask, kw["min_side"], kw["max_scales"], kw["px_budget"])
    out = []
    for im, mk in zip(images, masks):
        im_p, mk_p = R._pad_to_modulo(im, kw["modulo"]).to(dev), R._pad_to_modulo(mk, kw["modulo"]).to(dev)
        with torch.no_grad():
            out.append(front(torch.cat([im_p * (1 - mk_p), mk_p], dim=1)))
    return out


def time_rear(fn, z1, z2, reps=10):
    """ms per rear forward + backward (CUDA events, after two warm-up steps)."""
    a, b = z1.detach().clone().requires_grad_(True), z2.detach().clone().requires_grad_(True)

    def step():
        y = fn(a, b)
        y.backward(torch.ones_like(y))
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    from lama_b200 import engine as E, modules as M, refine as R
    from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_
    dev = torch.device("cuda:0")
    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to(dev)
    for p in gen.parameters():
        p.requires_grad_(False)
    g = torch.Generator().manual_seed(0)
    S = args.size
    img = torch.rand(1, 3, S, S, generator=g)
    mask = torch.zeros(1, 1, S, S)
    mask[..., S // 4: S // 2, S // 3: 2 * S // 3] = 1
    kw = dict(modulo=8, n_iters=args.iters, lr=0.002, min_side=512, max_scales=3, px_budget=1800000)
    os.environ["LAMA_B200_STRICT"] = "0"

    def run(arm, **over):
        os.environ["LAMA_B200_NATIVE_GRAD"] = "0" if arm == "torch" else "1"
        k = dict(kw, **over)
        if arm == "per_module":
            return refine_with_modules(R, img, mask, gen, **k)
        return R.refine_predict(img, mask, gen, **k)

    arms = ("native_rear", "per_module", "torch")
    out = {"card": card()}
    for arm in arms:
        run(arm, n_iters=2)                                   # warm-up: programs, cuDNN plans
    times = {a: [] for a in arms}
    res = {}
    for _ in range(args.reps):
        for arm in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res[arm] = run(arm)
            torch.cuda.synchronize()
            times[arm].append(time.perf_counter() - t0)
    for arm in arms:
        out[arm + "_s"] = [round(t, 3) for t in times[arm]]

    def diff(a, b):
        d = (res[a] - res[b]).abs()
        hole = torch.nn.functional.interpolate(mask, size=d.shape[2:], mode="nearest").expand_as(d) > 0   # px_budget
        return {"max": float(d.max()), "mean": float(d.mean()), "mean_in_hole": float(d[hole].mean())}
    out["native_rear_vs_per_module"] = diff("native_rear", "per_module")
    out["native_rear_vs_torch"] = diff("native_rear", "torch")
    os.environ["LAMA_B200_NATIVE_GRAD"] = "1"
    _, rear_mods = R.split_generator(gen.model)
    per_shape = []
    for z1, z2 in scale_shapes(R, img, mask, gen, kw):
        rec = {"z_hw": list(z1.shape[2:]), "native_supported": E.rear_grad_supported(gen, z1.shape, z2.shape)}
        if rec["native_supported"]:
            rec["native_rear_ms"] = round(time_rear(lambda a, b: E.generator_rear_with_input_grad(gen, a, b), z1, z2), 2)
        rec["per_module_ms"] = round(time_rear(lambda a, b: rear_mods((a, b)), z1, z2), 2)
        per_shape.append(rec)
    out["rear_fwd_bwd_per_scale"] = per_shape
    out.update(image=[S, S], n_iters=args.iters, scales="pyramid of refinement.py:176-226 (min_side 512)",
               timer="host wall clock around each refinement incl. its final .cpu(); rear: CUDA events")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
