#!/usr/bin/env python
"""High-resolution inference of big-lama at batch 1: the native path against the reference's operator sequence under
torch eager, on 4K-class photos whose bottleneck planes take the 8-channel FFT kernels (448..1024-point axes).

    python tools/highres_bench.py [--sizes 2160x3840,3000x4000,4096x4096,2160x3832,2160x4016] [--steps 10] [--out DIR]

Per size (the image sides are multiples of 8, so the generator and the predict driver see the same plane):
  * graph_ms      — CUDA-graph replay of the generator program (float in / out), CUDA events over ``--steps`` replays;
  * predict_ms    — ms per image through lama_b200.predict.BatchedInpainter (uint8 in and out, copies included),
                    host clock around ``inpaint`` of ``--images`` images (it returns after the last D2H);
  * eager_tf32_ms / eager_fp32_ms — oracle/ffc_torch_cpu.py's operator sequence (the reference's ffc.py) run by
                    torch eager on the same GPU (cuFFT / cuDNN), cudnn.allow_tf32 on / off;
  * fft_share     — share of the FFT kernels in the kernel time of one eager program step (every library call issued
                    once), from torch.profiler CUDA activities;
  * max_abs       — (first size only) max |native - CPU fp32 oracle| on the sigmoid output.
2160x3832 has a prime bottleneck width (479) and 2160x4016 a width of 502 = 2 * 251 (height 270): both run their rows
as Bluestein chirp-z transforms (1024-point convolutions).  The card's name and power limit are read
in the same run and printed with the numbers.  Nothing is written outside ``--out``.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def fft_share(ex):
    """(FFT kernels' share of the kernel time, kernel ms) of one eager step of the program: every library call issued
    once under torch.profiler; the FFT kernels are those with "fft" in their name (rfft_rows_kernel, fft_cols_*_kernel,
    irfft_rows_kernel and the 64x64 plane kernels)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from lama_b200 import _lib as L
    sc = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for n, fn, a in ex.calls:
            L.check(fn(*a, sc), n)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            trace = json.load(fh)
    kernels = [e for e in trace["traceEvents"] if e.get("cat") == "kernel"]
    total = sum(e["dur"] for e in kernels) / 1e3
    fft = sum(e["dur"] for e in kernels if "fft" in e["name"]) / 1e3
    return fft / total, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="2160x3840,3000x4000,4096x4096,2160x3832,2160x4016")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--eager-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import numpy as np
    import torch
    os.environ["LAMA_B200_STRICT"] = "1"
    from lama_b200 import engine as E, modules as M
    from lama_b200.predict import BatchedInpainter
    from lama_b200.testing import BIG_LAMA_KWARGS, generator_input, seeded_parameters_, synthetic_image_mask
    from oracle import ffc_torch_cpu as otc

    assert torch.cuda.is_available(), "highres_bench.py needs a GPU"
    dev = torch.device("cuda:0")
    info = {"card": card(), "torch": torch.__version__, "math": os.environ.get("LAMA_B200_MATH", "bf16x3"),
            "sizes": {}}
    print("card (name, power limit, max SM clock):", info["card"])
    g = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0)
    sd_cpu = {k: v.clone() for k, v in g.state_dict().items()}
    g = g.to(dev)
    for si, s in enumerate(a.sizes.split(",")):
        h, w = map(int, s.split("x"))
        r = {}
        img, mask = synthetic_image_mask(1, h, si, width=w)
        x_cpu = generator_input(img, mask)
        x = x_cpu.to(dev)
        # ---- native: graph replay of the generator program
        ex = E.get_executor(g, "generator", (x,))
        gp = E.GraphedProgram(ex)
        gp({"x0": x})
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            gp.graph.replay()
        e1.record()
        torch.cuda.synchronize()
        r["graph_ms"] = e0.elapsed_time(e1) / a.steps
        y = ex.outputs["y0"].cpu()
        r["fft_share"], r["eager_step_kernel_ms"] = fft_share(ex)
        del gp, ex
        E.invalidate(g)
        torch.cuda.empty_cache()
        # ---- native: the uint8 predict driver
        rng = np.random.default_rng(si)
        items = [(rng.integers(0, 256, (h, w, 3), dtype=np.uint8),
                  (rng.random((h, w)) < 0.2).astype(np.uint8) * 255) for _ in range(a.images)]
        inp = BatchedInpainter(g, max_batch=1)
        inp.inpaint(items[:1])
        t0 = time.perf_counter()
        inp.inpaint(items)
        r["predict_ms"] = (time.perf_counter() - t0) * 1e3 / a.images
        del inp
        E.invalidate(g)
        torch.cuda.empty_cache()
        # ---- reference operator sequence, torch eager on this GPU
        sd = {k: v.to(dev) for k, v in sd_cpu.items()}
        keep = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        try:
            for mode, tf32 in (("tf32", True), ("fp32", False)):
                torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32, False
                with torch.no_grad():
                    otc.ffc_resnet_generator(x, sd, **BIG_LAMA_KWARGS)
                    torch.cuda.synchronize()
                    e0.record()
                    for _ in range(a.eager_steps):
                        otc.ffc_resnet_generator(x, sd, **BIG_LAMA_KWARGS)
                    e1.record()
                    torch.cuda.synchronize()
                r[f"eager_{mode}_ms"] = e0.elapsed_time(e1) / a.eager_steps
                torch.cuda.empty_cache()
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = keep
        del sd, x
        torch.cuda.empty_cache()
        if si == 0:
            with torch.no_grad():
                ref = otc.ffc_resnet_generator(x_cpu, sd_cpu, **BIG_LAMA_KWARGS)
            r["max_abs"] = float((y - ref).abs().max())
        r["speedup_vs_eager_tf32"] = r["eager_tf32_ms"] / r["graph_ms"]
        info["sizes"][s] = r
        print(f"{s}: " + ", ".join(f"{k} {v:.4g}" for k, v in r.items()), flush=True)
    print(json.dumps(info))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "highres_bench.json"), "w") as fh:
            json.dump(info, fh, indent=1)


if __name__ == "__main__":
    main()
