#!/usr/bin/env python
"""LaMa-Regular generators (lama-regular, big-lama-regular; ``lama_b200.pix2pixhd.GlobalGenerator``) at 512x512, bs32.

    python tools/regular_bench.py [--steps 10] [--batch 32] [--size 512] [--out DIR]

Per model, seeded weights (gain 1.0), synthetic images and masks:
  * graph_img_s     — the native generator program (bf16x3 arm) as a CUDA-graph replay, CUDA events over ``--steps``;
  * pipeline_img_s  — ``GeneratorPipeline(u8=True)``: uint8 images + masks from pinned host memory to uint8 results,
                      copies overlapped with the replays, host clock over ``--steps`` batches ending in a synchronise;
  * eager_tf32_img_s / eager_fp32_img_s — torch eager on the same layers (``model.model``, cuDNN, benchmark mode) with
                      TF32 on and off;
  * launches        — kernel launches of one program replay (counted by the library);
  * conv512_ms / conv512_tflops — the median per-launch time of the 512 -> 512 3x3 block contractions (each call of
                      the program issued alone 20 times, CUDA events) and its algorithmic rate, 2*B*H*W*512*512*9
                      FLOP per launch (618.5 GFLOP at bs32 512x512);
  * bf16x3_vs_fp32  — max-abs difference between the outputs of the two arithmetic arms on the same batch.
The card's name, power limit and maximum SM clock are read in the same run.  Nothing is written outside ``--out``.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, steps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def bench_model(name, kw, a, dev):
    import numpy as np
    import torch
    from lama_b200 import _lib as L
    from lama_b200 import engine as E
    from lama_b200 import pix2pixhd as PX
    from lama_b200.serving import GeneratorPipeline
    from lama_b200.testing import generator_input, seeded_parameters_, synthetic_image_mask

    b, s = a.batch, a.size
    g = seeded_parameters_(PX.GlobalGenerator(**kw).eval(), 0, gain=1.0).to(dev)
    img, mask = synthetic_image_mask(b, s, 0)
    x = generator_input(img, mask).to(dev)
    r = {"model": name, "batch": b, "size": s}
    with torch.no_grad():
        ex = E.get_executor(g, "generator", (x,), math=L.MATH_BF16X3)
        ex.run({"x0": x})
        r["launches"] = ex.launches_per_run
        r["storage_gb"] = round(ex.storage_bytes / 1e9, 2)
        y_tc = ex.outputs["y0"].clone()
        graph = E.GraphedProgram(ex)
        graph({"x0": x})
        ms = timed(graph.graph.replay, a.steps)
        r["graph_ms"], r["graph_img_s"] = round(ms, 2), round(b * 1e3 / ms, 1)
        # the 512 -> 512 block contractions, each call alone
        stream = torch.cuda.current_stream().cuda_stream
        per = []
        for nm, fn, args in ex.calls:
            if nm.startswith("ffcb_conv:block"):
                fn(*args, stream)
                per.append(timed(lambda: fn(*args, stream), 20))
        med = statistics.median(per)
        flop = 2.0 * b * (s // 8) ** 2 * 512 * 512 * 9
        r["conv512_ms"], r["conv512_tflops"], r["conv512_gflop"] = round(med, 3), round(flop / med / 1e9, 1), \
            round(flop / 1e9, 1)
        r["conv512_share_of_step"] = round(med * len(per) / ms, 3)
        del graph
        E.invalidate(g)
        torch.cuda.empty_cache()
        ex32 = E.get_executor(g, "generator", (x,), math=L.MATH_FP32)
        y32 = ex32.run({"x0": x})["y0"]
        r["bf16x3_vs_fp32"] = float((y_tc - y32).abs().max())
        del ex32, y32
        E.invalidate(g)
        torch.cuda.empty_cache()

    # predict path: uint8 in / out through the overlapped pipeline
    rng = np.random.default_rng(0)
    pipe = GeneratorPipeline(g, b, s, s, u8=True)
    im = torch.from_numpy(rng.integers(0, 256, (b, s, s, 3), dtype=np.uint8)).pin_memory()
    mk = torch.from_numpy(((rng.random((b, s, s)) < 0.2) * 255).astype(np.uint8)).pin_memory()
    for _ in range(3):
        pipe.result(pipe.submit(im, mk))
    torch.cuda.synchronize()
    t = time.perf_counter()
    tickets = [pipe.submit(im, mk) for _ in range(a.steps)]
    pipe.result(tickets[-1])
    pipe.drain()
    r["pipeline_img_s"] = round(b * a.steps / (time.perf_counter() - t), 1)
    r["pipeline_launches"] = pipe.launches_per_batch
    E.drop_executor(pipe.ex)
    del pipe
    E.invalidate(g)
    torch.cuda.empty_cache()

    # torch eager, same layers
    torch.backends.cudnn.benchmark = True
    with torch.no_grad():
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            for _ in range(3):
                g.model(x)
            ms = timed(lambda: g.model(x), a.steps)
            r["eager_tf32_img_s" if tf32 else "eager_fp32_img_s"] = round(b * 1e3 / ms, 1)
    torch.backends.cudnn.allow_tf32 = True
    del g, x
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    os.environ["LAMA_B200_STRICT"] = "1"
    from lama_b200.testing import BIG_LAMA_REGULAR_KWARGS, LAMA_REGULAR_KWARGS

    assert torch.cuda.is_available(), "regular_bench.py needs a GPU"
    dev = torch.device("cuda:0")
    info = {"card": card(), "torch": torch.__version__, "models": []}
    print("card (name, power limit, max SM clock):", info["card"], flush=True)
    for name, kw in (("lama-regular", LAMA_REGULAR_KWARGS), ("big-lama-regular", BIG_LAMA_REGULAR_KWARGS)):
        r = bench_model(name, kw, a, dev)
        info["models"].append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "regular_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
