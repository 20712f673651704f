#!/usr/bin/env python
"""Where the time of one generator step goes, per library call, measured with torch.profiler (CUDA activities).

    python tools/step_breakdown.py [--batch 32] [--size 512] [--math bf16x3] [--out DIR] [--bn-sweep]

Runs one eager step of the big-lama generator (the program bench.py times) under the profiler.  Each call of the
program issues a known number of kernels (counted by the library's launch counter in a dry run), so the kernel
records, in launch order, map back to ``ex.calls[i][0]``.  Prints one table: kernel time per call name, its share of
the step's kernel time, launches and calls.  ``--bn-sweep`` also times the resblock local 3x3 contraction alone with
CUDA events at FFCB_TC_BN=64 and 128 (BN=64 moves 1.5x the operand bytes per FLOP of BN=128).
``--out DIR`` writes the table as DIR/step_breakdown.json.
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--math", default="bf16x3", choices=["fp32", "bf16x3"])
    ap.add_argument("--out", default=None)
    ap.add_argument("--bn-sweep", action="store_true")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    os.environ["LAMA_B200_MATH"] = args.math
    os.environ["LAMA_B200_STRICT"] = "1"
    from lama_b200 import _lib as L, engine as E, modules as M
    from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask, generator_input

    assert torch.cuda.is_available(), "step_breakdown.py needs a GPU"
    dev = torch.device("cuda:0")
    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to(dev)
    img, mask = synthetic_image_mask(args.batch, args.size, 0)
    x = generator_input(img, mask).to(dev)
    ex = E.get_executor(gen, "generator", (x,), math={"fp32": L.MATH_FP32, "bf16x3": L.MATH_BF16X3}[args.math])
    lib = L.get_lib()
    stream = torch.cuda.current_stream(dev)
    sc = stream.cuda_stream
    for _ in range(2):
        ex.run({"x0": x})
    torch.cuda.synchronize()

    def call(i):
        n, fn, a = ex.calls[i]
        rc = fn(*a, sc)
        if rc:
            L.check(rc, n)

    counts = []
    for i in range(len(ex.calls)):
        lib.ffcb_reset_launch_count()
        call(i)
        counts.append(int(lib.ffcb_launch_count()))
    torch.cuda.synchronize()

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(len(ex.calls)):
            call(i)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            trace = json.load(fh)
    kernels = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    if len(kernels) != sum(counts):
        sys.exit(f"{len(kernels)} kernel records, but the library counted {sum(counts)} launches")

    rows, k = {}, 0
    for i, c in enumerate(counts):
        name = ex.calls[i][0]
        r = rows.setdefault(name, {"ms": 0.0, "launches": 0, "calls": 0})
        r["ms"] += sum(e["dur"] for e in kernels[k:k + c]) / 1e3
        r["launches"] += c
        r["calls"] += 1
        k += c
    total = sum(r["ms"] for r in rows.values())
    span = (kernels[-1]["ts"] + kernels[-1]["dur"] - kernels[0]["ts"]) / 1e3
    table = sorted(rows.items(), key=lambda kv: -kv[1]["ms"])
    print(f"{'call':58s} {'ms':>9s} {'share':>7s} {'launches':>8s} {'calls':>6s}")
    for name, r in table:
        print(f"{name[:58]:58s} {r['ms']:9.3f} {100 * r['ms'] / total:6.1f}% {r['launches']:8d} {r['calls']:6d}")
    print(f"{'total kernel time':58s} {total:9.3f}   (first kernel start to last kernel end: {span:.3f} ms)")
    result = {"gpu": torch.cuda.get_device_name(dev), "batch": args.batch, "size": args.size, "math": args.math,
              "kernel_ms": total, "span_ms": span, "calls": {n: r for n, r in table}}

    if args.bn_sweep:
        idx = [i for i, (n, _f, _a) in enumerate(ex.calls) if n.startswith("ffcb_conv:convl2l+convg2l")]
        i0 = idx[len(idx) // 2]
        reps, sweep = 20, {}
        keep = os.environ.get("FFCB_TC_BN")
        try:
            for bn in ("128", "64", "128", "64"):          # alternated, each timed twice
                os.environ["FFCB_TC_BN"] = bn
                for _ in range(3):
                    call(i0)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(reps):
                    call(i0)
                e1.record(stream)
                torch.cuda.synchronize()
                sweep.setdefault(bn, []).append(e0.elapsed_time(e1) / reps)
        finally:
            if keep is None:
                os.environ.pop("FFCB_TC_BN", None)
            else:
                os.environ["FFCB_TC_BN"] = keep
        h = args.size // 8
        flops = 2.0 * args.batch * h * h * 128 * 9 * 512
        for bn, ts in sweep.items():
            print(f"local 3x3 contraction, FFCB_TC_BN={bn}: " + ", ".join(f"{t:.4f}" for t in ts) +
                  f" ms per launch ({flops / (min(ts) * 1e-3) / 1e12:.1f} TFLOP/s algorithmic)")
        result["local_contraction_ms_by_bn"] = sweep
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_breakdown.json"), "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
