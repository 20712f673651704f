"""FFT microbenchmark (CUDA events on the launch stream, warm, inputs larger than... see below):
  * the FourierUnit shape of the headline workload (B=32, C=192, 64x64 planes): the plane kernels against the
    two-pass kernels (FFCB_FFT_TWO_PASS), forward and inverse apart;
  * planes without a compile-time plan (row f2): direct DFT vs runtime mixed-radix Stockham.
Run on the GPU box:  python tools/fft_microbench.py  -> one JSON line per configuration."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lama_b200 import _lib as L          # noqa: E402
from lama_b200 import engine as E        # noqa: E402

KNOBS = ("FFCB_FFT_MIXED_RADIX", "FFCB_FFT_TWO_PASS")


def time_ops(b, c, h, w, env, which, reps=10, spec_fmt_split=True, warm=3):
    for k in KNOBS:
        os.environ.pop(k, None)
    os.environ.update(env)
    wf = w // 2 + 1
    # same formats as the FourierUnit of the generator program: real planes float32, forward spectrum split bf16
    # (GEMM operand), post-GEMM spectrum float32, inverse output split bf16 (operand of conv2)
    prog = E.Program("fft_bench", L.MATH_BF16X3)
    X = prog.buf("x", b, h, w, c)
    S = prog.buf("s", b, h, wf, 2 * c, gemm=spec_fmt_split)
    Z = prog.buf("z", b, h, wf, 2 * c)
    O = prog.buf("o", b, h, w, c, gemm=spec_fmt_split)
    if which == "fwd":
        prog.ops += [E.RfftOp(E.TV(X), E.TV(S))]
        alg = 4 * b * h * w * c + 4 * b * h * wf * 2 * c
    else:
        prog.ops += [E.IrfftOp(E.TV(Z), E.TV(X), E.TV(O))]
        alg = 4 * b * h * wf * 2 * c + 2 * 4 * b * h * w * c
    ex = E.CudaExecutor(prog, torch.device("cuda:0"))
    ex.storage[X.name].normal_()
    ex.storage[Z.name].normal_()
    for _ in range(warm):
        ex.run({})
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        ex.run({})
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return {"op": which, "plane": f"{h}x{w}", "B": b, "C": c, "env": env, "us": round(ms * 1e3, 1),
            "GBps_in_plus_out": round(alg / ms / 1e6, 1), "launches": ex.launches_per_run}


def time_fu_chain(b, c, h, w, planar, reps=20, warm=3, flush_mb=0):
    """rfft2 -> spectral 1x1 GEMM (+BN+ReLU) -> irfft2 (+residual) with the generator program's formats, each op timed
    alone and the chain as a whole; planar: channel-group planar layouts + second-generation plane kernels."""
    from lama_b200 import packing as P
    wf = w // 2 + 1
    prog = E.Program("fu_chain", L.MATH_BF16X3)
    T = prog.buf("t", b, h, w, c, cg=4 if planar else 0)
    S = prog.buf("s", b, h, wf, 2 * c, gemm=True, cg=8 if planar else 0)
    Z = prog.buf("z", b, h, wf, 2 * c, cg=8 if planar else 0)
    U = prog.buf("u", b, h, w, c, gemm=True, cg=8 if planar else 0)
    g = torch.Generator().manual_seed(0)
    pk = P.pack_conv([(torch.randn(2 * c, 2 * c, 1, 1, generator=g) * 0.05, 0, 0, 0)], torch.ones(2 * c).double(),
                     torch.zeros(2 * c).double(), act=L.ACT_RELU)
    prog.ops += [E.RfftOp(E.TV(T), E.TV(S)), E.ConvOp(pk, [E.TV(S), None], E.TV(Z), tag="fu.gemm"),
                 E.IrfftOp(E.TV(Z), E.TV(T), E.TV(U))]
    ex = E.CudaExecutor(prog, torch.device("cuda:0"))
    ex.storage[T.name].normal_()
    flush = torch.empty(flush_mb << 20, dtype=torch.uint8, device="cuda:0") if flush_mb else None
    stream = torch.cuda.current_stream().cuda_stream

    def run(idx):
        for i in idx:
            n, fn, a = ex.calls[i]
            rc = fn(*a, stream)
            assert rc == 0, (n, L.get_lib().ffcb_last_error())
    out = {"planar": planar, "B": b, "C": c, "plane": f"{h}x{w}", "l2": f"flush {flush_mb} MB" if flush_mb else "warm"}
    for name, idx in (("fwd_us", [0]), ("gemm_us", [1]), ("inv_us", [2]), ("chain_us", [0, 1, 2])):
        for _ in range(warm):
            run(idx)
        ts = []
        for _ in range(reps):
            if flush is not None:
                flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); run(idx); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        ts.sort()
        out[name] = round(ts[len(ts) // 2], 1)
    alg = 4.0 * b * h * w * 2 * c + 4.0 * (2 * c) * (2 * c) + 8.0 * 2 * c
    out["fu_algorithmic_GBps"] = round(alg / out["chain_us"] / 1e3, 1)
    return out


if __name__ == "__main__":
    fu = (32, 192, 64, 64)
    if "--chain" in sys.argv:            # FourierUnit chain of the headline workload: round-1 layout vs planar, warm / cold L2
        for planar in (False, True):
            for flush_mb in (0, 512):
                print(json.dumps(time_fu_chain(*fu, planar, flush_mb=flush_mb)), flush=True)
        sys.exit(0)
    if "--l2-hints" in sys.argv:         # planar chain with and without the L2 residency hints
        for hints in ("1", "0"):
            os.environ["FFCB_L2_HINTS"] = hints
            print(json.dumps({"FFCB_L2_HINTS": hints, **time_fu_chain(*fu, True, reps=10)}), flush=True)
        sys.exit(0)
    if "--chain-planar-once" in sys.argv:   # one pass of the planar chain (for ncu captures)
        print(json.dumps(time_fu_chain(*fu, True, reps=1, warm=1)), flush=True)
        sys.exit(0)
    if "--fu-only" in sys.argv:          # the shipped configuration only (for an ncu capture)
        print(json.dumps(time_ops(*fu, {}, "fwd", reps=1, warm=0)), flush=True)
        print(json.dumps(time_ops(*fu, {}, "inv", reps=1, warm=0)), flush=True)
        sys.exit(0)
    for which in ("fwd", "inv"):
        for env in [{}, {"FFCB_FFT_TWO_PASS": "1"}]:
            print(json.dumps(time_ops(*fu, env, which)), flush=True)
    for (h, w) in [(96, 128), (125, 188), (135, 240)]:
        for mixed in ("0", "1"):
            for which in ("fwd", "inv"):
                print(json.dumps(time_ops(8, 192, h, w, {"FFCB_FFT_MIXED_RADIX": mixed}, which, reps=5)), flush=True)
