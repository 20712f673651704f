#!/usr/bin/env python
"""bench.py — images/sec of the big-lama FFCResNetGenerator @512x512 bs32 per GPU (BASELINE.json
metric), through the drop-in modules -> libffc_b200.so.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--math fp32|bf16x3]
                    [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

One "step" = one forward pass of the generator over one batch of 32 synthetic 512x512 (image, mask)
pairs per GPU (weak scaling: every rank runs its own shard, no data-path collective; NCCL is used
only for the barrier and the max-over-ranks of the device time).

Reported on one JSON line by rank 0:
  value        images/s, inputs resident in HBM, CUDA-graph replay of the whole program, CUDA events
  e2e          same metric through the public module call with HOST (pinned) inputs: H2D of the
               (B,4,512,512) float input and D2H of the (B,3,512,512) result inside the timed region
  roofline     dominant kernel (the resblock local 3x3 contraction) vs the measured tensor peak, plus
               "fourier_unit": the FU sub-path (rfft2 -> pointwise GEMM -> irfft2) vs the HBM roofline
               with SURVEY.md §8(d)'s algorithmic bytes
  cpu_baseline the oracle's torch-CPU port (the reference's own operator sequence) on this box's host cores
`--impl reference` times that CPU port alone (bounded sample per step) as the reference arm.
`--dump-outputs DIR` writes what the last timed step computed (the generator output, rank 0) as DIR/<name>.npy in
float32, a fixed sample of it when the whole would exceed 64 MB; inputs and weights are seeded, so two builds run
with the same arguments can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

BATCH_PER_GPU = 32
SIZE = 512
METRIC = "images/sec FFCResNetGenerator @512x512 bs32"


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(p):
        with open(p) as fh:
            d = json.load(fh)
        return dict(hbm_gbs=d["hbm_gbs"], bf16_burst=d["bf16_tflops"], bf16_sustained=d["bf16_tflops_sustained"],
                    source="measured (MEASURED_PEAKS.json)")
    # NVIDIA H100 SXM data sheet (700 W): HBM3 3.35 TB/s, dense BF16 989 TFLOP/s — a denominator, not a reached rate
    return dict(hbm_gbs=3350.0, bf16_burst=989.0, bf16_sustained=989.0, source="fallback (H100 SXM data sheet)")


DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(directory, outputs):
    """Write {name: tensor} as <directory>/<name>.npy in float32.  An output larger than the 64 MB budget is
    replaced by a fixed sample of its elements (seed 0, sorted flat indices, <name>_sample.npy)."""
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    budget = DUMP_LIMIT_BYTES // max(1, len(outputs))
    for name, t in sorted(outputs.items()):
        a = t.detach().float().cpu().numpy()
        if a.nbytes > budget - 4096:                  # room for the .npy header
            n = (budget - 4096) // 4
            idx = np.sort(np.random.default_rng(0).choice(a.size, size=n, replace=False))
            a, name = a.reshape(-1)[idx], name + "_sample"
        np.save(os.path.join(directory, name + ".npy"), np.ascontiguousarray(a, dtype=np.float32))


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region (profiling recipe)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._pump, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None
        return self

    def _pump(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def __exit__(self, *a):
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:
                self.proc.kill()

    def summary(self):
        sm = sorted(int(float(r[1])) for r in self.rows if len(r) >= 8 and r[1].replace(".", "").isdigit())
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        mx = max(int(float(r[2])) for r in self.rows if len(r) >= 8)
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) >= 8 and r[4 + i].lower().startswith("active")
                                                         for r in self.rows)]
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": mx, "reasons": reasons, "samples": len(sm)}


def cpu_reference_step(images, threads=None):
    """One bounded sample of the workload on the host: the oracle's torch-CPU port of the reference
    generator on `images` 512x512 inputs.  Returns (seconds, n_images)."""
    import torch
    from oracle import ffc_torch_cpu as otc
    from lama_b200.testing import BIG_LAMA_KWARGS
    st = cpu_reference_step.state
    x = st["x"][:images]
    t0 = time.perf_counter()
    with torch.no_grad():
        otc.ffc_resnet_generator(x, st["sd"], **BIG_LAMA_KWARGS)
    return time.perf_counter() - t0, images


CPU_THREADS = int(os.environ.get("LAMA_B200_CPU_THREADS", "16"))
CPU_IMAGES_PER_STEP = 4


def _cpu_setup():
    """Build the CPU model once.  Thread count: FIXED at min(16, available) in both arms (stated in the JSON line).
    Round 1 calibrated it per run and the two arms disagreed (8 vs 16 threads on the same box); the box reports 128
    logical CPUs but oversubscribed intra-op pools are far slower than a right-sized one, so "all the host threads it
    can use" is 16 here."""
    import torch
    from lama_b200 import modules as M
    from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask, generator_input
    try:
        avail = len(os.sched_getaffinity(0))
    except AttributeError:
        avail = os.cpu_count() or 1
    n = max(1, min(CPU_THREADS, avail))
    torch.set_num_threads(n)
    g = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0)
    sd = {k: v for k, v in g.state_dict().items()}
    img, mask = synthetic_image_mask(CPU_IMAGES_PER_STEP, SIZE, 0)
    cpu_reference_step.state = {"sd": sd, "x": generator_input(img, mask)}
    return n


def torch_cuda_baseline(dev, B, S, steps=5, warmup=3):
    """The reference's own operator sequence (oracle/ffc_torch_cpu.py, bit-identical to ffc.py on CPU) run by torch
    EAGER on this GPU — cuFFT / cuDNN / ATen, the stack the reference uses on CUDA — with cudnn.allow_tf32 True (the
    torch default) and False (SURVEY.md §8d configs 1-3).  Baseline leg only: nothing of lama_b200 runs here.
    Returns {config: {"tf32": img/s or ms, "fp32": ...}}; timing: CUDA events, `warmup` + `steps` calls."""
    import torch
    from lama_b200 import modules as M
    from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask, generator_input
    from oracle import ffc_torch_cpu as otc
    g = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0)
    sd = {k: v.to(dev) for k, v in g.state_dict().items()}
    del g
    img, mask = synthetic_image_mask(B, S, 0)
    x = generator_input(img, mask).to(dev)
    h = S // 8
    gen = torch.Generator(device="cpu").manual_seed(0)
    xl = torch.randn(8, 128, h, h, generator=gen).to(dev)
    xg = torch.randn(8, 384, h, h, generator=gen).to(dev)
    t = torch.randn(B, 192, h, h, generator=gen).to(dev)
    x0 = torch.randn(1, 64, 256, 256, generator=gen).to(dev)
    blk = "model.10."
    fu = blk + "conv1.ffc.convg2g.fu."
    sd0 = {"conv_layer.weight": torch.randn(128, 128, 1, 1, generator=gen).to(dev) * 0.09,
           "bn.weight": torch.ones(128, device=dev), "bn.bias": torch.zeros(128, device=dev),
           "bn.running_mean": torch.zeros(128, device=dev), "bn.running_var": torch.ones(128, device=dev)}
    cases = {
        "generator_bs%d_%d" % (B, S): (lambda: otc.ffc_resnet_generator(x, sd, **BIG_LAMA_KWARGS), B, "images/s"),
        "resblock_bs8_%d" % S: (lambda: otc.ffc_resnet_block(xl, xg, sd, blk), None, "ms"),
        "fourier_unit_B%d_C192_%dx%d" % (B, h, h): (lambda: otc.fourier_unit(t, sd, fu), None, "ms"),
        "fourier_unit_1x64x256x256": (lambda: otc.fourier_unit(x0, sd0), None, "ms"),
    }
    out = {"stack": "torch %s eager (cuFFT/cuDNN/ATen), operator sequence of ffc.py (oracle/ffc_torch_cpu.py)" % torch.__version__}
    keep = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    try:
        for mode, tf32 in (("tf32", True), ("fp32", False)):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = False
            for name, (fn, imgs, unit) in cases.items():
                with torch.no_grad():
                    for _ in range(warmup):
                        fn()
                    torch.cuda.synchronize(dev)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(steps):
                        fn()
                    e1.record()
                    torch.cuda.synchronize(dev)
                ms = e0.elapsed_time(e1) / steps
                out.setdefault(name, {"unit": unit})[mode] = (imgs / (ms / 1e3)) if imgs else ms
                torch.cuda.empty_cache()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = keep
    # the same sub-path inputs through the drop-in modules (native programs), for the ours-vs-eager table
    try:
        blk_m = M.FFCResnetBlock(512, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                 activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75, enable_lfu=False)
        blk_m.load_state_dict({k[len(blk):]: v for k, v in sd.items() if k.startswith(blk)})
        blk_m = blk_m.eval().to(dev)
        fu_m = M.FourierUnit(192, 192)
        fu_m.load_state_dict({k[len(fu):]: v for k, v in sd.items() if k.startswith(fu)})
        fu_m = fu_m.eval().to(dev)
        fu0_m = M.FourierUnit(64, 64)
        fu0_m.load_state_dict(sd0)
        fu0_m = fu0_m.eval().to(dev)
        ours = {"resblock_bs8_%d" % S: lambda: blk_m((xl, xg)),
                "fourier_unit_B%d_C192_%dx%d" % (B, h, h): lambda: fu_m(t),
                "fourier_unit_1x64x256x256": lambda: fu0_m(x0)}
        for name, fn in ours.items():
            with torch.no_grad():
                for _ in range(warmup):
                    fn()
                torch.cuda.synchronize(dev)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(steps):
                    fn()
                e1.record()
                torch.cuda.synchronize(dev)
            out[name]["ours_module_call_ms"] = e0.elapsed_time(e1) / steps
            # same call in a serving loop that never touches the weights (LAMA_B200_TRUST_WEIGHTS=1: no per-call content
            # checksum of the weights, i.e. no host<->device round trip inside the call)
            os.environ["LAMA_B200_TRUST_WEIGHTS"] = "1"
            try:
                with torch.no_grad():
                    for _ in range(warmup):
                        fn()
                    torch.cuda.synchronize(dev)
                    e0.record()
                    for _ in range(steps):
                        fn()
                    e1.record()
                    torch.cuda.synchronize(dev)
                out[name]["ours_module_call_trusted_weights_ms"] = e0.elapsed_time(e1) / steps
            finally:
                os.environ.pop("LAMA_B200_TRUST_WEIGHTS", None)
        out["note_ours"] = ("ours_module_call_ms = the drop-in module called like the reference module (NCHW float in / out, "
                            "layout conversion + weight content checksum — one device->host scalar read — inside the "
                            "call); ..._trusted_weights_ms = same with LAMA_B200_TRUST_WEIGHTS=1")
    except Exception as ex_o:  # noqa: BLE001
        out["ours_error"] = f"{type(ex_o).__name__}: {ex_o}"[:300]
    return out


def run_reference(args, rank, world, out):
    """Reference arm: the reference's CPU path (oracle torch-CPU port; the reference tree itself cannot
    travel to the GPU box) on all host threads.  Rank 0 only."""
    if rank != 0:
        return
    cores = _cpu_setup()
    per_step = CPU_IMAGES_PER_STEP   # bounded sample of the bs32 step: one batch of 4 of its 32 images per step
    for _ in range(args.warmup):
        cpu_reference_step(per_step)
    t = 0.0
    for _ in range(args.steps):
        dt, _n = cpu_reference_step(per_step)
        t += dt
    v = per_step * args.steps / t
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": v, "unit": "images/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * t / args.steps, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "big-lama FFCResNetGenerator fwd, 512x512, seeded random weights",
                   "per_step_images": per_step, "device": "cpu", "threads": cores,
                   "sample": "each step = one batch of %d of the 32 images of the GPU arm's step" % per_step},
        "cpu_baseline": {"value": v, "unit": "images/s", "cores": cores, "kind": "port",
                         "sample": f"{per_step} images/step x {args.steps} steps, torch-CPU port of ffc.py (oracle/ffc_torch_cpu.py)"},
        "e2e": {"value": v, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }), file=out)
    out.flush()


def _claim_stdout():
    """The contract is ONE JSON line on stdout.  Libraries write there too (NCCL prints its version banner on
    init), so keep a private handle to the real stdout and point fd 1 at stderr for everything else."""
    sys.stdout.flush()
    real = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    sys.stdout = os.fdopen(os.dup(2), "w")
    return real


def main():
    out = _claim_stdout()
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--math", default=os.environ.get("LAMA_B200_MATH", "bf16x3"), choices=["fp32", "bf16x3"])
    ap.add_argument("--batch", type=int, default=BATCH_PER_GPU)
    ap.add_argument("--size", type=int, default=SIZE)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-fp32-arm", action="store_true", help="skip the CUDA-core fp32 reading of the same step")
    ap.add_argument("--no-torch-cuda-baseline", action="store_true",
                    help="skip the torch-eager (cuFFT/cuDNN) reading of the same operator sequence on this GPU")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the generator output of the last timed step as DIR/<name>.npy (float32, <= 64 MB)")
    ap.add_argument("--io", default=os.environ.get("LAMA_B200_BENCH_IO", "both"), choices=["f32", "both"],
                    help="both: also time the uint8 predict path (lama_b200.predict, SURVEY.md row f1) end to end")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference(args, rank, world, out)
        return

    import torch
    import torch.distributed as dist
    os.environ["LAMA_B200_MATH"] = args.math
    os.environ["LAMA_B200_STRICT"] = "1"
    from lama_b200 import _lib as L
    from lama_b200 import engine as E
    from lama_b200 import modules as M
    from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, synthetic_image_mask, generator_input

    assert torch.cuda.is_available(), "bench.py needs a GPU (no CPU fallback exists)"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        import datetime
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev,
                                timeout=datetime.timedelta(seconds=180))
    lib = L.get_lib()
    math = {"fp32": L.MATH_FP32, "bf16x3": L.MATH_BF16X3}[args.math]
    B, S = args.batch, args.size

    gen = seeded_parameters_(M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval(), 0).to(dev)
    img, mask = synthetic_image_mask(B, S, seed=rank)
    x_host = generator_input(img, mask).pin_memory()
    x_dev = x_host.to(dev)
    y_host = torch.empty(B, 3, S, S).pin_memory()

    ex = E.get_executor(gen, "generator", (x_dev,), math=math)
    graphed = E.GraphedProgram(ex, warmup=2)
    graphed.static_in["x0"].copy_(x_dev)
    stream = torch.cuda.current_stream(dev)

    def barrier():
        torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    def timed(fn, steps, collective=True):
        """CUDA-event time of `steps` calls.  collective=True (every rank must call it): barrier +
        synchronize on both sides and the MAX over ranks; collective=False: rank-local measurement
        (the rank-0-only roofline microbenchmarks — no rank may wait on a collective there)."""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if collective:
            barrier()
        else:
            torch.cuda.synchronize(dev)
        e0.record(stream)
        for _ in range(steps):
            fn()
        e1.record(stream)
        if collective:
            barrier()
        else:
            torch.cuda.synchronize(dev)
        ms = e0.elapsed_time(e1)
        if collective and world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
        return ms

    # ---- device-resident throughput (graph replay of the whole program)
    for _ in range(args.warmup):
        graphed.graph.replay()
    with ClockSampler(local) as clk:
        ms = timed(graphed.graph.replay, args.steps)
    clocks = clk.summary()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, ex.outputs)          # the program's outputs: the generator result
    value = world * B * args.steps / (ms / 1e3)

    # ---- end to end through the public serving API with HOST buffers: every step copies its pinned (B,4,S,S)
    # input to the device and its (B,3,S,S) result back; GeneratorPipeline overlaps those copies with the
    # kernels of the neighbouring steps (lama_b200/serving.py), all inside the timed region.
    from lama_b200.serving import GeneratorPipeline
    pipe = GeneratorPipeline(gen, B, S, S, device=dev, depth=2, math=math)
    for _ in range(3):
        pipe.result(pipe.submit(x_host))
    pipe.drain()
    import time as _time
    barrier()
    t0 = _time.perf_counter()
    tickets = []
    for _ in range(args.steps):
        tickets.append(pipe.submit(x_host))
        if len(tickets) > 1:
            y_host = pipe.result(tickets[-2])         # consume results as they complete
    y_host = pipe.result(tickets[-1])
    pipe.drain()
    barrier()
    ms_e2e = (_time.perf_counter() - t0) * 1e3
    if world > 1:
        t = torch.tensor([ms_e2e], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms_e2e = float(t.item())
    e2e = world * B * args.steps / (ms_e2e / 1e3)
    # the plain module call (what bin/predict.py does), serial copies, for comparison
    def serial_step():
        xd = x_host.to(dev, non_blocking=True)
        with torch.no_grad():
            y = gen(xd)
        y_host.copy_(y, non_blocking=True)
    serial_step()
    ms_serial = timed(serial_step, args.steps)

    # ---- dominant kernel + FourierUnit sub-path, timed alone with CUDA events on the launch stream
    conv_idx = [i for i, (n, _f, _a) in enumerate(ex.calls) if n.startswith("ffcb_conv:convl2l+convg2l")]
    fu_idx = [i for i, (n, _f, _a) in enumerate(ex.calls) if n == "ffcb_rfft2"]
    sc = stream.cuda_stream

    def run_calls(idx):
        for i in idx:
            n, fn, a = ex.calls[i]
            rc = fn(*a, sc)
            if rc:
                L.check(rc, n)
    peaks = _peaks()
    roof = None
    if conv_idx and rank == 0:
        i0 = conv_idx[len(conv_idx) // 2]
        reps = 10
        run_calls([i0] * 3)
        # (a) right after the timed steps: the GPU sits in its power cap (the state the sustained cuBLAS figure of
        #     MEASURED_PEAKS.json was taken in); (b) after two idle seconds, a short burst of launches — the protocol of
        #     the burst peak ("best of 10" on a cool GPU), which is the denominator the kernel-alone fraction is quoted on
        ms_c_hot = timed(lambda: run_calls([i0]), reps, collective=False) / reps
        torch.cuda.synchronize(dev)
        _time.sleep(2.0)
        run_calls([i0] * 2)
        ms_c = timed(lambda: run_calls([i0]), reps, collective=False) / reps
        h = S // 8
        flops = 2.0 * B * h * h * 128 * (9 * 512)
        ach = flops / (ms_c * 1e-3) / 1e12
        roof = {"kernel": "conv_simt_kernel" if math == L.MATH_FP32 else "conv_tc_kernel",
                "op": "resblock local 3x3 contraction (convl2l+convg2l+bn_l+relu): M=B*64*64, N=128, K=9*512",
                "bound": "tensor", "achieved": ach, "peak": peaks["bf16_burst"], "unit": "TFLOP/s",
                "frac": ach / peaks["bf16_burst"], "ms_per_launch": ms_c,
                "algorithmic_flops_per_launch": flops, "peak_source": peaks["source"] + ", bf16 burst",
                "ms_per_launch_hot": ms_c_hot,
                "frac_hot_vs_sustained_peak": flops / (ms_c_hot * 1e-3) / 1e12 / peaks["bf16_sustained"],
                "executed_over_algorithmic": 1.0 if math == L.MATH_FP32 else 3.0,
                "note": "fp32 CUDA-core arm (FFCB_MATH_FP32)" if math == L.MATH_FP32 else
                        "bf16x3 wgmma arm: 3 bf16 products per algorithmic MAC (frac <= 1/3 by construction); "
                        "ms_per_launch / frac: 10 launches after 2 idle seconds vs the burst peak; ms_per_launch_hot / "
                        "frac_hot_vs_sustained_peak: 10 launches right after the power-capped steps vs the back-to-back "
                        "cuBLAS figure of MEASURED_PEAKS.json"}
        if fu_idx:
            # one FourierUnit = a maximal run of {rfft2, spectral conv, irfft2} calls (3 calls, or 3 per batch chunk with
            # LAMA_B200_FU_CHUNK): take the run in the middle of the program
            is_fu = [n in ("ffcb_rfft2", "ffcb_irfft2") or n.startswith("ffcb_conv:fu.conv_layer") for n, _f, _a in ex.calls]
            runs, cur = [], []
            for i, f_ in enumerate(is_fu):
                if f_:
                    cur.append(i)
                elif cur:
                    runs.append(cur); cur = []
            if cur:
                runs.append(cur)
            fu_calls = runs[len(runs) // 2]
            run_calls(fu_calls * 3)
            c = 192
            fu_bytes = 4.0 * B * h * h * (c + c) + 4.0 * (2 * c) * (2 * c) + 8.0 * (2 * c)
            flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)     # 10x the 50 MB L2

            def fu_time(cold, idx):
                """median of `reps` single runs; cold: a 512 MB write evicts L2 before every run (outside the events)"""
                ts = []
                for _ in range(reps):
                    if cold:
                        flush.fill_(1)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    run_calls(idx)
                    e1.record(stream)
                    torch.cuda.synchronize(dev)
                    ts.append(e0.elapsed_time(e1))
                ts.sort()
                return ts[len(ts) // 2]
            ms_cold, ms_warm = fu_time(True, fu_calls), fu_time(False, fu_calls)
            kinds = {"rfft2": [k for k in fu_calls if ex.calls[k][0] == "ffcb_rfft2"],
                     "spectral_gemm": [k for k in fu_calls if ex.calls[k][0].startswith("ffcb_conv")],
                     "irfft2": [k for k in fu_calls if ex.calls[k][0] == "ffcb_irfft2"]}
            parts = {n: {"cold_ms": fu_time(True, ks), "warm_ms": fu_time(False, ks)} for n, ks in kinds.items()}
            del flush
            gbs = fu_bytes / (ms_cold * 1e-3) / 1e9
            roof["fourier_unit"] = {"bound": "hbm", "achieved": gbs, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                                    "frac": gbs / peaks["hbm_gbs"], "ms": ms_cold, "algorithmic_bytes": fu_bytes,
                                    "shape": [B, c, h, h], "launches": len(fu_calls),
                                    "l2": "cold (512 MB flush before each run)",
                                    "warm": {"ms": ms_warm, "achieved": fu_bytes / (ms_warm * 1e-3) / 1e9,
                                             "frac": fu_bytes / (ms_warm * 1e-3) / 1e9 / peaks["hbm_gbs"]},
                                    "per_kernel": parts,
                                    "layout": ("planar" if any(bf.cg for bf in ex.prog.bufs) else "nhwc"),
                                    "note": "SURVEY.md 8(d): algorithmic bytes = t in + u out + weights; spectrum "
                                            "intermediates not counted; graded figure = cold L2"}

    # ---- the CUDA-core fp32 arm of the same step (reference-grade arithmetic, LAMA_B200_MATH=fp32): same-arithmetic
    # reading beside the headline (rank 0, N=1 only; short: it is ~7x slower)
    fp32_arm = None
    if rank == 0 and world == 1 and math == L.MATH_BF16X3 and not args.no_fp32_arm:
        try:
            ex32 = E.get_executor(gen, "generator", (x_dev,), math=L.MATH_FP32)
            ex32.run({"x0": x_dev})
            ms32 = timed(lambda: ex32.run({"x0": x_dev}), 2, collective=False) / 2
            fp32_arm = {"value": B / (ms32 / 1e3), "unit": "images/s", "ms_per_step": ms32, "dtype": "f32",
                        "launches_per_step": ex32.launches_per_run}
            del ex32
            E.invalidate(gen)
            torch.cuda.empty_cache()
        except Exception as ex_f:  # noqa: BLE001
            fp32_arm = {"error": f"{type(ex_f).__name__}: {ex_f}"[:300]}

    # ---- CPU baseline (rank 0, N=1 only): bounded sample on all host cores
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        cores = _cpu_setup()
        cpu_reference_step(CPU_IMAGES_PER_STEP)
        n_img, t = 0, 0.0
        while t < 10.0 and n_img < 16:
            dt, n = cpu_reference_step(CPU_IMAGES_PER_STEP)
            t += dt; n_img += n
        cpu = {"value": n_img / t, "unit": "images/s", "cores": cores, "kind": "port",
               "sample": f"{n_img} images of 512x512 in batches of {CPU_IMAGES_PER_STEP}, torch-CPU port of the "
                         f"reference ops (oracle/ffc_torch_cpu.py), {cores} threads (fixed, same as --impl reference)"}

    # ---- the reference operator sequence under torch eager on this GPU (rank 0, N=1 only), TF32 on / off
    tcb = None
    if rank == 0 and world == 1 and not args.no_torch_cuda_baseline:
        try:
            tcb = torch_cuda_baseline(dev, B, S)
        except Exception as ex_t:  # noqa: BLE001
            tcb = {"error": f"{type(ex_t).__name__}: {ex_t}"[:300]}
        torch.cuda.empty_cache()

    # ---- the same step through the uint8 predict path (row f1): decoded bytes in, inpainted bytes out; /255, mask
    # multiply / concat, blend and x255 run inside the first / last kernels, PCIe carries 1 byte per sample.
    # Measured last and fenced: it is an extra reading, a failure here must not take the headline numbers down.
    u8_io = None
    if args.io == "both" and math == L.MATH_BF16X3 and world == 1:   # single-GPU reading (no collectives in here)
        try:
            img_h = (x_host[:, :3].permute(0, 2, 3, 1) * 255).round().to(torch.uint8).contiguous().pin_memory()
            msk_h = (x_host[:, 3] * 255).to(torch.uint8).contiguous().pin_memory()
            pipe8 = GeneratorPipeline(gen, B, S, S, device=dev, depth=2, math=math, u8=True)
            for _ in range(3):
                pipe8.result(pipe8.submit(img_h, msk_h))
            pipe8.drain()
            barrier()
            t0 = _time.perf_counter()
            tickets = []
            for _ in range(args.steps):
                tickets.append(pipe8.submit(img_h, msk_h))
                if len(tickets) > 1:
                    pipe8.result(tickets[-2])
            y8 = pipe8.result(tickets[-1])
            pipe8.drain()
            barrier()
            ms8 = (_time.perf_counter() - t0) * 1e3
            if world > 1:
                t = torch.tensor([ms8], device=dev)
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                ms8 = float(t.item())
            u8_io = {"value": world * B * args.steps / (ms8 / 1e3), "unit": "images/s",
                     "ms_per_step": ms8 / args.steps, "h2d_bytes_per_step": img_h.numel() + msk_h.numel(),
                     "d2h_bytes_per_step": y8.numel(), "launches_per_step": pipe8.launches_per_batch,
                     "api": "lama_b200.serving.GeneratorPipeline(u8=True) — the engine of lama_b200.predict"}
        except Exception as ex_u8:  # noqa: BLE001
            u8_io = {"error": f"{type(ex_u8).__name__}: {ex_u8}"[:300]}

    if rank == 0:
        print(json.dumps({
            "metric": METRIC, "value": value, "unit": "images/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32" if math == L.MATH_FP32 else "bf16x3(f32 accumulate)",
            "data": "synthetic",
            "config": {"workload": f"big-lama FFCResNetGenerator fwd (configs[2]), bs{B}/GPU {S}x{S}, seeded random weights",
                       "global_batch": B * world, "parallelism": f"batch-sharded x{world}, no data-path collective",
                       "math": args.math, "l2": "inputs+activations (>4 GB/step) exceed the 50 MB L2; no explicit flush",
                       "cuda_graph": True},
            "e2e": {"value": e2e, "unit": "images/s", "h2d_bytes_per_step": x_host.numel() * 4 * 1,
                    "d2h_bytes_per_step": y_host.numel() * 4, "ms_per_step": ms_e2e / args.steps,
                    "api": "lama_b200.serving.GeneratorPipeline (depth 2: copies overlap the neighbouring steps)",
                    "timer": "host wall clock around submit/result of all steps (copies are on side streams)",
                    "module_call_serial_copies": world * B * args.steps / (ms_serial / 1e3),
                    "u8_io": u8_io},
            "gpu_launches": ex.launches_per_run * args.steps,
            "launches_per_step": ex.launches_per_run,
            "clocks": clocks, "roofline": roof, "cpu_baseline": cpu, "torch_cuda_baseline": tcb,
            "fp32_arm": fp32_arm,
        }), file=out)
        out.flush()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
