"""CPU-only checks of the high-resolution path: FFT planes of 448..1024 points (the bottlenecks of 4K-class photos)
and predict batches sized to device memory.

* the 8-channel two-pass kernels' orchestration (fft_core.cuh compiled with g++, tests/host_emul/fft_narrow_emul.cpp)
  against a float64 DFT, and the runtime radix planner for every length up to 1024;
* the admission gates (fft_len_ok, plane_ok, generator_supported) at 4K-class sizes;
* a small generator program at a 270x480 bottleneck, interpreted (tests/spec_interp.py) against the oracle;
* BatchedInpainter's batch plan and lane policy under a memory budget, with a stand-in lane.
"""
import gc
import os
import subprocess
import weakref

import numpy as np
import pytest
import torch

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200 import predict as PR
from lama_b200.testing import BIG_LAMA_KWARGS, seeded_parameters_, small_lama_kwargs
from oracle import ffc_torch_cpu as otc
from spec_interp import SpecInterpreter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_host_emulation_of_the_8_channel_fft_kernels(tmp_path):
    """Forward and C2R inverse (non-Hermitian spectrum) at 448, 480, 500, 512, 540, 750, 960, 1000, 1024 and the
    primes 449, 479, 1021, as row and as column axis, and mixed planes (270x480, 375x500, ...), with several live and
    dead lanes of one 8-channel CTA: within 2e-6 of max |ref|.  The planner factors every n in 321..1024 into at most
    kMaxRtPasses radices >= 2 that multiply back to n."""
    exe = tmp_path / "fft_narrow_emul"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "host_emul", "fft_narrow_emul.cpp"), "-o", str(exe)])
    out = subprocess.run([str(exe), "v"], capture_output=True, text=True)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr


def test_fft_lengths_up_to_1024_are_native():
    assert all(E.fft_len_ok(n) for n in range(1, 1025))
    assert not E.fft_len_ok(1025) and not E.fft_len_ok(0) and not E.fft_len_ok(2048)
    for h, w in ((270, 480), (375, 500), (512, 512), (500, 750), (1024, 1024), (479, 270), (448, 96)):
        assert E.plane_ok(h, w) and E.plane_ok(w, h)
    assert not E.plane_ok(1025, 8) and not E.plane_ok(8, 1025) and not E.plane_ok(8, 1)


def test_big_lama_is_native_at_4k_class_sizes():
    big = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    for h, w in ((2160, 3840), (3000, 4000), (4096, 4096), (4000, 6000), (8192, 8192)):
        assert E.generator_supported(big, torch.empty(1, 4, h, w, device="meta")), (h, w)
    assert not E.generator_supported(big, torch.empty(1, 4, 8200, 8200, device="meta"))


def test_big_lama_program_storage_at_4k_class_sizes():
    """Device bytes of big-lama's uint8 predict program at batch 1 on the split-bf16 arm (computed from the buffer
    shapes, packed weights not counted), as quoted in the documentation."""
    big = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    got = {}
    for h, w in ((2160, 3840), (3000, 4000), (4096, 4096), (4000, 6000)):
        with torch.no_grad():
            prog = E.build_module_program(big, "generator_u8:8", ((1, h, w, 3), (1, h, w)), L.MATH_BF16X3)
        got[(h, w)] = E.program_storage_bytes(prog)
        print(f"big-lama generator_u8 program, batch 1, {h}x{w}: {got[(h, w)] / 1e9:.2f} GB")
    assert got[(2160, 3840)] < got[(3000, 4000)] < got[(4096, 4096)] < got[(4000, 6000)]
    assert 6e9 < got[(2160, 3840)] < 10e9


def test_small_generator_program_at_a_270x480_bottleneck():
    """The generator program interpreted op by op (the FFT ops at 480-point rows and 270-point columns) against the
    torch-CPU oracle port: one 540x960 image, one down-sampling, so the residual blocks run on 270x480 planes."""
    kw = small_lama_kwargs(ngf=16, n_blocks=1, n_downsampling=1)
    g = seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 3)
    sd = {k: v.clone() for k, v in g.state_dict().items()}
    x = torch.rand(1, 4, 540, 960, generator=torch.Generator().manual_seed(5))
    x[:, 3] = (x[:, 3] > 0.7).float()
    assert E.generator_supported(g, x)
    with torch.no_grad():
        prog = E.build_module_program(g, "generator", ((1, 4, 540, 960),), L.MATH_FP32)
        ref = otc.ffc_resnet_generator(x, sd, **kw)
    assert any(isinstance(o, E.RfftOp) for o in prog.ops)
    out = SpecInterpreter(prog).run({"x0": x})["y0"]
    err = float((out - ref).abs().max())
    print(f"small generator at a 270x480 bottleneck, interpreted vs oracle: max-abs {err:.2e}")
    assert err < 2e-5


# ------------------------------------------------------------------------------------------- predict batching
class _StandInLane:
    """Records what the inpainter builds and releases instead of allocating a pipeline."""

    def __init__(self, generator, b, h0, w0, device, depth, pad_mod):
        self.key = (b, h0, w0)
        self.bytes = 0
        self.closed = False

    def close(self):
        self.closed = True


def _inpainter(per_image, max_batch=32, mem_budget=None, max_pipelines=2):
    inp = PR.BatchedInpainter.__new__(PR.BatchedInpainter)
    inp.generator, inp.device = None, torch.device("cpu")
    inp.max_batch, inp.pad_mod, inp.depth, inp.max_pipelines = max_batch, 8, 2, max_pipelines
    inp.mem_budget = mem_budget
    inp._pipes = PR.OrderedDict()
    inp._per_image = dict(per_image)
    return inp


@pytest.mark.parametrize("n,fit", [(7, 3.5), (40, 9.2), (5, 1.0), (3, 0.4), (70, 32.0), (70, 100.0)])
def test_predict_batches_fit_the_budget(n, fit, monkeypatch):
    """Big images under a budget of ``fit`` images: balanced batches (sizes differ by at most one), every image once,
    and the lanes alive at any time, counted with the bytes the inpainter charges them, never pool more than the
    budget (except one image alone that exceeds it: it still runs at batch 1).  A budget that takes max_batch images
    gives exactly the batches of BatchedInpainter.plan."""
    monkeypatch.setattr(PR, "_Lane", _StandInLane)
    per = 8_000_000_000
    inp = _inpainter({(2157, 3838): per, (64, 64): per // 1000}, mem_budget=int(fit * per))
    sizes = [(2157, 3838)] * n + [(64, 64)] * 3
    got = list(inp.batches(sizes))
    big = [idx for hw, idx, _ in got if hw == (2157, 3838)]
    assert sorted(i for b in big for i in b) == list(range(n))
    assert max(map(len, big)) - min(map(len, big)) <= 1 or fit >= 32
    if fit >= 32:
        assert big == [idx for hw, idx in PR.BatchedInpainter.plan(sizes, 32) if hw == (2157, 3838)]
    else:
        nb = max(1, int(fit))
        assert max(map(len, big)) <= nb and len(big) == -(-n // nb)
    peak = 0
    for (h0, w0), idx, budget in got:
        inp._lane(len(idx), h0, w0, budget)
        peak = max(peak, inp._alive_bytes())
        assert len(inp._pipes) <= inp.max_pipelines
    assert peak <= max(int(fit * per), per), (peak, fit * per)


def test_predict_batches_without_memory_pressure_are_unchanged(monkeypatch):
    """Small images under a large budget: the batches, and the lanes built for them, are those the inpainter used
    before batches were sized to memory."""
    monkeypatch.setattr(PR, "_Lane", _StandInLane)
    sizes = [(45, 52)] * 5 + [(100, 75)] * 2 + [(45, 52)] * 2
    inp = _inpainter({(45, 52): 10_000, (100, 75): 30_000}, max_batch=2, mem_budget=10 ** 12)
    got = [(hw, idx) for hw, idx, _ in inp.batches(sizes)]
    assert got == PR.BatchedInpainter.plan(sizes, 2)
    for (h0, w0), idx in got:
        inp._lane(len(idx), h0, w0, 10 ** 12)
    assert list(inp._pipes) == [(1, 45, 52), (2, 100, 75)]


class _EchoPipe:
    """Stand-in pipeline: the result of a batch is its input image bytes."""

    def __init__(self):
        self._out = {}

    def submit(self, img, mask):
        self._out[len(self._out)] = img.clone()
        return len(self._out) - 1

    def result(self, ticket):
        return self._out[ticket]


class _TrackedLane(_StandInLane):
    """Stand-in lane that checks, when it is built, that every lane closed before it is unreachable (its device memory
    would otherwise still be held while the new program allocates)."""
    built = []

    def __init__(self, generator, b, h0, w0, device, depth, pad_mod):
        gc.collect()
        alive = [r() for r in _TrackedLane.built if r() is not None and r().closed]
        assert not alive, f"closed lane {alive[0].key} still alive while lane {(b, h0, w0)} is built"
        super().__init__(generator, b, h0, w0, device, depth, pad_mod)
        self.pipe = _EchoPipe()
        self._stage = (torch.zeros(b, h0, w0, 3, dtype=torch.uint8), torch.zeros(b, h0, w0, dtype=torch.uint8))
        _TrackedLane.built.append(weakref.ref(self))

    def stage(self):
        return self._stage


def test_inpaint_frees_released_lanes_before_building_the_next(monkeypatch):
    """Through ``inpaint``: eleven images under a budget of six cut into batches of 6 and 5, then a group of another
    shape.  Each new lane needs its predecessor released, and the released lane must be unreachable when the next one
    is built; the results come back in input order."""
    monkeypatch.setattr(PR, "_Lane", _TrackedLane)
    monkeypatch.setattr(_TrackedLane, "built", [])
    inp = _inpainter({(8, 8): 100, (8, 16): 100}, mem_budget=600)
    rng = np.random.default_rng(0)
    items = [(rng.integers(0, 256, (8, 8, 3), dtype=np.uint8), np.zeros((8, 8), np.uint8)) for _ in range(11)]
    items += [(rng.integers(0, 256, (8, 16, 3), dtype=np.uint8), np.zeros((8, 16), np.uint8)) for _ in range(3)]
    outs = inp.inpaint(items)
    assert all(np.array_equal(o, im) for o, (im, _) in zip(outs, items))
    assert [r() is None for r in _TrackedLane.built] == [True, True, False]
    assert list(inp._pipes) == [(3, 8, 16)]


def test_lanes_of_another_shape_are_released_when_they_would_not_fit(monkeypatch):
    monkeypatch.setattr(PR, "_Lane", _StandInLane)
    inp = _inpainter({(2160, 3840): 100, (64, 64): 10}, max_batch=8, mem_budget=1000, max_pipelines=3)
    a = inp._lane(8, 64, 64, 1000)               # 80 bytes
    b = inp._lane(5, 2160, 3840, 1000)           # 500 bytes: fits beside a
    assert not a.closed and set(inp._pipes) == {(8, 64, 64), (5, 2160, 3840)}
    c = inp._lane(9, 2160, 3840, 1000)           # 900 bytes: a and b are released, oldest first
    assert a.closed and b.closed and not c.closed and list(inp._pipes) == [(9, 2160, 3840)]
    assert inp._alive_bytes() == 900


def test_per_image_bytes_counts_program_and_staging():
    """One image's share: the batch-1 uint8 program's storage plus the pipeline's device staging slots."""
    g = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval()
    inp = _inpainter({})
    inp.generator = g
    with torch.no_grad():
        prog = E.build_module_program(g, "generator_u8:8", ((1, 45, 52, 3), (1, 45, 52)), E.default_math())
    want = E.program_storage_bytes(prog) + 3 * 4 * 45 * 52 + 2 * 3 * 45 * 52
    assert inp.per_image_bytes(45, 52) == want
    assert inp.per_image_bytes(45, 52) == want                    # cached


def test_budget_counts_the_inpainters_own_lanes(monkeypatch):
    """Default budget: 70 % of free device memory plus what this inpainter's alive lanes hold."""
    inp = _inpainter({})
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (1000, 2000))
    assert inp._budget() == 700
    lane = _StandInLane(None, 1, 8, 8, None, 2, 8)
    lane.bytes = 300
    inp._pipes[(1, 8, 8)] = lane
    assert inp._budget() == int(0.7 * (1000 + 300))
    inp.mem_budget = 123
    assert inp._budget() == 123
