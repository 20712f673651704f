"""Every C-ABI call a ``CudaExecutor`` issues, pinned on the CPU: programs of the small seeded generator and of a few
layers are bound on ``torch.device("cpu", 0)`` against a stub library, and each call is serialised as its name plus its
arguments (ctypes structures field by field, pointers normalised to what they point at) and compared with
``tests/golden/executor_calls.json`` by digest.  A change to the host layer that moves one launch argument fails here.

Running this module as a script (``PYTHONPATH=. python tests/test_executor_calls_cpu.py``) rewrites the golden; a
change that deliberately alters a program regenerates it and says why."""
import ctypes as C
import hashlib
import json
import os

import pytest
import torch
import torch.utils.deterministic

from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200.testing import seeded_parameters_, small_lama_kwargs

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "executor_calls.json")


class _StubLib:
    """Every symbol is a function that records nothing and returns 0."""

    def __getattr__(self, name):
        return lambda *args: 0


def _gen(**kw):
    return seeded_parameters_(M.FFCResNetGenerator(**small_lama_kwargs(**kw)).eval(), 5, gain=1.0)


def programs():
    """name -> Program.  Between them these contain every op type of the engine."""
    gen = _gen()
    sl, sg = (1, 16, 8, 8), (1, 48, 8, 8)
    ffc = seeded_parameters_(M.FFC_BN_ACT(64, 64, 3, 0.5, 0.5, stride=2, padding=1, activation_layer=torch.nn.ReLU,
                                          enable_lfu=True).eval(), 2, gain=1.0)
    fu = seeded_parameters_(M.FourierUnit(8, 8, spectral_pos_encoding=True).eval(), 3, gain=1.0)
    kw = small_lama_kwargs(ngf=16, n_blocks=1, n_downsampling=2)
    kw.update(out_ffc=True, out_ffc_kwargs=dict(ratio_gin=0.5, ratio_gout=0.5, enable_lfu=False))
    out_ffc = seeded_parameters_(M.FFCResNetGenerator(**kw).eval(), 4, gain=1.0)
    cases = {
        "generator_bf16x3_64x64": (gen, "generator", ((1, 4, 64, 64),), L.MATH_BF16X3),
        "generator_fp32_40x72": (gen, "generator", ((1, 4, 40, 72),), L.MATH_FP32),
        "generator_u8": (gen, "generator_u8:8", ((2, 45, 52, 3), (2, 45, 52)), L.MATH_BF16X3),
        "resnet_block_grad": (gen.model[5], "resnet_block_grad", (sl, sg), L.MATH_BF16X3),
        "generator_rear": (gen, "generator_rear", (sl, sg), L.MATH_BF16X3),
        "generator_rear_grad_fp32": (gen, "generator_rear_grad", (sl, sg), L.MATH_FP32),
        "generator_refine": (gen, "generator_refine:61x59", (sl, sg), L.MATH_BF16X3),
        "ffc_bn_act_lfu_s2": (ffc, "ffc_bn_act", ((1, 32, 16, 16), (1, 32, 16, 16)), L.MATH_BF16X3),
        "fourier_unit_pos": (fu, "fourier_unit", ((1, 8, 12, 16),), L.MATH_BF16X3),
        "generator_out_ffc": (out_ffc, "generator", ((1, 4, 32, 32),), L.MATH_BF16X3),
    }
    with torch.no_grad():
        return {k: E.build_module_program(m, kind, shapes, math) for k, (m, kind, shapes, math) in cases.items()}


class _Serialiser:
    """Normalises the pointers of one executor's calls: program buffers -> (storage slot, byte offset), outputs and the
    FFT workspace -> (name, offset), inputs -> their name, packed constants -> sha256 of their bytes, uninitialised
    scratch (NaN-filled under deterministic allocation) -> its size."""

    def __init__(self, ex, feed):
        self.regions = []                # (start, end, label(offset))
        for name, t in feed.items():
            self._add(t, lambda off, n=name: ["input", n] if off == 0 else ["input", n, off])
        for b in ex.prog.bufs:
            self._add(ex.storage[b.name], lambda off, s=ex.slots[b.name]: ["buf", s, off])
        for name, t in ex.outputs.items():
            self._add(t, lambda off, n=name: ["output", n, off])
        self._add(ex.ws, lambda off: ["workspace", off])
        for t in ex._keep:
            if torch.is_tensor(t):
                if t.is_floating_point() and bool(torch.isnan(t).all()):
                    self._add(t, lambda off, n=t.numel() * t.element_size(): ["scratch", n, off])
                else:
                    h = hashlib.sha256(t.detach().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()
                    self._add(t, lambda off, h=h, d=str(t.dtype), s=list(t.shape): ["const", h, d, s, off])

    def _add(self, t, label):
        p = t.data_ptr()
        self.regions.append((p, p + max(t.numel() * t.element_size(), 1), label))

    def ptr(self, p, strict=True):
        if p is None or p == 0:
            return None
        for lo, hi, label in self.regions:
            if lo <= p < hi:
                return label(p - lo)
        assert not strict, f"pointer {p:#x} into no known allocation"
        return p

    def value(self, v):
        if v is None:
            return None
        if isinstance(v, int) and not isinstance(v, bool):
            return self.ptr(v, strict=False)                  # an address, or a size / count (none is a valid address)
        if type(v).__name__ == "CArgObject":                 # ctypes.byref(structure)
            return self.struct(v._obj)
        if isinstance(v, C.Structure):
            return self.struct(v)
        raise TypeError(type(v))

    def struct(self, s):
        out = {}
        for f, ft in s._fields_:
            v = getattr(s, f)
            if f == "ptr" or ft is C.c_void_p:
                out[f] = self.ptr(v)
            elif isinstance(v, C.Array):
                items = list(v)[:s.nseg] if f == "seg" else list(v)
                out[f] = [self.struct(x) for x in items]
            elif isinstance(v, C.Structure):
                out[f] = self.struct(v)
            else:
                out[f] = v
        return out


def call_digests(prog):
    """[[call name, sha256 of the serialised arguments]] of a CudaExecutor of ``prog`` on the CPU with a stub library."""
    prev = torch.utils.deterministic.fill_uninitialized_memory, torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = True
    try:
        ex = E.CudaExecutor(prog, torch.device("cpu", 0))
    finally:
        torch.utils.deterministic.fill_uninitialized_memory = prev[0]
        torch.use_deterministic_algorithms(prev[1])
    feed = {k: torch.zeros(v, dtype=prog.dtypes.get(k, torch.float32)) for k, v in prog.inputs.items()}
    ex.bind_inputs(feed)
    ser = _Serialiser(ex, feed)
    out = []
    for name, _fn, args in ex.calls:
        blob = json.dumps([name, [ser.value(a) for a in args]], sort_keys=True, separators=(",", ":"))
        out.append([name, hashlib.sha256(blob.encode()).hexdigest()])
    return out


def _clean_env(setenv_del):
    for k in list(os.environ):
        if k.startswith(("LAMA_B200_", "FFCB_")):
            setenv_del(k)


@pytest.fixture
def stub_lib(monkeypatch):
    _clean_env(lambda k: monkeypatch.delenv(k, raising=False))
    monkeypatch.setattr(L, "get_lib", lambda: _StubLib())


def test_executor_calls_unchanged(stub_lib):
    """Each program binds to the same calls with the same arguments as when the golden was written."""
    with open(GOLDEN) as f:
        want = json.load(f)
    progs = programs()
    assert {type(op) for p in progs.values() for op in p.ops} == set(E.OP_TYPES)
    assert progs.keys() == want.keys()
    for k, prog in progs.items():
        got = call_digests(prog)
        assert [n for n, _ in got] == [n for n, _ in want[k]], k
        for i, (a, b) in enumerate(zip(got, want[k])):
            assert a == b, f"{k}: call {i} ({a[0]}) changed"


def test_every_op_type_is_declared_bound_and_interpreted():
    """Every op record of the engine is an ``Op`` in the one registry, declares the fields holding the views it reads
    and writes and its call, and has a case in the CPU interpreter."""
    import dataclasses
    from spec_interp import SpecInterpreter
    records = {v for v in vars(E).values() if isinstance(v, type) and dataclasses.is_dataclass(v)}
    assert records - {E.Buf, E.TV, E.Program, E.Ext} == set(E.OP_TYPES)
    for cls in E.OP_TYPES:
        assert {"reads", "writes", "bind"} <= set(vars(cls)), cls.__name__
        for f in cls.reads + cls.writes + cls.ring_in:
            assert f in cls.__dataclass_fields__, (cls.__name__, f)
        assert callable(getattr(SpecInterpreter, cls.__name__, None)), cls.__name__


if __name__ == "__main__":
    _clean_env(os.environ.pop)
    L.get_lib = lambda: _StubLib()
    with open(GOLDEN, "w") as f:
        json.dump({k: call_digests(p) for k, p in programs().items()}, f, indent=0)
    print("wrote", GOLDEN)
