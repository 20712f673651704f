"""``torch.library`` registration of the native generator call, so that a ``torch.jit.trace`` of the drop-in model
(the reference's ``bin/to_jit.py:49-60``) KEEPS the sm_90a kernels instead of silently baking in cuFFT / cuDNN.

A ctypes call is invisible to the tracer.  The op below makes the whole generator one node of the traced graph:

    lama_b200::ffc_generator(Tensor x, Tensor[] state, str spec) -> Tensor

``state`` is the generator's ``state_dict`` values in order (the tracer records them as parameters of the traced
module, so the saved TorchScript file carries the weights) and ``spec`` the JSON of the constructor arguments.  The
CUDA implementation rebuilds a shell ``FFCResNetGenerator`` around those tensors (once per set of storages) and runs
the native program; loading such a file needs ``import lama_b200.ops`` first (that registers the op — see
INTEGRATION.md).  CPU tensors never reach this op: on CPU the modules trace the reference's torch operator sequence,
exactly as before.
"""
from __future__ import annotations

import json
from typing import Dict, List, Tuple

import torch

_JSON_OK = (int, float, str, bool, type(None))


def spec_of(kwargs: dict):
    """JSON of the constructor arguments, or None when they are not plain data (custom layer classes): such models
    keep tracing through the torch operator sequence."""
    def plain(v):
        if isinstance(v, _JSON_OK):
            return True
        if isinstance(v, dict):
            return all(isinstance(k, str) and plain(x) for k, x in v.items())
        if isinstance(v, (list, tuple)):
            return all(plain(x) for x in v)
        return False
    return json.dumps(kwargs, sort_keys=True) if plain(kwargs) else None


_SHELLS: Dict[Tuple, torch.nn.Module] = {}
_MAX_SHELLS = 4


def _shell(state: List[torch.Tensor], spec: str):
    """FFCResNetGenerator whose parameters / buffers ARE the given tensors (no copy), cached by their storages."""
    from . import modules as M
    key = (spec, tuple(t.data_ptr() for t in state))
    g = _SHELLS.get(key)
    if g is None:
        with torch.device("meta"):
            g = M.FFCResNetGenerator(**json.loads(spec))
        names = list(g.state_dict().keys())
        if len(names) != len(state):
            raise RuntimeError(f"lama_b200::ffc_generator: {len(state)} state tensors for a model with {len(names)}")
        g.load_state_dict(dict(zip(names, state)), assign=True)
        g.eval()
        while len(_SHELLS) >= _MAX_SHELLS:
            _SHELLS.pop(next(iter(_SHELLS)))
        _SHELLS[key] = g
    return g


@torch.library.custom_op("lama_b200::ffc_generator", mutates_args=(), device_types="cuda")
def ffc_generator(x: torch.Tensor, state: List[torch.Tensor], spec: str) -> torch.Tensor:
    from . import engine as E
    g = _shell(state, spec)
    xc = x.contiguous()
    if not E.generator_supported(g, xc):
        raise RuntimeError(f"lama_b200::ffc_generator: {xc.shape[-2]}x{xc.shape[-1]} input / model outside the native "
                           f"path")
    with torch.no_grad():
        return E.run_module(g, "generator", (xc,))[0]


@ffc_generator.register_fake
def _(x, state, spec):
    out_nc = json.loads(spec)["output_nc"]
    return x.new_empty((x.shape[0], out_nc, x.shape[2], x.shape[3]))


def traced_generator_call(module, x: torch.Tensor):
    """What FFCResNetGenerator.forward does under torch.jit.trace on CUDA: one custom-op node."""
    return torch.ops.lama_b200.ffc_generator(x, list(module.state_dict(keep_vars=True).values()), module._ffcb_spec)
