"""CPU-only: the C-ABI library builds, loads and exports every symbol include/ffc_b200.h declares;
ctypes struct layouts match the C structs; no compute calls are made (no GPU here)."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from lama_b200 import _lib
    return _lib.get_lib()


def test_header_symbols_are_exported_and_bound(lib):
    from lama_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "ffc_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(ffcb_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    for name in declared:
        assert hasattr(lib, name)


def test_struct_layouts_match_c(tmp_path):
    from lama_b200 import _lib
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ffc_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu '
                   '%zu %zu %zu\\n",sizeof(ffcb_tensor),sizeof(ffcb_kseg),sizeof(ffcb_conv_desc),offsetof(ffcb_conv_desc,seg),'
                   'offsetof(ffcb_conv_desc,weight),sizeof(ffcb_conv_plan_info),offsetof(ffcb_conv_plan_info,m_tiles),'
                   'offsetof(ffcb_conv_plan_info,n_tiles));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    t, k, d, off_seg, off_w, p, off_m, off_n = map(int, subprocess.check_output([str(exe)]).split())
    assert ctypes.sizeof(_lib.Tensor) == t and ctypes.sizeof(_lib.KSeg) == k and ctypes.sizeof(_lib.ConvDesc) == d
    assert _lib.ConvDesc.seg.offset == off_seg and _lib.ConvDesc.weight.offset == off_w
    assert ctypes.sizeof(_lib.ConvPlanInfo) == p
    assert _lib.ConvPlanInfo.m_tiles.offset == off_m and _lib.ConvPlanInfo.n_tiles.offset == off_n


def test_version_and_error_plumbing(lib):
    from lama_b200 import _lib
    assert lib.ffcb_version() == _lib.VERSION
    # argument validation happens before any CUDA call, so it is testable without a GPU
    d = _lib.ConvDesc()
    assert lib.ffcb_conv(ctypes.byref(d), None) == _lib.EINVAL
    assert b"conv" in lib.ffcb_last_error()
    with pytest.raises(ValueError):
        _lib.check(_lib.EINVAL, "probe")
    assert lib.ffcb_fft2_workspace_bytes(2, 8, 8, 4) == 8 * 2 * 8 * 5 * 4


def test_missing_library_is_loud(monkeypatch, tmp_path):
    from lama_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.FFCBError):
        _lib.get_lib()


def test_host_emulation_of_fft_and_shipped_plane_kernels(tmp_path):
    """The FFT kernels' arithmetic (fft_core.cuh) compiled for the host and checked against a
    double-precision DFT for every supported size class (pow2 Stockham, direct DFT, runtime mixed-radix Stockham
    plans for composite / prime-power / prime lengths, C2R rule), and the per-thread steps of the 64x64 plane pair as
    rfft2_plane64_kernel / irfft2_plane64_v2_kernel run them."""
    exe = tmp_path / "fft_emul"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "host_emul", "fft_emul.cpp"), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr


def test_host_emulation_of_channel_group_planar_plane_kernels(tmp_path):
    """fft_plane_cg.cuh (the per-thread phases of the round-2 64x64 plane kernels) run for all 128 threads of a CTA
    on the host: swizzled in-place shared-memory layout, packed DC / Nyquist slot, C2R rule — vs a float64 DFT."""
    exe = tmp_path / "plane_cg_emul"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "host_emul", "plane_cg_emul.cpp"), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr


def test_cpu_tensor_never_touches_the_library():
    """On CPU tensors the modules run the torch composition (training / reference use); the CUDA
    library is only entered for CUDA tensors, where its absence raises."""
    import torch
    from lama_b200 import modules as M
    m = M.FourierUnit(8, 8).eval()
    with torch.no_grad():
        y = m(torch.randn(1, 8, 8, 8))
    assert y.shape == (1, 8, 8, 8)
