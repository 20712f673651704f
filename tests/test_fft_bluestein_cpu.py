"""CPU-only checks of the Bluestein (chirp-z) mode of the two-pass FFT kernels (lama_b200/csrc/fft.cu):

* the orchestration of one CTA (fft_core.cuh compiled with g++, tests/host_emul/fft_bluestein_emul.cpp) for every
  length 2..1024 the planner routes to Bluestein: row pass (two-for-one) and column pass, forward and C2R inverse,
  with dead lanes, against a float64 DFT;
* the planner's choices (make_bluestein_plan): which lengths take Bluestein, and that every other length keeps the
  runtime plan make_rt_plan gives it.
"""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    exe = tmp_path_factory.mktemp("bluestein") / "fft_bluestein_emul"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "host_emul", "fft_bluestein_emul.cpp"), "-o", str(exe)])
    return str(exe)


@pytest.fixture(scope="module")
def plans(emul):
    out = subprocess.run([emul, "plans"], capture_output=True, text=True, check=True).stdout
    got = {}
    for line in out.splitlines():
        head, radices = line.split("|")
        n, m, lanes, _cost, _direct = head.split()
        got[int(n)] = (int(m), int(lanes), [int(r) for r in radices.split()])
    return got


def test_host_emulation_of_the_bluestein_kernels(emul):
    """Every Bluestein length, row and column pass, both directions, 3 live lanes and the rest dead: within 2e-6 of
    max |ref| (the bound of the other FFT emulations)."""
    out = subprocess.run([emul, "v"], capture_output=True, text=True)
    print(out.stdout[-3000:])
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr


def test_planner_routes_large_prime_factors_to_bluestein(plans):
    """Bluestein convolves at the power of two m >= 2n - 1 (512 / 1024 with 8 channels per CTA, 2048 with 4)."""
    for n, m, lanes in ((479, 1024, 8), (251, 512, 8), (502, 1024, 8), (1021, 2048, 4), (997, 2048, 4), (211, 512, 8),
                        (263, 1024, 8)):
        assert plans[n][:2] == (m, lanes), (n, plans[n])
    for n, (m, lanes, _) in plans.items():
        if m:
            assert m >= 2 * n - 1 and m < 4 * n - 2 and lanes == (4 if m == 2048 else 8), (n, m, lanes)


# radices make_rt_plan gives these lengths (the plans they ran before the Bluestein mode)
KEEP = {480: [6, 5, 4, 4], 500: [5, 5, 5, 4], 512: [8, 4, 4, 4], 375: [5, 5, 5, 3], 270: [6, 5, 3, 3],
        135: [5, 3, 3, 3]}


def test_planner_keeps_the_runtime_plan_elsewhere(plans):
    for n, radices in KEEP.items():
        assert plans[n] == (0, 0, radices), (n, plans[n])
    for n in (4, 8, 16, 32, 64, 128, 256):                  # compile-time plans
        assert plans[n][0] == 0, n
    assert not any(plans[n][0] for n in range(2, 129))     # m would be below 512
