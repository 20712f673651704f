"""In-tree build of libffc_b200.so (sm_90a only) with nvcc.

``python -m lama_b200.build`` or ``__graft_entry__.build()``.  nvcc cross-compiles without a
GPU; the resulting ``lama_b200/libffc_b200.so`` and ``lama_b200/build/`` are git-ignored build products.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
LIB_PATH = os.path.join(HERE, "libffc_b200.so")
STAMP = LIB_PATH + ".stamp"
OBJ_DIR = os.path.join(HERE, "build")

SOURCES = ["api.cu", "fft.cu", "fft_plane.cu", "fft_plane_cg.cu", "conv_simt.cu", "conv_tc.cu", "shell.cu", "grad.cu",
           "refine.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [
    "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC", "-shared",
] + os.environ.get("LAMA_B200_NVCC_EXTRA", "").split()      # experiments only (e.g. --use_fast_math A/B)


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _file_hash(paths):
    h = hashlib.sha256()
    for f in paths:
        with open(f, "rb") as fh:
            h.update(os.path.basename(f).encode())
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _headers():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))] + [
        os.path.join(INCLUDE, "ffc_b200.h")]


def _fingerprint():
    return _file_hash([os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h"))] +
                      [os.path.join(INCLUDE, "ffc_b200.h")])


def is_current() -> bool:
    if not (os.path.isfile(LIB_PATH) and os.path.isfile(STAMP)):
        return False
    with open(STAMP) as fh:
        return fh.read().strip() == _fingerprint()


def _compile_one(src, verbose):
    """One translation unit -> build/<name>.o, skipped when the source, the headers and the flags are unchanged."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    obj = os.path.join(OBJ_DIR, src[:-3] + ".o")
    tag = _file_hash([os.path.join(CSRC, src)] + _headers())
    stamp = obj + ".stamp"
    if os.path.isfile(obj) and os.path.isfile(stamp) and open(stamp).read().strip() == tag:
        return obj, ""
    flags = [f for f in NVCC_FLAGS if f != "-shared"]
    cmd = [_nvcc()] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, src]
    proc = subprocess.run(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src}:\n" + proc.stdout[-6000:])
    with open(stamp, "w") as fh:
        fh.write(tag)
    return obj, proc.stdout


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile the library if sources changed (translation units in parallel, objects cached); returns its path."""
    if not force and is_current():
        return LIB_PATH
    if force and os.path.isdir(OBJ_DIR):
        shutil.rmtree(OBJ_DIR)
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=len(SOURCES)) as pool:
        results = list(pool.map(lambda s: _compile_one(s, verbose), SOURCES))
    if verbose:
        sys.stderr.write("".join(out for _o, out in results))
    cmd = [_nvcc(), "-shared"] + ARCH + ["-o", LIB_PATH] + [o for o, _ in results]
    proc = subprocess.run(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed linking libffc_b200.so:\n" + proc.stdout[-4000:])
    with open(STAMP, "w") as fh:
        fh.write(_fingerprint())
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
