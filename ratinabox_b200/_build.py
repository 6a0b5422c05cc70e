"""Build libriab_b200.so in-tree with nvcc for sm_90a (no torch extension machinery:
the library has a plain C ABI and is loaded with ctypes)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.environ.get("RIAB_LIB", os.path.join(HERE, "libriab_b200.so"))
SOURCES = ["riab_b200.cu", "riab_nnn.cu"]
HEADERS = None  # every csrc/*.cuh + include/riab_b200.h (see _headers)

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "--expt-relaxed-constexpr", "-split-compile", "0",
]


def _headers():
    import glob
    return sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [os.path.join(HERE, "..", "include", "riab_b200.h")]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(f) > t for f in [os.path.join(CSRC, f) for f in SOURCES] + _headers())


def build(force=False, verbose=False, extra=()):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + list(extra) + [os.path.join(CSRC, f) for f in SOURCES] + ["-o", LIB]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    build(force=True, verbose=True, extra=sys.argv[1:])
