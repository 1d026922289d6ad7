"""Builds libb200vis.so (CUDA kernels + C ABI) in-tree for sm_90a (H100).

nvcc cross-compiles without a GPU.  Numerics flags are part of the parity
contract (see csrc/kernels.cu): no FMA contraction on device or host, IEEE
division and square root, no flush-to-zero.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200vis.so")
SOURCES = ["kernels.cu", "api.cu", "host_view.cpp"]
HEADERS = ["device_types.cuh", "kernels.cuh", "tile_kernel_1b.cuh","host_view.hpp", os.path.join("..", "..", "include", "b200vis.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-O2,-ffp-contract=off,-fno-fast-math,-fvisibility=hidden",
    "-shared", "-cudart", "static",
]


def _newer_than_lib(paths):
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in paths)


def build(force=False, verbose=False):
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    deps = srcs + [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    if not force and not _newer_than_lib(deps):
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    tmp = LIB + ".tmp%d" % os.getpid()     # link into a scratch name, then rename: a reader never sees a half-written library
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + srcs
    env = dict(os.environ)
    env.pop("CC", None); env.pop("CXX", None)
    res = subprocess.run(cmd + ["-ccbin", "/usr/bin/g++"], env=env, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed building libb200vis.so")
    os.replace(tmp, LIB)
    if verbose:
        sys.stderr.write(res.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
