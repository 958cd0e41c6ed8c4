"""Build libgms_b200.so for sm_90a (H100), in the source tree next to the Python package that loads it.

    python gaussian-mesh-splatting_b200/build.py [--force] [--verbose]
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "gms_kernels.cu")
DEPS = [SRC] + sorted(glob.glob(os.path.join(HERE, "csrc", "*.cuh"))) + \
       [os.path.join(HERE, "..", "include", "gms_b200.h"), os.path.abspath(__file__)]    # this file: FLAGS (the target arch) live here
OUT = os.path.join(HERE, "gms_b200", "libgms_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--shared",
         "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++"]


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT, SRC]
    print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(OUT)
