"""Builds libx265cu.so (hand-written sm_90a CUDA, single translation unit) in-tree with nvcc."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libx265cu.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared",
              "-Xcompiler", "-ffp-contract=off"]          # host code: x265cu_aq_finish rounds as the reference does


def _newest_source():
    t = 0.0
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            if f.endswith((".cu", ".cuh", ".h")):
                t = max(t, os.path.getmtime(os.path.join(root, f)))
    return t


def build(force=False, verbose=False):
    if os.environ.get("X265CU_LIB"):          # experiment hook: use a specific prebuilt variant
        return os.environ["X265CU_LIB"]
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest_source():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        if os.path.exists(LIB):
            return LIB          # GPU box without nvcc on PATH: use the prebuilt library that travelled
        raise RuntimeError("nvcc not found and no prebuilt libx265cu.so")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", LIB, os.path.join(CSRC, "x265cu.cu")]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
