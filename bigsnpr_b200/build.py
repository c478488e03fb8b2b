"""Builds libbsgpu.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m bigsnpr_b200.build [--force]

The shared object lands next to this file (bigsnpr_b200/libbsgpu.so) and is git-ignored.  nvcc
cross-compiles without a GPU.
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libbsgpu.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O2,-Wall,-Wno-unused-function",
    "-shared",
    "-I", os.path.join(ROOT, "include"),
    "-I", CSRC,
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(ROOT, "include", "bsgpu.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + sources() + ["-lcublas"]
    env = dict(os.environ)
    r = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if verbose or r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode:
        raise RuntimeError("nvcc failed building libbsgpu.so")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
