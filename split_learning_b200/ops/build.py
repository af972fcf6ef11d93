"""Build the sm_90a kernel library in-tree: ``ops/_slb200.so`` (plain C ABI, loaded by
ctypes — no torch headers, seconds to compile, and it travels to the GPU box with the tree).

    python -m split_learning_b200.ops.build [--force]
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["umma_gemm.cu", "fused_cut.cu", "elementwise.cu", "transformer.cu", "allreduce.cu", "ticket.cu", "peer.cu"]
LIB = os.path.join(HERE, "_slb200.so")
STAMP = LIB + ".sha"
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "--shared", "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-lcudart"] + os.environ.get("SLB200_NVCC_EXTRA", "").split()


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def _digest() -> str:
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for f in sorted(os.listdir(CSRC)):
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(f.encode() + fh.read())
    return h.hexdigest()


def is_stale() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        return f.read().strip() != _digest()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    cmd = [_nvcc()] + NVCC_FLAGS + ["-o", LIB] + sources()
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(HERE, "_slb200.build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + log[-4000:])
    if verbose:
        print(log)
    with open(STAMP, "w") as f:
        f.write(_digest())
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
