"""Build libcalm_b200.so in-tree with nvcc for sm_90a (no JIT cache: the library is built once, next to the sources)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcalm_b200.so")
SOURCES = ["engine.cu"]
HEADERS = ["common.cuh", "stages.cuh", os.path.join("..", "..", "include", "calm_b200.h"), os.path.join("..", "..", "include", "calm_model.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-ccbin", "/usr/bin/g++",
         "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function", "-shared"]


def stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    deps += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return LIB
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu")]
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + sorted(srcs) + ["-o", LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building libcalm_b200.so")
    if verbose:
        sys.stderr.write(r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
