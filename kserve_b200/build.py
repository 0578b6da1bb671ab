"""In-tree build of the sm_90a shared library (nvcc cross-compiles without a GPU).

    python -m kserve_b200.build [--force]

Output: kserve_b200/lib/libkserve_b200.so (git-ignored, travels to the GPU box with the snapshot).
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libkserve_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-diag-suppress", "177",
]
SOURCES = ["engine.cu"]


def _newest_source_mtime() -> float:
    m = 0.0
    for root, _, files in os.walk(CSRC):
        for f in files:
            m = max(m, os.path.getmtime(os.path.join(root, f)))
    m = max(m, os.path.getmtime(os.path.join(os.path.dirname(HERE), "include", "kserve_b200.h")))
    return m


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIB_DIR, exist_ok=True)
    if not force and os.path.exists(LIB_PATH) and os.path.getmtime(LIB_PATH) >= _newest_source_mtime():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    cmd = [nvcc, *NVCC_FLAGS, *srcs, "-o", LIB_PATH, "-ldl", "-lpthread"]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
        print(" ".join(cmd))
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building libkserve_b200.so")
    if verbose:
        print(res.stderr)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
