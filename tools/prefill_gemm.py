"""Prefill GEMM throughput (TFLOP/s) through b200_op_gemm for the Llama-3-8B layer shapes at T=32768, next to
torch.mm (cuBLAS) on the same card; can load an alternative library build (B200_LIB_PATH) for A/B on the same box.

    python tools/prefill_gemm.py [--reps 20]
"""
import argparse
import ctypes as C
import os
import subprocess

import torch

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--no-cublas", action="store_true")
args = ap.parse_args()

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name()
path = os.environ.get("B200_LIB_PATH") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kserve_b200", "lib", "libkserve_b200.so")
lib = C.CDLL(path)
vp, i64 = C.c_void_p, C.c_int64
lib.b200_op_gemm.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, i64, vp]
lib.b200_last_error.restype = C.c_char_p
T = 32768
dev = "cuda"
p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


out = []
for name, N, K, epi in [("qkv", 6144, 4096, 0), ("o+res", 4096, 4096, 1), ("gate_up", 28672, 4096, 2), ("down+res", 4096, 14336, 1)]:
    A = torch.randn(T, K, device=dev, dtype=torch.bfloat16)
    W = torch.randn(N, K, device=dev, dtype=torch.bfloat16) * K ** -0.5
    ocols = N // 2 if epi == 2 else N
    O = torch.zeros(T, ocols, device=dev, dtype=torch.bfloat16)
    res = O if epi == 1 else None
    assert lib.b200_op_gemm(p(A), p(W), p(O), p(res), T, N, K, epi, 256, 1, ocols, None) == 0, lib.b200_last_error()
    ms = timed(lambda: lib.b200_op_gemm(p(A), p(W), p(O), p(res), T, N, K, epi, 256, 1, ocols, None), args.reps)
    flop = 2 * T * N * K
    s = f"{name}: {ms:.3f} ms {flop / ms / 1e9:.0f} TF/s"
    if not args.no_cublas:
        C_ = torch.empty(T, N, device=dev, dtype=torch.bfloat16)
        ms_ref = timed(lambda: torch.mm(A, W.t(), out=C_), args.reps)
        s += f" (cuBLAS mm {ms_ref:.3f} ms {flop / ms_ref / 1e9:.0f} TF/s)"
    out.append(s)
    del A, W, O
print(card, "|", os.path.basename(os.path.dirname(path)), "|", " | ".join(out), flush=True)
