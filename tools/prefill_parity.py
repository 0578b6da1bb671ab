"""Bitwise parity of the prefill GEMM epilogues between two library builds.

    B200_LIB_PATH=old.so python tools/prefill_parity.py --out old.json
    B200_LIB_PATH=new.so python tools/prefill_parity.py --out new.json
    python tools/prefill_parity.py --compare old.json new.json

Each case runs b200_op_gemm on seeded inputs into an output buffer that has 64 sentinel rows past M, and records
the sha256 of the whole buffer (sentinel rows included).  Cases: the four Llama-3-8B layer shapes at T = 32768 and
the tails M in {1, 127, 129, 300, 1000, 4100} of every row-major epilogue, with N / out_cols tails.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--out")
ap.add_argument("--compare", nargs=2)
args = ap.parse_args()

if args.compare:
    a, b = (json.load(open(f)) for f in args.compare)
    bad = [k for k in a if a[k] != b.get(k)]
    print(f"{len(a) - len(bad)}/{len(a)} cases bit-identical" + (f"; differ: {bad}" if bad else ""))
    sys.exit(1 if bad or set(a) != set(b) else 0)

import torch  # noqa: E402

path = os.environ.get("B200_LIB_PATH") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kserve_b200", "lib", "libkserve_b200.so")
lib = C.CDLL(path)
vp, i64 = C.c_void_p, C.c_int64
lib.b200_op_gemm.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, i64, vp]
lib.b200_last_error.restype = C.c_char_p
p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None


def rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def run(M, N, K, epi, seed):
    A = rand((M, K), seed)
    W = rand((N, K), seed + 1, K ** -0.5)
    ocols = N // 2 if epi == 2 else N
    O = rand((M + 64, ocols), seed + 2) if epi == 1 else torch.full((M + 64, ocols), -7.0, device="cuda", dtype=torch.bfloat16)
    res = O if epi == 1 else None
    rc = lib.b200_op_gemm(p(A), p(W), p(O), p(res), M, N, K, epi, 256, 1, ocols, None)
    assert rc == 0, lib.b200_last_error()
    torch.cuda.synchronize()
    return hashlib.sha256(O.view(torch.int16).cpu().numpy().tobytes()).hexdigest()


cases = {}
for name, N, K, epi in [("qkv", 6144, 4096, 0), ("o+res", 4096, 4096, 1), ("gate_up", 28672, 4096, 2), ("down+res", 4096, 14336, 1)]:
    cases[f"{name}/T32768"] = run(32768, N, K, epi, 11)
for M in (1, 127, 129, 300, 1000, 4100):
    for epi, N, K in ((0, 1031, 512), (0, 6144, 4096), (1, 520, 1024), (1, 4096, 4096), (2, 1056, 512), (2, 2 * 2816, 1024)):
        cases[f"epi{epi}/M{M}/N{N}/K{K}"] = run(M, N, K, epi, 100 + M)
with open(args.out, "w") as f:
    json.dump(cases, f, indent=1)
print(f"{len(cases)} cases -> {args.out}", flush=True)
