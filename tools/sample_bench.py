"""Time sample_kernel alone (b200_op_sample, CUDA events) and record the tokens it draws.

    python tools/sample_bench.py [--out DIR]        # B200_LIB_PATH selects the library build to measure

B = 64 rows of Gaussian bf16 logits (standard deviation 1.5 to 4), V = 128256, top_k 50 and 1024.  Prints one JSON line
with the card name and power limit read in the same run, the mean time per launch, and (with --out) writes the tokens
drawn on fixed seeds for several configurations, so two builds can be compared draw for draw."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kserve_b200 import _lib  # noqa: E402

CONFIGS = {"k50": dict(do_sample=1, top_k=50), "k1024": dict(do_sample=1, top_k=1024),
           "llama3_instruct": dict(do_sample=1, temperature=0.6, top_p=0.9, top_k=50),
           "qwen25_instruct": dict(do_sample=1, temperature=0.7, top_p=0.8, top_k=20, repetition_penalty=1.05),
           "p0.999": dict(do_sample=1, top_p=0.999, top_k=200), "t5": dict(do_sample=1, temperature=5.0, top_k=100)}


def params(c, seed):
    g = _lib.GenParams()
    g.repetition_penalty = c.get("repetition_penalty", 0.0)
    g.do_sample, g.temperature = c.get("do_sample", 0), c.get("temperature", 0.0)
    g.top_p, g.top_k, g.seed = c.get("top_p", 0.0), c.get("top_k", 0), seed
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    lib = _lib.load()
    B, V = 64, 128256
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(B, V, generator=g) * (1.5 + 2.5 * torch.rand(B, 1, generator=g))).bfloat16().cuda()
    seen = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, (V + 31) // 32), generator=g, dtype=torch.int32).cuda()
    out_val = torch.empty(B, dtype=torch.float32, device="cuda")
    out_idx = torch.empty(B, dtype=torch.int32, device="cuda")

    def launch(c, seed, step):
        rc = lib.b200_op_sample(x.data_ptr(), V, B, V, seen.data_ptr(), None, None, 1, C.byref(params(c, seed)), step,
                                out_val.data_ptr(), out_idx.data_ptr(), None)
        assert rc == 0, lib.b200_last_error().decode()

    res = {}
    for name in ("k50", "k1024"):
        for _ in range(20):
            launch(CONFIGS[name], 1, 0)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for i in range(a.iters):
            launch(CONFIGS[name], 1, i)
        t1.record()
        torch.cuda.synchronize()
        res[f"{name}_us"] = round(1000 * t0.elapsed_time(t1) / a.iters, 2)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps(dict(lib=os.path.basename(_lib.LIB_PATH), card=card, B=B, V=V, **res)))
    if a.out:
        toks = {}
        for name, c in CONFIGS.items():
            rows = []
            for step in range(10):
                launch(c, 100 + step, step)
                rows.append(out_idx.cpu().numpy())
            toks[name] = np.stack(rows)
        os.makedirs(a.out, exist_ok=True)
        np.savez(os.path.join(a.out, os.path.basename(_lib.LIB_PATH) + ".npz"), **toks)


if __name__ == "__main__":
    main()
