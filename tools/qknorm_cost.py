"""Cost of Qwen3's q / k norm in the prefill QKV epilogue: CUDA events over b200_op_qkv_rope_kv at Qwen3-8B's QKV shape
(H 4096, 32 q heads, 8 kv heads: N = 6144), T prompt tokens in 1024-token sequences, with the norm weights NULL and set,
the two alternated.  Prints one JSON line with the card's name and power limit.

    python tools/qknorm_cost.py [--tokens 32768] [--reps 20] [--kv-cache fp8]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=32768)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--kv-cache", choices=("bf16", "fp8"), default="bf16")
    args = ap.parse_args()
    import torch
    from kserve_b200 import _lib as L
    from kserve_b200.engine import hf_rope_tables
    from tools.model_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("qknorm_cost needs a CUDA device: there is no CPU path to time")
    lib, dev = L.load(), torch.device("cuda", 0)
    H, nh, nkv, T, S = 4096, 32, 8, args.tokens, 1024
    N = (nh + 2 * nkv) * 128
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(T, H, generator=g, device=dev).to(torch.bfloat16)
    w = (torch.randn(N, H, generator=g, device=dev) * H ** -0.5).to(torch.bfloat16)
    qn = (1 + torch.rand(128, generator=g, device=dev)).to(torch.bfloat16)
    kn = (1 + torch.rand(128, generator=g, device=dev)).to(torch.bfloat16)
    out = torch.empty(T, N, dtype=torch.bfloat16, device=dev)
    B = T // S
    pages = B * (S // 64)
    kv8 = args.kv_cache == "fp8"
    kc = torch.empty(pages, nkv, 64, 128, dtype=torch.uint8 if kv8 else torch.bfloat16, device=dev)
    vc = torch.empty_like(kc)
    pt = torch.arange(pages, dtype=torch.int32, device=dev).view(B, S // 64)
    seq = torch.arange(B, dtype=torch.int32, device=dev).repeat_interleave(S)
    pos = torch.arange(S, dtype=torch.int32, device=dev).repeat(B)
    cos, sin = (t.to(dev).contiguous() for t in hf_rope_tables(1000000.0, 128, S))
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None

    def launch(norm):
        rc = lib.b200_op_qkv_rope_kv(p(x), p(w), p(out), N, T, H, nh, nkv, None, p(qn) if norm else None,
                                     p(kn) if norm else None, 1e-6, p(kc), p(vc), int(kv8), p(pt), S // 64, p(seq), p(pos),
                                     p(cos), p(sin), None)
        assert rc == 0, lib.b200_last_error()

    def timed(norm, n=5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            launch(norm)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    for norm in (False, True, False, True):
        timed(norm, 3)
    off, on = [], []
    for _ in range(args.reps):
        off.append(timed(False))
        on.append(timed(True))
    flops = 2.0 * T * N * H
    mo, mn = statistics.median(off), statistics.median(on)
    print(json.dumps(dict(tokens=T, H=H, N=N, kv_cache=args.kv_cache, reps=args.reps, ms_no_norm=round(mo, 4),
                          ms_norm=round(mn, 4), norm_cost_pct=round(100 * (mn / mo - 1), 2),
                          ms_no_norm_range=[round(min(off), 4), round(max(off), 4)], ms_norm_range=[round(min(on), 4), round(max(on), 4)],
                          tflops_no_norm=round(flops / mo / 1e9, 1), tflops_norm=round(flops / mn / 1e9, 1), card=card())), flush=True)


if __name__ == "__main__":
    main()
