"""Throughput of one served model family on synthetic weights, timed the way bench.py times Llama-3-8B.

    python tools/model_bench.py                       # Qwen2.5-7B dims (28 layers), batch 32, 1024-in / 128-out
    python tools/model_bench.py --model qwen3_8b              # Qwen3-8B dims (36 layers, per-head q / k norms)
    python tools/model_bench.py --model llama3_8b --steps 3
    python tools/model_bench.py --model llama3_8b --weights fp8       # FP8 projections (e4m3 + a bf16 scale per row)
    python tools/model_bench.py --model llama3_8b --kv-cache fp8      # FP8 KV cache (one e4m3 code per K / V element)

The prompt is staged on the device once; each timed step is one prefill + (gen_len - 1) decode steps, measured with CUDA
events on the engine stream (b200_run_staged_timed).  Prints one JSON line: output tok/s, TTFT, decode ms/step, and the
shares of the H100's HBM bandwidth and dense BF16 tensor rate those times reach against the algorithmic bytes / FLOPs
(weights + KV bytes per decode step, GEMM + attention FLOPs of the prefill), with the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12     # H100 SXM data sheet
BF16_FLOPS = 989e12           # H100 SXM data sheet, dense


def algorithmic(cfg, B, S, T, fp8=False, kv8=False):
    H, I, V, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"], cfg["num_hidden_layers"]
    nh, nkv, d = cfg["num_attention_heads"], cfg["num_key_value_heads"], cfg.get("head_dim") or H // cfg["num_attention_heads"]
    layer = (nh + 2 * nkv) * d * H + H * nh * d + 3 * H * I       # q/k/v, o, gate/up/down weights
    gemm_params = L * layer + V * H                                # + LM head (the embedding is a gather)
    kv_per_token = 2 * L * nkv * d * (1 if kv8 else 2)           # k and v, bf16 or e4m3 codes
    mean_ctx = S + T / 2
    # FP8: one byte per projection weight plus a bf16 scale per row; the LM head stays bf16
    weight_bytes = (L * (layer + 2 * ((nh + 2 * nkv) * d + 2 * H + 2 * I)) + 2 * V * H) if fp8 else 2 * gemm_params
    decode_bytes = weight_bytes + B * mean_ctx * kv_per_token
    attn_flops = 4 * L * nh * d * (S * (S + 1) / 2) * B           # causal QK^T and PV
    prefill_flops = 2 * L * layer * B * S + 2 * V * H * B + attn_flops   # (the LM head runs on the last row only)
    return dict(weight_bytes=weight_bytes, kv_bytes_per_token=kv_per_token, decode_bytes_per_step=decode_bytes,
                prefill_flops=prefill_flops)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:     # the numbers are still printed; the card is then unknown
        return dict(name="unknown", error=str(e))


def device_weights(cfg, device, fp8=False):
    """random weights generated on the device one tensor at a time (the bench.py recipe; biases ~ N(0, 0.5)); with fp8
    every projection becomes e4m3 codes of the same draw and a per-row scale (amax / 448), the LM head stays bf16"""
    import torch
    from kserve_b200.model_spec import llama_tensor_specs
    if cfg.get("tie_word_embeddings"):
        raise SystemExit("tied checkpoints are not timed by this tool")
    g = torch.Generator(device=device).manual_seed(0)
    for name, shape, kind in llama_tensor_specs(cfg):
        if kind == "norm":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        elif kind == "embed":
            t = torch.randn(shape, generator=g, device=device)
        elif kind == "bias":
            t = 0.5 * torch.randn(shape, generator=g, device=device)
        else:
            t = torch.randn(shape, generator=g, device=device) * (shape[-1] ** -0.5)
        if fp8 and kind == "linear" and name.startswith("model.layers."):
            scale = (t.abs().amax(dim=1, keepdim=True) / 448.0).to(torch.bfloat16)
            yield name, (t / scale.float()).to(torch.float8_e4m3fn)
            yield name + "_scale", scale
            del t
            continue
        yield name, t.to(torch.bfloat16)
        del t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="qwen2_7b", help="a tools/synth_weights.py CONFIGS name")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--prompt-len", type=int, default=1024)
    ap.add_argument("--gen-len", type=int, default=128)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--weights", choices=("bf16", "fp8"), default="bf16")
    ap.add_argument("--kv-cache", choices=("bf16", "fp8"), default="bf16")
    args = ap.parse_args()
    from tools.synth_weights import CONFIGS
    cfg = CONFIGS[args.model]
    B, S, T = args.batch, args.prompt_len, args.gen_len
    fp8 = args.weights == "fp8"
    kv8 = args.kv_cache == "fp8"
    alg = algorithmic(cfg, B, S, T, fp8, kv8)

    import torch
    from kserve_b200.engine import B200Engine
    if not torch.cuda.is_available():
        raise SystemExit("model_bench needs a CUDA device: there is no CPU path to time")
    eng = B200Engine(cfg, max_batch=B, max_seq_len=S + T, max_prefill_tokens=B * S, weight_format=1 if fp8 else 0,
                     kv_cache_dtype=1 if kv8 else 0)
    eng.load_weights(device_weights(cfg, torch.device("cuda", 0), fp8))
    torch.cuda.empty_cache()
    g = torch.Generator().manual_seed(1234)
    ids = torch.randint(3, min(128000, cfg["vocab_size"] - 8), (B, S), generator=g, dtype=torch.int64).pin_memory()
    eng.stage(ids, None, max_new_tokens=T, pad_token_id=cfg["vocab_size"] - 1)
    for _ in range(args.warmup):
        eng.run_staged_timed(T - 1)
    torch.cuda.synchronize()
    pre, dec = [], []
    for _ in range(args.steps):
        a, b = eng.run_staged_timed(T - 1)
        pre.append(a)
        dec.append(b)
    eng.close()
    step_ms = (sum(pre) + sum(dec)) / args.steps
    ttft = statistics.median(pre)
    dec_step = statistics.median(dec) / (T - 1)
    line = dict(
        model=args.model, weights=args.weights, kv_cache=args.kv_cache, batch=B, prompt_len=S, gen_len=T, steps=args.steps, warmup=args.warmup,
        tok_per_s=round(B * T / (step_ms / 1e3), 1), ttft_ms=round(ttft, 1), decode_ms_per_step=round(dec_step, 3),
        ttft_ms_all=[round(x, 1) for x in pre], decode_ms_per_step_all=[round(x / (T - 1), 3) for x in dec],
        decode_bytes_per_step=alg["decode_bytes_per_step"], weight_bytes=alg["weight_bytes"],
        kv_bytes_per_token=alg["kv_bytes_per_token"], prefill_flops=alg["prefill_flops"],
        decode_hbm_fraction=round(alg["decode_bytes_per_step"] / HBM_BYTES_PER_S / (dec_step / 1e3), 3),
        decode_floor_ms=round(alg["decode_bytes_per_step"] / HBM_BYTES_PER_S * 1e3, 3),
        prefill_tensor_fraction=round(alg["prefill_flops"] / BF16_FLOPS / (ttft / 1e3), 3),
        card=card())
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
