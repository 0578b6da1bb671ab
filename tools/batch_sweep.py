"""BASELINE.json configs[1]: Llama-3-8B bf16 on 1xH100, batch sweep 1-64, 1024-in/128-out.  One engine, every batch
size timed like bench.py (device-resident prompt, CUDA events on the engine stream) plus the end-to-end call."""
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import LLAMA3_8B, algorithmic, gpu_weights, load_peaks  # noqa: E402
from kserve_b200.engine import B200Engine  # noqa: E402


def main():
    S, T = 1024, 128
    cfg = LLAMA3_8B
    eng = B200Engine(cfg, max_batch=64, max_seq_len=S + T, max_prefill_tokens=64 * S)
    eng.load_weights(gpu_weights(cfg, torch.device("cuda")))
    peaks = load_peaks()
    g = torch.Generator().manual_seed(1234)
    rows = []
    for B in (1, 2, 4, 8, 16, 32, 64):
        ids = torch.randint(3, 128000, (B, S), generator=g, dtype=torch.int64)
        eng.stage(ids, None, max_new_tokens=T, pad_token_id=cfg["vocab_size"] - 1)
        for _ in range(3):
            eng.run_staged_timed(T - 1)
        pre, dec = [], []
        for _ in range(3):
            a, b = eng.run_staged_timed(T - 1)
            pre.append(a); dec.append(b)
        t0 = time.perf_counter()
        eng.generate(ids, None, max_new_tokens=T, pad_token_id=cfg["vocab_size"] - 1)
        torch.cuda.synchronize()
        e2e = time.perf_counter() - t0
        alg = algorithmic(cfg, B, S, T)
        step_ms = statistics.mean(dec) / (T - 1)
        ttft = statistics.median(pre)
        total_ms = statistics.mean([p + d for p, d in zip(pre, dec)])
        rows.append(dict(batch=B, tokens_per_s=round(B * T / (total_ms / 1e3), 1), ttft_ms=round(ttft, 2),
                         decode_ms_per_step=round(step_ms, 4), decode_tokens_per_s=round(B / (step_ms / 1e3), 1),
                         hbm_frac=round(alg["decode_bytes_per_step"] / (step_ms * 1e-3) / 1e9 / peaks["hbm_gbs"], 4),
                         tensor_frac=round(alg["prefill_flops"] / (ttft * 1e-3) / 1e12 / peaks["tf_sustained"], 4),
                         e2e_tokens_per_s=round(B * T / e2e, 1)))
        print(json.dumps(rows[-1]), flush=True)
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out", "batch_sweep.json")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    json.dump(dict(workload="Llama-3-8B bf16 random-init, 1024-in/128-out, greedy, 1xH100", peaks=peaks, rows=rows), open(out, "w"), indent=1)


if __name__ == "__main__":
    main()
