"""CPU oracle and golden fixtures for the FP8 KV cache (`--kv_cache_dtype fp8`; TEST INFRASTRUCTURE ONLY, like oracle/).

HF's attention modules (LlamaAttention, Qwen2Attention, MixtralAttention) attend over the tensors their cache's `update()`
returns, in prefill and in every decode step.  `Fp8KVCache.update` rounds the k (after RoPE) and v states it is handed
with `kserve_b200.fp8.quantize_kv` before storing them, so transformers' own generate computes exactly what an FP8 KV
cache holds: bf16(e4m3(clamp(x, -448, 448))).  The oracle model is hooked so that the unchanged
`OracleGenerativeModel.create_completion` passes a fresh Fp8KVCache to each `generate` call.

Each fixture `<twin>_kv8.npz` repeats an existing bf16 fixture `<twin>.npz` (same config, seed, prompts, lengths) with the
FP8 cache, so every pair is also a negative control: the logits of the two differ by more than the parity tolerance.
(`tiny_kv8_*` are unrelated: the 8-KV-head config.)  Run from the repo root:

    python -m tools.kv8_oracle            # the tiny cases (~1 min)
    python -m tools.kv8_oracle --big      # + the Llama-3-8B-shape 4 x 1024 case (a few minutes, ~12 GB RAM)
    python -m tools.kv8_oracle --only tiny_g4_ids
"""
from __future__ import annotations

import argparse
import functools
import json
import os
import sys

import numpy as np
import torch
import transformers
from transformers import DynamicCache

from kserve_b200.fp8 import quantize_kv
from oracle.hf_oracle import OracleGenerativeModel
from oracle.make_goldens import GOLDEN, sub_columns, topk_pack
from tools import synth_weights as W
from tools.qwen2_oracle import build_model

TINY = ("tiny_g4_ids", "tiny_g4_peaked", "tiny_qwen2_ids", "tiny_qwen2_peaked", "tiny_moe_ids")
BIG = ("llama3_8b_2l_b4",)


class Fp8KVCache(DynamicCache):
    """a DynamicCache that stores (and hands back to attention) the FP8 KV cache's values of k and v"""

    def update(self, key_states, value_states, layer_idx, *args, **kwargs):
        return super().update(quantize_kv(key_states).to(key_states.dtype), quantize_kv(value_states).to(value_states.dtype),
                              layer_idx, *args, **kwargs)


def kv8_name(twin: str) -> str:
    return twin + "_kv8"


def twin_case(twin: str):
    """(meta, prompt rows) of the bf16 fixture"""
    z = np.load(os.path.join(GOLDEN, twin + ".npz"))
    meta = json.loads(str(z["meta"]))
    ids = z["output_ids"]
    S = ids.shape[1] - meta["completion_tokens"] // ids.shape[0]
    return meta, ids[:, :S].tolist()


def oracle_model(meta, kv8: bool = True):
    cfg = W.CONFIGS[meta["cfg"]]
    sd = W.synth_state_dict(cfg, meta["seed"])
    model = build_model(cfg, sd)
    if kv8:
        gen = model.generate
        model.generate = functools.wraps(gen)(lambda *a, **kw: gen(*a, past_key_values=Fp8KVCache(), **kw))
    return model, sd


def run(twin: str):
    """-> (meta, OracleResult) of the FP8-KV oracle on the twin's case"""
    meta, prompt = twin_case(twin)
    model, sd = oracle_model(meta)
    orc = OracleGenerativeModel(model, pad_token_id=meta["pad_token_id"])
    res = orc.create_completion(prompt, max_tokens=meta["max_tokens"], stop=(), temperature=0, want_logits=True)
    return meta, res, model, sd


def gen_case(twin: str, big: bool = False):
    meta, res, model, sd = run(twin)
    cfg = W.CONFIGS[meta["cfg"]]
    tv, ti = topk_pack(res.step_logits)
    out = dict(output_ids=res.output_ids.numpy(), topk_vals=tv, topk_idx=ti,
               meta=json.dumps(dict(
                   meta, name=kv8_name(twin), twin=twin, kv_cache_dtype="fp8", finish_reason=res.finish_reason,
                   prompt_tokens=res.prompt_tokens, completion_tokens=res.completion_tokens, texts=res.texts,
                   weights_checksum=None if big else W.checksum(sd), transformers=transformers.__version__,
                   torch=torch.__version__, threads=torch.get_num_threads())))
    logits = torch.stack(res.step_logits, 1)                     # [B, T, V]
    if big:
        cols = sub_columns(cfg["vocab_size"])
        out["sub_cols"] = cols.numpy().astype(np.int32)
        out["sub_logits"] = logits[..., cols].numpy().astype(np.float16)
    else:
        assert logits.numel() * 4 <= (1 << 20), f"{twin}: full logits would exceed 1 MB"
        out["step_logits"] = logits.numpy().astype(np.float32)
    path = os.path.join(GOLDEN, kv8_name(twin) + ".npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: ids {out['output_ids'].shape} margins(top1-top2) min={float((tv[..., 0] - tv[..., 1]).min()):.4f}",
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big", action="store_true")
    ap.add_argument("--only", default=None, help="comma separated twin names: generate just these")
    args = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    names = list(TINY) + (list(BIG) if args.big else [])
    if args.only:
        names = [n for n in args.only.split(",")]
    for n in names:
        gen_case(n, big=n in BIG)


if __name__ == "__main__":
    sys.exit(main())
