"""CPU oracle and golden fixtures for FP8 (compressed-tensors) checkpoints (TEST INFRASTRUCTURE ONLY, like oracle/).

Each FP8 config of tools/synth_weights.py is written as a real compressed-tensors checkpoint directory (safetensors +
config.json with its quantization_config) and loaded with `AutoModelForCausalLM.from_pretrained` on the CPU — the call
the reference makes — so transformers' own decompression, not a restatement of it, produces the fixtures.  They have the
layout tests/helpers.py reads.  Run from the repo root:

    python -m tools.fp8_oracle            # the tiny FP8 cases (~30 s)
    python -m tools.fp8_oracle --big      # + the Llama-3-8B-shape cases (a few minutes, ~12 GB RAM, ~2.5 GB temp disk)
    python -m tools.fp8_oracle --only tiny_g4_fp8_ids
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch
import transformers

from oracle.hf_oracle import OracleGenerativeModel
from oracle.make_goldens import GOLDEN, ids_prompt, sub_columns, topk_pack
from tools import synth_weights as W


def write_checkpoint(d: str, cfg_name: str, seed: int, scale_override=None) -> str:
    """the seeded FP8 config as a compressed-tensors directory.  scale_override(name, scale) -> scale replaces the
    weight_scale tensors (negative controls)"""
    from safetensors.torch import save_file
    cfg = W.CONFIGS[cfg_name]
    sd = {}
    for name, t in W.iter_state_dict(cfg, seed):
        if scale_override is not None and name.endswith(".weight_scale"):
            t = scale_override(name, t)
        sd[name] = t.contiguous()
    save_file(sd, os.path.join(d, "model.safetensors"))
    hf = dict(W.hf_config_dict(cfg), torch_dtype="bfloat16", hidden_act="silu", eos_token_id=None, bos_token_id=None,
              pad_token_id=None, tie_word_embeddings=bool(cfg.get("tie_word_embeddings")),
              quantization_config=W.fp8_quantization_config(cfg["_fp8"]))
    hf.setdefault("model_type", "llama")
    hf["architectures"] = ["Qwen2ForCausalLM" if hf["model_type"] == "qwen2" else "LlamaForCausalLM"]
    if hf["model_type"] == "qwen2":
        hf["use_sliding_window"] = False
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(hf, f)
    return d


def load_oracle(cfg_name: str, seed: int, scale_override=None):
    """transformers' model of the FP8 checkpoint (weights decompressed to bf16 by its compressed-tensors integration)"""
    from transformers import AutoModelForCausalLM
    with tempfile.TemporaryDirectory() as d:
        write_checkpoint(d, cfg_name, seed, scale_override)
        model = AutoModelForCausalLM.from_pretrained(d, dtype=torch.bfloat16)
    model.eval()
    with torch.no_grad():
        model(torch.tensor([[1, 2]]))           # the first forward decompresses every projection
    return model


ONLY = None


def gen_case(name, cfg_name, seed, prompt, max_tokens, pad_token_id, sub_logits=False):
    if ONLY is not None and name not in ONLY:
        return
    cfg = W.CONFIGS[cfg_name]
    model = load_oracle(cfg_name, seed)
    orc = OracleGenerativeModel(model, pad_token_id=pad_token_id)
    res = orc.create_completion(prompt, max_tokens=max_tokens, stop=(), temperature=0, want_logits=True)
    tv, ti = topk_pack(res.step_logits)
    out = dict(
        output_ids=res.output_ids.numpy(), topk_vals=tv, topk_idx=ti,
        meta=json.dumps(dict(
            name=name, cfg=cfg_name, seed=seed, max_tokens=max_tokens, finish_reason=res.finish_reason,
            prompt_tokens=res.prompt_tokens, completion_tokens=res.completion_tokens, texts=res.texts,
            pad_token_id=orc.pad_token_id, vocab_rows=int(model.get_input_embeddings().weight.shape[0]),
            weights_checksum=W.checksum(W.synth_state_dict(cfg, seed)) if not sub_logits else None, stop=[], prompt=None,
            echo=False, presence_penalty=None, transformers=transformers.__version__, torch=torch.__version__,
            threads=torch.get_num_threads())))
    logits = torch.stack(res.step_logits, 1)                     # [B, T, V]
    if sub_logits:
        cols = sub_columns(cfg["vocab_size"])
        out["sub_cols"] = cols.numpy().astype(np.int32)
        out["sub_logits"] = logits[..., cols].numpy().astype(np.float16)
    else:
        assert logits.numel() * 2 <= (1 << 20), f"{name}: full logits would exceed 1 MB"
        out["step_logits"] = logits.numpy().astype(np.float32)
    path = os.path.join(GOLDEN, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: ids {out['output_ids'].shape} finish={res.finish_reason} "
          f"margins(top1-top2) min={float((tv[..., 0] - tv[..., 1]).min()):.4f}", flush=True)


# name -> (config, seed, prompt args (B, S, vocab_hi, seed), max_tokens, pad); prompts of the peaked case cross 128-token chunks
TINY_CASES = {
    "tiny_g4_fp8_ids": ("tiny_g4_fp8", 4, (4, 70, 2000, 404), 16, 2047),
    "tiny_g4_fp8_peaked": ("tiny_g4_fp8_peaked", 4, (4, 300, 2000, 414), 16, 2047),
    "tiny_qwen2_fp8_ids": ("tiny_qwen2_fp8", 7, (4, 70, 1000, 727), 16, 1030),
    "tiny_g2_fp8_tensor_ids": ("tiny_g2_fp8_tensor", 2, (3, 90, 1000, 202), 16, 1030),
}
BIG_CASES = {
    "llama3_8b_2l_fp8_b4": ("llama3_8b_2l_fp8", 0, (4, 1024, 128000, 2027), 16, 128255),
    "llama3_8b_2l_fp8_peaked_b4": ("llama3_8b_2l_fp8_peaked", 0, (4, 1024, 128000, 2027), 16, 128255),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big", action="store_true")
    ap.add_argument("--only", default=None, help="comma separated case names: generate just these")
    args = ap.parse_args()
    global ONLY
    ONLY = set(args.only.split(",")) if args.only else None
    torch.set_num_threads(os.cpu_count())
    for name, (cfg_name, seed, pr, T, pad) in TINY_CASES.items():
        gen_case(name, cfg_name, seed, ids_prompt(*pr), T, pad)
    if args.big:
        for name, (cfg_name, seed, pr, T, pad) in BIG_CASES.items():
            gen_case(name, cfg_name, seed, ids_prompt(*pr), T, pad, sub_logits=True)


if __name__ == "__main__":
    sys.exit(main())
