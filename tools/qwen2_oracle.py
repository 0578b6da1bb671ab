"""CPU oracle and golden fixtures for Qwen2 / Qwen2.5 decoders (TEST INFRASTRUCTURE ONLY, like oracle/).

transformers' Qwen2ForCausalLM, built from the seeded synthetic checkpoints of tools/synth_weights.py, stands where the
reference's `AutoModelForCausalLM.from_pretrained` would load a Qwen2 checkpoint.  The fixtures have the layout of
oracle/make_goldens.py's (tests/helpers.py: load_case reads both).  Run from the repo root:

    python -m tools.qwen2_oracle            # the tiny Qwen2 cases (~20 s)
    python -m tools.qwen2_oracle --big      # + the Qwen2.5-7B-shape cases (~1 min, 10 GB RAM)
    python -m tools.qwen2_oracle --only tiny_qwen2_ids,tiny_qwen2_peaked
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from typing import Dict

import numpy as np
import torch
import transformers

from oracle.hf_oracle import OracleGenerativeModel
from oracle.hf_oracle import build_model as build_llama_family
from oracle.make_goldens import GOLDEN, ids_prompt, sub_columns, topk_pack
from tools import synth_weights as W


def build_qwen2(cfg: dict, state_dict: Dict[str, torch.Tensor], dtype=torch.bfloat16):
    """Qwen2ForCausalLM (q / k / v projections with bias) from config + seeded weights; full attention, the lm_head tied
    to the embedding when the config says so (the checkpoint then has no lm_head.weight)."""
    from transformers import Qwen2Config, Qwen2ForCausalLM
    cfg = {k: v for k, v in cfg.items() if not k.startswith("_") and k != "model_type"}
    cfg["use_sliding_window"] = False
    cfg.setdefault("tie_word_embeddings", False)
    hf_cfg = Qwen2Config(**cfg, eos_token_id=None, bos_token_id=None, pad_token_id=None)
    with torch.device("meta"):
        model = Qwen2ForCausalLM(hf_cfg)
    model = model.to_empty(device="cpu").to(dtype)
    missing, unexpected = model.load_state_dict(state_dict, strict=False, assign=True)
    assert not unexpected, unexpected
    if hf_cfg.tie_word_embeddings:
        model.lm_head.weight = model.model.embed_tokens.weight
        missing = [m for m in missing if m != "lm_head.weight"]
    # rotary inv_freq is a non-persistent buffer: to_empty() left it uninitialised, and it stays fp32
    n_fixed = 0
    for mod in model.modules():
        if hasattr(mod, "inv_freq"):
            inv_freq, scaling = type(mod).compute_default_rope_parameters(mod.config, "cpu")
            mod.register_buffer("inv_freq", inv_freq.float(), persistent=False)
            mod.register_buffer("original_inv_freq", inv_freq.float().clone(), persistent=False)
            mod.attention_scaling = scaling
            n_fixed += 1
    assert n_fixed >= 1
    assert not [m for m in missing if "inv_freq" not in m], missing
    model.eval()
    return model


def build_model(cfg: dict, state_dict, dtype=torch.bfloat16):
    """Qwen2 configs (model_type "qwen2") -> Qwen2ForCausalLM; everything else as oracle.hf_oracle.build_model"""
    if cfg.get("model_type") == "qwen2":
        return build_qwen2(cfg, state_dict, dtype)
    return build_llama_family(cfg, state_dict, dtype)


ONLY = None         # --only: the case names to (re)generate


def gen_case(name, cfg_name, seed, prompt, max_tokens, pad_token_id, sub_logits=False, build=None):
    """greedy generate of the oracle with every step's logits -> tests/golden/<name>.npz (full logits, or for a big
    vocabulary the logits on make_goldens.sub_columns + the top-16); `build` (config, state dict) -> model, default
    build_model"""
    if ONLY is not None and name not in ONLY:
        return
    cfg = W.CONFIGS[cfg_name]
    sd = W.synth_state_dict(cfg, seed)
    model = (build or build_model)(cfg, sd)
    orc = OracleGenerativeModel(model, pad_token_id=pad_token_id)
    res = orc.create_completion(prompt, max_tokens=max_tokens, stop=(), temperature=0, want_logits=True)
    tv, ti = topk_pack(res.step_logits)
    out = dict(
        output_ids=res.output_ids.numpy(), topk_vals=tv, topk_idx=ti,
        meta=json.dumps(dict(
            name=name, cfg=cfg_name, seed=seed, max_tokens=max_tokens, finish_reason=res.finish_reason,
            prompt_tokens=res.prompt_tokens, completion_tokens=res.completion_tokens, texts=res.texts,
            pad_token_id=orc.pad_token_id, vocab_rows=int(model.get_input_embeddings().weight.shape[0]),
            weights_checksum=W.checksum(sd), stop=[], prompt=None, echo=False, presence_penalty=None,
            transformers=transformers.__version__, torch=torch.__version__, threads=torch.get_num_threads())))
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
          f"margins(top1-top2) min={float((tv[..., 0] - tv[..., 1]).min()):.4f}")


def qwen2_prompts(B, S, vocab_hi, seed):
    """token-id prompts whose row 2 repeats row 0's first two 128-token blocks (prefix reuse in the continuous batcher)"""
    rows = ids_prompt(B, S, vocab_hi, seed)
    if B > 2 and S > 256:
        rows[2][:256] = rows[0][:256]
    return rows


def qwen2_cases():
    """GQA groups 7 (split-K decode QKV), 6 (tied embeddings) and 5, and 80 m-tiles of decode QKV (bf16 EPI_T_STORE
    epilogue).  The peaked case's 300-token prompts cross 128-token chunks."""
    gen_case("tiny_qwen2_ids", "tiny_qwen2", 7, ids_prompt(4, 70, 1000, 707), 16, pad_token_id=1030)
    gen_case("tiny_qwen2_peaked", "tiny_qwen2_peaked", 7, qwen2_prompts(4, 300, 1000, 717), 16, pad_token_id=1030)
    gen_case("tiny_qwen2_g6_tied_ids", "tiny_qwen2_g6_tied", 8, ids_prompt(3, 100, 1000, 808), 16, pad_token_id=1030)
    gen_case("tiny_qwen2_g5_ids", "tiny_qwen2_g5", 9, ids_prompt(3, 65, 1000, 909), 16, pad_token_id=1030)
    gen_case("tiny_qwen2_wide_ids", "tiny_qwen2_wide", 10, ids_prompt(4, 70, 1000, 1010), 16, pad_token_id=1030)


def qwen2_big_cases():
    """Qwen2.5-7B layer shapes (2 layers): 4 x 1024-token prompts, V = 152064"""
    pad = 152063
    for name, cfg_name in (("qwen2_7b_2l_b4", "qwen2_7b_2l"), ("qwen2_7b_2l_peaked_b4", "qwen2_7b_2l_peaked")):
        gen_case(name, cfg_name, 0, ids_prompt(4, 1024, 150000, 2026), 16, pad_token_id=pad, sub_logits=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big", action="store_true")
    ap.add_argument("--only", default=None, help="comma separated case names: generate just these")
    args = ap.parse_args()
    global ONLY
    ONLY = set(args.only.split(",")) if args.only else None
    torch.set_num_threads(os.cpu_count())
    qwen2_cases()
    if args.big:
        qwen2_big_cases()


if __name__ == "__main__":
    sys.exit(main())
