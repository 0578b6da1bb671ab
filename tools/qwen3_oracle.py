"""CPU oracle and golden fixtures for dense Qwen3 decoders (TEST INFRASTRUCTURE ONLY, like oracle/).

transformers' Qwen3ForCausalLM, built from the seeded synthetic checkpoints of tools/synth_weights.py (q_norm / k_norm
drawn far from 1, q / k projections with an RMS away from 1), stands where the reference's
`AutoModelForCausalLM.from_pretrained` would load a Qwen3 checkpoint.  The fixtures have the layout tests/helpers.py's
load_case reads; tools/qwen2_oracle.gen_case writes them.  Run from the repo root:

    python -m tools.qwen3_oracle            # the tiny Qwen3 cases (~20 s)
    python -m tools.qwen3_oracle --big      # + the Qwen3-8B-shape cases (a few minutes, ~12 GB RAM)
    python -m tools.qwen3_oracle --only tiny_qwen3_ids,tiny_qwen3_peaked
"""
from __future__ import annotations

import argparse
import os
import sys
from typing import Dict

import torch

from oracle.make_goldens import ids_prompt
from tools import qwen2_oracle as Q2


def build_qwen3(cfg: dict, state_dict: Dict[str, torch.Tensor], dtype=torch.bfloat16):
    """Qwen3ForCausalLM (per-head q / k RMSNorm before RoPE, no projection biases) from config + seeded weights; full
    attention, the lm_head tied to the embedding when the config says so (the checkpoint then has no lm_head.weight)."""
    from transformers import Qwen3Config, Qwen3ForCausalLM
    cfg = {k: v for k, v in cfg.items() if not k.startswith("_") and k != "model_type"}
    cfg["use_sliding_window"] = False
    cfg.setdefault("tie_word_embeddings", False)
    hf_cfg = Qwen3Config(**cfg, eos_token_id=None, bos_token_id=None, pad_token_id=None)
    with torch.device("meta"):
        model = Qwen3ForCausalLM(hf_cfg)
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
    """Qwen3 configs (model_type "qwen3") -> Qwen3ForCausalLM; everything else as tools.qwen2_oracle.build_model"""
    if cfg.get("model_type") == "qwen3":
        return build_qwen3(cfg, state_dict, dtype)
    return Q2.build_model(cfg, state_dict, dtype)


def qwen3_cases():
    """G = 2 with q dim 2H, tied embeddings and split-K decode QKV (tiny_qwen3); G = 4, 5 and 8 (80 m-tiles of decode QKV:
    the bf16 EPI_T_STORE epilogue).  The peaked case's 300-token prompts cross 128-token chunks, and its row 2 shares
    row 0's first 256 tokens."""
    gen_case = Q2.gen_case
    gen_case("tiny_qwen3_ids", "tiny_qwen3", 11, ids_prompt(4, 70, 1000, 1111), 16, pad_token_id=1030, build=build_model)
    gen_case("tiny_qwen3_peaked", "tiny_qwen3_peaked", 11, Q2.qwen2_prompts(4, 300, 1000, 1121), 16, pad_token_id=1030,
             build=build_model)
    gen_case("tiny_qwen3_g4_ids", "tiny_qwen3_g4", 12, ids_prompt(3, 100, 1000, 1212), 16, pad_token_id=1030, build=build_model)
    gen_case("tiny_qwen3_g5_ids", "tiny_qwen3_g5", 13, ids_prompt(3, 65, 1000, 1313), 16, pad_token_id=1030, build=build_model)
    gen_case("tiny_qwen3_wide_ids", "tiny_qwen3_wide", 14, ids_prompt(4, 70, 1000, 1414), 16, pad_token_id=1030,
             build=build_model)


def qwen3_big_cases():
    """Qwen3-8B layer shapes (2 layers): 4 x 1024-token prompts, V = 151936"""
    pad = 151935
    for name, cfg_name in (("qwen3_8b_2l_b4", "qwen3_8b_2l"), ("qwen3_8b_2l_peaked_b4", "qwen3_8b_2l_peaked")):
        Q2.gen_case(name, cfg_name, 0, ids_prompt(4, 1024, 150000, 2027), 16, pad_token_id=pad, sub_logits=True,
                    build=build_model)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big", action="store_true")
    ap.add_argument("--only", default=None, help="comma separated case names: generate just these")
    args = ap.parse_args()
    Q2.ONLY = set(args.only.split(",")) if args.only else None
    torch.set_num_threads(os.cpu_count())
    qwen3_cases()
    if args.big:
        qwen3_big_cases()


if __name__ == "__main__":
    sys.exit(main())
