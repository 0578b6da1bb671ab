"""Llama-family tensor table: HF state_dict names and shapes the engine expects
(what AutoModelForCausalLM.from_pretrained loads in the reference, generative_model.py:249-254).
Qwen2 configs (model_type "qwen2") add the q / k / v projection biases, Qwen3 configs (model_type "qwen3") the per-head
q / k norm weights, and a tied checkpoint has no lm_head.weight."""
from __future__ import annotations

from typing import Iterator, Tuple


def llama_tensor_specs(cfg: dict) -> Iterator[Tuple[str, Tuple[int, ...], str]]:
    """Yield (name, shape, kind); kind in {embed, linear, norm, bias}."""
    H, I, V = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]
    nh, nkv = cfg["num_attention_heads"], cfg["num_key_value_heads"]
    d = cfg.get("head_dim") or H // nh
    E = int(cfg.get("num_local_experts", 0) or 0)
    qwen2 = cfg.get("model_type") == "qwen2"
    qwen3 = cfg.get("model_type") == "qwen3"
    yield "model.embed_tokens.weight", (V, H), "embed"
    for i in range(cfg["num_hidden_layers"]):
        if E:   # Mixtral-style sparse MoE (transformers 5.x fused-expert state_dict)
            p = f"model.layers.{i}."
            yield p + "input_layernorm.weight", (H,), "norm"
            yield p + "self_attn.q_proj.weight", (nh * d, H), "linear"
            yield p + "self_attn.k_proj.weight", (nkv * d, H), "linear"
            yield p + "self_attn.v_proj.weight", (nkv * d, H), "linear"
            yield p + "self_attn.o_proj.weight", (H, nh * d), "linear"
            yield p + "post_attention_layernorm.weight", (H,), "norm"
            yield p + "mlp.gate.weight", (E, H), "linear"
            yield p + "mlp.experts.gate_up_proj", (E, 2 * I, H), "linear"
            yield p + "mlp.experts.down_proj", (E, H, I), "linear"
            continue
        p = f"model.layers.{i}."
        yield p + "input_layernorm.weight", (H,), "norm"
        yield p + "self_attn.q_proj.weight", (nh * d, H), "linear"
        if qwen2:
            yield p + "self_attn.q_proj.bias", (nh * d,), "bias"
        yield p + "self_attn.k_proj.weight", (nkv * d, H), "linear"
        if qwen2:
            yield p + "self_attn.k_proj.bias", (nkv * d,), "bias"
        if qwen3:
            yield p + "self_attn.q_norm.weight", (d,), "norm"
            yield p + "self_attn.k_norm.weight", (d,), "norm"
        yield p + "self_attn.v_proj.weight", (nkv * d, H), "linear"
        if qwen2:
            yield p + "self_attn.v_proj.bias", (nkv * d,), "bias"
        yield p + "self_attn.o_proj.weight", (H, nh * d), "linear"
        yield p + "post_attention_layernorm.weight", (H,), "norm"
        yield p + "mlp.gate_proj.weight", (I, H), "linear"
        yield p + "mlp.up_proj.weight", (I, H), "linear"
        yield p + "mlp.down_proj.weight", (H, I), "linear"
    yield "model.norm.weight", (H,), "norm"
    if not cfg.get("tie_word_embeddings"):
        yield "lm_head.weight", (V, H), "linear"
