"""Deterministic synthetic Llama checkpoints (test / bench infrastructure; re-exported as oracle.weights).

There is no network and no checkpoint on disk, so both the CPU oracle and the
CUDA engine are fed the same seeded tensors.  Each tensor gets its own CPU
``torch.Generator`` (seed derived from the tensor's index in a canonical
order) so that tensors can be produced one at a time without holding a whole
fp32 model in memory, and so that the bytes are identical on every box.

Names follow the HF Llama ``state_dict`` (what the reference's
``AutoModelForCausalLM.from_pretrained`` would load,
python/huggingfaceserver/huggingfaceserver/generative_model.py:249-254).
"""
from __future__ import annotations

import math
from typing import Dict, Iterator, Tuple

import torch

# Named model shapes used by tests / bench.  ``llama3_8b`` is BASELINE.json's
# flagship; the tiny ones exercise GQA group sizes 2 and 4 and a vocabulary
# that is not a multiple of any tile size.
CONFIGS: Dict[str, dict] = {
    "tiny_g2": dict(vocab_size=1031, hidden_size=512, intermediate_size=1024,
                    num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                    head_dim=128, max_position_embeddings=2048, rms_norm_eps=1e-5,
                    rope_theta=500000.0),
    "tiny_g4": dict(vocab_size=2048, hidden_size=1024, intermediate_size=2816,
                    num_hidden_layers=3, num_attention_heads=8, num_key_value_heads=2,
                    head_dim=128, max_position_embeddings=2048, rms_norm_eps=1e-5,
                    rope_theta=500000.0),
    "llama3_8b": dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336,
                      num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=8,
                      head_dim=128, max_position_embeddings=8192, rms_norm_eps=1e-5,
                      rope_theta=500000.0),
    # same layer shapes as llama3_8b, 2 layers: the largest thing the CPU oracle
    # can run in seconds while still hitting every full-size GEMM / vocab shape.
    "llama3_8b_2l": dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336,
                         num_hidden_layers=2, num_attention_heads=32, num_key_value_heads=8,
                         head_dim=128, max_position_embeddings=8192, rms_norm_eps=1e-5,
                         rope_theta=500000.0),
}


MOE_CONFIGS: Dict[str, dict] = {
    # Mixtral-style sparse MoE (BASELINE.json configs[3]) at test size: 4 experts, top-2
    "tiny_moe": dict(vocab_size=1031, hidden_size=512, intermediate_size=1024, num_hidden_layers=2,
                     num_attention_heads=4, num_key_value_heads=2, head_dim=128, max_position_embeddings=2048,
                     rms_norm_eps=1e-5, rope_theta=1000000.0, num_local_experts=4, num_experts_per_tok=2),
    "tiny_moe8": dict(vocab_size=2048, hidden_size=1024, intermediate_size=1536, num_hidden_layers=2,
                      num_attention_heads=8, num_key_value_heads=2, head_dim=128, max_position_embeddings=2048,
                      rms_norm_eps=1e-5, rope_theta=1000000.0, num_local_experts=8, num_experts_per_tok=2),
}
CONFIGS.update(MOE_CONFIGS)

# 8 KV heads: the smallest shapes every tensor-parallel degree of BASELINE configs[2] (TP = 2 / 4 / 8) can shard
# (TP=8 -> one KV head and two query heads per GPU); the vocabulary is odd on purpose (uneven vocab-parallel shards).
CONFIGS["tiny_kv8"] = dict(vocab_size=4099, hidden_size=1024, intermediate_size=2048, num_hidden_layers=2,
                           num_attention_heads=16, num_key_value_heads=8, head_dim=128, max_position_embeddings=2048,
                           rms_norm_eps=1e-5, rope_theta=500000.0)
# Llama-3.1-style rope scaling (rope_type "llama3"): the tables differ from the default ones at every position
CONFIGS["tiny_g2_rope3"] = dict(CONFIGS["tiny_g2"], max_position_embeddings=4096,
                                rope_scaling=dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
                                                  original_max_position_embeddings=256))

# "Peaked" variants: lm_head row v = embed row perm[v].  The final hidden state still carries the current token's
# embedding (the residual stream starts from it), so one logit towers over the rest the way a trained model's does and
# the greedy choice is decisive at (nearly) every step: greedy ids can then be compared EXACTLY, not just where a
# random-weight near-tie happens to be wide enough.  All other tensors are those of the base config, so the layers are
# exercised identically and the full logits are still compared element-wise (tests/helpers.py: logits_tol_elementwise).
for _base in ("tiny_g2", "tiny_g4", "tiny_kv8", "llama3_8b_2l"):
    CONFIGS[_base + "_peaked"] = dict(CONFIGS[_base], _peaked=True)

# Qwen2 / Qwen2.5 decoders: Llama layers plus q / k / v projection biases (theta 1e6, eps 1e-6).  GQA groups 7, 6 and 5
# are those of Qwen2-0.5B / Qwen2.5-3B / Qwen2.5-32B.  tiny_qwen2's decode QKV projection (18 m-tiles) takes split-K;
# tiny_qwen2_wide's (qkv_cols 10240 = 80 m-tiles) takes the bf16 EPI_T_STORE epilogue, as 72B-class models do.
_QWEN2 = dict(model_type="qwen2", head_dim=128, max_position_embeddings=2048, rms_norm_eps=1e-6, rope_theta=1000000.0,
              use_sliding_window=False)
QWEN2_CONFIGS: Dict[str, dict] = {
    "tiny_qwen2": dict(_QWEN2, vocab_size=1031, hidden_size=896, intermediate_size=4864, num_hidden_layers=2,
                       num_attention_heads=14, num_key_value_heads=2),
    "tiny_qwen2_g6_tied": dict(_QWEN2, vocab_size=1031, hidden_size=768, intermediate_size=2048, num_hidden_layers=2,
                               num_attention_heads=12, num_key_value_heads=2, tie_word_embeddings=True),
    "tiny_qwen2_g5": dict(_QWEN2, vocab_size=1031, hidden_size=640, intermediate_size=1536, num_hidden_layers=2,
                          num_attention_heads=10, num_key_value_heads=2),
    "tiny_qwen2_wide": dict(_QWEN2, vocab_size=1031, hidden_size=512, intermediate_size=1024, num_hidden_layers=2,
                            num_attention_heads=64, num_key_value_heads=8),
    # Qwen2.5-7B layer and vocabulary shapes, 2 layers
    "qwen2_7b_2l": dict(_QWEN2, vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=2,
                        num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=32768),
    # Qwen2.5-7B, all 28 layers (tools/model_bench.py)
    "qwen2_7b": dict(_QWEN2, vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
                     num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=32768),
}
for _base in ("tiny_qwen2", "qwen2_7b_2l"):
    QWEN2_CONFIGS[_base + "_peaked"] = dict(QWEN2_CONFIGS[_base], _peaked=True)
CONFIGS.update(QWEN2_CONFIGS)

# Qwen3 dense decoders: Llama layers plus a per-head RMSNorm of q and of k (q_norm / k_norm, [128] each) before RoPE, no
# projection biases, theta 1e6, eps 1e-6.  tiny_qwen3 has 0.6B's q dim = 2H, G = 2 and tied embeddings, and its decode
# QKV projection (16 m-tiles) takes split-K; g4 / g5 are 8B's and 14B's groups; tiny_qwen3_wide (G = 8, qkv_cols 10240
# = 80 m-tiles) takes the bf16 EPI_T_STORE decode epilogue, as the 32B class does.
_QWEN3 = dict(model_type="qwen3", head_dim=128, max_position_embeddings=2048, rms_norm_eps=1e-6, rope_theta=1000000.0,
              use_sliding_window=False)
QWEN3_CONFIGS: Dict[str, dict] = {
    "tiny_qwen3": dict(_QWEN3, vocab_size=1031, hidden_size=512, intermediate_size=1536, num_hidden_layers=2,
                       num_attention_heads=8, num_key_value_heads=4, tie_word_embeddings=True),
    "tiny_qwen3_g4": dict(_QWEN3, vocab_size=1031, hidden_size=1024, intermediate_size=2048, num_hidden_layers=2,
                          num_attention_heads=8, num_key_value_heads=2),
    "tiny_qwen3_g5": dict(_QWEN3, vocab_size=1031, hidden_size=640, intermediate_size=1536, num_hidden_layers=2,
                          num_attention_heads=10, num_key_value_heads=2),
    "tiny_qwen3_wide": dict(_QWEN3, vocab_size=1031, hidden_size=512, intermediate_size=1024, num_hidden_layers=2,
                            num_attention_heads=64, num_key_value_heads=8),
    # Qwen3-8B layer and vocabulary shapes, 2 layers
    "qwen3_8b_2l": dict(_QWEN3, vocab_size=151936, hidden_size=4096, intermediate_size=12288, num_hidden_layers=2,
                        num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=40960),
    # Qwen3-8B, all 36 layers (tools/model_bench.py)
    "qwen3_8b": dict(_QWEN3, vocab_size=151936, hidden_size=4096, intermediate_size=12288, num_hidden_layers=36,
                     num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=40960),
}
# (a peaked head is a permuted embedding, so the peaked tiny case is untied)
QWEN3_CONFIGS["tiny_qwen3_peaked"] = dict(QWEN3_CONFIGS["tiny_qwen3"], tie_word_embeddings=False, _peaked=True)
QWEN3_CONFIGS["qwen3_8b_2l_peaked"] = dict(QWEN3_CONFIGS["qwen3_8b_2l"], _peaked=True)
CONFIGS.update(QWEN3_CONFIGS)

# FP8 checkpoints (compressed-tensors float-quantized, kserve_b200/fp8.py): the SAME seeded bf16 tensors as the base
# config, each q/k/v/o/gate/up/down projection quantized to float8_e4m3fn with a scale amax / 448 per row ("channel") or
# per tensor ("tensor"), in bf16 or fp32; everything else (embeddings, norms, lm_head, Qwen2 biases) stays bf16.
# iter_state_dict yields `<proj>.weight` codes followed by `<proj>.weight_scale`, as such a checkpoint holds them.
FP8_CONFIGS: Dict[str, dict] = {
    "tiny_g4_fp8": dict(CONFIGS["tiny_g4"], _fp8="channel"),
    "tiny_g4_fp8_peaked": dict(CONFIGS["tiny_g4_peaked"], _fp8="channel"),
    "tiny_qwen2_fp8": dict(CONFIGS["tiny_qwen2"], _fp8="channel"),                               # biases, G = 7
    "tiny_g2_fp8_tensor": dict(CONFIGS["tiny_g2"], _fp8="tensor", _fp8_scale="float32"),
    "tiny_qwen2_g6_tied_fp8": dict(CONFIGS["tiny_qwen2_g6_tied"], _fp8="channel", _fp8_scale="float32"),
    "llama3_8b_2l_fp8": dict(CONFIGS["llama3_8b_2l"], _fp8="channel"),
    "llama3_8b_2l_fp8_peaked": dict(CONFIGS["llama3_8b_2l_peaked"], _fp8="channel"),
    "tiny_qwen3_fp8": dict(CONFIGS["tiny_qwen3"], _fp8="channel"),                               # q/k norms, tied, G = 2
}
CONFIGS.update(FP8_CONFIGS)
FP8_PROJECTIONS = ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight", "self_attn.o_proj.weight",
                   "mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight")


def fp8_quantize(t: torch.Tensor, strategy: str = "channel", scale_dtype=torch.bfloat16):
    """(e4m3 codes, weight_scale) of a weight: scale = amax / 448 ([out, 1] per row, [1] per tensor), codes = w / scale"""
    t = t.float()
    amax = t.abs().amax(dim=1, keepdim=True) if strategy == "channel" else t.abs().amax().reshape(1)
    scale = (amax / 448.0).clamp_min(1e-12).to(scale_dtype)
    codes = (t / (scale.float() if strategy == "channel" else scale.float()[0])).clamp(-448.0, 448.0)
    return codes.to(torch.float8_e4m3fn), scale


def fp8_quantization_config(strategy: str) -> dict:
    """config.json's quantization_config of an FP8 config (what llm-compressor writes for weight-only FP8)"""
    return dict(quant_method="compressed-tensors", format="float-quantized", quantization_status="compressed",
                ignore=["lm_head"], kv_cache_scheme=None,
                config_groups={"group_0": dict(targets=["Linear"], input_activations=None, output_activations=None,
                                               weights=dict(num_bits=8, type="float", symmetric=True, strategy=strategy,
                                                            dynamic=False))})


def hf_config_dict(cfg: dict) -> dict:
    """the keys a transformers config understands (drops this module's private `_...` markers)"""
    return {k: v for k, v in cfg.items() if not k.startswith("_")}


def moe_tensor_specs(cfg: dict) -> Iterator[Tuple[str, Tuple[int, ...], str]]:
    """HF MixtralForCausalLM state_dict (transformers 5.x fused-expert layout)."""
    H, I, V, E = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"], cfg["num_local_experts"]
    nh, nkv, d = cfg["num_attention_heads"], cfg["num_key_value_heads"], cfg["head_dim"]
    yield "model.embed_tokens.weight", (V, H), "embed"
    for i in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{i}."
        yield p + "input_layernorm.weight", (H,), "norm"
        yield p + "self_attn.q_proj.weight", (nh * d, H), "linear"
        yield p + "self_attn.k_proj.weight", (nkv * d, H), "linear"
        yield p + "self_attn.v_proj.weight", (nkv * d, H), "linear"
        yield p + "self_attn.o_proj.weight", (H, nh * d), "linear"
        yield p + "post_attention_layernorm.weight", (H,), "norm"
        yield p + "mlp.gate.weight", (E, H), "router"
        yield p + "mlp.experts.gate_up_proj", (E, 2 * I, H), "linear"
        yield p + "mlp.experts.down_proj", (E, H, I), "linear"
    yield "model.norm.weight", (H,), "norm"
    yield "lm_head.weight", (V, H), "linear"


def tensor_specs(cfg: dict) -> Iterator[Tuple[str, Tuple[int, ...], str]]:
    """Yield (name, shape, kind) in canonical order. kind in {embed, linear, norm, bias}.  Qwen2 biases follow their
    weight, Qwen3's q_norm / k_norm follow k_proj, and a tied checkpoint has no lm_head.weight; the Llama / Mixtral order
    (and so every seed) is unchanged."""
    H, I, V = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]
    nh, nkv, d = cfg["num_attention_heads"], cfg["num_key_value_heads"], cfg["head_dim"]
    if "num_local_experts" in cfg:
        yield from moe_tensor_specs(cfg)
        return
    qwen2 = cfg.get("model_type") == "qwen2"
    qwen3 = cfg.get("model_type") == "qwen3"
    yield "model.embed_tokens.weight", (V, H), "embed"
    for i in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{i}."
        yield p + "input_layernorm.weight", (H,), "norm"
        for proj, rows in (("q", nh * d), ("k", nkv * d), ("v", nkv * d)):
            yield p + f"self_attn.{proj}_proj.weight", (rows, H), "linear"
            if qwen2:
                yield p + f"self_attn.{proj}_proj.bias", (rows,), "bias"
            if qwen3 and proj == "k":
                yield p + "self_attn.q_norm.weight", (d,), "norm"
                yield p + "self_attn.k_norm.weight", (d,), "norm"
        yield p + "self_attn.o_proj.weight", (H, nh * d), "linear"
        yield p + "post_attention_layernorm.weight", (H,), "norm"
        yield p + "mlp.gate_proj.weight", (I, H), "linear"
        yield p + "mlp.up_proj.weight", (I, H), "linear"
        yield p + "mlp.down_proj.weight", (H, I), "linear"
    yield "model.norm.weight", (H,), "norm"
    if not cfg.get("tie_word_embeddings"):
        yield "lm_head.weight", (V, H), "linear"


def synth_bias(index: int, shape, name: str, seed: int, dtype=torch.bfloat16) -> torch.Tensor:
    """Qwen2 q / k / v biases.  HF initialises them to zero, so they are drawn large enough that a dropped, doubled or
    misplaced (after RoPE) bias moves the logits: q, v ~ N(0, 0.5); k ~ N(0, 2) with a few entries near +-20, the
    outliers real Qwen k biases have."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed * 1000003 + index * 7919 + 17)
    if ".k_proj." in name:
        t = 2.0 * torch.randn(shape, generator=g, dtype=torch.float32)
        idx = torch.randperm(shape[0], generator=g)[: max(2, shape[0] // 64)]
        t[idx] = torch.sign(t[idx] + 1e-3) * (18.0 + 4.0 * torch.rand(idx.shape, generator=g))
    else:
        t = 0.5 * torch.randn(shape, generator=g, dtype=torch.float32)
    return t.to(dtype)


def synth_qk_norm(index: int, shape, name: str, seed: int, dtype=torch.bfloat16) -> torch.Tensor:
    """Qwen3 q_norm / k_norm weights.  HF initialises them to ones, so they are drawn far from 1 (log-uniform over
    [0.2, 4]) that a dropped, post-RoPE or swapped norm moves the logits; k_norm also gets two entries near +-10..20, the
    outliers real Qwen3 k_norm weights have."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed * 1000003 + index * 7919 + 17)
    t = torch.exp(math.log(0.2) + (math.log(4.0) - math.log(0.2)) * torch.rand(shape, generator=g, dtype=torch.float32))
    if ".k_norm." in name:
        idx = torch.randperm(shape[0], generator=g)[:2]
        t[idx] = torch.sign(torch.randn(idx.shape, generator=g)) * (10.0 + 10.0 * torch.rand(idx.shape, generator=g))
    return t.to(dtype)


# Qwen3 q / k projections: an RMS well away from 1 (the norm removes it; a dropped norm does not)
QWEN3_QK_SCALE = {"self_attn.q_proj.weight": 3.0, "self_attn.k_proj.weight": 0.3}


def synth_tensor(index: int, shape, kind: str, seed: int, dtype=torch.bfloat16) -> torch.Tensor:
    g = torch.Generator(device="cpu")
    g.manual_seed(seed * 1000003 + index * 7919 + 17)
    if kind == "norm":
        t = 1.0 + 0.1 * torch.randn(shape, generator=g, dtype=torch.float32)
    elif kind == "embed":
        t = torch.randn(shape, generator=g, dtype=torch.float32)
    elif kind == "router":  # moderately peaky routing: the 2nd expert carries real weight, 2nd/3rd margins mostly above bf16 noise
        t = torch.randn(shape, generator=g, dtype=torch.float32) * (2.5 / math.sqrt(shape[-1]))
    else:  # linear: variance preserving, so attention / logits are not near-uniform
        t = torch.randn(shape, generator=g, dtype=torch.float32) * (1.0 / math.sqrt(shape[-1]))
    return t.to(dtype)


def peaked_perm(vocab: int, seed: int) -> torch.Tensor:
    g = torch.Generator(device="cpu")
    g.manual_seed(seed * 7727 + 4241)
    return torch.randperm(vocab, generator=g)


def iter_state_dict(cfg: dict, seed: int = 0, dtype=torch.bfloat16):
    """Yield (name, tensor) one tensor at a time (bounded memory)."""
    if cfg.get("_fp8"):
        base = {k: v for k, v in cfg.items() if k not in ("_fp8", "_fp8_scale")}
        sdt = getattr(torch, cfg.get("_fp8_scale", "bfloat16"))
        for name, t in iter_state_dict(base, seed, dtype):
            if name.split(".", 3)[-1] in FP8_PROJECTIONS:
                codes, scale = fp8_quantize(t, cfg["_fp8"], sdt)
                yield name, codes
                yield name + "_scale", scale
            else:
                yield name, t
        return
    for idx, (name, shape, kind) in enumerate(tensor_specs(cfg)):
        if name == "lm_head.weight" and cfg.get("_peaked"):
            embed = synth_tensor(0, shape, "embed", seed, dtype)      # index 0 == model.embed_tokens.weight
            yield name, embed[peaked_perm(shape[0], seed)].contiguous()
            continue
        if kind == "bias":
            yield name, synth_bias(idx, shape, name, seed, dtype)
            continue
        if cfg.get("model_type") == "qwen3":
            if name.endswith(("self_attn.q_norm.weight", "self_attn.k_norm.weight")):
                yield name, synth_qk_norm(idx, shape, name, seed, dtype)
                continue
            qk = QWEN3_QK_SCALE.get(name.split(".", 3)[-1])
            if qk is not None:
                yield name, (synth_tensor(idx, shape, kind, seed, torch.float32) * qk).to(dtype)
                continue
        yield name, synth_tensor(idx, shape, kind, seed, dtype)


def synth_state_dict(cfg: dict, seed: int = 0, dtype=torch.bfloat16) -> Dict[str, torch.Tensor]:
    return dict(iter_state_dict(cfg, seed, dtype))


def checksum(sd: Dict[str, torch.Tensor]) -> float:
    """Cheap fingerprint recorded in golden files to prove both sides loaded the same bytes."""
    s = 0.0
    third = "model.layers.0.mlp.down_proj.weight"
    if third not in sd:   # MoE checkpoints have fused expert tensors instead
        third = "model.layers.0.self_attn.o_proj.weight"
    for name in ("model.embed_tokens.weight", "lm_head.weight", third):
        t = sd[name] if name in sd else sd["model.embed_tokens.weight"]   # (tied checkpoints have no lm_head.weight)
        s += float(t[: 64].float().sum()) + float(t[-1].float().abs().sum())
    return s
