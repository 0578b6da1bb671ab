"""Checkpoint-config helpers of the runtime model: the served context length and the rotary tables.

`get_and_verify_max_len` restates what `HuggingfaceGenerativeModel.load` calls at
python/huggingfaceserver/huggingfaceserver/generative_model.py:206 (`_get_and_verify_max_len(model_config, max_length)`,
python/huggingfaceserver/huggingfaceserver/utils.py:28-159) for plain-dict configs: same key list, same derivation
order, same error text and the same ALLOW_LONG_MAX_MODEL_LEN override.

`rope_inv_freq` / `hf_rope_tables` compute cos/sin exactly as transformers' LlamaRotaryEmbedding does for the rope
types Llama-family checkpoints ship with ("default", "linear", "llama3"); anything else is refused — an ignored
`rope_scaling` produces fluent but wrong tokens, which is worse than not loading.
"""
from __future__ import annotations

import logging
import math
import os
from typing import Any, Dict, List, Optional, Tuple, Union

import torch

logger = logging.getLogger("kserve_b200")

ALLOW_LONG_MAX_MODEL_LEN = "ALLOW_LONG_MAX_MODEL_LEN"

# order matters only for the name reported in the error message (utils.py:37-55)
_MAX_LEN_KEYS = ("max_position_embeddings", "n_positions", "max_seq_len", "seq_length", "model_max_length",
                 "max_sequence_length", "max_seq_length", "seq_len")


def rope_parameters(cfg: Dict[str, Any]) -> Dict[str, Any]:
    """The rope dict of a config in either spelling: transformers <= 4.x `rope_scaling` (+ top-level `rope_theta`,
    `type` as an old alias of `rope_type`) or 5.x `rope_parameters`."""
    rp = dict(cfg.get("rope_parameters") or cfg.get("rope_scaling") or {})
    if "rope_type" not in rp:
        rp["rope_type"] = rp.pop("type", None) or "default"
    if "rope_theta" not in rp:
        rp["rope_theta"] = cfg.get("rope_theta", 10000.0)
    return rp


def get_min_sliding_window(sliding_window: Union[int, List[Optional[int]]]) -> int:
    if isinstance(sliding_window, list):
        return min(s for s in sliding_window if s is not None)
    return sliding_window


def get_and_verify_max_len(hf_config: Dict[str, Any], max_model_len: Optional[int], disable_sliding_window: bool = False,
                           sliding_window_len: Optional[Union[int, List[Optional[int]]]] = None) -> int:
    """utils.py:28-159 for a dict config (the speculative-draft and encoder arguments of the original never apply
    to the generative runtime and are not carried)."""
    derived = float("inf")
    key_of_min = None
    for key in _MAX_LEN_KEYS:
        v = hf_config.get(key)
        if v is None:
            continue
        if v < derived:
            key_of_min = key
        derived = min(derived, v)
    if disable_sliding_window and sliding_window_len is not None:
        w = get_min_sliding_window(sliding_window_len)
        if w < derived:
            key_of_min = "sliding_window"
        derived = min(derived, w)
    if derived == float("inf"):
        if max_model_len is not None:
            return max_model_len
        default_max_len = 2048
        logger.warning("The model's config.json does not contain any of the following keys to determine the original "
                       "maximum length of the model: %s. Assuming the model's maximum length is %d.",
                       list(_MAX_LEN_KEYS), default_max_len)
        derived = default_max_len
    has_rope = hf_config.get("rope_scaling") is not None or (
        hf_config.get("rope_parameters") is not None and rope_parameters(hf_config)["rope_type"] != "default")
    if has_rope:
        rp = rope_parameters(hf_config)
        rope_type = rp["rope_type"]
        if rope_type not in ("su", "longrope", "llama3"):
            if disable_sliding_window:
                raise NotImplementedError("Disabling sliding window is not supported for models with rope_scaling. "
                                          "Please raise an issue so we can investigate.")
            if rope_type == "yarn":
                derived = rp["original_max_position_embeddings"]
            derived *= rp.get("factor", 1.0)      # "default" defines no factor
    if max_model_len is None:
        return int(derived)
    if max_model_len > derived:
        model_max_length = hf_config.get("model_max_length")
        if model_max_length is not None and max_model_len <= model_max_length:
            if disable_sliding_window:
                raise NotImplementedError("Disabling sliding window is not supported for models model_max_length in "
                                          "the config. Please raise an issue so we can investigate.")
        else:
            msg = (f"User-specified max_model_len ({max_model_len}) is greater than the derived max_model_len "
                   f"({key_of_min}={derived} or model_max_length={model_max_length} in model's config.json). "
                   "This may lead to incorrect model outputs or CUDA errors.")
            if int(os.environ.get(ALLOW_LONG_MAX_MODEL_LEN, 0)) == 1:
                logger.warning("%s Make sure the value is correct and within the model context size.", msg)
            else:
                raise ValueError(f"{msg} To allow overriding this maximum, set the env var ALLOW_LONG_MAX_MODEL_LEN=1")
    return int(max_model_len)


SUPPORTED_ROPE_TYPES = ("default", "linear", "llama3")


def rope_inv_freq(cfg: Dict[str, Any], head_dim: int) -> torch.Tensor:
    """fp32 inverse frequencies, op for op what transformers computes (modeling_rope_utils.py:
    `_compute_default_rope_parameters`, `_compute_linear_scaling_rope_parameters`, `_compute_llama3_parameters`)."""
    rp = rope_parameters(cfg)
    kind = rp["rope_type"]
    if kind not in SUPPORTED_ROPE_TYPES:
        raise ValueError(f"rope_scaling type '{kind}' is not supported by the H100 runtime (supported: "
                         f"{', '.join(SUPPORTED_ROPE_TYPES)}); refusing to load a model that would generate wrong tokens")
    if float(rp.get("partial_rotary_factor", cfg.get("partial_rotary_factor", 1.0)) or 1.0) != 1.0:
        raise ValueError("partial_rotary_factor != 1 is not supported by the H100 runtime")
    base = float(rp["rope_theta"])
    inv_freq = 1.0 / (base ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(torch.float) / head_dim))
    if kind == "linear":
        inv_freq = inv_freq / rp["factor"]
    elif kind == "llama3":
        factor, lo, hi = rp["factor"], rp["low_freq_factor"], rp["high_freq_factor"]
        old_len = rp.get("original_max_position_embeddings") or cfg["max_position_embeddings"]
        wavelen = 2 * math.pi / inv_freq
        scaled = torch.where(wavelen > old_len / lo, inv_freq / factor, inv_freq)
        smooth = (old_len / wavelen - lo) / (hi - lo)
        blended = (1 - smooth) * scaled / factor + smooth * scaled
        medium = ~(wavelen < old_len / hi) * ~(wavelen > old_len / lo)
        inv_freq = torch.where(medium, blended, scaled)
    return inv_freq


def hf_rope_tables(cfg: Dict[str, Any], head_dim: int, max_pos: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """bf16 cos/sin [max_pos, head_dim/2] as LlamaRotaryEmbedding.forward yields them for a bf16 model
    (transformers modeling_llama.py: fp32 inv_freq x fp32 position -> cos/sin in fp32 (x attention_scaling == 1 for
    the supported types) -> cast to the activation dtype)."""
    inv_freq = rope_inv_freq(cfg, head_dim)
    pos = torch.arange(max_pos, dtype=torch.float32)
    freqs = pos[:, None] * inv_freq[None, :]
    return freqs.cos().to(torch.bfloat16).contiguous(), freqs.sin().to(torch.bfloat16).contiguous()


def plan_memory(cfg: Dict[str, Any], vocab_rows: int, max_batch: int, max_len: int, tp_size: int, free_bytes: int,
                max_prefill_tokens: Optional[int] = None, reserve_bytes: int = 3 << 30) -> Tuple[int, int]:
    """-> (max_prefill_tokens, num_kv_pages) that fit `free_bytes` of device memory next to the weights.

    The engine preallocates its activation buffers for `max_prefill_tokens` packed prompt tokens and a pool of 64-token
    KV pages; sizing both as max_batch x max_model_len (a Llama-3.1 config says 131072) would not fit any GPU, so the
    prefill buffers are capped (one full-length prompt always fits) and the page pool takes what is left, at most
    max_batch full-length sequences and at least one."""
    H, I, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
    nh, nkv = cfg["num_attention_heads"], cfg["num_key_value_heads"]
    d = cfg.get("head_dim") or H // nh
    E = int(cfg.get("num_local_experts", 0) or 0)
    nh_l, nkv_l, I_l = nh // tp_size, nkv // tp_size, I // tp_size
    qkv_cols = (nh_l + 2 * nkv_l) * d
    layer = qkv_cols * H + H * nh_l * d + (E * (3 * H * I_l) + E * H if E else 3 * H * I_l) + 2 * H
    weights = 2 * (L * layer + vocab_rows * H + -(-vocab_rows // tp_size) * H + H)
    per_tok = 2 * (3 * H + qkv_cols + nh_l * d + I_l) + 16 + (2 * (3 * H + 2 * I_l) + 24 if E else 0)
    page = L * 2 * nkv_l * 64 * d * 2
    pages_per_seq = -(-max_len // 64)
    want_pages = max_batch * pages_per_seq
    fixed = reserve_bytes + 3 * 8 * max_batch * max_len + 2 * 4 * max_batch * max_len + 2 * max_batch * -(-vocab_rows // tp_size)
    cap_t = max_prefill_tokens or min(max_batch * max_len, max(max_len, 32768))
    avail = free_bytes - weights - fixed - cap_t * per_tok
    pages = min(want_pages, avail // page) if avail > 0 else 0
    if pages < pages_per_seq:
        raise ValueError(f"not enough device memory for one sequence of max_model_len={max_len}: weights "
                         f"{weights / 2**30:.1f} GiB + buffers leave room for {max(pages, 0)} KV pages, {pages_per_seq} needed; "
                         "pass a smaller --max_model_len")
    return int(cap_t), int(pages)
