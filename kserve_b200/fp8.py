"""FP8 checkpoints: which `quantization_config` the H100 runtime serves, and the dequantization rule it computes.

Served: compressed-tensors `float-quantized` checkpoints (what llm-compressor writes) whose config groups quantize the
`Linear` layers' weights to symmetric 8-bit floats (float8_e4m3fn) with a `channel` or `tensor` scale, and leave
`lm_head` (and so the embeddings, norms and Qwen2's q/k/v biases) in bf16.  Each projection then arrives as
`<name>.weight` (e4m3 codes [out, in]) plus `<name>.weight_scale` ([out, 1] for channel, [1] or a scalar for tensor).

Numerics: transformers loads the scale into the bf16 model (an fp32 scale is rounded to bf16) and its compressed-tensors
decompression computes `dequantize(w, scale) = w.to(scale.dtype) * scale`, i.e. W' = bf16(code) * bf16(scale) in bf16
arithmetic, rounded once.  The engine multiplies exactly this W', so an FP8 engine is bit-identical to a bf16 engine
loaded with W' (`dequantize_reference`).

FP8 engines run on one GPU (tensor parallelism is refused).  Activations stay bf16: a checkpoint with dynamic per-token
FP8 input activations ("FP8-dynamic") is served as W8A16 and its outputs are not those of a runtime that quantizes
activations.  Static activation scales are refused.

FP8 KV cache (`--kv_cache_dtype fp8`, independent of the checkpoint's format): the KV pages hold float8_e4m3fn codes of
k after RoPE and v, `quantize_kv` of the bf16 values a bf16 cache would hold (per-tensor scale 1, what vLLM does for a
checkpoint without calibrated KV scales), and attention reads bf16(code), which is exact.
"""
from __future__ import annotations

import logging
from typing import Any, Dict, Optional

import torch

logger = logging.getLogger("kserve_b200")

PROJECTIONS = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj",
               "mlp.gate_proj", "mlp.up_proj", "mlp.down_proj")


class UnsupportedQuantization(ValueError):
    pass


# --kv_cache_dtype names (vLLM's) -> b200_model_config_t.kv_cache_dtype
KV_CACHE_DTYPES = {"auto": 0, "bfloat16": 0, "fp8": 1, "fp8_e4m3": 1}


def kv_cache_format(name: str, tp_size: int = 1) -> int:
    """--kv_cache_dtype -> 0 (bf16 KV pages) or 1 (float8_e4m3fn codes); raises UnsupportedQuantization"""
    if name == "fp8_e5m2":
        raise UnsupportedQuantization("--kv_cache_dtype fp8_e5m2 is not supported (the FP8 KV cache is float8_e4m3fn: "
                                      "use fp8 or fp8_e4m3)")
    if name not in KV_CACHE_DTYPES:
        raise UnsupportedQuantization(f"--kv_cache_dtype {name!r} is not one of {sorted(KV_CACHE_DTYPES)}")
    fmt = KV_CACHE_DTYPES[name]
    if fmt == 1 and tp_size > 1:
        raise UnsupportedQuantization(f"an FP8 KV cache with tensor parallelism (tensor_parallel_size={tp_size}) is not "
                                      "supported")
    return fmt


def quantize_kv(x: torch.Tensor) -> torch.Tensor:
    """The code an FP8 KV cache stores for each element of x: e4m3(clamp(x, -448, 448)), round to nearest even (NaN stays
    NaN; torch's plain cast would turn |x| >= 464 into NaN)"""
    return x.float().clamp(-448.0, 448.0).to(torch.float8_e4m3fn)


def _refuse(msg: str):
    raise UnsupportedQuantization(f"{msg}; the H100 runtime serves compressed-tensors FP8 checkpoints "
                                  "(float8_e4m3fn weights with channel or tensor scales, lm_head in bf16) only")


def _is_lm_head(pat) -> bool:
    return pat == "lm_head" or (isinstance(pat, str) and pat.startswith("re:") and "lm_head" in pat)


def parse_quantization_config(cfg: Dict[str, Any], tp_size: int = 1) -> Optional[Dict[str, Any]]:
    """-> None for an unquantized checkpoint, else {"strategy": "channel" | "tensor", "activations": None | "dynamic"}.
    Raises UnsupportedQuantization, naming what the runtime cannot serve."""
    qc = cfg.get("quantization_config")
    if not qc:
        return None
    method = qc.get("quant_method")
    if method != "compressed-tensors":
        blocks = qc.get("weight_block_size")   # quant_method "fp8" with 128 x 128 blocks: the official Qwen3-*-FP8 checkpoints
        _refuse(f"quantization_config.quant_method={method!r} is not supported"
                + (f" (block-scaled FP8, weight_block_size={blocks})" if blocks else ""))
    if qc.get("format") != "float-quantized":
        _refuse(f"quantization_config.format={qc.get('format')!r} is not supported")
    if qc.get("kv_cache_scheme"):
        _refuse("an FP8 KV cache (quantization_config.kv_cache_scheme) is not supported")
    if int(cfg.get("num_local_experts", 0) or 0) or cfg.get("model_type") == "mixtral":
        _refuse("FP8 Mixtral (sparse MoE experts) is not supported")
    if tp_size > 1:
        _refuse(f"FP8 weights with tensor parallelism (tensor_parallel_size={tp_size}) are not supported")
    groups = qc.get("config_groups") or {}
    if not groups:
        _refuse("quantization_config has no config_groups")
    strategies, acts = set(), set()
    for gname, g in groups.items():
        if g.get("format") not in (None, "float-quantized"):
            _refuse(f"config group {gname}: format={g.get('format')!r} is not supported")
        if list(g.get("targets") or []) != ["Linear"]:
            _refuse(f"config group {gname}: targets={g.get('targets')!r} (only ['Linear'] is supported)")
        w = g.get("weights") or {}
        if w.get("type") != "float" or int(w.get("num_bits", 0)) != 8:
            _refuse(f"config group {gname}: {w.get('num_bits')}-bit {w.get('type')} weights are not supported")
        if not w.get("symmetric", False) or w.get("dynamic"):
            _refuse(f"config group {gname}: asymmetric or dynamic weight quantization is not supported")
        if w.get("strategy") not in ("channel", "tensor"):
            _refuse(f"config group {gname}: weight strategy={w.get('strategy')!r} (block / group scales, e.g. the official "
                    "Qwen3-*-FP8 checkpoints' 128x128 blocks) is not supported")
        strategies.add(w["strategy"])
        if g.get("output_activations"):
            _refuse(f"config group {gname}: output activation quantization is not supported")
        a = g.get("input_activations")
        if a:
            if not a.get("dynamic"):
                _refuse(f"config group {gname}: static input activation scales (input_scale) are not supported")
            if a.get("type") != "float" or int(a.get("num_bits", 0)) != 8:
                _refuse(f"config group {gname}: {a.get('num_bits')}-bit {a.get('type')} input activations are not supported")
            acts.add("dynamic")
        else:
            acts.add(None)
    ignore = list(qc.get("ignore") or [])
    if not any(_is_lm_head(p) for p in ignore):
        _refuse("an FP8 lm_head is not supported (quantization_config.ignore must list lm_head)")
    rest = [p for p in ignore if not _is_lm_head(p)]
    if rest:
        # every projection of every layer must be FP8: the engine holds one weight format for all of them
        _refuse(f"quantization_config.ignore leaves {rest} unquantized; mixed bf16 / FP8 projections are not supported")
    return {"strategy": "channel" if "channel" in strategies else "tensor",
            "activations": "dynamic" if "dynamic" in acts else None}


def log_activation_scheme(q: Dict[str, Any]) -> None:
    if q.get("activations") == "dynamic":
        logger.warning("FP8 checkpoint with dynamic per-token FP8 input activations: the H100 runtime keeps activations "
                       "in bf16 (W8A16), so outputs differ from a runtime that quantizes activations")


def row_scales(scale: torch.Tensor, rows: int) -> torch.Tensor:
    """a checkpoint's weight_scale ([out, 1], [out], [1] or a scalar) as one contiguous value per weight row"""
    s = scale.reshape(-1)
    if s.numel() == 1:
        s = s.expand(rows)
    if s.numel() != rows:
        raise UnsupportedQuantization(f"weight_scale with {scale.numel()} values for {rows} weight rows: "
                                      "only channel or tensor scales are supported")
    return s.contiguous()


def dequantize_reference(w: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """W' exactly as transformers' compressed-tensors decompression gives it to a bf16 model (see the module docstring)"""
    return w.to(torch.bfloat16) * row_scales(scale, w.shape[0]).to(torch.bfloat16)[:, None]
