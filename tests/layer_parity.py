"""Engine parity at the final hidden state (helper module of tests/test_layer_parity_cpu.py and _gpu.py).

A checkpoint with vocab_size = H and an untied lm_head = eye(H) makes the engine's bf16 logits exactly its final-normed
hidden state: every logit of the swap-AB LM-head GEMM is one non-zero product summed in fp32 (split-K or stream-K
included), so generate(..., want_logits=True) returns the hidden state per element with no ABI or engine change.

That state is compared with two transformers runs of the same weights: a float64 model (the reference) and a bf16
model (the yardstick; HF's rounding points, which the engine follows).  With d_eng = eng - ref64 and
d_hf = hf16 - ref64 the engine must be no less accurate than transformers' own bf16 model:

  per (step, row)                 rms(d_eng) <= A * rms(d_hf)
  per (step, row, 128 columns)    the same rule, the same A (catches column-range bugs: GEMM tails, norm chunks)
  per element                     |d_eng| <= M * max over its 128-column block of |d_hf| + half a bf16 ulp of ref64
  over the case                   mean of the per-(step, row) ratios <= MEAN_RATIO

A and M are fixed here, before any engine run.  Two things calibrate and check them:

  the permuted twin   the hidden and intermediate channels permuted through every tensor: a model mathematically
                      identical to the yardstick whose bf16 run sums every reduction in another order.  Un-permuted, it
                      passes the criterion against the yardstick: the thresholds accept a legitimate bf16 implementation.
  negative controls   small weight or position perturbations given to both references (not to the engine or the
                      twin): each makes the criterion fail.

The test draws its own seeded weights (not tools/synth_weights.py's), scaled so that each layer's attention and MLP
update has an RMS comparable to the residual stream's (UPDATE_RMS_RANGE, checked in float64 by the CPU test);
otherwise an error inside a layer would be diluted by the embedding that starts the residual stream.
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch

A = 2.0               # per (step, row) and per (step, row, 128-column block) rms ratio to the bf16 yardstick
M = 4.0               # per element: multiple of the block's largest yardstick error
MEAN_RATIO = 1.3      # mean per-(step, row) ratio of a whole case
BLOCK = 128
PERTURB = 2.0 ** -4   # the negative controls' relative perturbation
UPDATE_RMS_RANGE = (0.4, 2.5)   # rms(layer update) / rms(residual stream entering it), each attention and MLP block of each row

# weight gains (times 1/sqrt(fan-in)): q / k make the attention scores O(2) so heads attend selectively rather than
# average (an average of v shrinks the attention update); o / down bring the updates to the residual stream's RMS, and
# in layer 1 by LAYER1_GAIN more, since layer 0's updates have about doubled the residual stream by then
GAIN = {"q_proj": 1.4, "k_proj": 1.4, "v_proj": 1.0, "o_proj": 2.2, "gate_proj": 1.0, "up_proj": 1.0, "down_proj": 3.0}
LAYER1_GAIN = 1.8

# layer shape -> (family, H, I, nh, nkv); head_dim 128 everywhere (the engine's only head size)
SHAPES = {
    "tiny_g2": ("llama", 512, 1024, 4, 2),
    "tiny_g4": ("llama", 1024, 2816, 8, 2),
    "llama3_8b": ("llama", 4096, 14336, 32, 8),
    "llama32_3b": ("llama", 3072, 8192, 24, 8),        # Llama-3.2-3B-like: G = 3
    "tiny_qwen2": ("qwen2", 512, 1024, 8, 2),
    "qwen25_0p5b": ("qwen2", 896, 4864, 14, 2),        # (Qwen2.5-0.5B's head_dim is 64; the engine serves 128)
    "qwen25_1p5b": ("qwen2", 1536, 8960, 12, 2),
    "qwen25_7b": ("qwen2", 3584, 18944, 28, 4),
    "qwen25_14b": ("qwen2", 5120, 13824, 40, 8),
    "tiny_qwen3": ("qwen3", 512, 1024, 8, 4),
    "qwen3_0p6b": ("qwen3", 1024, 3072, 16, 8),
    "qwen3_4b": ("qwen3", 2560, 9728, 32, 8),
    "qwen3_8b": ("qwen3", 4096, 12288, 32, 8),
    "qwen3_32b": ("qwen3", 5120, 25600, 64, 8),
}


def config(shape: str) -> dict:
    fam, H, I, nh, nkv = SHAPES[shape]
    assert H % BLOCK == 0
    cfg = dict(vocab_size=H, hidden_size=H, intermediate_size=I, num_hidden_layers=2, num_attention_heads=nh,
               num_key_value_heads=nkv, head_dim=128, max_position_embeddings=8192)
    if fam == "llama":
        cfg.update(rms_norm_eps=1e-5, rope_theta=500000.0)
    else:
        cfg.update(model_type=fam, rms_norm_eps=1e-6, rope_theta=1000000.0, use_sliding_window=False)
    return cfg


def family(cfg: dict) -> str:
    return cfg.get("model_type", "llama")


def draw_weights(cfg: dict, seed: int, device="cpu") -> Dict[str, torch.Tensor]:
    """seeded bf16 state dict with the identity LM head (drawn on `device`; the same seed gives the same tensors on the
    same device type)"""
    from tools.synth_weights import tensor_specs
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for name, shape, kind in tensor_specs(dict(cfg, tie_word_embeddings=False)):
        if name == "lm_head.weight":
            t = torch.eye(shape[0], shape[1], device=device)
        elif kind == "embed":
            t = torch.randn(shape, generator=g, device=device)
        elif name.endswith(("q_norm.weight", "k_norm.weight")):
            t = 1.0 + torch.rand(shape, generator=g, device=device)      # [1, 2]: q / k come out of the norm with RMS ~1.5
        elif kind == "norm":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        elif kind == "bias":
            t = 0.5 * torch.randn(shape, generator=g, device=device)
        else:
            proj = name.rsplit(".", 2)[-2]
            gain = GAIN[proj] * (LAYER1_GAIN if proj in ("o_proj", "down_proj") and ".layers.0." not in name else 1.0)
            t = torch.randn(shape, generator=g, device=device) * (gain / math.sqrt(shape[1]))
        sd[name] = t.to(torch.bfloat16)
    return sd


# ---- the permuted twin ------------------------------------------------------------------------------------------------
def permutations(cfg: dict, seed: int, device="cpu"):
    g = torch.Generator(device="cpu").manual_seed(seed + 99991)
    return (torch.randperm(cfg["hidden_size"], generator=g).to(device),
            torch.randperm(cfg["intermediate_size"], generator=g).to(device))


def permute(sd: Dict[str, torch.Tensor], p: torch.Tensor, q: torch.Tensor) -> Dict[str, torch.Tensor]:
    """hidden channels by p (embedding and q / k / v / gate / up / LM-head input columns, o / down output rows, every
    hidden norm weight), intermediate channels by q (gate / up rows, down columns); the residual stream of the result is
    x[p] wherever the original's is x"""
    out = {}
    for n, t in sd.items():
        if n.endswith(("input_layernorm.weight", "post_attention_layernorm.weight", "model.norm.weight")):
            t = t[p]
        elif n.endswith(("embed_tokens.weight", "q_proj.weight", "k_proj.weight", "v_proj.weight", "lm_head.weight")):
            t = t[:, p]
        elif n.endswith("o_proj.weight"):
            t = t[p]
        elif n.endswith(("gate_proj.weight", "up_proj.weight")):
            t = t[q][:, p]
        elif n.endswith("down_proj.weight"):
            t = t[p][:, q]
        out[n] = t.contiguous()
    return out


# ---- negative controls ------------------------------------------------------------------------------------------------
def _scaled(sd, name, index, factor=1.0 + PERTURB):
    sd = dict(sd)
    t = sd[name].double().clone()
    t[index] *= factor
    sd[name] = t
    return sd


def controls(cfg: dict) -> Dict[str, dict]:
    """name -> dict(edit=state dict -> perturbed state dict (float64 where edited), shift_last=bool): what both
    references get; the engine (or on the CPU the twin standing in for it) keeps the original weights"""
    fam = family(cfg)
    c = {
        "v_rows_kv_head0_layer0": dict(edit=lambda sd: _scaled(sd, "model.layers.0.self_attn.v_proj.weight", slice(0, 128))),
        "o_cols_q_head0_layer1": dict(edit=lambda sd: _scaled(sd, "model.layers.1.self_attn.o_proj.weight",
                                                               (slice(None), slice(0, 128)))),
        "final_norm_block1": dict(edit=lambda sd: _scaled(sd, "model.norm.weight", slice(BLOCK, 2 * BLOCK))),
        "rope_last_token_pos_plus1": dict(edit=None, shift_last=True),
    }
    if fam == "qwen2":
        c["q_bias_head0_dropped_layer0"] = dict(edit=lambda sd: _scaled(sd, "model.layers.0.self_attn.q_proj.bias",
                                                                       slice(0, 128), 0.0))
    if fam == "qwen3":
        c["k_norm_16_dims_layer0"] = dict(edit=lambda sd: _scaled(sd, "model.layers.0.self_attn.k_norm.weight", slice(0, 16)))
    return c


# ---- transformers references ------------------------------------------------------------------------------------------
def build_hf(cfg: dict, sd: Dict[str, torch.Tensor], dtype, device="cpu"):
    """transformers model of `sd` in `dtype` on `device`, eager attention (SDPA / flash would keep P in fp32 and make the
    bf16 yardstick more precise than HF's eager bf16 model is)"""
    from oracle.hf_oracle import build_llama
    from tools.qwen2_oracle import build_qwen2
    from tools.qwen3_oracle import build_qwen3
    builder = {"llama": build_llama, "qwen2": build_qwen2, "qwen3": build_qwen3}[family(cfg)]
    model = builder(cfg, {n: t.to(dtype) for n, t in sd.items()}, dtype).to(device)
    model.set_attn_implementation("eager")
    return model


@torch.no_grad()
def final_hidden(model, ids: List[int], n_steps: int, shift_last: bool = False) -> torch.Tensor:
    """final-normed hidden state [n_steps, H] (float64) at positions len(ids) - n_steps .. len(ids) - 1 of one unpadded
    causal pass; `shift_last` runs the last token at position + 1"""
    dev = next(model.parameters()).device
    x = torch.tensor(ids, dtype=torch.int64, device=dev)[None]
    pos = torch.arange(len(ids), device=dev)
    if shift_last:
        pos[-1] += 1
    h = model.model(input_ids=x, position_ids=pos[None]).last_hidden_state[0]
    return h[-n_steps:].double()


def sequences(prompts: List[List[int]], forced: torch.Tensor, T: int) -> List[List[int]]:
    """prompt + the first T forced tokens of each row: its outputs at positions S - 1 .. S - 1 + T are steps 0 .. T"""
    return [list(p) + forced[b, :T].tolist() for b, p in enumerate(prompts)]


def run_rows(model, seqs: List[List[int]], T: int, shift_last: bool = False) -> List[torch.Tensor]:
    """per row [T + 1, H] float64 on the CPU"""
    return [final_hidden(model, s, T + 1, shift_last).cpu() for s in seqs]


def prompt_pool(n: int, vocab: int, seed: int, fixed=(1, 63, 64, 65, 127, 128, 129), lo=2, hi=300) -> List[List[int]]:
    """n prompts: the boundary lengths first, then seeded lengths in [lo, hi]; token ids in [0, vocab)"""
    g = torch.Generator().manual_seed(seed)
    lens = list(fixed[:n]) + torch.randint(lo, hi + 1, (max(0, n - len(fixed)),), generator=g).tolist()
    return [torch.randint(0, vocab, (L,), generator=g).tolist() for L in lens]


def forced_tokens(n: int, T: int, vocab: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed + 7)
    return torch.randint(0, vocab, (n, T + 1), generator=g)


# ---- the criterion ----------------------------------------------------------------------------------------------------
def _half_ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 8)


def judge(eng: torch.Tensor, hf: torch.Tensor, ref: torch.Tensor) -> dict:
    """eng / hf / ref [..., H] (any leading shape, e.g. steps x rows): the ratios of the criterion and whether it holds"""
    H = ref.shape[-1]
    eng, hf, ref = (t.double().reshape(-1, H) for t in (eng, hf, ref))
    de, dh = eng - ref, hf - ref
    row = de.pow(2).mean(-1).sqrt() / dh.pow(2).mean(-1).sqrt()
    deb, dhb = de.view(-1, H // BLOCK, BLOCK), dh.view(-1, H // BLOCK, BLOCK)
    block = deb.pow(2).mean(-1).sqrt() / dhb.pow(2).mean(-1).sqrt()
    bound = M * dhb.abs().amax(-1, keepdim=True) + _half_ulp_bf16(ref).view(-1, H // BLOCK, BLOCK)
    elem = deb.abs() / bound
    r = dict(row=float(row.max()), block=float(block.max()), elem=float(elem.max()), mean=float(row.mean()),
             finite=bool(torch.isfinite(eng).all()))
    r["ok"] = r["finite"] and r["row"] <= A and r["block"] <= A and r["elem"] <= 1.0 and r["mean"] <= MEAN_RATIO
    return r


def fmt(r: dict) -> str:
    return (f"row {r['row']:.3f} block {r['block']:.3f} elem {r['elem']:.3f} mean {r['mean']:.3f}"
            f"{'' if r['finite'] else ' NON-FINITE'} -> {'pass' if r['ok'] else 'FAIL'}")


def logits_check_catches(eng: torch.Tensor, oracle: torch.Tensor, vocab: int, seed: int) -> bool:
    """tests/helpers.py's teacher-forced logits check (max |err| <= 4 ulps x max |logit|) through a random LM head
    (the synthetic checkpoints' N(0, 1/H) rows) on two sets of bf16 final hidden states [..., H]: True if it fails"""
    from helpers import logits_tol
    H = oracle.shape[-1]
    g = torch.Generator().manual_seed(seed)
    head = (torch.randn(vocab, H, generator=g) / math.sqrt(H)).to(torch.bfloat16).float()
    le = (eng.float().to(torch.bfloat16).float() @ head.T).to(torch.bfloat16).float()
    lo = (oracle.float().to(torch.bfloat16).float() @ head.T).to(torch.bfloat16).float()
    return float((le - lo).abs().max()) > logits_tol(lo)
