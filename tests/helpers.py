"""Shared helpers for the parity tests (golden fixture loading, engine construction)."""
import json
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# Stated bf16 tolerance for logits (SURVEY.md §8c(ii)): both sides run a bf16 pipeline with fp32
# accumulation; they differ in accumulation order only.  One bf16 ulp is 2^-8 relative; after L layers of
# residual updates the logits of the two pipelines are observed to differ by a few ulps of the largest
# logit.  TOL_ULPS * 2^-8 * max|logit| is the absolute tolerance used everywhere below.
TOL_ULPS = 4.0


def logits_tol(ref_logits: torch.Tensor) -> float:
    return TOL_ULPS * 2.0 ** -8 * float(ref_logits.abs().max())


def logits_tol_elementwise(ref: torch.Tensor, row_floor: torch.Tensor = None) -> torch.Tensor:
    """Per-element tolerance for PEAKED logits: TOL_ULPS bf16 ulps of max(|logit|, the row's 2nd-largest |logit|).
    One logit towers over the rest there, so a tolerance relative to the row maximum would be vacuous for the bulk; the
    2nd-largest magnitude is the scale of everything but the peak, and the peak itself is held to its own ulps."""
    if row_floor is None:
        row_floor = ref.abs().topk(2, dim=-1).values[..., 1]
    return TOL_ULPS * 2.0 ** -8 * torch.maximum(ref.abs(), row_floor.abs().unsqueeze(-1))


def load_case(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    out = torch.from_numpy(z["output_ids"].astype(np.int64))
    T = meta["completion_tokens"] // out.shape[0]
    S = out.shape[1] - T
    case = dict(meta=meta, output_ids=out, S=S, T=T, input_ids=out[:, :S].contiguous(), gen=out[:, S:].contiguous(),
                topk_vals=torch.from_numpy(z["topk_vals"]), topk_idx=torch.from_numpy(z["topk_idx"]))
    if "step_logits" in z:
        case["step_logits"] = torch.from_numpy(z["step_logits"])  # [B, T, V]
    if "step_logits_bf16" in z:   # the same logits (bf16 values) as 16-bit patterns, rows split over <name>.npz and <name>.2.npz
        parts = [z["step_logits_bf16"]]
        more = os.path.join(GOLDEN, name + ".2.npz")
        if os.path.exists(more):
            parts.append(np.load(more)["step_logits_bf16"])
        case["step_logits"] = torch.from_numpy(np.concatenate(parts)).view(torch.bfloat16).float()
    if "step0_logits" in z:
        case["step0_logits"] = torch.from_numpy(z["step0_logits"].astype(np.float32))
    if "sub_logits" in z:     # big-vocabulary cases: every step's logits on a fixed subset of the columns, [B, T, n]
        case["sub_logits"] = torch.from_numpy(z["sub_logits"].astype(np.float32))
        case["sub_cols"] = torch.from_numpy(z["sub_cols"].astype(np.int64))
    pad = meta["pad_token_id"]
    mask = (case["input_ids"] != pad).long() if pad is not None else torch.ones_like(case["input_ids"])
    case["mask"] = mask
    case["margin"] = case["topk_vals"][..., 0] - case["topk_vals"][..., 1]  # [B, T]
    return case


def make_engine(cfg_name, seed, vocab_rows=None, **kw):
    from oracle import weights as W  # the oracle package also owns the synthetic checkpoint generator
    from kserve_b200.engine import B200Engine
    cfg = W.CONFIGS[cfg_name]
    eng = B200Engine(cfg, vocab_rows=vocab_rows, **kw)

    def gen():
        for name, t in W.iter_state_dict(cfg, seed):
            if vocab_rows and name in ("model.embed_tokens.weight", "lm_head.weight"):
                t = t[:vocab_rows] if t.shape[0] >= vocab_rows else torch.cat(
                    [t, torch.zeros(vocab_rows - t.shape[0], t.shape[1], dtype=t.dtype)])
            yield name, t
    eng.load_weights(gen())
    return eng
