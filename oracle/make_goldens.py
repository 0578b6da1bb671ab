"""Generate tests/golden/* by running the oracle (transformers CPU backend) here.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Run from the repo root:

    python -m oracle.make_goldens            # all small cases (~1 min)
    python -m oracle.make_goldens --big      # + llama3_8b_2l case (~few min, 10 GB RAM)

The fixtures are committed; the GPU tests compare the CUDA engine with them and
the CPU tests re-run the oracle against them (determinism of the checker).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch
import transformers

from . import weights as W
from .hf_oracle import OracleGenerativeModel, build_llama, build_model

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

CHAT_TEMPLATE = (
    "{% for message in messages %}<|{{ message['role'] }}|>{{ message['content'] }}\n{% endfor %}"
    "{% if add_generation_prompt %}<|assistant|>{% endif %}"
)


def build_byte_tokenizer(out_dir: str):
    """A 256-byte + specials byte-level tokenizer built from scratch (no Hub).

    It has NO pad token on purpose, so loading it exercises the reference's
    fallback ``[PAD]`` + ``resize_token_embeddings`` path
    (generative_model.py:256-265, tests/test_model.py:502-509).
    """
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast

    alphabet = sorted(pre_tokenizers.ByteLevel.alphabet())
    vocab = {ch: i for i, ch in enumerate(alphabet)}
    tok = Tokenizer(models.BPE(vocab=vocab, merges=[]))
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)
    tok.decoder = decoders.ByteLevel()
    fast = PreTrainedTokenizerFast(tokenizer_object=tok, bos_token=None, eos_token=None, unk_token=None)
    fast.chat_template = CHAT_TEMPLATE
    os.makedirs(out_dir, exist_ok=True)
    fast.save_pretrained(out_dir)
    return fast


def load_byte_tokenizer():
    from transformers import AutoTokenizer
    return AutoTokenizer.from_pretrained(os.path.join(GOLDEN, "byte_tokenizer"))


def topk_pack(step_logits, k=16):
    vals, idx = [], []
    for l in step_logits:
        v, i = torch.topk(l, k, dim=-1)
        vals.append(v.numpy())
        idx.append(i.numpy())
    return np.stack(vals, 1), np.stack(idx, 1)  # [B, T, k]


ONLY = None         # --only: the case names to (re)generate

SUB_COLS = 4096     # big-vocabulary cases keep every step's logits on this many fixed pseudo-random columns (+ the top-16)


def sub_columns(vocab: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(99)
    return torch.randperm(vocab, generator=g)[:SUB_COLS].sort().values


def gen_case(name, cfg_name, seed, prompt, max_tokens, stop=(), tokenizer=None, pad_token_id=None,
             full_logits=True, echo=False, stop_from=None, presence_penalty=None, sub_logits=False):
    if ONLY is not None and name not in ONLY:
        return
    cfg = W.CONFIGS[cfg_name]
    sd = W.synth_state_dict(cfg, seed)
    model = build_model(cfg, sd)
    orc = OracleGenerativeModel(model, tokenizer=tokenizer, pad_token_id=pad_token_id)
    if stop_from is not None:  # derive a stop sequence that is guaranteed to occur: (row, i, j) of a free run
        row, i, j = stop_from
        free = orc.create_completion(prompt, max_tokens=max_tokens, temperature=0)
        S = free.output_ids.shape[1] - max_tokens
        stop = [free.output_ids[row, S + i:S + j].tolist()]
    res = orc.create_completion(prompt, max_tokens=max_tokens, stop=stop, echo=echo, temperature=0,
                                want_logits=True, presence_penalty=presence_penalty)
    # top-k of the PROCESSED scores: what argmax saw (identical to the raw logits unless a logits processor ran)
    tv, ti = topk_pack(res.extra["step_scores"] if presence_penalty else res.step_logits)
    out = dict(
        output_ids=res.output_ids.numpy(),
        topk_vals=tv, topk_idx=ti,
        meta=json.dumps(dict(
            name=name, cfg=cfg_name, seed=seed, max_tokens=max_tokens,
            finish_reason=res.finish_reason, prompt_tokens=res.prompt_tokens,
            completion_tokens=res.completion_tokens, texts=res.texts,
            pad_token_id=orc.pad_token_id, vocab_rows=int(model.get_input_embeddings().weight.shape[0]),
            weights_checksum=W.checksum(sd), stop=[list(s) if not isinstance(s, str) else s for s in stop],
            prompt=prompt if isinstance(prompt, (str, list)) and (isinstance(prompt, str) or isinstance(prompt[0], str)) else None,
            echo=echo, presence_penalty=presence_penalty,
            transformers=transformers.__version__, torch=torch.__version__,
            threads=torch.get_num_threads())),
    )
    if "num_local_experts" in cfg:
        # router decisiveness per position (min over layers of p(2nd) - p(3rd)): a flipped expert choice is a discrete
        # change, so logits are only comparable up to the first position whose margin is inside bf16 noise
        with torch.no_grad():
            fw = model(input_ids=res.output_ids, output_router_logits=True)
        risk = []
        for rl in fw.router_logits:            # [B*S_total, E] bf16 logits per layer
            pr = rl.float()                       # transformers 5.x returns the softmaxed router output here
            if not torch.allclose(pr.sum(-1), torch.ones(pr.shape[0]), atol=1e-3):
                pr = torch.softmax(pr, -1)
            pr = pr.view(res.output_ids.shape[0], res.output_ids.shape[1], -1)
            top = torch.topk(pr, 3, dim=-1).values
            margin = top[..., 1] - top[..., 2]                 # 2nd vs 3rd expert probability
            w2 = top[..., 1] / (top[..., 0] + top[..., 1])     # renormalised weight the 2nd expert carries
            # a flip between the 2nd and 3rd expert matters iff the margin is inside bf16 noise AND the expert has weight
            risk.append(torch.where(w2 > 0.01, margin, torch.ones_like(margin)))
        out["router_margin"] = torch.stack(risk, 0).min(0).values.numpy().astype(np.float32)   # [B, S+T]
    if sub_logits:      # [B, T, SUB_COLS] fp16 (exact for bf16 values in range) + the columns
        cols = sub_columns(cfg["vocab_size"])
        out["sub_cols"] = cols.numpy().astype(np.int32)
        out["sub_logits"] = torch.stack(res.step_logits, 1)[..., cols].numpy().astype(np.float16)
    more = None
    if full_logits:
        logits = torch.stack(res.step_logits, 1)                                        # [B, T, V]
        if logits.numel() * 2 <= (1 << 20):
            out["step_logits"] = logits.numpy().astype(np.float32)
        else:   # bf16 values, stored as their 16-bit patterns; rows split over two files so that each stays under 1 MB
            as_bf16 = logits.to(torch.bfloat16)
            assert torch.equal(as_bf16.float(), logits.float()), f"{name}: logits are not bf16 values, the 16-bit store would round them"
            bits = as_bf16.view(torch.int16).numpy()
            out["step_logits_bf16"], more = bits[:bits.shape[0] // 2], bits[bits.shape[0] // 2:]
    elif not sub_logits:
        out["step0_logits"] = res.step_logits[0].numpy().astype(np.float16)
    path = os.path.join(GOLDEN, name + ".npz")
    np.savez_compressed(path, **out)
    more_path = os.path.join(GOLDEN, name + ".2.npz")
    if more is not None:
        np.savez_compressed(more_path, step_logits_bf16=more)
    elif os.path.exists(more_path):   # left from an earlier, larger version of this case: tests/helpers.py would append its rows
        os.remove(more_path)
    print(f"wrote {path}: ids {out['output_ids'].shape} finish={res.finish_reason} "
          f"{res.seconds:.2f}s  margins(top1-top2) min={float((tv[..., 0]-tv[..., 1]).min()):.4f}")


MOE_DECISIVE = 0.005  # 2nd-vs-3rd expert probability margin regarded as safely above bf16 noise (~0.003)


def _moe_risk(model, ids):
    with torch.no_grad():
        fw = model(input_ids=ids, output_router_logits=True)
    risk = []
    for rl in fw.router_logits:
        pr = rl.float()
        if not torch.allclose(pr.sum(-1), torch.ones(pr.shape[0]), atol=1e-3):
            pr = torch.softmax(pr, -1)
        pr = pr.view(ids.shape[0], ids.shape[1], -1)
        top = torch.topk(pr, 3, dim=-1).values
        margin = top[..., 1] - top[..., 2]
        w2 = top[..., 1] / (top[..., 0] + top[..., 1])
        m12 = top[..., 0] - top[..., 1]     # order of the two chosen experts decides the accumulation order only
        risk.append(torch.where(w2 > 0.01, margin, torch.ones_like(margin)))
    return torch.stack(risk, 0).min(0).values


def find_decisive_moe_prompt(cfg_name, seed, B, S, T, vocab_hi, pad):
    cfg = W.CONFIGS[cfg_name]
    model = build_model(cfg, W.synth_state_dict(cfg, seed))
    orc = OracleGenerativeModel(model, pad_token_id=pad)
    good = []
    for trial in range(8000):
        row = ids_prompt(1, S, vocab_hi, 100000 + trial)
        out = orc.create_completion(row, max_tokens=T).output_ids
        if float(_moe_risk(model, out).min()) >= 1.5 * MOE_DECISIVE:
            good.append(row[0])
            if len(good) >= B:
                batch = good[-B:]
                outb = orc.create_completion(batch, max_tokens=T).output_ids
                if float(_moe_risk(model, outb).min()) >= MOE_DECISIVE:
                    print(f"{cfg_name}: decisive batch found after {trial + 1} candidate prompts")
                    return batch
    raise RuntimeError("no decisive MoE prompt found")


def ids_prompt(B, S, vocab_hi, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(3, vocab_hi, (B, S), generator=g).tolist()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big", action="store_true")
    ap.add_argument("--only", default=None, help="comma separated case names: generate just these (new fixtures without touching the old ones)")
    args = ap.parse_args()
    global ONLY
    ONLY = set(args.only.split(",")) if args.only else None
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count())

    if ONLY is None:
        build_byte_tokenizer(os.path.join(GOLDEN, "byte_tokenizer"))

    # (a) equal-length token-id prompts (generative_model.py:552-555 path), group size 2
    gen_case("tiny_g2_ids", "tiny_g2", 0, ids_prompt(4, 48, 1000, 1234), 16, pad_token_id=1030)
    # (b) ragged string prompts -> tokenizer, left padding, fallback [PAD] + embedding resize
    tok = load_byte_tokenizer()
    gen_case("tiny_g2_text", "tiny_g2", 0,
             ["Hello world", "The quick brown fox jumps over the lazy dog.", "KServe on B200!", "a"],
             12, tokenizer=tok)
    # (c) stop sequence as token ids: take case (a)'s 5th+6th generated token of row 2 -> must stop the batch
    gen_case("tiny_g2_stop", "tiny_g2", 0, ids_prompt(4, 48, 1000, 1234), 16, stop_from=(2, 4, 6), pad_token_id=1030)
    # presence_penalty > 0 -> repetition_penalty (generative_model.py:388-402): a logits processor under GREEDY decoding;
    # prompts drawn from 40 token ids so that repeats (and therefore penalised logits) occur
    gen_case("tiny_g2_reppen", "tiny_g2", 0, ids_prompt(4, 48, 40, 77), 24, pad_token_id=1030, presence_penalty=1.8)
    # (d) group size 4, 3 layers, odd batch, longer prompt (crosses KV page boundary of 64)
    gen_case("tiny_g4_ids", "tiny_g4", 1, ids_prompt(3, 100, 2048, 99), 40, pad_token_id=0)
    # (e) single sequence, batch 1, long decode crossing pages
    gen_case("tiny_g4_b1", "tiny_g4", 1, ids_prompt(1, 17, 2048, 5), 80, pad_token_id=0)
    # (f) token-id prompts that contain the pad id => transformers infers a mask (quirk q4)
    p = ids_prompt(2, 32, 1000, 77)
    p[0][:5] = [1030] * 5
    gen_case("tiny_g2_padinfer", "tiny_g2", 0, p, 8, pad_token_id=1030)
    # (g) Mixtral-style sparse MoE (BASELINE configs[3] architecture at test size).  An expert choice is a discrete
    # decision: where the oracle's own 2nd/3rd-expert margin is inside bf16 noise the two bf16 pipelines may
    # legitimately route differently.  The fixtures therefore use prompts (searched here, deterministically) on
    # which every position of every row is decisive, so the full logits comparison applies to them.
    for name, cfg_name, seed, B, S, T, vhi, pad in (("tiny_moe_ids", "tiny_moe", 3, 3, 14, 6, 1000, 1030),
                                                     ("tiny_moe8_ids", "tiny_moe8", 4, 2, 12, 6, 2048, 0)):
        if ONLY is not None and name not in ONLY:
            continue
        prompt = find_decisive_moe_prompt(cfg_name, seed, B, S, T, vhi, pad)
        gen_case(name, cfg_name, seed, prompt, T, pad_token_id=pad)
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        assert float(z["router_margin"].min()) >= MOE_DECISIVE, "search result is not decisive in the batched run"
    # (h) 8 KV heads: shards under TP = 2 / 4 / 8 (tests/test_tp_gpu.py, bench.py's in-run parity check); S crosses a KV page
    gen_case("tiny_kv8_ids", "tiny_kv8", 5, ids_prompt(4, 70, 4000, 4321), 16, pad_token_id=4098)
    # (i) peaked logits (lm_head = permuted embedding): >= 95 % of the steps are decisive, greedy ids compare exactly
    gen_case("tiny_g2_peaked", "tiny_g2_peaked", 0, ids_prompt(4, 48, 1000, 1234), 16, pad_token_id=1030)
    gen_case("tiny_g4_peaked", "tiny_g4_peaked", 1, ids_prompt(3, 100, 2048, 99), 40, pad_token_id=0)
    gen_case("tiny_kv8_peaked", "tiny_kv8_peaked", 5, ids_prompt(4, 70, 4000, 4321), 16, pad_token_id=4098)
    # (j) rope_scaling "llama3" (Llama-3.1 checkpoints), prompt longer than original_max_position_embeddings
    gen_case("tiny_g2_rope3", "tiny_g2_rope3", 0, ids_prompt(2, 300, 1000, 55), 8, pad_token_id=1030)
    # (k) boundary lengths: rows of 1 / 63 / 64 / 65 / 127 / 128 prompt tokens (one KV page = 64 tokens, one attention query
    # tile = 128), left padded with the pad id, decoded until prompt + generated = 192 = exactly three full pages — the
    # GPU test runs it on an engine whose max_seq_len is that 192 (the "maximum size" case)
    rows = ids_prompt(6, 128, 2048, 4242)
    rows = [[0] * (128 - n) + r[128 - n:] for r, n in zip(rows, (1, 63, 64, 65, 127, 128))]
    gen_case("tiny_g4_peaked_edges", "tiny_g4_peaked", 1, rows, 64, pad_token_id=0)
    if args.big:
        gen_case("llama3_8b_2l_ids", "llama3_8b_2l", 0, ids_prompt(2, 96, 128000, 1234), 8,
                 pad_token_id=128255, full_logits=False)
        big_cases()


def big_cases():
    """BASELINE.json's headline shapes on the 2-layer Llama-3-8B-dims model: 1024-token prompts (16 KV tiles through the
    prefill attention, M = 4096 rows through the prefill GEMMs), decode at context 1025..1040, V = 128256."""
    pad = 128255
    gen_case("llama3_8b_2l_b4", "llama3_8b_2l", 0, ids_prompt(4, 1024, 128000, 2024), 16, pad_token_id=pad,
             full_logits=False, sub_logits=True)
    gen_case("llama3_8b_2l_peaked_b4", "llama3_8b_2l_peaked", 0, ids_prompt(4, 1024, 128000, 2024), 16, pad_token_id=pad,
             full_logits=False, sub_logits=True)
    # ragged U[512, 1024] prompts, left padded with the pad id (token-id prompts carry no mask: transformers infers it, q4)
    g = torch.Generator().manual_seed(31)
    lens = torch.randint(512, 1025, (4,), generator=g).tolist()
    lens[1] = 1024
    rows = ids_prompt(4, 1024, 128000, 2025)
    rows = [[pad] * (1024 - n) + r[1024 - n:] for r, n in zip(rows, lens)]
    gen_case("llama3_8b_2l_peaked_ragged", "llama3_8b_2l_peaked", 0, rows, 16, pad_token_id=pad,
             full_logits=False, sub_logits=True)


if __name__ == "__main__":
    sys.exit(main())
