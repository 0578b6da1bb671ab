"""sample_kernel (sampling.cuh) as the engine launches it, through b200_op_sample, against tests/sampling_ref.py.

Every draw is checked exactly: the Philox uniform is reproduced bit for bit, so the reference knows which token the
kept set and its CDF give.  Greedy rows must match argmax of the fp32 processed scores bit for bit; sampled rows must give
the expected token and its processed score, except within the reference's rounding band, which must stay under 1 % of
draws.  Covered: V = 1000 (k capped at V), 1031, 128256 and 152064, ld > V, B = 1, 7 and 64, the static-batch launch
(one config, RNG counter (step, row)) and the continuous-batching launch (per-slot configs and bitmaps, counter
(n_gen[slot], 0)), the instruct checkpoints' defaults and the edges of every processor, rows built so that ties at the
k-th value, signed zeros, -inf and tied maxima carry most of the probability, and a replay of whole generate calls."""
import numpy as np
import pytest
import torch

import sampling_ref as R
from kserve_b200 import _lib

pytestmark = pytest.mark.gpu

LLAMA3_INSTRUCT = dict(do_sample=1, temperature=0.6, top_p=0.9, top_k=50)
QWEN25_INSTRUCT = dict(do_sample=1, temperature=0.7, top_p=0.8, top_k=20, repetition_penalty=1.05)
CONFIGS = {
    "llama3_instruct": LLAMA3_INSTRUCT,
    "qwen25_instruct": QWEN25_INSTRUCT,
    "k1024": dict(do_sample=1, top_k=1024),
    "p0.01": dict(do_sample=1, top_p=0.01, top_k=50),
    "p0.999": dict(do_sample=1, top_p=0.999, top_k=200),
    "t1e-3": dict(do_sample=1, temperature=1e-3, top_k=50),
    "t5": dict(do_sample=1, temperature=5.0, top_k=100, top_p=0.95),
    "pen1.8": dict(do_sample=1, repetition_penalty=1.8, top_k=50),
    "pen0.7": dict(do_sample=1, repetition_penalty=0.7, top_k=50, temperature=1.2),
    "greedy": dict(do_sample=0),
    "greedy_pen1.8": dict(do_sample=0, repetition_penalty=1.8),
}
STATS = {"draws": 0, "band": 0}


def _params(cfgs):
    arr = (_lib.GenParams * len(cfgs))()
    for g, c in zip(arr, cfgs):
        g.repetition_penalty = c.get("repetition_penalty", 0.0)
        g.do_sample = c.get("do_sample", 0)
        g.temperature = c.get("temperature", 0.0)
        g.top_p = c.get("top_p", 0.0)
        g.top_k = c.get("top_k", 0)
        g.seed = c.get("seed", 0)
    return arr


def run_op(lib, logits, V, cfgs, seen=None, row_slot=None, n_gen=None, step=0):
    """logits: cuda bf16 [B, ld]; seen: cuda int32 [rows, words] or None; returns (idx, val) on the host"""
    B = logits.shape[0]
    out_val = torch.full((B,), float("nan"), dtype=torch.float32, device="cuda")
    out_idx = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    ptr = lambda t: t.data_ptr() if t is not None else None
    rc = lib.b200_op_sample(logits.data_ptr(), logits.stride(0), B, V, ptr(seen), ptr(row_slot), ptr(n_gen), len(cfgs),
                            _params(cfgs), step, out_val.data_ptr(), out_idx.data_ptr(), None)
    assert rc == 0, lib.b200_last_error().decode()
    torch.cuda.synchronize()
    return out_idx.cpu(), out_val.cpu()


def check_row(logits_row, seen_mask, cfg, c0, c1, idx, val, what=""):
    """one decision against the reference; returns True when it was exact (outside the band)"""
    c = R.config(**cfg)
    toks, exact, scores = R.expected(logits_row, seen_mask, c, c0, c1)
    assert int(idx) in toks, f"{what}: token {int(idx)}, expected {sorted(toks)[:8]} (counter {c0}, {c1})"
    if not c["do_sample"]:
        assert np.float32(val).view(np.int32) == np.float32(scores[int(idx)]).view(np.int32), f"{what}: greedy value"
    else:
        assert float(val) == scores[int(idx)], f"{what}: out_val {float(val)} is not the processed score {scores[int(idx)]}"
    STATS["draws"] += 1
    STATS["band"] += 0 if exact else 1
    return exact


def assert_band_small(n_exact, n):
    assert n - n_exact <= max(1, 0.01 * n), f"{n - n_exact} of {n} draws fell in the rounding band"


def gauss_rows(B, V, seed):
    g = torch.Generator().manual_seed(seed)
    std = 1.5 + 2.5 * torch.rand(B, 1, generator=g)
    x = torch.randn(B, V, generator=g) * std
    x[:, torch.randperm(V, generator=g)[:8]] = 0.0          # exact zeros for the penalty to keep
    return x.bfloat16()


def seen_bits(rows, V, seed, frac=0.1):
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(rows, V, generator=g) < frac
    m[:, :64] = True                                         # a fixed block, so zeros set above may be hit too
    bits = np.stack([R.mask_to_bits(r.numpy()) for r in m])
    return m, torch.from_numpy(bits.view(np.int32)).cuda()


def to_device(x, ld):
    out = torch.full((x.shape[0], ld), float("nan"), dtype=torch.bfloat16, device="cuda")   # columns past V are NaN
    out[:, :x.shape[1]] = x.cuda()
    return out


@pytest.mark.parametrize("V,ld", [(1031, 1031 + 13), (128256, 128256), (152064, 152064 + 64)])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_static_batch(lib, V, ld, name):
    B, steps = 64, 3
    x = gauss_rows(B, V, V + len(name))
    mask, seen = seen_bits(B, V, V)
    d = to_device(x, ld)
    n = n_exact = 0
    for step in range(steps):
        cfg = dict(CONFIGS[name], seed=1000 * step + 17)
        idx, val = run_op(lib, d, V, [cfg], seen=seen, step=step)
        for b in range(B):
            n_exact += check_row(x[b], mask[b], cfg, step, b, idx[b], val[b], f"{name} V={V} step {step} row {b}")
            n += 1
    assert_band_small(n_exact, n)


@pytest.mark.parametrize("B", [1, 7])
@pytest.mark.parametrize("name", ["llama3_instruct", "qwen25_instruct", "greedy_pen1.8"])
def test_small_batches(lib, B, name):
    V = 128256
    n = n_exact = 0
    for rep in range(40 if B == 1 else 8):
        x = gauss_rows(B, V, 7 * rep + B)
        mask, seen = seen_bits(B, V, rep)
        cfg = dict(CONFIGS[name], seed=rep * 31 + 5)
        idx, val = run_op(lib, to_device(x, V), V, [cfg], seen=seen, step=rep)
        for b in range(B):
            n_exact += check_row(x[b], mask[b], cfg, rep, b, idx[b], val[b], f"{name} B={B} rep {rep} row {b}")
            n += 1
    assert n - n_exact <= max(1, 0.01 * n)


def test_top_k_capped_at_vocabulary(lib):
    """V = 1000 < top_k = 1024: every token is kept"""
    V, B = 1000, 64
    x = gauss_rows(B, V, 3)
    n = n_exact = 0
    for step in range(6):
        cfg = dict(do_sample=1, top_k=1024, seed=step)
        idx, val = run_op(lib, to_device(x, V + 24), V, [cfg], step=step)
        for b in range(B):
            n_exact += check_row(x[b], None, cfg, step, b, idx[b], val[b], f"step {step} row {b}")
            n += 1
    assert_band_small(n_exact, n)


@pytest.mark.parametrize("V", [1031, 152064])
def test_continuous_batching_slots_and_static_form(lib, V):
    """row_slot a permutation with gaps; greedy slots among sampling ones; the same rows in the static form"""
    B, slots = 64, 90
    g = torch.Generator().manual_seed(V)
    names = list(CONFIGS)
    x = gauss_rows(B, V, V + 1)
    d = to_device(x, V + 5)
    mask, seen = seen_bits(slots, V, V + 2)
    n = n_exact = 0
    for rep in range(5):
        row_slot = torch.randperm(slots, generator=g)[:B].to(torch.int32)
        n_gen = torch.randint(0, 5000, (slots,), generator=g, dtype=torch.int32)
        cfgs = [dict(CONFIGS[names[(s + rep) % len(names)]], seed=s * 7919 + rep) for s in range(slots)]
        idx, val = run_op(lib, d, V, cfgs, seen=seen, row_slot=row_slot.cuda(), n_gen=n_gen.cuda())
        for b in range(B):
            s = int(row_slot[b])
            n_exact += check_row(x[b], mask[s], cfgs[s], int(n_gen[s]), 0, idx[b], val[b], f"slot {s} row {b} rep {rep}")
            n += 1
        # the static form of the same rows: one config, bitmap row = batch row, counter (step, row)
        cfg = dict(QWEN25_INSTRUCT, seed=rep + 11)
        sseen = seen[row_slot.long().cuda()].contiguous()
        idx, val = run_op(lib, d, V, [cfg], seen=sseen, step=rep + 3)
        for b in range(B):
            n_exact += check_row(x[b], mask[int(row_slot[b])], cfg, rep + 3, b, idx[b], val[b], f"static row {b} rep {rep}")
            n += 1
    assert_band_small(n_exact, n)


# ---- adversarial rows: the tokens a wrong kept set would mishandle carry most of the probability

def _draw_rows(lib, rows, cfg, steps, V, ld=None):
    B = rows.shape[0]
    d = to_device(rows, ld or V)
    n = n_exact = 0
    for step in range(steps):
        c = dict(cfg, seed=step * 101 + 7)
        idx, val = run_op(lib, d, V, [c], step=step)
        for b in range(B):
            n_exact += check_row(rows[b], None, c, step, b, idx[b], val[b], f"step {step} row {b}")
            n += 1
    return n, n_exact


def _place(V, groups, rest, seed):
    """a bf16 row: groups = [(value, count)] at random positions, `rest` elsewhere"""
    g = torch.Generator().manual_seed(seed)
    x = torch.full((V,), rest, dtype=torch.float32)
    perm = torch.randperm(V, generator=g)
    o = 0
    for v, cnt in groups:
        x[perm[o:o + cnt]] = v
        o += cnt
    return x.bfloat16()


def test_ties_at_kth_value_beyond_1024_candidates(lib):
    """k = 1024: 1000 values one bf16 ulp above 1.0 and 100 at 1.0 -> transformers keeps 1100 tokens"""
    V = 128256
    rows = torch.stack([_place(V, [(1.0078125, 1000), (1.0, 100)], -30.0, s) for s in range(16)])
    n, n_exact = _draw_rows(lib, rows, dict(do_sample=1, top_k=1024), 16, V)
    assert_band_small(n_exact, n)


def test_constant_row_keeps_the_whole_vocabulary(lib):
    """k = 50 on a constant row: every token ties with the 50th, so the draw is uniform over all V in index order"""
    V = 152064
    rows = torch.full((8, V), 0.5).bfloat16()
    n, n_exact = _draw_rows(lib, rows, dict(do_sample=1, top_k=50), 24, V)
    assert_band_small(n_exact, n)


def test_signed_zero_ties_at_kth_value(lib):
    """k-th value +0.0 with 60 tokens at -0.0 (44 % of the mass); transformers keeps them, -0.0 < 0.0 being false"""
    V = 1031
    rows = []
    for s in range(32):
        r = _place(V, [(0.5, 10), (0.0, 60), (0.0, 60)], -40.0, s).float()
        r[torch.nonzero(r == 0.0).flatten()[::2]] = -0.0
        rows.append(r.bfloat16())
    rows = torch.stack(rows)
    assert int((rows.float() == 0).sum(1).min()) == 120 and int(torch.signbit(rows.float()).logical_and(rows.float() == 0).sum(1).min()) == 60
    n, n_exact = _draw_rows(lib, rows, dict(do_sample=1, top_k=50), 12, V, ld=V + 1)
    assert_band_small(n_exact, n)


def test_minus_inf_logits_with_k_beyond_the_finite_ones(lib):
    """30 finite logits, k = 50: the k-th value is -inf, every token is kept, only the finite ones can be drawn"""
    V = 128256
    g = torch.Generator().manual_seed(5)
    rows = torch.stack([_place(V, [(float(v), 1) for v in torch.randn(30, generator=g) * 2], float("-inf"), s)
                        for s in range(16)])
    n, n_exact = _draw_rows(lib, rows, dict(do_sample=1, top_k=50), 16, V)
    assert_band_small(n_exact, n)


def test_top_p_cut_inside_a_tie_run(lib):
    """8 tokens tied at the maximum, everything else -inf, top_p = 0.5: the tails are exact multiples of 1/8, the cut
    keeps exactly 4 of the run, the 4 lowest indices"""
    V = 152064
    rows = torch.stack([_place(V, [(2.0, 8)], float("-inf"), s) for s in range(16)])
    n, n_exact = _draw_rows(lib, rows, dict(do_sample=1, top_k=50, top_p=0.5), 16, V)
    assert n_exact == n


def test_top_k_1_draws_among_tied_maxima(lib):
    """top_k = 1 under do_sample keeps every token tied at the maximum (TopKLogitsWarper); it is not argmax"""
    V = 128256
    rows = []
    for s in range(32):
        r = gauss_rows(1, V, s)[0].float().clamp(max=2.0)
        r[torch.randperm(V, generator=torch.Generator().manual_seed(s))[:3]] = 3.0
        rows.append(r.bfloat16())
    rows = torch.stack(rows)
    n, n_exact = _draw_rows(lib, rows, dict(do_sample=1, top_k=1, temperature=1.7), 8, V)
    assert n_exact == n


# ---- the engine: every step of generate replayed on its own logits

def _engine(cfg_name, vocab_rows):
    from oracle import weights as W
    from kserve_b200.engine import B200Engine
    cfg = W.CONFIGS[cfg_name]
    eng = B200Engine(cfg, vocab_rows=vocab_rows, max_batch=4, max_seq_len=256)

    def gen():
        embed = None
        for name, t in W.iter_state_dict(cfg, 0):
            if name == "model.embed_tokens.weight":
                embed = t
            yield name, t
        if cfg.get("tie_word_embeddings"):
            yield "lm_head.weight", embed
    eng.load_weights(gen())
    return eng


@pytest.mark.parametrize("cfg_name,V,pad,sampling", [("llama3_8b_2l", 128256, 128255, LLAMA3_INSTRUCT),
                                                     ("qwen2_7b_2l", 152064, 152063, QWEN25_INSTRUCT)])
def test_generate_replay(cfg_name, V, pad, sampling):
    """batch 4 with one left-padded row, 32 steps: each sampled token is the one the reference draws from that step's
    logits, with the penalty bitmap = prompt + pads + tokens generated so far and the counter (step, row)"""
    S, T = 48, 32
    g = torch.Generator().manual_seed(V)
    ids = torch.randint(0, V - 1, (4, S), generator=g)
    mask = torch.ones_like(ids)
    ids[1, :13] = pad
    mask[1, :13] = 0
    eng = _engine(cfg_name, V)
    try:
        compared = 0
        for seed in (1, 2):
            cfg = dict(sampling, seed=seed)
            r = eng.generate(ids, mask, max_new_tokens=T, pad_token_id=pad, want_logits=True, do_sample=True,
                             temperature=cfg["temperature"], top_p=cfg["top_p"], top_k=cfg["top_k"],
                             repetition_penalty=cfg.get("repetition_penalty"), seed=seed)
            assert r.num_generated == T
            gen = r.output_ids[:, S:]
            for b in range(4):
                seen = torch.zeros(V, dtype=torch.bool)
                seen[ids[b]] = True
                for t in range(T):
                    tok = int(gen[b, t])
                    exact = check_row(r.logits[t, b], seen, cfg, t, b, tok,
                                      R.process(r.logits[t, b], seen, R.config(**cfg))[tok], f"{cfg_name} seed {seed} row {b} step {t}")
                    compared += 1
                    if not exact:
                        break
                    seen[tok] = True
        assert compared >= 200, f"only {compared} decisions compared"
    finally:
        eng.close()


def test_report_band_fraction():
    """runs last in this file: the share of all draws above that fell in the rounding band"""
    if STATS["draws"]:
        frac = STATS["band"] / STATS["draws"]
        print(f"\nsampling draws checked: {STATS['draws']}, in the rounding band: {STATS['band']} ({100 * frac:.3f} %)")
        assert frac <= 0.01
