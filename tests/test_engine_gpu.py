"""End-to-end parity of the CUDA engine (through the C ABI) against the committed oracle fixtures.

Protocol (SURVEY.md §8c): (i) teacher-forced per-step logits within the stated bf16 tolerance,
(ii) greedy ids equal wherever the oracle's top-1/top-2 margin exceeds 2x that tolerance,
(iii) free-running ids equal up to the first step whose oracle margin is inside the tolerance,
(iv) stop / length / usage bookkeeping equal.  bf16 CPU results themselves move by an ulp with the
host's thread count, so bit-exact ids on near-tie steps are not a property either side has.
"""
import json
import os

import pytest
import torch

from helpers import load_case, logits_tol, logits_tol_elementwise, make_engine

pytestmark = pytest.mark.gpu

STATS = {}


def _record(name, **kw):
    """Parity statistics of the run; written as JSON to the file KSERVE_PARITY_STATS names, if set."""
    STATS[name] = kw
    path = os.environ.get("KSERVE_PARITY_STATS")
    if path:
        with open(path, "w") as f:
            json.dump(STATS, f, indent=1)


CASES = ["tiny_g2_ids", "tiny_g2_text", "tiny_g2_padinfer", "tiny_g4_ids", "tiny_g4_b1",
         "tiny_moe_ids", "tiny_moe8_ids",   # Mixtral-style sparse MoE (BASELINE configs[3] architecture)
         "tiny_kv8_ids",                    # 8 KV heads (the TP = 4 / 8 test shapes), odd vocabulary
         "tiny_g2_rope3"]                   # rope_scaling "llama3" (Llama-3.1), prompt past original_max_position_embeddings
# lm_head = permuted embedding: one logit towers over the rest as in a trained model, so (nearly) every step is decisive
# and greedy ids are compared EXACTLY (VERDICT r01 weak #3); logits are held to a per-element tolerance
PEAKED = ["tiny_g2_peaked", "tiny_g4_peaked", "tiny_kv8_peaked"]


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(case):
        m = case["meta"]
        key = (m["cfg"], m["seed"], m["vocab_rows"])
        if key not in cache:
            cache[key] = make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], max_batch=8, max_seq_len=512)
        return cache[key]
    yield get
    for e in cache.values():
        e.close()


@pytest.mark.parametrize("name", CASES)
def test_teacher_forced_logits_and_greedy(engines, name):
    c = load_case(name)
    eng = engines(c)
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=c["meta"]["pad_token_id"],
                     forced_tokens=c["gen"], want_logits=True)
    assert r.num_generated == c["T"]
    assert torch.equal(r.output_ids, c["output_ids"]), "forced tokens must be echoed verbatim"
    got = r.logits.float().permute(1, 0, 2)          # [B, T, V]
    ref = c["step_logits"]
    tol = logits_tol(ref)
    err = (got - ref).abs()
    _record(name + ":teacher_forced", max_err=float(err.max()), mean_err=float(err.mean()), tol=tol,
            max_logit=float(ref.abs().max()), frac_within_1ulp=float((err <= 2.0 ** -8 * ref.abs().max()).float().mean()))
    assert not torch.isnan(got).any()
    assert float(err.max()) <= tol, f"max logits error {float(err.max()):.4f} > tol {tol:.4f}"
    # greedy ids equal wherever the oracle margin is decisive
    pred = got.argmax(-1)
    decisive = c["margin"] > 2 * tol
    agree = pred == c["gen"]
    assert bool(agree[decisive].all()), "argmax differs on a step whose oracle margin exceeds 2x tolerance"
    _record(name + ":greedy_tf", steps=int(agree.numel()), agree=int(agree.sum()), decisive=int(decisive.sum()))


@pytest.mark.parametrize("name", CASES)
def test_free_running_ids(engines, name):
    c = load_case(name)
    eng = engines(c)
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=c["meta"]["pad_token_id"])
    assert r.num_generated == c["T"]
    assert torch.equal(r.output_ids[:, :c["S"]], c["input_ids"])
    tol = logits_tol(c["step_logits"])
    gen = r.output_ids[:, c["S"]:]
    exact_rows = 0
    for b in range(gen.shape[0]):
        neq = (gen[b] != c["gen"][b]).nonzero()
        if len(neq) == 0:
            exact_rows += 1
            continue
        t = int(neq[0])
        assert float(c["margin"][b, t]) <= 2 * tol, (
            f"row {b} diverges at step {t} where the oracle margin {float(c['margin'][b, t]):.4f} is decisive")
    _record(name + ":free_running", rows=int(gen.shape[0]), exact_rows=exact_rows,
            token_match=float((gen == c["gen"]).float().mean()))
    # determinism of the engine itself: same call twice -> identical ids
    r2 = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=c["meta"]["pad_token_id"])
    assert torch.equal(r.output_ids, r2.output_ids)


def _check_peaked(eng, c, name):
    pad = c["meta"]["pad_token_id"]
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"], want_logits=True)
    got = r.logits.float().permute(1, 0, 2)
    ref = c["step_logits"]
    tol = logits_tol_elementwise(ref)
    err = (got - ref).abs()
    assert bool((err <= tol).all()), f"worst element: err/tol = {float((err / tol).max()):.2f}"
    decisive = c["margin"] > 2 * logits_tol(ref)
    assert float(decisive.float().mean()) >= 0.95
    assert bool((got.argmax(-1) == c["gen"])[decisive].all())
    free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
    exact = free.output_ids[:, c["S"]:] == c["gen"]
    _record(name + ":peaked", decisive_frac=float(decisive.float().mean()), free_running_exact_match=float(exact.float().mean()),
            worst_err_over_tol=float((err / tol).max()), max_err_bulk=float(err.max()), steps=int(exact.numel()))
    if bool(decisive.all()):
        assert bool(exact.all()), "every step is decisive: free-running greedy ids must equal the oracle's exactly"
    else:
        first_soft = (~decisive).float().argmax(1)          # rows may legitimately diverge from their first soft step on
        for b in range(exact.shape[0]):
            upto = int(first_soft[b]) if not bool(decisive[b].all()) else exact.shape[1]
            assert bool(exact[b, :upto].all())


@pytest.mark.parametrize("name", PEAKED)
def test_peaked_logits_greedy_ids_exact(engines, name):
    c = load_case(name)
    _check_peaked(engines(c), c, name)


def test_boundary_lengths_on_an_engine_sized_exactly_for_them():
    """rows of 1 / 63 / 64 / 65 / 127 / 128 prompt tokens (KV page = 64 tokens, attention query tile = 128), left padded,
    decoded until prompt + generated = 192 tokens = three full pages, on an engine whose max_seq_len IS 192 and whose
    max_batch is the batch: every page and tile boundary and the maximum size in one oracle fixture"""
    c = load_case("tiny_g4_peaked_edges")
    m = c["meta"]
    assert c["S"] + c["T"] == 192 and c["mask"].sum(1).tolist() == [1, 63, 64, 65, 127, 128]
    eng = make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], max_batch=c["input_ids"].shape[0], max_seq_len=c["S"] + c["T"])
    try:
        _check_peaked(eng, c, "tiny_g4_peaked_edges")
        with pytest.raises(Exception):      # one token more than the engine was sized for is refused, not truncated
            eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"] + 1, pad_token_id=m["pad_token_id"])
    finally:
        eng.close()


HEADLINE = ["llama3_8b_2l_b4", "llama3_8b_2l_peaked_b4", "llama3_8b_2l_peaked_ragged"]


@pytest.fixture(scope="module")
def headline_engines():
    """2-layer Llama-3-8B-dims engines for BASELINE.json's headline shapes (4 x 1024-token prompts, V = 128256)."""
    cache = {}

    def get(case):
        m = case["meta"]
        if m["cfg"] not in cache:
            for e in cache.values():      # one 3.5 GB model at a time
                e.close()
            cache.clear()
            cache[m["cfg"]] = make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], max_batch=4, max_seq_len=1152)
        return cache[m["cfg"]]
    yield get
    for e in cache.values():
        e.close()


@pytest.mark.slow
@pytest.mark.parametrize("name", HEADLINE)
def test_headline_shapes_1024_prompt_tokens(headline_engines, name):
    """VERDICT r01 weak #1: the headline configuration's shapes against the oracle — S = 1024 (16 KV tiles through
    attn_prefill_tc_kernel, 4096 packed rows through the 256-column prefill GEMMs), decode at context 1025..1040, a ragged
    U[512,1024] left-padded batch, V = 128256.  Teacher-forced: every step's logits on 4096 fixed columns + the oracle's
    top-16; peaked cases additionally require the free-running greedy ids to be the oracle's, token for token."""
    c = load_case(name)
    eng = headline_engines(c)
    pad = c["meta"]["pad_token_id"]
    peaked = "peaked" in name
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"], want_logits=True)
    assert torch.equal(r.output_ids, c["output_ids"])
    got = r.logits.float().permute(1, 0, 2)                  # [B, T, V]
    assert not torch.isnan(got).any()
    sub = got[..., c["sub_cols"]]
    topv = torch.gather(got, 2, c["topk_idx"].long())
    if peaked:
        floor = c["topk_vals"][..., 1]
        ok_sub = (sub - c["sub_logits"]).abs() <= logits_tol_elementwise(c["sub_logits"], floor)
        ok_top = (topv - c["topk_vals"]).abs() <= logits_tol_elementwise(c["topk_vals"], floor)
        tol_scalar = float(logits_tol(c["topk_vals"]))
    else:
        tol_scalar = float(logits_tol(c["topk_vals"]))      # max |logit| of the case is in the top-k
        ok_sub = (sub - c["sub_logits"]).abs() <= tol_scalar
        ok_top = (topv - c["topk_vals"]).abs() <= tol_scalar
    err_sub, err_top = float((sub - c["sub_logits"]).abs().max()), float((topv - c["topk_vals"]).abs().max())
    decisive = c["margin"] > 2 * tol_scalar
    agree = got.argmax(-1) == c["gen"]
    stats = dict(max_err_sub=err_sub, max_err_topk=err_top, tol=tol_scalar, max_logit=float(c["topk_vals"].abs().max()),
                 decisive=int(decisive.sum()), steps=int(decisive.numel()), agree_tf=int(agree.sum()))
    assert bool(ok_sub.all()) and bool(ok_top.all()), stats
    assert bool(agree[decisive].all()), stats
    free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
    exact = free.output_ids[:, c["S"]:] == c["gen"]
    stats["free_running_exact_match"] = float(exact.float().mean())
    _record(name + ":headline", **stats)
    if peaked:
        assert float(decisive.float().mean()) >= 0.95, stats
        if bool(decisive.all()):
            assert bool(exact.all()), stats
    else:
        for b in range(exact.shape[0]):
            neq = (~exact[b]).nonzero()
            if len(neq):
                assert not bool(decisive[b, int(neq[0])]), f"row {b} diverges at a decisive step"


def test_stop_sequence_batch_wide(engines):
    """stop_sequence_stopping_criteria.py:36-48: any row matching stops every row; finish_reason 'stop'."""
    c = load_case("tiny_g2_stop")
    eng = engines(c)
    stop = c["meta"]["stop"]
    max_new = c["meta"]["max_tokens"]
    forced = torch.cat([c["gen"], torch.zeros((c["gen"].shape[0], max_new - c["T"]), dtype=torch.int64)], 1)
    r = eng.generate(c["input_ids"], None, max_new_tokens=max_new, pad_token_id=c["meta"]["pad_token_id"],
                     stop_sequences=stop, forced_tokens=forced)
    assert r.stop_triggered and c["meta"]["finish_reason"] == "stop"
    assert r.num_generated == c["T"], (r.num_generated, c["T"])
    assert torch.equal(r.output_ids, c["output_ids"])
    # without the stop sequence the same request runs to max_new_tokens
    r = eng.generate(c["input_ids"], None, max_new_tokens=max_new, pad_token_id=c["meta"]["pad_token_id"], forced_tokens=forced)
    assert not r.stop_triggered and r.num_generated == max_new


def test_eos_rows_are_padded(engines):
    """transformers utils.py:2796-2797: after EOS a row emits pad_token_id; all rows EOS -> generation ends."""
    c = load_case("tiny_g2_ids")
    eng = engines(c)
    eos = int(c["gen"][1, 2])
    r = eng.generate(c["input_ids"], None, max_new_tokens=c["T"], pad_token_id=1030, eos_token_ids=[eos],
                     forced_tokens=c["gen"])
    row = r.output_ids[1, c["S"]:]
    assert int(row[2]) == eos and bool((row[3:] == 1030).all())
    allsame = c["gen"].clone()
    allsame[:, 3] = eos
    r = eng.generate(c["input_ids"], None, max_new_tokens=c["T"], pad_token_id=1030, eos_token_ids=[eos], forced_tokens=allsame)
    assert r.num_generated <= 4 + 0 and not r.stop_triggered


def test_streamer_callback(engines):
    c = load_case("tiny_g2_ids")
    eng = engines(c)
    seen = []
    r = eng.generate(c["input_ids"], None, max_new_tokens=6, pad_token_id=1030, forced_tokens=c["gen"][:, :6],
                     streamer=lambda step, toks: seen.append((step, list(toks))) and False)
    assert [s for s, _ in seen] == list(range(6))
    assert torch.tensor([t for _, t in seen]).T.tolist() == c["gen"][:, :6].tolist()


@pytest.mark.slow
def test_llama3_8b_shapes_two_layers():
    """Full-size Llama-3-8B layer / vocabulary shapes (2 layers): every production GEMM shape, 128256-row LM head."""
    c = load_case("llama3_8b_2l_ids")
    m = c["meta"]
    eng = make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], max_batch=4, max_seq_len=256)
    try:
        r = eng.generate(c["input_ids"], None, max_new_tokens=c["T"], pad_token_id=m["pad_token_id"],
                         forced_tokens=c["gen"], want_logits=True)
        got = r.logits.float().permute(1, 0, 2)      # [B, T, V]
        ref0 = c["step0_logits"]                      # fp16-stored bf16 logits of step 0
        tol = logits_tol(ref0)
        err0 = (got[:, 0] - ref0).abs()
        # top-k values of every step
        idx = c["topk_idx"].long()
        gv = torch.gather(got, 2, idx)
        errk = (gv - c["topk_vals"]).abs()
        _record("llama3_8b_2l:teacher_forced", max_err_step0=float(err0.max()), max_err_topk=float(errk.max()), tol=tol,
                max_logit=float(ref0.abs().max()))
        assert float(err0.max()) <= tol and float(errk.max()) <= tol
        pred = got.argmax(-1)
        decisive = c["margin"] > 2 * tol
        assert bool((pred == c["gen"])[decisive].all())
        _record("llama3_8b_2l:greedy_tf", steps=int(pred.numel()), agree=int((pred == c["gen"]).sum()), decisive=int(decisive.sum()))
    finally:
        eng.close()


def test_kv_host_offload_tier_roundtrip(engines):
    """BASELINE configs[3] 'host-DRAM KV-offload tier': swap every sequence's KV pages out to pinned host memory
    (scrubbing the device copy), swap them back in, and decoding continues bit-identically."""
    c = load_case("tiny_g4_ids")
    eng = engines(c)
    T = 24
    eng.stage(c["input_ids"], None, max_new_tokens=T, pad_token_id=0)
    eng.run_staged(True, T - 1)
    ref = eng.fetch_staged().clone()
    eng.stage(c["input_ids"], None, max_new_tokens=T, pad_token_id=0)
    eng.run_staged(True, 9)
    for b in range(c["input_ids"].shape[0]):
        eng.kv_swap_out(b, scrub=True)
    for b in range(c["input_ids"].shape[0]):
        eng.kv_swap_in(b)
    eng.run_staged(False, T - 1 - 9)
    assert torch.equal(eng.fetch_staged(), ref)


@pytest.mark.parametrize("name,use_mask", [("tiny_g2_ids", False), ("tiny_g2_text", True)])   # plain / left-padded rows
def test_staged_prompt_replays_like_generate(engines, name, use_mask):
    """b200_run_staged(do_prefill=1) replays the staged prompt from what staging left on the device, as bench.py times
    it: every replay gives generate's ids.  Continuous batching overwrites the packed prompt and the page table, so a
    replay after a continuous-batching session is refused."""
    from kserve_b200._lib import B200Error
    c = load_case(name)
    eng = engines(c)
    pad, T = c["meta"]["pad_token_id"], c["T"]
    mask = c["mask"] if use_mask else None
    ref = eng.generate(c["input_ids"], mask, max_new_tokens=T, pad_token_id=pad).output_ids
    eng.stage(c["input_ids"], mask, max_new_tokens=T, pad_token_id=pad)
    for _ in range(3):
        eng.run_staged(True, T - 1)
        assert torch.equal(eng.fetch_staged(), ref)
    eng.cb_begin(pad)
    eng.cb_end()
    with pytest.raises(B200Error, match="no staged prompt"):
        eng.run_staged(True, T - 1)


def test_long_context_3968_prompt_tokens():
    """A 3968-token prompt (31 query tiles of 128) plus 64 generated tokens on tiny_g2_rope3, whose max_position of 4096
    bounds both: every step's logits against the oracle's forward (on the CPU) over the engine's own ids, at the stated
    tolerance; then the same greedy ids through the continuous batcher with 1024-token prefill chunks and the prefix
    cache, alongside a second prompt that shares the first 2048 tokens (chunks start at kv_off 1024 ... 3072)."""
    from oracle import weights as W
    from oracle.hf_oracle import OracleGenerativeModel, build_model
    S, T, pad = 3968, 64, 1030
    g = torch.Generator().manual_seed(3968)
    ids = torch.randint(3, 1000, (1, S), generator=g)
    other = ids.clone()
    other[0, 2048:] = torch.randint(3, 1000, (S - 2048,), generator=g)
    eng = make_engine("tiny_g2_rope3", 0, max_batch=2, max_seq_len=S + T)
    try:
        r = eng.generate(ids, None, max_new_tokens=T, pad_token_id=pad, want_logits=True)
        assert r.num_generated == T
        ref_other = eng.generate(other, None, max_new_tokens=T, pad_token_id=pad).output_ids[0, S:].tolist()
        cfg = W.CONFIGS["tiny_g2_rope3"]
        orc = OracleGenerativeModel(build_model(cfg, W.synth_state_dict(cfg, 0)), pad_token_id=pad)
        ref = orc.forward_logits(r.output_ids[:, :-1])[:, S - 1:]          # [1, T, V]: step t sees prompt + t engine ids
        got = r.logits.float().permute(1, 0, 2)
        tol = logits_tol(ref)
        err = float((got - ref).abs().max())
        _record("long_context_3968:teacher_forced", max_err=err, tol=tol)
        assert err <= tol, f"max logits error {err:.4f} > tol {tol:.4f}"

        eng.cb_begin(pad, [])
        eng.cb_config(1024, True)
        try:
            a = eng.cb_admit([ids[0].tolist()], [T])[0]
            for _ in range(T + 8):
                if eng.cb_poll()[1][a]:
                    break
                eng.cb_step(1)
            assert eng.cb_read(a, 0, T) == r.output_ids[0, S:].tolist()
            eng.cb_release(a)
            b = eng.cb_admit([other[0].tolist()], [T])[0]
            assert eng.cb_stats()["prefix_hit_tokens"] == 2048
            for _ in range(T + 8):
                if eng.cb_poll()[1][b]:
                    break
                eng.cb_step(1)
            assert eng.cb_read(b, 0, T) == ref_other
            eng.cb_release(b)
        finally:
            eng.cb_end()
    finally:
        eng.close()
