"""The continuous batcher's final hidden state per element against a float64 decoder, at served layer shapes, through
joins and leaves, a rotating decode window, chunked prefill, prefix reuse and host swap (criterion, weights and
references: tests/layer_parity.py; schedules: tests/cb_parity.py).

Each engine has 2 layers, vocab_size = H and lm_head = eye(H), so its bf16 logits are its final-normed hidden state.
b200_cb_logits_tap copies the logits of every batcher LM-head pass — the head of a prefill pass that ends prompts, and
each decode step's — to a [slot][step][H] buffer, and each sequence's rows [0, n_gen) are judged against the float64
model and the bf16 yardstick on its prompt plus the tokens it generated (greedy: the batcher takes no forced tokens).
The driver follows a plan made by a model of the engine's bookkeeping and compares every slot's polled n_gen with it
after every step.

  A  join and leave      no chunking, no prefix cache, 96 slots: the resident count is driven through 1, 5, 16, 17,
                         32, 33, 64, 64, 80, 90, 90, admitting the difference each step (1..300-token prompts, the
                         boundary lengths first, max_new 3..10) and releasing each sequence the step after it finishes;
                         later admits land in released slots, and above 64 resident the 64-row window rotates
  B  chunked + prefix    chunks of 512 and of 1024 tokens with the prefix cache: 8 short rows decode while two
                         prompts of 4001 / 3968 tokens and a 1000-token prompt P are prefilled in chunks; then one admit
                         of P[:256]+37, P[:896]+1, P, P[:640] (every block cached, the last recomputed) and a prompt
                         that leaves P inside block 1; prefix_hit_tokens, prefill_passes and prefilled_tokens must equal
                         the plan's
  C  host swap           inside B: P[:896]+1 (leading pages shared with the cache), P and the broken-chain row are
                         swapped out to host memory for two steps and back in
  D  FP8 weights         scenario A on an FP8 engine and on a bf16 engine loaded with W' = bf16(code) * bf16(scale):
                         same ids, same schedule, bit-identical tapped logits

Shapes (decode plans as in test_layer_parity_gpu.py): tiny_g4; qwen25_0p5b (o / down split-K 14 / 16, biases);
qwen3_0p6b (gate/up split-K 2 + swiglu_reduce_kernel, q/k norm); llama3_8b (gate/up stream-K); qwen25_7b (G = 7,
biases); qwen3_8b (q/k norm); qwen25_14b and qwen3_32b are slow.  Rows stay at or under ~4000 tokens: the eager float64
reference holds an L x L score matrix per head.

Negative controls (both references edited, the engine not), at the 8-head control shapes on scenario B with 512-token
chunks: `wrong_prefix_block` gives the P[:896]+1 row block 2 of the first long prompt instead of P's, as a page-table
row pointing at another prompt's pages would; `chunk_offset` runs the tokens of P's second chunk one position later.
Each must fail the criterion on its row.

Measured on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit), worst ratios (row / block / element / mean; limits
2 / 2 / 1 / 1.3) of scenario A and of B + C over both chunk sizes:

  shape          A (135 sequences, 20 steps)     B + C (16 sequences, 30 / 20 steps)
  tiny_g4        1.26 / 1.55 / 0.51 / 0.83       1.11 / 1.37 / 0.42 / 0.82
  qwen25_0p5b    1.20 / 1.34 / 0.49 / 0.86       1.08 / 1.26 / 0.42 / 0.88
  qwen3_0p6b     1.19 / 1.36 / 0.44 / 0.83       1.11 / 1.25 / 0.47 / 0.83
  llama3_8b      1.07 / 1.30 / 0.49 / 0.82       1.04 / 1.27 / 0.53 / 0.83
  qwen25_7b      1.03 / 1.30 / 0.51 / 0.86       1.10 / 1.26 / 0.50 / 0.87
  qwen3_8b       1.12 / 1.36 / 0.50 / 0.82       1.05 / 1.22 / 0.43 / 0.81
  qwen25_14b     1.03 / 1.27 / 0.50 / 0.86       1.03 / 1.28 / 0.52 / 0.87
  qwen3_32b      1.05 / 1.25 / 0.48 / 0.81       1.01 / 1.20 / 0.47 / 0.81

The controls (row ratio; every one fails): tiny_g4 wrong_prefix_block 32.2, chunk_offset 19.7; tiny_qwen2 25.0, 10.8;
tiny_qwen3 27.4, 17.7.  Scenario D: 135 of 135 sequences bit-identical at tiny_g4 and qwen25_0p5b.  Wall time: 1 min
38 s for the non-slow tests, 1 min 7 s for the two slow shapes (engine weight loads and references included)."""

import pytest
import torch

import cb_parity as CB
import layer_parity as LP

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
SEED = 2
POOL = 200
SHAPES = ["tiny_g4", "qwen25_0p5b", "qwen3_0p6b", "llama3_8b", "qwen25_7b", "qwen3_8b",
          pytest.param("qwen25_14b", marks=pytest.mark.slow), pytest.param("qwen3_32b", marks=pytest.mark.slow)]
CONTROL_SHAPES = ["tiny_g4", "tiny_qwen2", "tiny_qwen3"]
FP8_SHAPES = ["tiny_g4", "qwen25_0p5b"]
KV_PAGES = 768
MAX_SEQ = 4096


@pytest.fixture
def precision():
    """cuBLAS bf16 GEMMs of the yardstick with fp32 reductions throughout (restored afterwards)"""
    old = torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
    yield
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = old


def _free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


class References:
    """the float64 reference and the bf16 yardstick of one state dict (optionally edited), cached by token sequence
    and position ids: (ref64, hf16) [n, H] float64 on the CPU"""
    KEEP = 16

    def __init__(self, cfg, sd, edit=None):
        sd = edit(sd) if edit else sd
        self.models = [LP.build_hf(cfg, sd, dt, DEV) for dt in (torch.float64, torch.bfloat16)]
        self.cache = {}

    def get(self, seq, n, pos=None):
        assert n <= self.KEEP
        key = (tuple(seq), None if pos is None else tuple(pos))
        if key not in self.cache:
            k = min(self.KEEP, len(seq))
            self.cache[key] = [CB.hidden_at(m, seq, k, pos) for m in self.models]
        return [h[-n:] for h in self.cache[key]]

    def close(self):
        del self.models
        _free()


def make_engine(cfg, sd, **kw):
    from kserve_b200.engine import B200Engine
    eng = B200Engine(cfg, max_batch=CB.A_MAX_BATCH, max_seq_len=MAX_SEQ, max_prefill_tokens=CB.MAX_PREFILL_TOKENS,
                     num_kv_pages=KV_PAGES, **kw)
    eng.load_weights(sd.items() if isinstance(sd, dict) else sd)
    return eng


def drive(eng, plan):
    """runs the plan through b200_cb_*: {row: (generated ids, tapped logits bf16 [n_gen, V] on the CPU)}, cb_stats"""
    rows = plan.rows
    tap = eng.cb_logits_tap(max(r.max_new for r in rows))
    out = {}
    eng.cb_begin(0, [])
    try:
        eng.cb_config(plan.chunk, plan.prefix)
        for k, s in enumerate(plan.steps):
            for i in s.release:
                slot = rows[i].slot
                gen = eng.cb_read(slot, 0, rows[i].max_new)
                assert len(gen) == rows[i].max_new, f"row {i}: {len(gen)} tokens, max_new {rows[i].max_new}"
                out[i] = (gen, tap[slot, :len(gen)].cpu())
                eng.cb_release(slot)
            for i in s.swap_out:
                eng.cb_swap_out(rows[i].slot)
            for i in s.swap_in:
                eng.cb_swap_in(rows[i].slot)
            if s.admit:
                slots = eng.cb_admit([rows[i].prompt for i in s.admit], [rows[i].max_new for i in s.admit])
                assert slots == [rows[i].slot for i in s.admit], f"step {k}: slots {slots}"
            if not s.run:
                break
            eng.cb_step(1)
            n_gen, _, _ = eng.cb_poll()
            got = {i: n_gen[rows[i].slot] for i in s.n_gen}
            bad = {i: (got[i], n) for i, n in s.n_gen.items() if got[i] != n}
            assert not bad, f"step {k} ({s.resident} resident): row -> (n_gen, planned) {dict(list(bad.items())[:8])}"
        stats = eng.cb_stats()
    finally:
        eng.cb_end()
        eng.cb_logits_tap(0)
    assert sorted(out) == list(range(len(rows)))
    return out, stats


def judge(refs, plan, out, rids=None, seqs=None, pos=None):
    """the criterion over the tapped rows of `rids` (default all); seqs / pos: per row, the reference's token sequence
    and position ids instead of the row's own"""
    eng, hf, ref = [], [], []
    for i in (range(len(plan.rows)) if rids is None else rids):
        gen, tapped = out[i]
        seq = (seqs or {}).get(i) or CB.reference_sequence(plan.rows[i], gen)
        r64, r16 = refs.get(seq, len(gen), (pos or {}).get(i))
        eng.append(tapped.double())
        hf.append(r16)
        ref.append(r64)
    return LP.judge(torch.cat(eng), torch.cat(hf), torch.cat(ref))


def _inputs(cfg):
    H = cfg["hidden_size"]
    pool = LP.prompt_pool(POOL, H, SEED)
    shorts = LP.prompt_pool(8, H, SEED + 2)
    longs = LP.prompt_pool(2, H, SEED + 1, fixed=CB.LONG)
    P = LP.prompt_pool(1, H, SEED + 3, fixed=(CB.P_LEN,))[0]
    return pool, (shorts, longs, P, H, SEED)


def _chunked_run(eng, chunked_args, chunk):
    plan = CB.plan_chunked(*chunked_args, chunk)
    out, stats = drive(eng, plan)
    want = dict(prefix_hit_tokens=plan.hit_tokens, prefill_passes=plan.passes, prefilled_tokens=plan.prefilled,
                swap_outs=len(plan.swapped), swap_ins=len(plan.swapped))
    got = {k: stats[k] for k in want}
    assert got == want, f"chunk {chunk}: cb_stats {got}, plan {want}"
    return plan, out


@pytest.mark.parametrize("shape", SHAPES)
def test_batcher_final_hidden_state(precision, shape):
    cfg = LP.config(shape)
    sd = LP.draw_weights(cfg, SEED, DEV)
    pool, chunked_args = _inputs(cfg)
    eng = make_engine(cfg, sd)
    try:
        plan_a = CB.plan_join_leave(pool, SEED)
        runs = [("A join/leave", plan_a, drive(eng, plan_a)[0])]
        for chunk in (512, 1024):
            plan, out = _chunked_run(eng, chunked_args, chunk)
            runs.append((f"B+C chunk {chunk}", plan, out))
    finally:
        eng.close()
        _free()
    refs = References(cfg, sd)
    failures = []
    try:
        for name, plan, out in runs:
            r = judge(refs, plan, out)
            print(f"{shape} {name} ({len(plan.rows)} sequences, {len(plan.steps)} steps): {LP.fmt(r)}")
            if not r["ok"]:
                bad = [i for i in range(len(plan.rows)) if not judge(refs, plan, out, [i])["ok"]]
                failures.append(f"{name}: {LP.fmt(r)}; failing rows {bad[:8]} "
                                f"(lens {[len(plan.rows[i].prompt) for i in bad[:8]]})")
    finally:
        refs.close()
    assert not failures, f"{shape}: " + " | ".join(failures)


@pytest.mark.parametrize("shape", CONTROL_SHAPES)
def test_batcher_negative_controls(precision, shape):
    """scenario B (512-token chunks) passes on the engine; each batcher control, given to both references, fails"""
    cfg = LP.config(shape)
    sd = LP.draw_weights(cfg, SEED, DEV)
    _, chunked_args = _inputs(cfg)
    eng = make_engine(cfg, sd)
    try:
        plan, out = _chunked_run(eng, chunked_args, 512)
    finally:
        eng.close()
        _free()
    refs = References(cfg, sd)
    try:
        r = judge(refs, plan, out)
        print(f"{shape} engine: {LP.fmt(r)}")
        assert r["ok"], f"engine: {LP.fmt(r)}"
        i = plan.family[1]                                        # P[:896] + 1: blocks 0..6 from the cache
        seq = CB.reference_sequence(plan.rows[i], out[i][0])
        longp = plan.rows[8].prompt
        seq = seq[:2 * CB.BLOCK] + longp[2 * CB.BLOCK:3 * CB.BLOCK] + seq[3 * CB.BLOCK:]
        ctl = {"wrong_prefix_block": judge(refs, plan, out, [i], seqs={i: seq})}
        p = plan.p_row
        start, count = plan.rows[p].chunks[1]
        seq = CB.reference_sequence(plan.rows[p], out[p][0])
        pos = list(range(len(seq)))
        pos[start:start + count] = [q + 1 for q in pos[start:start + count]]
        ctl["chunk_offset"] = judge(refs, plan, out, [p], pos={p: pos})
    finally:
        refs.close()
    for name, r in ctl.items():
        print(f"{shape} control {name}: {LP.fmt(r)}")
    missed = [n for n, r in ctl.items() if r["ok"]]
    assert not missed, f"controls the criterion did not detect: {missed}"


def _fp8_pair(cfg, sd):
    from kserve_b200.fp8 import PROJECTIONS, dequantize_reference
    from test_fp8_gpu import quantize
    q, wp = [], []
    for name, t in sd.items():
        if any(name.endswith(p + ".weight") for p in PROJECTIONS):
            codes, scale = quantize(t)
            q += [(name, codes), (name + "_scale", scale)]
            wp.append((name, dequantize_reference(codes, scale)))
        else:
            q.append((name, t))
            wp.append((name, t))
    return make_engine(cfg, q, weight_format=1), make_engine(cfg, wp)


@pytest.mark.parametrize("shape", FP8_SHAPES)
def test_fp8_batcher_bit_identical_to_bf16_on_w_prime(shape):
    cfg = LP.config(shape)
    sd = LP.draw_weights(cfg, SEED, DEV)
    pool, _ = _inputs(cfg)
    plan = CB.plan_join_leave(pool, SEED)
    e8, e16 = _fp8_pair(cfg, sd)
    try:
        got8, _ = drive(e8, plan)
        got16, _ = drive(e16, plan)
    finally:
        e8.close()
        e16.close()
        _free()
    diff = []
    for i in range(len(plan.rows)):
        (g8, t8), (g16, t16) = got8[i], got16[i]
        assert torch.isfinite(t8.float()).all(), f"row {i}: a tapped step was not written"
        if g8 != g16 or not torch.equal(t8.view(torch.int16), t16.view(torch.int16)):
            diff.append(i)
    print(f"{shape} fp8 vs W': {len(plan.rows)} sequences, {len(diff)} differ")
    assert not diff, f"rows whose ids or tapped logits differ: {diff[:8]}"
