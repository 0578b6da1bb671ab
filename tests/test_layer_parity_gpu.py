"""The engine's final hidden state per element against a float64 transformers decoder, at served layer shapes and decode
batches of 1 to 64 (criterion, weights, twin and controls: tests/layer_parity.py).

Each case is a 2-layer engine with vocab_size = H and lm_head = eye(H), so the teacher-forced bf16 logits are the
final-normed hidden state.  A pool of 64 prompts (1, 63, 64, 65, 127, 128, 129 tokens, then seeded 2..300) with 6 forced
decode steps runs through generate() left-padded on its first B rows, B in BATCHES (decode GEMM column blocks of 16, 32
and 64 with their tails), and 2 rows of ~4000 tokens run on their own (8-way split decode attention over 63 pages).
Step 0 is the prefill's last row of each sequence, steps 1..6 the decode passes; with 2 layers every prefill row of
layer 0 reaches the output through layer 1's K / V.  The references are computed once per shape, on the GPU, one
unpadded causal pass per row, and every batch size reuses them.

Decode plans these shapes reach on a 132-SM H100 (engine.cu: pick_splits, the gate/up stream-K rule, the attention
split count; launch_rmsnorm's kernel choice):

  tiny_g2 / tiny_g4   G = 2 / 4, the tiny fixtures' shapes
  llama3_8b           G = 4, gate/up stream-K at 224 tiles
  llama32_3b          G = 3; gate/up 128 tiles (plain SwiGLU, just under the stream-K rule); down split 5
  qwen25_0p5b         G = 7; o / down split-K 14 / 16 (sum_partials8 past 4 splits); norm H = 896 on >= 256 prefill rows
                      (rmsnorm_kernel, not the rows kernel)
  qwen25_1p5b         G = 6; gate/up stream-K at 140 tiles (8 past one wave)
  qwen25_7b           G = 7, q dim 3584 = H
  qwen25_14b (slow)   G = 5; rmsnorm_kernel with H > 4096 (strided weight path) in decode and prefill
  qwen3_0p6b          q dim 2048 != H (o_proj K = 2048); gate/up split-K 2 + swiglu_reduce_kernel
  qwen3_4b / 8b       G = 4, q dim 4096 != H (4b)
  qwen3_32b (slow)    q / k norm with the bf16 EPI_T_STORE decode QKV (80 tiles); gate/up stream-K at 400 tiles

The twin and the negative controls run again at one shape per family (CONTROL_SHAPES) on the first 16 rows, the
engine standing where the CPU test has the twin.  Results are printed (pytest -s) as one line per case.

Measured on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit): the engine's worst ratios over every batch size and
the long rows (row / block / element / mean; limits 2 / 2 / 1 / 1.3)

  tiny_g2      1.41 / 1.57 / 0.54 / 0.93      qwen25_0p5b  1.25 / 1.39 / 0.48 / 1.01      qwen3_0p6b  1.18 / 1.36 / 0.42 / 0.97
  tiny_g4      1.33 / 1.48 / 0.45 / 0.96      qwen25_1p5b  1.15 / 1.42 / 0.52 / 0.97      qwen3_4b    1.07 / 1.25 / 0.52 / 0.94
  llama3_8b    1.08 / 1.25 / 0.49 / 0.94      qwen25_7b    1.06 / 1.28 / 0.48 / 0.97      qwen3_8b    1.09 / 1.25 / 0.45 / 1.00
  llama32_3b   1.06 / 1.30 / 0.49 / 0.98      qwen25_14b   1.03 / 1.27 / 0.54 / 0.93      qwen3_32b   1.07 / 1.28 / 0.44 / 0.97

and at the control shapes (row / block / element):

  tiny_g4     twin 1.24 / 1.39 / 0.41; controls (row): v head 5.5, o head 2.6, final norm 2.8 (block 6.3), rope 25.2
  tiny_qwen2  twin 1.15 / 1.26 / 0.40; controls: v head 5.4, o head 2.6, final norm 4.1 (block 7.5), rope 22.6, q bias 19.4
  tiny_qwen3  twin 1.28 / 1.35 / 0.41; controls: v head 4.3, o head 2.4, final norm 3.9 (block 6.7), rope 17.3, k_norm 4.7"""

import pytest
import torch

import layer_parity as LP

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
T = 6                                   # forced decode steps (max_new_tokens = T + 1: step 0 is the prefill's)
POOL = 64
BATCHES = [1, 5, 16, 17, 32, 33, 64]
LONG = (4001, 3968)                      # tokens of the two long rows
SEED = 2

SHAPES = ["tiny_g2", "tiny_g4", "llama3_8b", "llama32_3b",
          "qwen25_0p5b", "qwen25_1p5b", "qwen25_7b", pytest.param("qwen25_14b", marks=pytest.mark.slow),
          "qwen3_0p6b", "qwen3_4b", "qwen3_8b", pytest.param("qwen3_32b", marks=pytest.mark.slow)]
# 8 q heads each: the o_proj control (2^-4 on one of layer 1's nh heads) moves the output by ~1/sqrt(nh) of that
# layer's attention update, which at nh >= 14 is under twice the bf16 yardstick's own error (on an H100: ratio 1.78 at
# qwen25_0p5b, 1.69 at qwen3_0p6b), so the controls run where the criterion can resolve one head
CONTROL_SHAPES = ["tiny_g4", "tiny_qwen2", "tiny_qwen3"]
CONTROL_ROWS = 16


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


def references(cfg, sd, seqs, edit=None, shift_last=False):
    """(ref64, hf16): per row [T + 1, H] float64 on the CPU; each model is freed before the next is built"""
    out = []
    for dtype in (torch.float64, torch.bfloat16):
        model = LP.build_hf(cfg, edit(sd) if edit else sd, dtype, DEV)
        out.append(torch.stack(LP.run_rows(model, seqs, T, shift_last)))
        del model
        _free()
    return out


def make_engine(cfg, sd, rows):
    """sized for `rows` (token lists): explicit max_prefill_tokens and KV pages (the 64 x max_seq_len default would not
    fit an I = 25600 hbuf)"""
    from kserve_b200.engine import B200Engine
    longest = max(len(r) for r in rows) + T + 1
    max_seq = -(-longest // 64) * 64
    eng = B200Engine(cfg, max_batch=POOL, max_seq_len=max_seq, max_prefill_tokens=sum(len(r) for r in rows),
                     num_kv_pages=POOL * (max_seq // 64))
    eng.load_weights(sd.items())
    return eng


def engine_hidden(eng, prompts, forced):
    """generate() on the rows left-padded: [B, T + 1, H] float64 on the CPU"""
    B, S = len(prompts), max(len(p) for p in prompts)
    ids = torch.zeros((B, S), dtype=torch.int64)
    mask = torch.zeros((B, S), dtype=torch.int64)
    for b, p in enumerate(prompts):
        ids[b, S - len(p):] = torch.tensor(p)
        mask[b, S - len(p):] = 1
    r = eng.generate(ids, mask, max_new_tokens=T + 1, pad_token_id=0, forced_tokens=forced[:B], want_logits=True)
    assert r.num_generated == T + 1 and r.logits.shape == (T + 1, B, eng.vocab)
    return r.logits.permute(1, 0, 2).double()


def _where(eng, hf, ref):
    """(row, step) pairs that fail the criterion on their own"""
    bad = []
    for b in range(ref.shape[0]):
        for t in range(ref.shape[1]):
            if not LP.judge(eng[b, t], hf[b, t], ref[b, t])["ok"]:
                bad.append((b, t))
    return bad[:8]


def _case(shape):
    cfg = LP.config(shape)
    H = cfg["hidden_size"]
    sd = LP.draw_weights(cfg, SEED, DEV)
    prompts = LP.prompt_pool(POOL, H, SEED)
    long = LP.prompt_pool(len(LONG), H, SEED + 1, fixed=LONG)
    forced = LP.forced_tokens(POOL + len(LONG), T, H, SEED)
    return cfg, sd, prompts, long, forced


@pytest.mark.parametrize("shape", SHAPES)
def test_engine_final_hidden_state(precision, shape):
    cfg, sd, prompts, long, forced = _case(shape)
    rows = prompts + long
    ref, hf = references(cfg, sd, LP.sequences(rows, forced, T))
    eng = make_engine(cfg, sd, rows)
    try:
        runs = [(f"B={B}", engine_hidden(eng, prompts[:B], forced[:B]), slice(0, B)) for B in BATCHES]
        runs.append((f"long {LONG}", engine_hidden(eng, long, forced[POOL:]), slice(POOL, POOL + len(LONG))))
    finally:
        eng.close()
        _free()
    failures = []
    for name, got, sl in runs:
        r = LP.judge(got, hf[sl], ref[sl])
        print(f"{shape} {name}: {LP.fmt(r)}")
        if not r["ok"]:
            failures.append(f"{name}: {LP.fmt(r)}; failing (row, step): {_where(got, hf[sl], ref[sl])}")
    assert not failures, f"{shape}: " + " | ".join(failures)


@pytest.mark.parametrize("shape", CONTROL_SHAPES)
def test_twin_and_negative_controls(precision, shape):
    """the permuted twin passes against the yardstick; every control (both references perturbed, the engine not)
    fails; the old logits check's verdict on each control is printed beside it"""
    cfg, sd, prompts, _, forced = _case(shape)
    prompts, forced = prompts[:CONTROL_ROWS], forced[:CONTROL_ROWS]
    seqs = LP.sequences(prompts, forced, T)
    ref, hf = references(cfg, sd, seqs)
    p, q = LP.permutations(cfg, SEED, DEV)
    model = LP.build_hf(cfg, LP.permute(sd, p, q), torch.bfloat16, DEV)
    twin = torch.stack(LP.run_rows(model, seqs, T))[..., torch.argsort(p).cpu()]
    del model
    _free()
    r = LP.judge(twin, hf, ref)
    print(f"{shape} twin: {LP.fmt(r)}")
    assert r["ok"], f"twin: {LP.fmt(r)}"
    eng = make_engine(cfg, sd, prompts)
    try:
        got = engine_hidden(eng, prompts, forced)
    finally:
        eng.close()
        _free()
    r = LP.judge(got, hf, ref)
    print(f"{shape} engine (B={CONTROL_ROWS}): {LP.fmt(r)}")
    assert r["ok"], f"engine: {LP.fmt(r)}"
    missed = []
    for name, ctl in LP.controls(cfg).items():
        ref_c, hf_c = references(cfg, sd, seqs, ctl["edit"], ctl.get("shift_last", False))
        r = LP.judge(got, hf_c, ref_c)
        caught = LP.logits_check_catches(got, hf_c, 1031, SEED)
        print(f"{shape} control {name}: {LP.fmt(r)}; old logits check catches it: {caught}")
        if r["ok"]:
            missed.append(name)
    assert not missed, f"controls the criterion did not detect: {missed}"
