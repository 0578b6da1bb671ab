"""Qwen2 / Qwen2.5 decoders on the GPU: the q / k / v projection biases through every place the engine forms the QKV
projection, against the oracle fixtures (tools/synth_weights.py draws the biases large, with k outliers, so a dropped,
doubled or post-RoPE bias fails these comparisons; tests/test_qwen2_cpu.py checks that it would).

  prefill  : EPI_ROPE_KV (bias before RoPE), or EPI_STORE + rope_kv_kernel under B200_NO_ROPE_FUSION=1
  decode   : split-K partials + the attention prologue (tiny_qwen2, G = 7; qwen2_7b_2l), or the bf16 EPI_T_STORE
             epilogue (tiny_qwen2_wide, 80 m-tiles); GQA groups 5, 6 and 7 through the decode attention
Same protocol as tests/test_engine_gpu.py."""
import json
import os
import subprocess
import sys

import pytest
import torch

from helpers import load_case, logits_tol, logits_tol_elementwise

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def make_engine(cfg_name, seed, vocab_rows=None, **kw):
    """helpers.make_engine plus tied embeddings: a tied checkpoint's head is its embedding matrix"""
    from oracle import weights as W
    from kserve_b200.engine import B200Engine
    cfg = W.CONFIGS[cfg_name]
    eng = B200Engine(cfg, vocab_rows=vocab_rows, **kw)

    def gen():
        embed = None
        for name, t in W.iter_state_dict(cfg, seed):
            if name == "model.embed_tokens.weight":
                embed = t
            yield name, t
        if cfg.get("tie_word_embeddings"):
            yield "lm_head.weight", embed
    eng.load_weights(gen())
    return eng


CASES = ["tiny_qwen2_ids",          # G = 7, decode QKV by split-K partials (bias in the attention prologue)
         "tiny_qwen2_wide_ids",     # 80 m-tiles: decode QKV by the bf16 EPI_T_STORE epilogue
         "tiny_qwen2_g6_tied_ids",  # G = 6, tied embeddings
         "tiny_qwen2_g5_ids"]       # G = 5


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(case):
        m = case["meta"]
        key = (m["cfg"], m["seed"])
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
    assert r.num_generated == c["T"] and torch.equal(r.output_ids, c["output_ids"])
    got = r.logits.float().permute(1, 0, 2)
    ref = c["step_logits"]
    tol = logits_tol(ref)
    assert not torch.isnan(got).any()
    err = float((got - ref).abs().max())
    assert err <= tol, f"max logits error {err:.4f} > tol {tol:.4f}"
    decisive = c["margin"] > 2 * tol
    assert bool((got.argmax(-1) == c["gen"])[decisive].all())


@pytest.mark.parametrize("name", CASES)
def test_free_running_ids(engines, name):
    c = load_case(name)
    eng = engines(c)
    pad = c["meta"]["pad_token_id"]
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
    assert r.num_generated == c["T"]
    tol = logits_tol(c["step_logits"])
    gen = r.output_ids[:, c["S"]:]
    for b in range(gen.shape[0]):
        neq = (gen[b] != c["gen"][b]).nonzero()
        if len(neq):
            t = int(neq[0])
            assert float(c["margin"][b, t]) <= 2 * tol, f"row {b} diverges at decisive step {t}"
    r2 = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
    assert torch.equal(r.output_ids, r2.output_ids)


def _check_peaked(eng, c):
    pad = c["meta"]["pad_token_id"]
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"], want_logits=True)
    got = r.logits.float().permute(1, 0, 2)
    ref = c["step_logits"]
    err = (got - ref).abs()
    tol = logits_tol_elementwise(ref)
    assert bool((err <= tol).all()), f"worst element: err/tol = {float((err / tol).max()):.2f}"
    decisive = c["margin"] > 2 * logits_tol(ref)
    assert bool(decisive.all())
    free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
    assert torch.equal(free.output_ids[:, c["S"]:], c["gen"])


def test_peaked_greedy_ids_exact(engines):
    c = load_case("tiny_qwen2_peaked")
    _check_peaked(engines(c), c)


def test_peaked_without_rope_fusion():
    """B200_NO_ROPE_FUSION=1: the prefill QKV projection stores bf16(acc + bias) (EPI_STORE) and rope_kv_kernel rotates it;
    the switch is read once per process, hence the subprocess"""
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from helpers import load_case\n"
            "import test_qwen2_gpu as t\n"
            "c = load_case('tiny_qwen2_peaked'); m = c['meta']\n"
            "e = t.make_engine(m['cfg'], m['seed'], vocab_rows=m['vocab_rows'], max_batch=8, max_seq_len=512)\n"
            "t._check_peaked(e, c); e.close(); print('NO_FUSION_OK')\n") % (ROOT, HERE)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, B200_NO_ROPE_FUSION="1"))
    assert res.returncode == 0 and "NO_FUSION_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


def _run_until_done(e, slots, max_iters=400):
    for _ in range(max_iters):
        n_gen, fin, stop = e.cb_poll()
        if all(fin[s] for s in slots):
            return n_gen
        e.cb_step(1)
    raise AssertionError("sequences did not finish")


def test_continuous_batching_chunked_prefill_and_prefix_reuse(engines):
    """b200_cb_*: two rows start, two join the running batch; 300-token prompts go through 128-token chunks with the prefix
    cache on (row 2 shares row 0's first two blocks).  Every step of the fixture is decisive: ids equal the oracle's."""
    c = load_case("tiny_qwen2_peaked")
    e = engines(c)
    T = c["T"]
    rows = [r.tolist() for r in c["input_ids"]]
    e.cb_begin(c["meta"]["pad_token_id"], [])
    e.cb_config(128, True)
    try:
        slots = e.cb_admit(rows[:2], [T, T])
        e.cb_step(8)                                      # both prompts prefilled (3 chunks each), their blocks cached
        slots += e.cb_admit(rows[2:], [T, T])
        n_gen = _run_until_done(e, slots)
        assert e.cb_stats()["prefix_hit_tokens"] >= 256
        for b, s in enumerate(slots):
            assert n_gen[s] == T
            assert e.cb_read(s, 0, T) == c["gen"][b].tolist(), f"row {b}"
        for s in slots:
            e.cb_release(s)
    finally:
        e.cb_end()


def test_partial_bias_set_is_refused_at_finalize():
    from oracle import weights as W
    from kserve_b200 import _lib
    from kserve_b200.engine import B200Engine
    cfg = W.CONFIGS["tiny_qwen2"]
    eng = B200Engine(cfg, max_batch=2, max_seq_len=256)
    try:
        with pytest.raises(_lib.B200Error, match="model.layers.1.self_attn.k_proj.bias"):
            eng.load_weights((n, t) for n, t in W.iter_state_dict(cfg, 0) if n != "model.layers.1.self_attn.k_proj.bias")
    finally:
        eng.close()


def test_served_from_a_qwen2_checkpoint_directory(tmp_path):
    """B200GenerativeModel.load() from a directory holding a Qwen2 config.json (tied embeddings, the sliding-window fields
    of real Qwen2 configs) and a safetensors file without lm_head.weight; /openai/v1/completions returns the fixture's ids"""
    from fastapi.testclient import TestClient
    from safetensors.torch import save_file
    from oracle import weights as W
    from kserve_b200.generative_model import B200GenerativeModel
    from kserve_b200.kserve_api import ModelServer
    c = load_case("tiny_qwen2_g6_tied_ids")
    m = c["meta"]
    cfg = W.CONFIGS[m["cfg"]]
    hf = dict(W.hf_config_dict(cfg), architectures=["Qwen2ForCausalLM"], model_type="qwen2", use_sliding_window=False,
              sliding_window=131072, max_window_layers=21, tie_word_embeddings=True, torch_dtype="bfloat16",
              hidden_act="silu", eos_token_id=None)
    with open(tmp_path / "config.json", "w") as f:
        json.dump(hf, f)
    sd = dict(W.iter_state_dict(cfg, m["seed"]))
    assert "lm_head.weight" not in sd
    save_file(sd, str(tmp_path / "model.safetensors"))
    model = B200GenerativeModel("qwen", str(tmp_path), pad_token_id=m["pad_token_id"], max_model_len=512, max_batch=4)
    assert model.load() and model.max_length == 512
    try:
        with TestClient(ModelServer().create_application([model])) as client:
            r = client.post("/openai/v1/completions", json={"model": "qwen", "prompt": c["input_ids"].tolist(),
                                                            "max_tokens": m["max_tokens"], "temperature": 0})
            assert r.status_code == 200, r.text
            j = r.json()
            assert [ch["text"] for ch in j["choices"]] == [" ".join(str(int(t)) for t in row) for row in c["gen"]]
            assert j["usage"] == {"prompt_tokens": m["prompt_tokens"], "completion_tokens": m["completion_tokens"],
                                  "total_tokens": m["prompt_tokens"] + m["completion_tokens"]}
    finally:
        model.stop()


# ---- b200_op_gemm_bias --------------------------------------------------------------------------------------------
def _lib():
    from kserve_b200 import _lib as L
    return L.load()


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _assert_one_rounding(got, acc, bias):
    """got == bf16(acc + bias) up to the accumulation order: one bf16 ulp of the fp32 reference, plus 1e-4 for the
    fp32 sums of K = 3584 products taken in another order (a dropped or doubled bias would be off by O(0.5))"""
    ref = acc + bias
    err = (got.float() - ref).abs()
    assert bool((err <= 2.0 ** -7 * ref.abs() + 1e-4).all()), float((err - 2.0 ** -7 * ref.abs()).max())


@pytest.mark.parametrize("M", [1, 127, 129, 300, 1000, 4100])
@pytest.mark.parametrize("N, K", [(1031, 512), (4608, 3584)])
def test_op_gemm_bias_prefill_store(M, N, K):
    """epi 0, block_n 256: out[m][n] = bf16(A[m] . W[n] + bias[n]); the 64 sentinel rows after M stay untouched"""
    lib = _lib()
    A = _rand((M, K), M)
    W = _rand((N, K), M + 1, K ** -0.5)
    b = _rand((N,), M + 2)
    O = torch.full((M + 64, N), -7.0, device="cuda", dtype=torch.bfloat16)
    assert lib.b200_op_gemm_bias(_ptr(A), _ptr(W), _ptr(O), None, M, N, K, 0, 256, 1, N, _ptr(b), None) == 0, lib.b200_last_error()
    torch.cuda.synchronize()
    _assert_one_rounding(O[:M], A.float() @ W.float().T, b.float())
    assert bool((O[M:] == -7.0).all())
    O2 = torch.full((M + 64, N), -7.0, device="cuda", dtype=torch.bfloat16)     # no bias: b200_op_gemm, bf16(acc)
    assert lib.b200_op_gemm(_ptr(A), _ptr(W), _ptr(O2), None, M, N, K, 0, 256, 1, N, None) == 0
    torch.cuda.synchronize()
    assert not torch.equal(O, O2)


@pytest.mark.parametrize("M, N, bn", [(1031, 13, 16), (4608, 32, 32), (10240, 64, 64), (10240, 5, 16),
                                      (17024 + 128 * 3 + 7, 16, 16)])   # the last: 137 m-tiles > 132 SMs -> stream-K
def test_op_gemm_bias_decode_transposed_store(M, N, bn):
    """epi 3 (swap-AB): out[n][m] = bf16(W[m] . x[n] + bias[m]).  Without stream-K the fp32 accumulator of the same
    tile schedule is available exactly (epi 5, one split), so the result must be bf16(acc + bias) bit for bit."""
    lib = _lib()
    K = 512
    Wt = _rand((M, K), M, K ** -0.5)
    x = _rand((N, K), M + 1)
    b = _rand((M,), M + 2)
    O = torch.full((N + 8, M), -7.0, device="cuda", dtype=torch.bfloat16)
    assert lib.b200_op_gemm_bias(_ptr(Wt), _ptr(x), _ptr(O), None, M, N, K, 3, bn, 1, M, _ptr(b), None) == 0, lib.b200_last_error()
    acc = torch.zeros((N, M), device="cuda", dtype=torch.float32)
    assert lib.b200_op_gemm(_ptr(Wt), _ptr(x), _ptr(acc), None, M, N, K, 5, bn, 1, M, None) == 0, lib.b200_last_error()
    torch.cuda.synchronize()
    assert bool((O[N:] == -7.0).all())
    m_tiles = -(-M // 128)
    if m_tiles < torch.cuda.get_device_properties(0).multi_processor_count:
        assert torch.equal(O[:N], (acc + b.float()).to(torch.bfloat16))
    else:
        _assert_one_rounding(O[:N], (x.float() @ Wt.float().T), b.float())


def test_op_gemm_bias_refuses_other_epilogues():
    lib = _lib()
    A, W, b = _rand((128, 64), 1), _rand((512, 64), 2), _rand((512,), 3)
    O = torch.empty((128, 256), device="cuda", dtype=torch.bfloat16)
    assert lib.b200_op_gemm_bias(_ptr(A), _ptr(W), _ptr(O), None, 128, 512, 64, 2, 256, 1, 256, _ptr(b), None) != 0


# ---- Qwen2.5-7B layer shapes ----------------------------------------------------------------------------------------
@pytest.mark.slow
@pytest.mark.parametrize("name", ["qwen2_7b_2l_b4", "qwen2_7b_2l_peaked_b4"])
def test_qwen2_7b_shapes_1024_prompt_tokens(name):
    """Qwen2.5-7B layer shapes (2 layers, 28 / 4 heads, I = 18944, V = 152064): 4 x 1024-token prompts, 16 decode steps.
    Teacher-forced logits on 4096 fixed columns + the oracle's top-16; the peaked case's free-running ids exactly."""
    c = load_case(name)
    m = c["meta"]
    eng = make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], max_batch=4, max_seq_len=1152)
    try:
        pad = m["pad_token_id"]
        peaked = "peaked" in name
        r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"], want_logits=True)
        assert torch.equal(r.output_ids, c["output_ids"])
        got = r.logits.float().permute(1, 0, 2)
        assert not torch.isnan(got).any()
        sub = got[..., c["sub_cols"]]
        topv = torch.gather(got, 2, c["topk_idx"].long())
        tol = float(logits_tol(c["topk_vals"]))
        if peaked:
            floor = c["topk_vals"][..., 1]
            ok_sub = (sub - c["sub_logits"]).abs() <= logits_tol_elementwise(c["sub_logits"], floor)
            ok_top = (topv - c["topk_vals"]).abs() <= logits_tol_elementwise(c["topk_vals"], floor)
        else:
            ok_sub = (sub - c["sub_logits"]).abs() <= tol
            ok_top = (topv - c["topk_vals"]).abs() <= tol
        stats = dict(err_sub=float((sub - c["sub_logits"]).abs().max()), err_top=float((topv - c["topk_vals"]).abs().max()), tol=tol)
        assert bool(ok_sub.all()) and bool(ok_top.all()), stats
        decisive = c["margin"] > 2 * tol
        assert bool((got.argmax(-1) == c["gen"])[decisive].all()), stats
        free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
        exact = free.output_ids[:, c["S"]:] == c["gen"]
        if peaked:
            assert bool(decisive.all()) and bool(exact.all()), stats
        else:
            for b in range(exact.shape[0]):
                neq = (~exact[b]).nonzero()
                if len(neq):
                    assert not bool(decisive[b, int(neq[0])]), f"row {b} diverges at a decisive step"
    finally:
        eng.close()


# ---- tensor parallel ------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tp2_qwen2_matches_oracle_fixture():
    """TP = 2: each rank holds half of the q / k / v heads and the matching slices of their biases"""
    names = ["tiny_qwen2_ids", "tiny_qwen2_wide_ids"]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29641", os.path.join(HERE, "tp_worker.py"), ",".join(names)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    ret = json.loads([l for l in res.stdout.splitlines() if l.startswith("TPRESULT ")][0][len("TPRESULT "):])
    for name in names:
        c = load_case(name)
        tol = logits_tol(c["step_logits"])
        assert torch.equal(torch.tensor(ret[name + ":forced"]), c["output_ids"])
        assert ret[name + ":max_err"] <= tol
        gen = torch.tensor(ret[name])[:, c["S"]:]
        for b in range(gen.shape[0]):
            neq = (gen[b] != c["gen"][b]).nonzero()
            if len(neq):
                assert float(c["margin"][b, int(neq[0])]) <= 2 * tol
