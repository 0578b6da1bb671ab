"""FP8 (compressed-tensors float8_e4m3fn) checkpoints on the GPU.

The engine multiplies exactly W' = bf16(code) * bf16(scale) (kserve_b200/fp8.py), so an FP8 engine must be
bit-identical to a bf16 engine loaded with W' — prefill and decode, logits and ids — whatever path a projection takes:
the FP8 swap-AB decode GEMM (BLOCK_N 16 / 32 / 64, split-K partials, stream-K, the SwiGLU and transposed-store epilogues,
the Qwen2 bias) and the per-layer dequantize feeding the unchanged prefill GEMM.  tests/test_fp8_cpu.py ties W' to
what transformers computes for the same checkpoint; the engine's bf16 path is held to the oracle by the existing tests."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = torch.device("cuda", 0)
E4M3_MAX = 448.0


def quantize(t, scale_dtype=torch.bfloat16, strategy="channel"):
    """e4m3 codes of a bf16 weight with a channel (per-row) or tensor scale, as llm-compressor forms them"""
    t = t.float()
    amax = t.abs().amax(dim=1, keepdim=True) if strategy == "channel" else t.abs().amax().reshape(1)
    scale = (amax / E4M3_MAX).clamp_min(1e-12).to(scale_dtype)
    codes = (t / scale.float().reshape(-1, 1) if strategy == "channel" else t / scale.float()).clamp(-E4M3_MAX, E4M3_MAX)
    return codes.to(torch.float8_e4m3fn), scale


def fp8_state_dicts(cfg, seed, scale_dtype=torch.bfloat16, strategy="channel", device="cpu"):
    """(FP8 checkpoint tensors, the bf16 tensors of W') from the seeded synthetic checkpoint"""
    from oracle import weights as W
    from kserve_b200.fp8 import PROJECTIONS, dequantize_reference
    q, ref = [], []
    embed = None
    for name, t in W.iter_state_dict(cfg, seed):
        t = t.to(device)
        if name == "model.embed_tokens.weight":
            embed = t
        if any(name.endswith(p + ".weight") for p in PROJECTIONS):
            codes, scale = quantize(t, scale_dtype, strategy)
            q += [(name, codes), (name + "_scale", scale)]
            ref.append((name, dequantize_reference(codes, scale)))
        else:
            q.append((name, t))
            ref.append((name, t))
    if cfg.get("tie_word_embeddings"):
        q.append(("lm_head.weight", embed))
        ref.append(("lm_head.weight", embed))
    return q, ref


def engine_pair(cfg_name, seed=0, scale_dtype=torch.bfloat16, strategy="channel", device="cpu", **kw):
    from oracle import weights as W
    from kserve_b200.engine import B200Engine
    cfg = W.CONFIGS[cfg_name]
    q, ref = fp8_state_dicts(cfg, seed, scale_dtype, strategy, device)
    e8 = B200Engine(cfg, weight_format=1, **kw)
    e8.load_weights(iter(q))
    e16 = B200Engine(cfg, **kw)
    e16.load_weights(iter(ref))
    return cfg, e8, e16


def prompts(cfg, B, S, seed=1):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, cfg["vocab_size"] - 1, (B, S), generator=g)
    mask = torch.ones_like(ids)
    for b in range(B):                              # ragged, left padded
        mask[b, : (b * 7) % max(1, S // 2)] = 0
    ids[mask == 0] = 0
    return ids, mask


def assert_same_generation(e8, e16, cfg, B, S, T):
    ids, mask = prompts(cfg, B, S)
    forced = torch.randint(3, cfg["vocab_size"] - 1, (B, T), generator=torch.Generator().manual_seed(7))
    a = e8.generate(ids, mask, max_new_tokens=T, pad_token_id=0, forced_tokens=forced, want_logits=True)
    b = e16.generate(ids, mask, max_new_tokens=T, pad_token_id=0, forced_tokens=forced, want_logits=True)
    assert torch.equal(a.logits.view(torch.int16), b.logits.view(torch.int16)), "teacher-forced logits differ"
    a = e8.generate(ids, mask, max_new_tokens=T, pad_token_id=0)
    b = e16.generate(ids, mask, max_new_tokens=T, pad_token_id=0)
    assert torch.equal(a.output_ids, b.output_ids)


# ---- kernels -------------------------------------------------------------------------------------------------
def _lib():
    from kserve_b200 import _lib as L
    return L.load()


def all_codes():
    c = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn)
    return c[~c.float().isnan()]


def test_dequant_kernel_equals_the_rule_on_every_code_and_scale_class():
    from kserve_b200.fp8 import dequantize_reference
    codes = all_codes()
    scales = torch.tensor([1e-30, 3e-39, 1e-8, 3.7e-3, 0.0173, 1.0, 2.5, 255.0, 1e5, 3e38, -0.5], dtype=torch.float32)
    K = 16 * ((codes.numel() + 15) // 16)
    w = torch.zeros(len(scales), K, dtype=torch.float8_e4m3fn)
    w[:, : codes.numel()] = codes
    for sd in (torch.bfloat16, torch.float32):
        s = scales.to(sd)
        ref = dequantize_reference(w, s)
        wd, sb = w.to(DEV), s.to(torch.bfloat16).to(DEV)
        out = torch.empty(len(scales), K, dtype=torch.bfloat16, device=DEV)
        assert _lib().b200_op_dequant_fp8(wd.data_ptr(), sb.data_ptr(), out.data_ptr(), len(scales), K, None) == 0
        torch.cuda.synchronize()
        assert torch.equal(out.cpu().view(torch.int16), ref.view(torch.int16))


def _gemm(fp8, A, sc, Bm, M, N, K, epi, bn, splits, bias=None):
    ldo = M if epi != 4 else M // 2
    rows_out = N * splits if epi == 5 else N
    dt = torch.float32 if epi == 5 else torch.bfloat16
    out = torch.full((rows_out + 3, ldo), -7.0, dtype=dt, device=DEV)    # rows past the output are sentinels
    bp = bias.data_ptr() if bias is not None else None
    lib = _lib()
    if fp8:
        rc = lib.b200_op_gemm_fp8(A.data_ptr(), sc.data_ptr(), Bm.data_ptr(), out.data_ptr(), bp, M, N, K, epi, bn, splits, ldo, None)
    elif bias is not None:
        rc = lib.b200_op_gemm_bias(A.data_ptr(), Bm.data_ptr(), out.data_ptr(), None, M, N, K, epi, bn, splits, ldo, bp, None)
    else:
        rc = lib.b200_op_gemm(A.data_ptr(), Bm.data_ptr(), out.data_ptr(), None, M, N, K, epi, bn, splits, ldo, None)
    assert rc == 0, lib.b200_last_error()
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("M", [1, 127, 129, 300, 2304])
@pytest.mark.parametrize("epi", [3, 4, 5])
def test_fp8_gemm_equals_bf16_gemm_on_w_prime(M, epi):
    from kserve_b200.fp8 import dequantize_reference
    if epi == 4:
        M = 32 * ((M + 31) // 32)                    # 16-row gate / up interleave
    g = torch.Generator(device=DEV).manual_seed(M + 10 * epi)
    K = 1024
    w = torch.randn(M, K, generator=g, device=DEV) * 0.05
    A, sc = quantize(w)
    Wp = dequantize_reference(A, sc)
    for N in [1, 2, 7, 15, 16, 17, 31, 32, 33, 47, 63, 64]:
        bn = 16 if N <= 16 else (32 if N <= 32 else 64)
        Bm = torch.randn(N, K, generator=g, device=DEV).to(torch.bfloat16)
        for splits in ([1] if epi != 5 else [2, 5]):
            for bias in ([None, torch.randn(M, generator=g, device=DEV).to(torch.bfloat16)] if epi == 3 else [None]):
                a = _gemm(True, A, sc, Bm, M, N, K, epi, bn, splits, bias)
                b = _gemm(False, Wp, None, Bm, M, N, K, epi, bn, splits, bias)
                assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                                   b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32)), (N, splits, bias is not None)
                assert bool((a[-3:] == -7.0).all()), "rows past the output were written"
                a2 = _gemm(True, A, sc, Bm, M, N, K, epi, bn, splits, bias)
                assert torch.equal(a, a2)


def test_fp8_gemm_stream_k_equals_bf16():
    """single-split swap-AB GEMMs with more weight tiles than SMs are cut into balanced stream-K pieces"""
    from kserve_b200.fp8 import dequantize_reference
    g = torch.Generator(device=DEV).manual_seed(3)
    M, K = 128 * 150, 512
    A, sc = quantize(torch.randn(M, K, generator=g, device=DEV) * 0.05)
    Wp = dequantize_reference(A, sc)
    for epi, N in [(3, 5), (4, 24), (3, 40)]:
        bn = 16 if N <= 16 else (32 if N <= 32 else 64)
        Bm = torch.randn(N, K, generator=g, device=DEV).to(torch.bfloat16)
        assert torch.equal(_gemm(True, A, sc, Bm, M, N, K, epi, bn, 1), _gemm(False, Wp, None, Bm, M, N, K, epi, bn, 1))


# ---- the engine -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def g4_pair():
    cfg, e8, e16 = engine_pair("tiny_g4", 0, max_batch=64, max_seq_len=512)
    yield cfg, e8, e16
    e8.close()
    e16.close()


@pytest.mark.parametrize("B", [1, 3, 20, 40, 64])     # split-K decode, and every BLOCK_N class
def test_engine_bit_identical_to_bf16_engine_on_w_prime(g4_pair, B):
    cfg, e8, e16 = g4_pair
    assert_same_generation(e8, e16, cfg, B, 37, 9)


@pytest.mark.parametrize("cfg_name, scale_dtype, strategy", [
    ("tiny_qwen2", torch.bfloat16, "channel"),        # q/k/v biases, G = 7
    ("tiny_qwen2_g6_tied", torch.float32, "channel"),  # fp32 scales (rounded to bf16 at load), tied embeddings
    ("tiny_g2", torch.float32, "tensor"),              # one scale per tensor, broadcast to the rows
])
def test_engine_bit_identical_other_configs(cfg_name, scale_dtype, strategy):
    cfg, e8, e16 = engine_pair(cfg_name, 0, scale_dtype, strategy, max_batch=32, max_seq_len=256)
    try:
        for B in (2, 24):
            assert_same_generation(e8, e16, cfg, B, 50, 8)
    finally:
        e8.close()
        e16.close()


def test_engine_stream_k_paths_bit_identical(monkeypatch):
    """B200_STREAMK_ANY: every single-split decode GEMM (gate/up, o, down, LM head) takes the stream-K schedule"""
    monkeypatch.setenv("B200_STREAMK_ANY", "1")
    cfg, e8, e16 = engine_pair("tiny_g4", 0, max_batch=32, max_seq_len=256)
    try:
        assert_same_generation(e8, e16, cfg, 24, 40, 6)
    finally:
        e8.close()
        e16.close()


def test_continuous_batching_chunked_prefill_matches_static(g4_pair):
    """chunked prefill (128-token chunks) with prefix reuse runs the per-layer dequantize once per chunk pass"""
    cfg, e8, _ = g4_pair
    g = torch.Generator().manual_seed(5)
    shared = torch.randint(3, cfg["vocab_size"] - 1, (256,), generator=g).tolist()
    rows = [shared + torch.randint(3, cfg["vocab_size"] - 1, (n,), generator=g).tolist() for n in (5, 140, 61)]
    T = 6
    want = [e8.generate(torch.tensor([r]), None, max_new_tokens=T, pad_token_id=0).output_ids[0, len(r):].tolist() for r in rows]
    e8.cb_begin(0, [])
    try:
        e8.cb_config(128, True)
        slots = e8.cb_admit(rows[:1], [T])
        for _ in range(50):                          # the first prompt's prefill completes: its blocks are cached
            e8.cb_step(1)
            if e8.cb_poll()[1][slots[0]]:
                break
        slots += e8.cb_admit(rows[1:], [T, T])
        for _ in range(200):
            e8.cb_step(1)
            n_gen, fin, _ = e8.cb_poll()
            if all(fin[s] for s in slots):
                break
        got = [e8.cb_read(s)[:T] for s in slots]
        for s in slots:
            e8.cb_release(s)
        assert e8.cb_stats()["prefix_hit_tokens"] > 0
    finally:
        e8.cb_end()
    assert got == want


def test_without_rope_fusion_subprocess():
    env = dict(os.environ, B200_NO_ROPE_FUSION="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "test_engine_bit_identical_to_bf16_engine_on_w_prime"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def test_prefetcher_is_refused_with_fp8_weights():
    code = ("import torch, sys; sys.path.insert(0, 'tests'); from test_fp8_gpu import engine_pair, prompts\n"
            "cfg, e8, e16 = engine_pair('tiny_g2', 0, max_batch=4, max_seq_len=128)\n"
            "ids, mask = prompts(cfg, 2, 20)\n"
            "try:\n    e8.generate(ids, mask, max_new_tokens=4, pad_token_id=0)\nexcept Exception as e:\n    print('REFUSED', e)\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, B200_PREFETCHER="1"),
                       capture_output=True, text=True, timeout=600)
    assert "REFUSED" in r.stdout and "B200_PREFETCHER" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.slow
def test_llama3_8b_shapes_4x1024_bit_identical():
    """Llama-3-8B layer shapes (2 layers, 128k vocabulary): gate/up takes the stream-K schedule natively (224 tiles)"""
    cfg, e8, e16 = engine_pair("llama3_8b_2l", 0, device=DEV, max_batch=4, max_seq_len=1024 + 8, max_prefill_tokens=4 * 1024)
    try:
        assert_same_generation(e8, e16, cfg, 4, 1024, 8)
    finally:
        e8.close()
        e16.close()


# ---- the transformers oracle (tools/fp8_oracle.py fixtures) ---------------------------------------------------------
from helpers import load_case, logits_tol, logits_tol_elementwise, make_engine  # noqa: E402

GOLDEN_CASES = ["tiny_g4_fp8_ids", "tiny_qwen2_fp8_ids", "tiny_g2_fp8_tensor_ids"]


@pytest.fixture(scope="module")
def oracle_engines():
    cache = {}

    def get(case):
        m = case["meta"]
        key = (m["cfg"], m["seed"])
        if key not in cache:
            from oracle import weights as W
            from kserve_b200.engine import B200Engine
            cfg = W.CONFIGS[m["cfg"]]
            eng = B200Engine(cfg, weight_format=1, vocab_rows=m["vocab_rows"], max_batch=8, max_seq_len=512)
            eng.load_weights(W.iter_state_dict(cfg, m["seed"]))
            cache[key] = eng
        return cache[key]
    yield get
    for e in cache.values():
        e.close()


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_teacher_forced_logits_and_greedy_vs_oracle(oracle_engines, name):
    c = load_case(name)
    eng = oracle_engines(c)
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=c["meta"]["pad_token_id"],
                     forced_tokens=c["gen"], want_logits=True)
    assert r.num_generated == c["T"] and torch.equal(r.output_ids, c["output_ids"])
    got = r.logits.float().permute(1, 0, 2)
    tol = logits_tol(c["step_logits"])
    err = float((got - c["step_logits"]).abs().max())
    assert err <= tol, f"max logits error {err:.4f} > tol {tol:.4f}"
    decisive = c["margin"] > 2 * tol
    assert bool((got.argmax(-1) == c["gen"])[decisive].all())


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_free_running_ids_vs_oracle(oracle_engines, name):
    c = load_case(name)
    eng = oracle_engines(c)
    pad = c["meta"]["pad_token_id"]
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
    tol = logits_tol(c["step_logits"])
    gen = r.output_ids[:, c["S"]:]
    for b in range(gen.shape[0]):
        neq = (gen[b] != c["gen"][b]).nonzero()
        if len(neq):
            assert float(c["margin"][b, int(neq[0])]) <= 2 * tol, f"row {b} diverges at decisive step {int(neq[0])}"


def test_peaked_ids_exact_vs_oracle(oracle_engines):
    c = load_case("tiny_g4_fp8_peaked")
    eng = oracle_engines(c)
    pad = c["meta"]["pad_token_id"]
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"], want_logits=True)
    got = r.logits.float().permute(1, 0, 2)
    err = (got - c["step_logits"]).abs()
    assert bool((err <= logits_tol_elementwise(c["step_logits"])).all())
    assert bool((c["margin"] > 2 * logits_tol(c["step_logits"])).all())
    free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
    assert torch.equal(free.output_ids[:, c["S"]:], c["gen"])


@pytest.mark.slow
@pytest.mark.parametrize("name", ["llama3_8b_2l_fp8_b4", "llama3_8b_2l_fp8_peaked_b4"])
def test_llama3_8b_shapes_4x1024_vs_oracle(name):
    """Llama-3-8B layer shapes, FP8 projections: 4 x 1024-token prompts, 16 steps; logits on 4096 fixed columns + the
    oracle's top-16; the peaked case's free-running ids exactly"""
    from oracle import weights as W
    from kserve_b200.engine import B200Engine
    c = load_case(name)
    m = c["meta"]
    cfg = W.CONFIGS[m["cfg"]]
    eng = B200Engine(cfg, weight_format=1, vocab_rows=m["vocab_rows"], max_batch=4, max_seq_len=1152)
    eng.load_weights(W.iter_state_dict(cfg, m["seed"]))
    try:
        pad = m["pad_token_id"]
        peaked = "peaked" in name
        r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"], want_logits=True)
        got = r.logits.float().permute(1, 0, 2)
        sub = got[..., c["sub_cols"]]
        topv = torch.gather(got, 2, c["topk_idx"].long())
        tol = float(logits_tol(c["topk_vals"]))
        if peaked:
            floor = c["topk_vals"][..., 1]
            ok = ((sub - c["sub_logits"]).abs() <= logits_tol_elementwise(c["sub_logits"], floor)).all() and \
                ((topv - c["topk_vals"]).abs() <= logits_tol_elementwise(c["topk_vals"], floor)).all()
        else:
            ok = ((sub - c["sub_logits"]).abs() <= tol).all() and ((topv - c["topk_vals"]).abs() <= tol).all()
        assert bool(ok), dict(err_sub=float((sub - c["sub_logits"]).abs().max()), tol=tol)
        decisive = c["margin"] > 2 * tol
        assert bool((got.argmax(-1) == c["gen"])[decisive].all())
        free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
        exact = free.output_ids[:, c["S"]:] == c["gen"]
        if peaked:
            assert bool(decisive.all()) and bool(exact.all())
        else:
            for b in range(exact.shape[0]):
                neq = (~exact[b]).nonzero()
                if len(neq):
                    assert not bool(decisive[b, int(neq[0])]), f"row {b} diverges at a decisive step"
    finally:
        eng.close()


# ---- serving a compressed-tensors checkpoint directory -----------------------------------------------------------
def test_checkpoint_directory_served_over_openai_completions(tmp_path):
    """the oracle's own checkpoint directory (tools/fp8_oracle.write_checkpoint) through B200GenerativeModel and
    /openai/v1/completions: every step of the peaked fixture is decisive, so the served text is the oracle's ids"""
    from fastapi.testclient import TestClient
    from tools.fp8_oracle import write_checkpoint
    from kserve_b200.generative_model import B200GenerativeModel
    from kserve_b200.kserve_api import ModelServer
    c = load_case("tiny_g4_fp8_peaked")
    m = c["meta"]
    d = write_checkpoint(str(tmp_path), m["cfg"], m["seed"])
    rows = [r[mk.bool()].tolist() for r, mk in zip(c["input_ids"], c["mask"])]
    model = B200GenerativeModel("fp8", d, pad_token_id=m["pad_token_id"], max_model_len=512, max_batch=4)
    assert model.load()
    try:
        with TestClient(ModelServer().create_application([model])) as client:
            for b, row in enumerate(rows):
                r = client.post("/openai/v1/completions", json={"model": "fp8", "prompt": row, "max_tokens": m["max_tokens"],
                                                                "temperature": 0})
                assert r.status_code == 200, r.text
                assert r.json()["choices"][0]["text"] == " ".join(str(int(t)) for t in c["gen"][b]), f"row {b}"
    finally:
        model.stop()
