"""The FP8 KV cache (kv_cache_dtype 1: float8_e4m3fn codes) on the GPU.

- attn_prefill_tc_kernel<true> on a code cache C gives the bits attn_prefill_tc_kernel gives on the bf16 cache bf16(C);
- attn_decode_kernel<true> against fp32 attention over the dequantized cache (the bounds of test_attention_gpu.py), with
  the appended codes equal to kserve_b200.fp8.quantize_kv of HF RoPE in bf16, byte for byte;
- 0x7F codes (NaN in e4m3fn) in every slot outside the contexts change no bit of either kernel's output;
- the engine against the oracle fixtures of tools/kv8_oracle.py (HF generate with a quantizing cache), the switches and
  paths that write or move the cache, and a checkpoint served with kv_cache_dtype="fp8".
"""
import json
import os
import subprocess
import sys

import pytest
import torch

from helpers import load_case, logits_tol, logits_tol_elementwise, make_engine
from test_attention_gpu import (DEC_CTX, DEV, HEADS, MODES, PREFILL_HEADS, DecodeCase, Paged, _check, _close, _merges,
                                _prefill_inputs, _ptr, _ref, _same)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def q8(x):
    from kserve_b200.fp8 import quantize_kv
    return quantize_kv(x)


def dq(x):
    """the bf16 values an FP8 cache holds for x"""
    return q8(x).to(torch.bfloat16)


class Codes:
    """the e4m3 code caches of a bf16 Paged whose keys are e4m3 values: every slot outside the contexts (NaN in a Paged
    built with stale="nan") becomes the NaN code 0x7F"""

    def __init__(self, paged):
        self.pt, self.max_pages, self.num_pages, self.slot = paged.pt, paged.max_pages, paged.num_pages, paged.slot
        self.kc, self.vc = (self._codes(c) for c in (paged.kc, paged.vc))

    @staticmethod
    def _codes(c):
        u = q8(c).view(torch.uint8).clone()
        u[torch.isnan(c)] = 0x7F
        return u


# ---------------------------------------------------------------------------------------------------------------- prefill
def _prefill(lib, q, cache, lens, offs, nh, nkv, kv8):
    B = len(lens)
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    slot = torch.arange(B, dtype=torch.int32, device=DEV)
    off = torch.tensor(offs, dtype=torch.int32, device=DEV) if offs is not None else None
    out = torch.full((q.shape[0], nh * 128), float("nan"), dtype=torch.bfloat16, device=DEV)
    fn = lib.b200_op_attn_prefill_tc_kv8 if kv8 else lib.b200_op_attn_prefill_tc_off
    _check(lib, fn(_ptr(q), nh * 128, q.shape[0], _ptr(out), nh * 128, _ptr(cache.kc), _ptr(cache.vc), cache.num_pages,
                   _ptr(cache.pt), cache.max_pages, _ptr(cu), _ptr(slot), _ptr(off), B, max(lens), nh, nkv, None),
           "attn_prefill_tc" + ("_kv8" if kv8 else "_off"))
    torch.cuda.synchronize()
    return out


def _prefill_case(lib, nh, nkv, lens, offs, seed):
    ks, vs, q = _prefill_inputs(nh, nkv, lens, offs, seed)
    ks, vs = [dq(k) for k in ks], [dq(v) for v in vs]
    want = _prefill(lib, q, Paged(ks, vs, "zero", seed), lens, offs, nh, nkv, kv8=False)
    got = _prefill(lib, q, Codes(Paged(ks, vs, "zero", seed)), lens, offs, nh, nkv, kv8=True)
    _same(f"prefill kv8 nh {nh} nkv {nkv} lens {lens}", got, want)
    poisoned = _prefill(lib, q, Codes(Paged(ks, vs, "nan", seed)), lens, offs, nh, nkv, kv8=True)
    _same(f"prefill kv8 nh {nh} nkv {nkv}: 0x7F codes outside the contexts", poisoned, got)


@pytest.mark.parametrize("nh,nkv", PREFILL_HEADS)
@pytest.mark.parametrize("with_off", [False, True])
def test_prefill_kv8_bit_identical_to_bf16_on_dequantized_cache(lib, nh, nkv, with_off):
    lens = [1, 127, 128, 129, 200, 63]
    offs = [4096, 128, 1024, 0, 128, 1024] if with_off else None
    _prefill_case(lib, nh, nkv, lens, offs, seed=nh * 31 + nkv)


def test_prefill_kv8_8192_tokens(lib):
    _prefill_case(lib, 28, 4, [8192], None, seed=77)


# ----------------------------------------------------------------------------------------------------------------- decode
class DecodeCase8(DecodeCase):
    """DecodeCase on a code cache: the cached keys are e4m3 values, the kernel appends e4m3 codes"""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.ks, self.vs = [dq(k) for k in self.ks], [dq(v) for v in self.vs]

    def paged(self, stale, seed=11):
        return Codes(super().paged("nan" if stale != "zero" else "zero", seed))

    def run(self, lib, paged, mode, splits, fold, part_fill="zero", reps=1):
        class Kv8Lib:           # DecodeCase.run launches b200_op_attn_decode_fused: point it at the kv8 entry point
            b200_op_attn_decode_fused = lib.b200_op_attn_decode_fused_kv8
            b200_last_error = lib.b200_last_error
        return super().run(Kv8Lib, paged, mode, splits, fold, part_fill, reps)

    def check(self, name, paged, out, raw):
        q, k, v = self.roped(raw)
        for b, c in enumerate(self.ctxs):
            page, s = paged.slot(b, c - 1)
            assert torch.equal(paged.kc[page, :, s], q8(k[b]).view(torch.uint8)), f"{name}: appended k codes of sequence {b}"
            assert torch.equal(paged.vc[page, :, s], q8(v[b]).view(torch.uint8)), f"{name}: appended v codes of sequence {b}"
            kk = torch.cat([self.ks[b], dq(k[b])[:, None]], 1)
            vv = torch.cat([self.vs[b], dq(v[b])[:, None]], 1)
            ref, pv = _ref(q[b][:, None], kk, vv, torch.tensor([c - 1], device=DEV))
            _close(f"{name} seq {b} ctx {c}", out[b:b + 1], ref, pv)


@pytest.mark.parametrize("splits", [1, 2, 5, 8])
@pytest.mark.parametrize("nh,nkv", HEADS)
def test_decode_kv8_vs_fp32(lib, nh, nkv, splits):
    """every input mode and both merges at contexts 1 .. 32768; the appended codes; split counters back at zero and a
    second launch bit-identical (DecodeCase.run); 0x7F codes outside the contexts: bit-identical"""
    dc = DecodeCase8(nh, nkv, DEC_CTX, seed=nh * 13 + nkv + splits)
    for mode in MODES:
        for fold in _merges(splits):
            name = f"decode kv8 G{dc.G} splits {splits} {mode} {'folded' if fold else 'combine kernel'}"
            paged = dc.paged("zero")
            base, again = dc.run(lib, paged, mode, splits, fold, reps=2)
            _same(f"{name}: second launch", again, base)
            dc.check(name, paged, base, dc.raw(mode == "partial+bias"))
            got, = dc.run(lib, dc.paged("7f"), mode, splits, fold)
            _same(f"{name} 0x7F codes outside the contexts", got, base)


def test_decode_kv8_large_k_saturates():
    """k values past +-448 (and past +-464, where torch's plain cast gives NaN) are stored as +-448"""
    from kserve_b200 import _lib
    lib = _lib.load()
    dc = DecodeCase8(16, 8, [1, 65, 1000], seed=3)
    dc.partial[0, :dc.B, dc.nh * 128:(dc.nh + 2 * dc.nkv) * 128] *= 300.0      # k and v rows up to ~2400
    paged = dc.paged("zero")
    out, = dc.run(lib, paged, "partial", 1, True)
    dc.check("decode kv8 saturated", paged, out, dc.raw(False))
    assert int((paged.kc == 0x7E).sum() + (paged.kc == 0xFE).sum()) > 0, "no code saturated at +-448"


# ----------------------------------------------------------------------------------------------------------------- engine
def _engine(c, **kw):
    m = c["meta"]
    if m["cfg"].startswith("tiny_qwen2"):
        import test_qwen2_gpu as t
        return t.make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], kv_cache_dtype=1, **kw)
    return make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], kv_cache_dtype=1, **kw)


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(c):
        key = (c["meta"]["cfg"], c["meta"]["seed"])
        if key not in cache:
            cache[key] = _engine(c, max_batch=8, max_seq_len=512)
        return cache[key]
    yield get
    for e in cache.values():
        e.close()


@pytest.mark.parametrize("name", ["tiny_g4_ids_kv8", "tiny_qwen2_ids_kv8", "tiny_moe_ids_kv8"])
def test_engine_kv8_teacher_forced_and_greedy(engines, name):
    c = load_case(name)
    eng = engines(c)
    pad = c["meta"]["pad_token_id"]
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"], want_logits=True)
    got = r.logits.float().permute(1, 0, 2)
    ref = c["step_logits"]
    tol = logits_tol(ref)
    err = float((got - ref).abs().max())
    assert err <= tol, f"max logits error {err:.4f} > tol {tol:.4f}"
    decisive = c["margin"] > 2 * tol
    assert bool((got.argmax(-1) == c["gen"])[decisive].all())
    free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad).output_ids[:, c["S"]:]
    for b in range(free.shape[0]):
        neq = (free[b] != c["gen"][b]).nonzero()
        if len(neq):
            assert float(c["margin"][b, int(neq[0])]) <= 2 * tol, f"row {b} diverges on a decisive step"


def _check_peaked(eng, c):
    pad = c["meta"]["pad_token_id"]
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"], want_logits=True)
    got = r.logits.float().permute(1, 0, 2)
    ref = c["step_logits"]
    err = (got - ref).abs()
    assert bool((err <= logits_tol_elementwise(ref)).all()), "peaked logits out of tolerance"
    free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
    assert torch.equal(free.output_ids, c["output_ids"]), "free-running greedy ids differ from the oracle's"


@pytest.mark.parametrize("name", ["tiny_g4_peaked_kv8", "tiny_qwen2_peaked_kv8"])
def test_engine_kv8_peaked_ids_exact(engines, name):
    c = load_case(name)
    assert bool((c["margin"] > 2 * logits_tol(c["step_logits"])).all()), "fixture: every step decisive"
    _check_peaked(engines(c), c)


@pytest.mark.slow
def test_engine_kv8_llama3_8b_shapes_4x1024():
    c = load_case("llama3_8b_2l_b4_kv8")
    m = c["meta"]
    eng = make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], max_batch=4, max_seq_len=c["S"] + c["T"],
                      kv_cache_dtype=1)
    try:
        r = eng.generate(c["input_ids"], None, max_new_tokens=c["T"], pad_token_id=m["pad_token_id"], forced_tokens=c["gen"],
                         want_logits=True)
        got = r.logits.float().permute(1, 0, 2)[..., c["sub_cols"]]
        ref = c["sub_logits"]
        tol = logits_tol(ref)
        assert float((got - ref).abs().max()) <= tol
        decisive = c["margin"] > 2 * tol
        assert bool((r.logits.float().permute(1, 0, 2).argmax(-1) == c["gen"])[decisive].all())
    finally:
        eng.close()


def test_engine_kv8_without_rope_fusion_is_bit_identical(engines):
    """B200_NO_ROPE_FUSION=1 (EPI_STORE + rope_kv_kernel<true>) writes the codes the fused epilogue writes; the switch is
    read once per process, hence the subprocess"""
    c = load_case("tiny_qwen2_peaked_kv8")
    pad = c["meta"]["pad_token_id"]
    r = engines(c).generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"],
                            want_logits=True)
    code = ("import sys, torch; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from helpers import load_case\n"
            "import test_kv8_gpu as t\n"
            "c = load_case('tiny_qwen2_peaked_kv8')\n"
            "e = t._engine(c, max_batch=8, max_seq_len=512)\n"
            "r = e.generate(c['input_ids'], c['mask'], max_new_tokens=c['T'], pad_token_id=c['meta']['pad_token_id'], "
            "forced_tokens=c['gen'], want_logits=True)\n"
            "torch.save(r.logits.cpu(), sys.argv[1]); e.close()\n") % (ROOT, HERE)
    path = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"kv8_nofusion_{os.getpid()}.pt")
    try:
        res = subprocess.run([sys.executable, "-c", code, path], capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, B200_NO_ROPE_FUSION="1"))
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
        other = torch.load(path)
    finally:
        if os.path.exists(path):
            os.remove(path)
    assert torch.equal(r.logits.cpu().view(torch.int16), other.view(torch.int16))


def test_engine_fp8_weights_with_kv8_equal_bf16_weights_with_kv8():
    from test_fp8_gpu import assert_same_generation, engine_pair
    cfg, e8, e16 = engine_pair("tiny_g4", max_batch=8, max_seq_len=256, kv_cache_dtype=1)
    try:
        assert_same_generation(e8, e16, cfg, B=5, S=100, T=12)
    finally:
        e8.close()
        e16.close()


def _run_until_done(e, slots, max_iters=400):
    for _ in range(max_iters):
        n_gen, fin, _ = e.cb_poll()
        if all(fin[s] for s in slots):
            return n_gen
        e.cb_step(1)
    raise AssertionError("sequences did not finish")


def test_continuous_batching_chunks_prefix_cache_and_host_swap_match_static(engines):
    """128-token prefill chunks, the prefix cache (row 2 shares row 0's first two 128-token blocks: shared pages hold the
    same codes) and a swap-out / swap-in of a running sequence through host DRAM (page_bytes of codes): ids identical to
    a one-pass static prefill on the same engine"""
    c = load_case("tiny_qwen2_peaked_kv8")
    e = engines(c)
    pad, T = c["meta"]["pad_token_id"], c["T"]
    ref = e.generate(c["input_ids"], None, max_new_tokens=T, pad_token_id=pad).output_ids[:, c["S"]:]
    rows = [r.tolist() for r in c["input_ids"]]
    e.cb_begin(pad, [])
    e.cb_config(128, True)
    try:
        slots = e.cb_admit(rows[:2], [T, T])
        e.cb_step(8)
        slots += e.cb_admit(rows[2:], [T, T])
        e.cb_step(4)
        e.cb_swap_out(slots[0])
        e.cb_step(2)
        e.cb_swap_in(slots[0])
        _run_until_done(e, slots)
        st = e.cb_stats()
        assert st["prefix_hit_tokens"] >= 256 and st["swap_outs"] == 1 and st["swap_ins"] == 1
        for b, s in enumerate(slots):
            assert e.cb_read(s, 0, T) == ref[b].tolist(), f"row {b}"
            e.cb_release(s)
    finally:
        e.cb_end()


def test_pool_sized_exactly_admits_the_sequences():
    """an FP8-KV engine whose pool holds exactly the pages of its sequences (3 x ceil(140 / 64)) generates the fixture"""
    c = load_case("tiny_g4_peaked_kv8")
    e = _engine(c, max_batch=3, max_seq_len=c["S"] + c["T"], num_kv_pages=3 * -(-(c["S"] + c["T"]) // 64))
    try:
        r = e.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=c["meta"]["pad_token_id"])
        assert torch.equal(r.output_ids, c["output_ids"])
    finally:
        e.close()


def test_served_with_kv_cache_dtype_fp8(tmp_path):
    """B200GenerativeModel(kv_cache_dtype="fp8") loaded from a checkpoint directory: /openai/v1/completions returns the
    FP8-KV fixture's ids"""
    from fastapi.testclient import TestClient
    from safetensors.torch import save_file
    from oracle import weights as W
    from kserve_b200.generative_model import B200GenerativeModel
    from kserve_b200.kserve_api import ModelServer
    c = load_case("tiny_qwen2_peaked_kv8")
    m = c["meta"]
    cfg = W.CONFIGS[m["cfg"]]
    hf = dict(W.hf_config_dict(cfg), architectures=["Qwen2ForCausalLM"], model_type="qwen2", use_sliding_window=False,
              torch_dtype="bfloat16", hidden_act="silu", eos_token_id=None)
    with open(tmp_path / "config.json", "w") as f:
        json.dump(hf, f)
    save_file(dict(W.iter_state_dict(cfg, m["seed"])), str(tmp_path / "model.safetensors"))
    model = B200GenerativeModel("qwen", str(tmp_path), pad_token_id=m["pad_token_id"], max_model_len=512, max_batch=4,
                                kv_cache_dtype="fp8")
    assert model.load() and model._engine.kv_cache_dtype == 1
    try:
        with TestClient(ModelServer().create_application([model])) as client:
            r = client.post("/openai/v1/completions", json={"model": "qwen", "prompt": c["input_ids"].tolist(),
                                                            "max_tokens": m["max_tokens"], "temperature": 0})
            assert r.status_code == 200, r.text
            assert [ch["text"] for ch in r.json()["choices"]] == [" ".join(str(int(t)) for t in row) for row in c["gen"]]
    finally:
        model.stop()
