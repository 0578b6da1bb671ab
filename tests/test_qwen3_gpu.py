"""Dense Qwen3 decoders on the GPU: the per-head q / k RMSNorm in the three places the engine forms q and k, against fp32
references and the oracle fixtures (tools/synth_weights.py draws the norm weights far from 1 and the q / k projections
with an RMS far from 1, so a dropped, post-RoPE or swapped norm fails these comparisons; tests/test_qwen3_cpu.py checks
that it would).

  prefill  : the EPI_ROPE_KV epilogue of the QKV GEMM (gemm_prefill_kernel<.., QKNORM>), or EPI_STORE + rope_kv_kernel
             under B200_NO_ROPE_FUSION=1; bf16 and e4m3 caches
  decode   : the attn_decode_kernel prologue, on split-K partials and on the bf16 EPI_T_STORE row, G = 2, 4, 5 and 8
Same protocol as tests/test_qwen2_gpu.py."""
import ctypes as C
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
DEV = torch.device("cuda", 0)
EPS = 1e-6


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


# ---- kernels --------------------------------------------------------------------------------------------------------
def _lib():
    from kserve_b200 import _lib as L
    return L.load()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _check(lib, rc, what):
    assert rc == 0, f"{what}: {lib.b200_last_error().decode()}"


def _grid(shape, lo, hi, step, seed):
    """integers in [lo, hi) times `step`, bf16: every fp32 dot product of two such operands is exact in any order"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randint(lo, hi, shape, generator=g, device=DEV).float() * step).to(torch.bfloat16)


def _norm_weights(seed):
    from oracle import weights as W
    q = W.synth_qk_norm(0, (128,), "q_norm", seed).to(DEV)
    k = W.synth_qk_norm(1, (128,), "self_attn.k_norm.weight", seed).to(DEV)
    return q, k


def _tables(n):
    from kserve_b200.engine import hf_rope_tables
    cos, sin = hf_rope_tables(1000000.0, 128, n)
    return cos.to(DEV).contiguous(), sin.to(DEV).contiguous()


def ref_qknorm(x, w):
    """Qwen3RMSNorm of bf16 heads x [.., 128]: fp32 statistics, bf16 before the weight multiply, bf16 after"""
    a = x.float()
    n = (a * torch.rsqrt(a.pow(2).mean(-1, keepdim=True) + EPS)).to(torch.bfloat16)
    return (n.float() * w.float()).to(torch.bfloat16)


def ref_rope(x, cos, sin, pos):
    """HF apply_rotary_pos_emb in bf16 arithmetic; x bf16 [T][heads][128], pos [T]"""
    c = torch.cat([cos, cos], -1)[pos.long()][:, None, :]
    s = torch.cat([sin, sin], -1)[pos.long()][:, None, :]
    return x * c + torch.cat((-x[..., 64:], x[..., :64]), -1) * s


def _assert_rounding_points(what, got, ref):
    """got == ref (the fp32 reference with the bf16 rounding points) up to rsqrtf and the order of the 128 squares: at most
    one bf16 ulp of the normalised value moves each output, and nearly every element is exact"""
    got, ref = got.float(), ref.float()
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output"
    err = (got - ref).abs()
    tol = 2.0 ** -6 * ref.abs().amax(-1, keepdim=True).clamp_min(1e-3)
    assert bool((err <= tol).all()), f"{what}: worst err/tol {float((err / tol).max()):.2f}"
    exact = float((err == 0).float().mean())
    assert exact > 0.98, f"{what}: only {exact:.4f} of the elements are exact"


class PrefillCase:
    """T prompt tokens of two sequences (positions 0.. of each), paged caches with shuffled page ids and sentinel slots"""

    def __init__(self, T, H, nh, nkv, seed):
        self.T, self.H, self.nh, self.nkv = T, H, nh, nkv
        self.N = (nh + 2 * nkv) * 128
        self.x = _grid((T, H), -8, 8, 2.0 ** -3, seed)
        self.w = _grid((self.N, H), -8, 8, 2.0 ** -6, seed + 1)
        self.qn, self.kn = _norm_weights(seed)
        t0 = T // 2
        self.seq = torch.tensor([0] * t0 + [1] * (T - t0), dtype=torch.int32, device=DEV)
        self.pos = torch.tensor(list(range(t0)) + list(range(T - t0)), dtype=torch.int32, device=DEV)
        self.max_pages = (max(t0, T - t0) + 63) // 64 + 1
        self.num_pages = 2 * self.max_pages + 3
        perm = torch.randperm(self.num_pages, generator=torch.Generator().manual_seed(seed))
        self.pt = perm[:2 * self.max_pages].view(2, self.max_pages).to(torch.int32).to(DEV)
        self.cos, self.sin = _tables(max(t0, T - t0) + 64)

    def caches(self, kv8):
        dt = torch.uint8 if kv8 else torch.int16
        fill = 0x5A if kv8 else 0x7F7F
        shape = (self.num_pages, self.nkv, 64, 128)
        return torch.full(shape, fill, dtype=dt, device=DEV), torch.full(shape, fill, dtype=dt, device=DEV)

    def out(self):
        return torch.full((self.T + 64, self.N), -7.0, dtype=torch.bfloat16, device=DEV)   # 64 sentinel rows past T

    def fused(self, lib, kv8, norm=True):
        o = self.out()
        kc, vc = self.caches(kv8)
        _check(lib, lib.b200_op_qkv_rope_kv(_ptr(self.x), _ptr(self.w), _ptr(o), self.N, self.T, self.H, self.nh, self.nkv, None,
                                            _ptr(self.qn) if norm else None, _ptr(self.kn) if norm else None, EPS,
                                            _ptr(kc), _ptr(vc), int(kv8), _ptr(self.pt), self.max_pages, _ptr(self.seq),
                                            _ptr(self.pos), _ptr(self.cos), _ptr(self.sin), None), "qkv_rope_kv")
        torch.cuda.synchronize()
        return o, kc, vc

    def unfused(self, lib, kv8):
        """EPI_STORE + rope_kv_kernel with norms, in place, as the engine runs it under B200_NO_ROPE_FUSION=1"""
        o = self.out()
        kc, vc = self.caches(kv8)
        _check(lib, lib.b200_op_gemm(_ptr(self.x), _ptr(self.w), _ptr(o), None, self.T, self.N, self.H, 0, 256, 1, self.N, None),
               "gemm")
        _check(lib, lib.b200_op_rope_kv_norm(_ptr(o), self.N, _ptr(o), self.N, _ptr(kc), _ptr(vc), int(kv8), _ptr(self.pt),
                                             self.max_pages, _ptr(self.seq), _ptr(self.pos), _ptr(self.cos), _ptr(self.sin),
                                             _ptr(self.qn), _ptr(self.kn), EPS, self.T, self.nh, self.nkv, None), "rope_kv_norm")
        torch.cuda.synchronize()
        return o, kc, vc

    def reference(self):
        """fp32 GEMM (exact on the grid), bf16 rounding, q / k norm, RoPE: q [T][nh][128], k / v [T][nkv][128] bf16"""
        acc = (self.x.float() @ self.w.float().T).to(torch.bfloat16).view(self.T, -1, 128)
        nh, nkv = self.nh, self.nkv
        q = ref_rope(ref_qknorm(acc[:, :nh], self.qn), self.cos, self.sin, self.pos)
        k = ref_rope(ref_qknorm(acc[:, nh:nh + nkv], self.kn), self.cos, self.sin, self.pos)
        return q, k, acc[:, nh + nkv:]

    def rows(self, cache):
        """[T][nkv][128] cache rows of the tokens"""
        page = self.pt[self.seq.long(), (self.pos // 64).long()].long()
        return cache[page, :, (self.pos % 64).long()]

    def untouched(self, cache, fill):
        mask = torch.ones(cache.shape[0], cache.shape[2], dtype=torch.bool, device=DEV)
        page = self.pt[self.seq.long(), (self.pos // 64).long()].long()
        mask[page, (self.pos % 64).long()] = False
        return bool((cache.permute(0, 2, 1, 3)[mask] == fill).all())


PREFILL_SHAPES = [(1024, 8, 4),      # G = 2, q dim 2H (Qwen3-0.6B's ratio)
                  (1024, 5, 1)]      # odd nh: the 256-column tile of heads 4 and 5 holds the last q head and the k head


@pytest.mark.parametrize("H, nh, nkv", PREFILL_SHAPES)
@pytest.mark.parametrize("M", [1, 127, 129, 300, 4100])
def test_op_qkv_rope_kv_norm_vs_fp32(M, H, nh, nkv):
    lib = _lib()
    pc = PrefillCase(M, H, nh, nkv, seed=M + nh)
    q, k, v = pc.reference()
    o, kc, vc = pc.fused(lib, kv8=False)
    _assert_rounding_points("q rows", o[:M, :nh * 128].view(M, nh, 128), q)
    _assert_rounding_points("cached k", pc.rows(kc).view(torch.bfloat16), k)
    assert torch.equal(pc.rows(vc).view(torch.bfloat16), v), "cached v is the bf16 projection"
    assert bool((o[M:] == -7.0).all()), "rows past M were written"
    assert bool((o[:M, nh * 128:] == -7.0).all()), "k / v columns of the q rows are not written"
    assert pc.untouched(kc, 0x7F7F) and pc.untouched(vc, 0x7F7F), "cache slots of no token were written"
    # e4m3 cache: the codes of the bf16 path's values, bit for bit, and the same q rows
    o8, kc8, vc8 = pc.fused(lib, kv8=True)
    from kserve_b200.fp8 import quantize_kv
    assert torch.equal(o8, o)
    assert torch.equal(pc.rows(kc8), quantize_kv(pc.rows(kc).view(torch.bfloat16)).view(torch.uint8))
    assert torch.equal(pc.rows(vc8), quantize_kv(pc.rows(vc).view(torch.bfloat16)).view(torch.uint8))
    assert pc.untouched(kc8, 0x5A) and pc.untouched(vc8, 0x5A)
    # the norm is there: without it q differs
    o0, _, _ = pc.fused(lib, kv8=False, norm=False)
    assert not torch.equal(o0[:M, :nh * 128], o[:M, :nh * 128])


@pytest.mark.parametrize("H, nh, nkv", PREFILL_SHAPES + [(512, 64, 8)])
@pytest.mark.parametrize("kv8", [False, True], ids=["bf16_cache", "e4m3_cache"])
def test_fused_epilogue_equals_store_plus_rope_kv_kernel(H, nh, nkv, kv8):
    """the same bits from the QKNORM epilogue and from EPI_STORE + rope_kv_kernel: q rows and cache bytes"""
    lib = _lib()
    pc = PrefillCase(300, H, nh, nkv, seed=nh * 7 + int(kv8))
    o, kc, vc = pc.fused(lib, kv8)
    o2, kc2, vc2 = pc.unfused(lib, kv8)
    assert torch.equal(o[:300, :nh * 128].view(torch.int16), o2[:300, :nh * 128].view(torch.int16))
    assert torch.equal(kc, kc2) and torch.equal(vc, vc2)


def test_op_qkv_rope_kv_refuses_norms_with_a_bias():
    lib = _lib()
    pc = PrefillCase(16, 512, 2, 1, seed=3)
    b = torch.zeros(pc.N, dtype=torch.bfloat16, device=DEV)
    o = pc.out()
    kc, vc = pc.caches(False)
    assert lib.b200_op_qkv_rope_kv(_ptr(pc.x), _ptr(pc.w), _ptr(o), pc.N, pc.T, pc.H, pc.nh, pc.nkv, _ptr(b), _ptr(pc.qn),
                                   _ptr(pc.kn), EPS, _ptr(kc), _ptr(vc), 0, _ptr(pc.pt), pc.max_pages, _ptr(pc.seq),
                                   _ptr(pc.pos), _ptr(pc.cos), _ptr(pc.sin), None) != 0


DECODE_HEADS = [(16, 8), (32, 8), (40, 8), (64, 8)]    # G = 2, 4, 5, 8


@pytest.mark.parametrize("nh, nkv", DECODE_HEADS)
@pytest.mark.parametrize("kv8", [False, True], ids=["bf16_cache", "e4m3_cache"])
def test_decode_prologue_norm(nh, nkv, kv8):
    """b200_op_attn_decode_fused_norm on the bf16 row and on split-K partials, 1-5 splits: the appended k / v bytes equal
    rope_kv_kernel's for the same bf16 row and position, and the output is within test_attention_gpu's fp32 tolerance of
    attention with rope_kv_kernel's q over the cache plus that k / v"""
    from test_attention_gpu import DecodeCase, QKV_SPLITS, _close, _ref
    from kserve_b200.fp8 import quantize_kv
    lib = _lib()
    dc = DecodeCase(nh, nkv, [1, 63, 64, 65, 200], seed=nh + 100 * int(kv8), kscale=0.5)
    qn, kn = _norm_weights(nh)
    B, G = dc.B, dc.G
    raw = dc.raw(False)
    # reference: rope_kv_kernel with the norm on the same bf16 row and positions
    paged = dc.paged("zero")
    to_cache = (lambda t: quantize_kv(t.view(torch.bfloat16)).view(torch.uint8)) if kv8 else (lambda t: t.clone())
    kc_r, vc_r = to_cache(paged.kc), to_cache(paged.vc)
    qo = torch.empty((B, nh * 128), dtype=torch.bfloat16, device=DEV)
    seq = torch.arange(B, dtype=torch.int32, device=DEV)
    _check(lib, lib.b200_op_rope_kv_norm(_ptr(raw), dc.cols, _ptr(qo), nh * 128, _ptr(kc_r), _ptr(vc_r), int(kv8), _ptr(paged.pt),
                                         paged.max_pages, _ptr(seq), _ptr(dc.pos), _ptr(dc.cos), _ptr(dc.sin), _ptr(qn), _ptr(kn),
                                         EPS, B, nh, nkv, None), "rope_kv_norm")
    torch.cuda.synchronize()
    deq = (lambda t: t.view(torch.float8_e4m3fn).float().to(torch.bfloat16)) if kv8 else (lambda t: t)
    for mode in ("bf16", "partial"):
        for splits in range(1, 6):
            name = f"G{G} {mode} splits {splits} {'e4m3' if kv8 else 'bf16'} cache"
            kc, vc = to_cache(paged.kc), to_cache(paged.vc)
            out = torch.full((B, nh * 128), float("nan"), dtype=torch.bfloat16, device=DEV)
            po = torch.zeros(B * nkv * splits * G * 128, dtype=torch.float32, device=DEV)
            pml = torch.zeros(B * nkv * splits * G * 2, dtype=torch.float32, device=DEV)
            cnt = torch.zeros(B * nkv, dtype=torch.int32, device=DEV)
            if mode == "bf16":
                qkv = torch.zeros((B, dc.cols + 64), dtype=torch.bfloat16, device=DEV)
                qkv[:, :dc.cols] = raw
                src = (_ptr(qkv), qkv.shape[1], None, 0, 0, 0, None)
            else:
                src = (None, 0, _ptr(dc.partial), QKV_SPLITS, dc.split_stride, dc.ld_partial, None)
            _check(lib, lib.b200_op_attn_decode_fused_norm(*src, _ptr(qn), _ptr(kn), EPS, _ptr(dc.cos), _ptr(dc.sin), _ptr(out),
                                                           nh * 128, _ptr(kc), _ptr(vc), int(kv8), _ptr(paged.pt), paged.max_pages,
                                                           _ptr(seq), _ptr(dc.pos), B, nh, nkv, splits, _ptr(po), _ptr(pml),
                                                           _ptr(cnt), None), "attn_decode_fused_norm")
            torch.cuda.synchronize()
            assert torch.equal(kc, kc_r), f"{name}: appended k differs from rope_kv_kernel's"
            assert torch.equal(vc, vc_r), f"{name}: appended v differs from rope_kv_kernel's"
            for b, c in enumerate(dc.ctxs):
                page, s = paged.slot(b, c - 1)
                k_now, v_now = deq(kc_r[page, :, s]), deq(vc_r[page, :, s])
                kk = torch.cat([deq(to_cache(dc.ks[b])), k_now[:, None]], 1)
                vv = torch.cat([deq(to_cache(dc.vs[b])), v_now[:, None]], 1)
                q = qo[b].view(nh, 1, 128)
                ref, pv = _ref(q, kk.view(torch.bfloat16), vv.view(torch.bfloat16), torch.tensor([c - 1], device=DEV))
                _close(f"{name} seq {b} ctx {c}", out[b:b + 1], ref, pv)
    # the norm is there: rope_kv_kernel without it appends another k
    kc0 = to_cache(paged.kc)
    _check(lib, lib.b200_op_rope_kv_norm(_ptr(raw), dc.cols, _ptr(qo), nh * 128, _ptr(kc0), _ptr(to_cache(paged.vc)), int(kv8),
                                         _ptr(paged.pt), paged.max_pages, _ptr(seq), _ptr(dc.pos), _ptr(dc.cos), _ptr(dc.sin),
                                         None, None, EPS, B, nh, nkv, None), "rope_kv")
    torch.cuda.synchronize()
    assert not torch.equal(kc0, kc_r)


# ---- engine ---------------------------------------------------------------------------------------------------------
CASES = ["tiny_qwen3_ids",          # G = 2, q dim 2H, tied; decode QKV by split-K partials (norm in the attention prologue)
         "tiny_qwen3_wide_ids",     # G = 8, 80 m-tiles: decode QKV by the bf16 EPI_T_STORE epilogue
         "tiny_qwen3_g4_ids",       # G = 4, untied
         "tiny_qwen3_g5_ids"]       # G = 5


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(case, **kw):
        m = case["meta"]
        key = (m["cfg"], m["seed"], tuple(sorted(kw.items())))
        if key not in cache:
            cache[key] = make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], max_batch=8, max_seq_len=512, **kw)
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
    """elementwise logits at 2x the peaked rule of tests/helpers.py: the drawn k_norm outliers (+-10..20) make the
    attention scores of this 512-wide model large, so the engine's and the oracle's bf16 q / k (same rounding points,
    other accumulation orders) move the softmax more than in the Llama / Qwen2 fixtures (worst element 1.47x the 1x rule
    on an H100); the free-running ids are exact"""
    pad = c["meta"]["pad_token_id"]
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad, forced_tokens=c["gen"], want_logits=True)
    got = r.logits.float().permute(1, 0, 2)
    ref = c["step_logits"]
    err = (got - ref).abs()
    tol = 2 * logits_tol_elementwise(ref)
    assert bool((err <= tol).all()), f"worst element: err/tol = {float((err / tol).max()):.2f}"
    decisive = c["margin"] > 2 * logits_tol(ref)
    assert bool(decisive.all())
    free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=pad)
    assert torch.equal(free.output_ids[:, c["S"]:], c["gen"])
    return r.logits, free.output_ids


def test_peaked_greedy_ids_exact(engines):
    c = load_case("tiny_qwen3_peaked")
    _check_peaked(engines(c), c)


@pytest.mark.parametrize("kv8", [0, 1], ids=["bf16_cache", "e4m3_cache"])
def test_without_rope_fusion_bit_identical(engines, tmp_path, kv8):
    """B200_NO_ROPE_FUSION=1 (read once per process, hence the subprocess): EPI_STORE + rope_kv_kernel with the norms gives
    the fused path's logits and ids bit for bit, with either cache format"""
    c = load_case("tiny_qwen3_peaked")
    m = c["meta"]
    out = tmp_path / "nofusion.pt"
    code = ("import sys, torch; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from helpers import load_case\n"
            "import test_qwen3_gpu as t\n"
            "c = load_case('tiny_qwen3_peaked'); m = c['meta']\n"
            "e = t.make_engine(m['cfg'], m['seed'], vocab_rows=m['vocab_rows'], max_batch=8, max_seq_len=512, kv_cache_dtype=%d)\n"
            "r = e.generate(c['input_ids'], c['mask'], max_new_tokens=c['T'], pad_token_id=m['pad_token_id'], forced_tokens=c['gen'], want_logits=True)\n"
            "f = e.generate(c['input_ids'], c['mask'], max_new_tokens=c['T'], pad_token_id=m['pad_token_id'])\n"
            "torch.save(dict(logits=r.logits.cpu(), ids=f.output_ids.cpu()), %r); e.close(); print('NO_FUSION_OK')\n"
            ) % (ROOT, HERE, kv8, str(out))
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, B200_NO_ROPE_FUSION="1"))
    assert res.returncode == 0 and "NO_FUSION_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]
    eng = engines(c, kv_cache_dtype=kv8)
    r = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=m["pad_token_id"], forced_tokens=c["gen"],
                     want_logits=True)
    f = eng.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=m["pad_token_id"])
    want = torch.load(out)
    assert torch.equal(r.logits.cpu().view(torch.int16), want["logits"].view(torch.int16))
    assert torch.equal(f.output_ids.cpu(), want["ids"])
    if kv8 == 0:
        assert torch.equal(f.output_ids[:, c["S"]:].cpu(), c["gen"])


def _run_until_done(e, slots, max_iters=400):
    for _ in range(max_iters):
        n_gen, fin, stop = e.cb_poll()
        if all(fin[s] for s in slots):
            return n_gen
        e.cb_step(1)
    raise AssertionError("sequences did not finish")


def test_continuous_batching_chunked_prefill_and_prefix_reuse(engines):
    """two rows start, two join the running batch; 300-token prompts go through 128-token chunks with the prefix cache on
    (row 2 shares row 0's first two blocks).  Every step of the fixture is decisive: ids equal the oracle's."""
    c = load_case("tiny_qwen3_peaked")
    e = engines(c)
    T = c["T"]
    rows = [r.tolist() for r in c["input_ids"]]
    e.cb_begin(c["meta"]["pad_token_id"], [])
    e.cb_config(128, True)
    try:
        slots = e.cb_admit(rows[:2], [T, T])
        e.cb_step(8)
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


def test_preempt_to_host_and_resume_bit_identical(engines):
    """a running sequence swapped out to host memory (its pages reused by others) and back continues with its ids"""
    c = load_case("tiny_qwen3_peaked")
    e = engines(c)
    T = c["T"]
    rows = [r.tolist() for r in c["input_ids"]]
    e.cb_begin(c["meta"]["pad_token_id"], [])
    e.cb_config(0, False)
    try:
        a = e.cb_admit([rows[0]], [T])[0]
        e.cb_step(4)
        e.cb_swap_out(a)
        others = e.cb_admit(rows[1:], [T, T, T])
        e.cb_step(5)
        e.cb_swap_in(a)
        assert e.cb_stats()["swap_ins"] == 1
        _run_until_done(e, [a] + others)
        assert e.cb_read(a, 0, T) == c["gen"][0].tolist()
        for i, s in enumerate(others):
            assert e.cb_read(s, 0, T) == c["gen"][i + 1].tolist()
        for s in [a] + others:
            e.cb_release(s)
    finally:
        e.cb_end()


def test_fp8_engine_bit_identical_to_bf16_engine_on_w_prime():
    """tiny_qwen3_fp8's weights: e4m3 projections with channel scales (bf16 q / k norms, tied head) against a bf16 engine
    loaded with W' = dequant(codes, scales)"""
    from test_fp8_gpu import assert_same_generation, engine_pair
    from oracle import weights as W
    assert W.CONFIGS["tiny_qwen3_fp8"]["_fp8"] == "channel"
    cfg, e8, e16 = engine_pair("tiny_qwen3", 0, max_batch=32, max_seq_len=256)
    try:
        for B in (2, 24):
            assert_same_generation(e8, e16, cfg, B, 50, 8)
    finally:
        e8.close()
        e16.close()


@pytest.mark.parametrize("drop, add, match", [
    ("model.layers.1.self_attn.k_norm.weight", None, "model.layers.1.self_attn.k_norm.weight"),
    ("model.layers.0.self_attn.q_norm.weight", None, "model.layers.0.self_attn.q_norm.weight"),
    (None, "model.layers.0.self_attn.q_proj.bias", "biases together with q/k norm"),
])
def test_partial_norm_set_and_norms_with_biases_are_refused_at_finalize(drop, add, match):
    from oracle import weights as W
    from kserve_b200 import _lib as L
    from kserve_b200.engine import B200Engine
    cfg = W.CONFIGS["tiny_qwen3_g4"]
    eng = B200Engine(cfg, max_batch=2, max_seq_len=256)

    def tensors():
        for n, t in W.iter_state_dict(cfg, 0):
            if n != drop:
                yield n, t
        if add:
            yield add, torch.zeros(cfg["num_attention_heads"] * 128, dtype=torch.bfloat16)
    try:
        with pytest.raises(L.B200Error, match=match):
            eng.load_weights(tensors())
    finally:
        eng.close()


def test_served_from_a_qwen3_checkpoint_directory(tmp_path):
    """B200GenerativeModel.load() from a directory holding a Qwen3 config.json (tied embeddings, the fields of real Qwen3
    configs) and a safetensors file without lm_head.weight; /openai/v1/completions returns the fixture's ids"""
    from fastapi.testclient import TestClient
    from safetensors.torch import save_file
    from oracle import weights as W
    from kserve_b200.generative_model import B200GenerativeModel
    from kserve_b200.kserve_api import ModelServer
    c = load_case("tiny_qwen3_ids")
    m = c["meta"]
    cfg = W.CONFIGS[m["cfg"]]
    hf = dict(W.hf_config_dict(cfg), architectures=["Qwen3ForCausalLM"], model_type="qwen3", use_sliding_window=False,
              sliding_window=None, max_window_layers=28, tie_word_embeddings=True, torch_dtype="bfloat16", attention_bias=False,
              hidden_act="silu", eos_token_id=None, layer_types=["full_attention"] * cfg["num_hidden_layers"])
    with open(tmp_path / "config.json", "w") as f:
        json.dump(hf, f)
    sd = dict(W.iter_state_dict(cfg, m["seed"]))
    assert "lm_head.weight" not in sd and "model.layers.0.self_attn.q_norm.weight" in sd
    save_file(sd, str(tmp_path / "model.safetensors"))
    model = B200GenerativeModel("qwen3", str(tmp_path), pad_token_id=m["pad_token_id"], max_model_len=512, max_batch=4)
    assert model.load() and model.max_length == 512
    try:
        with TestClient(ModelServer().create_application([model])) as client:
            r = client.post("/openai/v1/completions", json={"model": "qwen3", "prompt": c["input_ids"].tolist(),
                                                            "max_tokens": m["max_tokens"], "temperature": 0})
            assert r.status_code == 200, r.text
            j = r.json()
            tol = logits_tol(c["step_logits"])
            for b, ch in enumerate(j["choices"]):
                got = [int(t) for t in ch["text"].split()]
                neq = [i for i, (x, y) in enumerate(zip(got, c["gen"][b].tolist())) if x != y]
                assert len(got) == m["max_tokens"]
                assert not neq or float(c["margin"][b, neq[0]]) <= 2 * tol, f"row {b}"
    finally:
        model.stop()


# ---- Qwen3-8B layer shapes --------------------------------------------------------------------------------------------
@pytest.mark.slow
@pytest.mark.parametrize("name", ["qwen3_8b_2l_b4", "qwen3_8b_2l_peaked_b4"])
def test_qwen3_8b_shapes_1024_prompt_tokens(name):
    """Qwen3-8B layer shapes (2 layers, 32 / 8 heads, I = 12288, V = 151936): 4 x 1024-token prompts, 16 decode steps.
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
def test_tp2_qwen3_matches_oracle_fixture():
    """TP = 2: each rank holds half of the q / k / v heads and the full (replicated) q / k norm weights"""
    names = ["tiny_qwen3_g4_ids", "tiny_qwen3_wide_ids"]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29643", os.path.join(HERE, "tp_worker.py"), ",".join(names)]
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
