"""The attention kernels as the engine runs them, against plain fp32 attention computed with torch on the same device.

- attn_prefill_tc_kernel (the engine's prefill attention), with and without kv_off (chunked prefill / prefix reuse),
  through b200_op_attn_prefill_tc_off on a q buffer of exactly T rows (as the engine's q at T = cap_T);
- attn_decode_kernel with RoPE and the KV append fused, from bf16 q|k|v rows or fp32 split-K partials plus the Qwen2
  bias, with the split merge folded into the last-arriving CTA or done by attn_combine_kernel, through
  b200_op_attn_decode_fused (the parameters engine.cu sets for the decode step);
at GQA groups 1-8, ragged batches, page and query-tile boundaries, contexts up to 32768, stale or poisoned memory outside
the contexts, and softmax inputs whose scores span about +-40.

Tolerance of the fp32 comparisons, per element: the kernels round every p to bf16 before P.V (relative error <= 2^-8
each) and the output to bf16 (<= 2^-8 of |O|); scores, softmax statistics and accumulators are fp32.  So
|O - O_ref| <= 2^-8 (P |V|) + 2^-8 |O_ref| up to fp32 rounding; the checks allow 1.25x that.  One key wrongly in or out
of the softmax moves O by only ~|v| / L, which this bound cannot see at long contexts, so masks and page boundaries are
held to bit-exact checks instead: perturbing keys a row must not see changes no bit of it, and poisoning every KV slot,
page-table entry and split partial outside the contexts with NaN or 0x7F7F changes no bit of any output.
"""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
SCALE = 1.0 / math.sqrt(128)
STALE = ("nan", "7f7f")       # 0x7F7F (3.4e38) is the pattern b200_kv_swap_out(scrub=1) leaves in a page
# (nh, nkv) at every group size the decode kernel supports; 28/4, 12/2, 40/8 and 64/8 are Qwen2-7B, Qwen2.5-3B,
# Qwen2.5-14B and Llama-3-70B / Qwen2-72B
HEADS = [(8, 8), (16, 8), (12, 4), (32, 8), (40, 8), (12, 2), (28, 4), (64, 8)]
PREFILL_HEADS = [hp for hp in HEADS if hp != (12, 4)]     # G in {1, 2, 4, 5, 6, 7, 8}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _check(lib, rc, what):
    assert rc == 0, f"{what}: {lib.b200_last_error().decode()}"


def _randn(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(torch.bfloat16)


def _fill(kind, shape, dtype=torch.bfloat16):
    """zero, NaN or the 0x7F7F bit pattern (bf16 3.39e38; for fp32 buffers the 0x7F7F7F7F pattern, 3.39e38 too)"""
    if kind == "zero":
        return torch.zeros(shape, dtype=dtype, device=DEV)
    if kind == "nan":
        return torch.full(shape, float("nan"), dtype=dtype, device=DEV)
    if dtype == torch.bfloat16:
        return torch.full(shape, 0x7F7F, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    return torch.full(shape, 0x7F7F7F7F, dtype=torch.int32, device=DEV).view(torch.float32)


class Paged:
    """K / V of B sequences (ks[b], vs[b]: [nkv][n_b][128]) in paged caches [num_pages][nkv][64][128] with shuffled page
    ids.  Sequence b owns ceil(alloc[b] / 64) pages; its page-table row lists two more pages that nobody owns.  Every slot
    that holds no key of a sequence (the tail of its last page, the unowned pages) holds `stale`."""

    def __init__(self, ks, vs, stale="zero", seed=0, alloc=None):
        B, nkv = len(ks), ks[0].shape[0]
        alloc = alloc or [k.shape[1] for k in ks]
        npg = [max(1, (a + 63) // 64) for a in alloc]
        self.max_pages = max(npg) + 2
        self.num_pages = B * self.max_pages + 3
        perm = torch.randperm(self.num_pages, generator=torch.Generator().manual_seed(seed))
        self.pt = perm[:B * self.max_pages].view(B, self.max_pages).to(torch.int32).to(DEV)
        self.kc = _fill(stale, (self.num_pages, nkv, 64, 128))
        self.vc = _fill(stale, (self.num_pages, nkv, 64, 128))
        for b in range(B):
            for src, dst in ((ks[b], self.kc), (vs[b], self.vc)):
                n = src.shape[1]
                full = torch.cat([src, _fill(stale, (nkv, npg[b] * 64 - n, 128))], 1)
                dst[self.pt[b, :npg[b]].long()] = full.view(nkv, npg[b], 64, 128).transpose(0, 1)

    def slot(self, b, pos):
        return int(self.pt[b, pos // 64]), pos % 64


def _ref(q, k, v, qpos):
    """q [nh][n][128], k / v [nkv][L][128] (bf16); query i sees keys 0 .. qpos[i].
    -> fp32 (O, P|V|), each [n][nh * 128]"""
    nh, n, _ = q.shape
    G = nh // k.shape[0]
    masked = torch.arange(k.shape[1], device=DEV)[None, :] > qpos[:, None]
    out, pv = [], []
    for h in range(nh):
        kf, vf = k[h // G].float(), v[h // G].float()
        s = (q[h].float() @ kf.T) * SCALE
        p = torch.softmax(s.masked_fill(masked, float("-inf")), -1)
        out.append(p @ vf)
        pv.append(p @ vf.abs())
    return torch.stack(out, 1).reshape(n, nh * 128), torch.stack(pv, 1).reshape(n, nh * 128)


def _close(what, got, ref, pv):
    got = got.float()
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output"
    err = (got - ref).abs()
    tol = 1.25 * 2.0 ** -8 * (pv + ref.abs()) + 1e-6
    bad = err > tol
    if bad.any():
        i = int((err / tol).flatten().argmax())
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements out of tolerance; worst at flat index {i}: "
                             f"ref {float(ref.flatten()[i]):.6f} got {float(got.flatten()[i]):.6f} tol {float(tol.flatten()[i]):.2e}")


def _same(what, got, want):
    assert bool(torch.isfinite(got.float()).all()), f"{what}: non-finite output"
    if not torch.equal(got.view(torch.int16), want.view(torch.int16)):
        d = (got.view(torch.int16) != want.view(torch.int16)).nonzero()
        raise AssertionError(f"{what}: {len(d)} elements differ from the reference run, first at {d[0].tolist()}")


# ---------------------------------------------------------------------------------------------------------------- prefill
def _prefill(lib, q, paged, lens, offs, nh, nkv):
    """the wgmma prefill attention on packed q [T][nh*128] (exactly T rows); offs = kv_off per sequence or None"""
    B = len(lens)
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    slot = torch.arange(B, dtype=torch.int32, device=DEV)
    off = torch.tensor(offs, dtype=torch.int32, device=DEV) if offs is not None else None
    out = torch.full((q.shape[0], nh * 128), float("nan"), dtype=torch.bfloat16, device=DEV)
    _check(lib, lib.b200_op_attn_prefill_tc_off(_ptr(q), nh * 128, q.shape[0], _ptr(out), nh * 128, _ptr(paged.kc), _ptr(paged.vc),
                                                paged.num_pages, _ptr(paged.pt), paged.max_pages, _ptr(cu), _ptr(slot), _ptr(off),
                                                B, max(lens), nh, nkv, None), "attn_prefill_tc_off")
    torch.cuda.synchronize()
    return out


def _prefill_inputs(nh, nkv, lens, offs, seed, kscale=1.0):
    offs = offs or [0] * len(lens)
    ks = [_randn((nkv, o + l, 128), seed + 2 * b, kscale) for b, (l, o) in enumerate(zip(lens, offs))]
    vs = [_randn((nkv, o + l, 128), seed + 2 * b + 1) for b, (l, o) in enumerate(zip(lens, offs))]
    q = _randn((sum(lens), nh * 128), seed + 1000)
    return ks, vs, q


def _prefill_vs_ref(name, out, q, ks, vs, lens, offs, nh, rows_cap=None):
    offs = offs or [0] * len(lens)
    t0 = 0
    for b, (l, o) in enumerate(zip(lens, offs)):
        rows = torch.arange(l, device=DEV)
        if rows_cap and l > rows_cap:          # long sequences: every k-th row plus the last tile (the reference is O(L^2))
            rows = torch.unique(torch.cat([rows[::l // rows_cap], rows[-130:]]))
        qb = q[t0:t0 + l][rows].view(len(rows), nh, 128).transpose(0, 1)
        ref, pv = _ref(qb, ks[b], vs[b], rows + o)
        _close(f"{name} seq {b} len {l} kv_off {o}", out[t0:t0 + l][rows], ref, pv)
        t0 += l


def _prefill_all_fills(lib, name, q, ks, vs, lens, offs, nh, nkv, seed):
    """zero-filled run, then NaN / 0x7F7F in every slot outside the contexts: bit-identical, finite"""
    base = _prefill(lib, q, Paged(ks, vs, "zero", seed), lens, offs, nh, nkv)
    for kind in STALE:
        _same(f"{name} stale={kind}", _prefill(lib, q, Paged(ks, vs, kind, seed), lens, offs, nh, nkv), base)
    return base


@pytest.mark.parametrize("nh,nkv", PREFILL_HEADS)
@pytest.mark.parametrize("with_off", [False, True])
def test_prefill_ragged_vs_fp32(lib, nh, nkv, with_off):
    lens = [1, 127, 128, 129, 200, 63]
    offs = [4096, 128, 1024, 0, 128, 1024] if with_off else None
    ks, vs, q = _prefill_inputs(nh, nkv, lens, offs, seed=nh * 31 + nkv)
    out = _prefill_all_fills(lib, "prefill", q, ks, vs, lens, offs, nh, nkv, seed=5)
    _prefill_vs_ref("prefill", out, q, ks, vs, lens, offs, nh)


@pytest.mark.parametrize("L,off", [(8192, 0), (3969, 4096)])
def test_prefill_long_vs_fp32(lib, L, off):
    nh, nkv = 28, 4
    offs = [off] if off else None
    ks, vs, q = _prefill_inputs(nh, nkv, [L], offs, seed=77)
    out = _prefill_all_fills(lib, "prefill long", q, ks, vs, [L], offs, nh, nkv, seed=6)
    _prefill_vs_ref("prefill long", out, q, ks, vs, [L], offs, nh, rows_cap=512)


@pytest.mark.parametrize("off", [0, 1024])
def test_prefill_causality_and_page_boundaries_exact(lib, off):
    """Keys at positions >= P are perturbed by a large amount: every row at a position < P keeps every bit, the row at P
    changes (key P is visible to query P), and the other sequence of the batch keeps every bit."""
    nh, nkv, L = 8, 2, 300
    lens, offs = [L, 129], ([off, 128] if off else None)
    ks, vs, q = _prefill_inputs(nh, nkv, lens, offs, seed=3)
    base = _prefill(lib, q, Paged(ks, vs, "zero", 9), lens, offs, nh, nkv)
    cuts = [off + p for p in (1, 63, 64, 65, 127, 128, 129, L - 1)] + ([0, off - 1] if off else [])
    for P in cuts:
        k2, v2 = [k.clone() for k in ks], [v.clone() for v in vs]
        k2[0][:, P:] += 4.0
        v2[0][:, P:] += 16.0
        got = _prefill(lib, q, Paged(k2, v2, "zero", 9), lens, offs, nh, nkv)
        first = max(P - off, 0)                  # chunk row of the first query that sees a perturbed key
        _same(f"rows before position {P}", got[:first], base[:first])
        assert not torch.equal(got[first], base[first]), f"row at position {off + first} does not see key {P}"
        _same(f"other sequence (cut {P})", got[L:], base[L:])


@pytest.mark.parametrize("hot", ["first", "last"])
@pytest.mark.parametrize("off", [0, 1024])
def test_prefill_peaked_softmax(lib, hot, off):
    """Scores spanning about +-40: one key per kv head scores +40 and one -40 against every query, the rest ~N(0, 2.5^2).
    With the hot key in the first KV tile every later tile is exp(-30) small; in the last tile it arrives after the
    running maximum settled near 10, so a missing or misapplied online-softmax rescale is off by O(1)."""
    nh, nkv, L = 28, 4, 300
    offs = [off] if off else None
    ks, vs, _ = _prefill_inputs(nh, nkv, [L], offs, seed=41, kscale=2.5)
    G = nh // nkv
    u = _randn((nkv, 128), 42)                                   # every query row of kv group g is u[g]
    q = u.repeat_interleave(G, 0).reshape(1, nh * 128).repeat(L, 1).contiguous()
    uf = u.float()
    hot_pos = 3 if hot == "first" else off + L - 5
    cold_pos = off + L // 2
    for pos, target in ((hot_pos, 40.0), (cold_pos, -40.0)):
        ks[0][:, pos] = (uf * (target / SCALE / (uf * uf).sum(-1, keepdim=True))).to(torch.bfloat16)
    out = _prefill_all_fills(lib, "peaked prefill", q, ks, vs, [L], offs, nh, nkv, seed=7)
    _prefill_vs_ref("peaked prefill", out, q, ks, vs, [L], offs, nh)


# ----------------------------------------------------------------------------------------------------------------- decode
DEC_CTX = [1, 63, 64, 65, 1000, 4097, 32768]
QKV_SPLITS = 3


class DecodeCase:
    """B sequences at contexts `ctxs`: the cache holds keys 0 .. ctx-2, the current token (position ctx-1) arrives as its raw
    q|k|v projection row.  The raw rows are multiples of 2^-10 below 8 in magnitude, given either as bf16 rows or as
    QKV_SPLITS fp32 partials on that grid, and the bias too: every fp32 sum is exact in any order, so bf16(sum + bias)
    has exactly one correct value."""

    def __init__(self, nh, nkv, ctxs, seed, kscale=1.0):
        self.nh, self.nkv, self.G, self.ctxs, self.B = nh, nkv, nh // nkv, ctxs, len(ctxs)
        self.cols = (nh + 2 * nkv) * 128
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.ks = [_randn((nkv, c - 1, 128), seed + 2 * b, kscale) for b, c in enumerate(ctxs)]
        self.vs = [_randn((nkv, c - 1, 128), seed + 2 * b + 1) for b, c in enumerate(ctxs)]
        ld_p = self.cols + 8
        self.partial = torch.zeros((QKV_SPLITS, self.B + 1, ld_p), dtype=torch.float32, device=DEV)   # row B: padding
        self.partial[:, :self.B, :self.cols] = torch.randint(-2048, 2048, (QKV_SPLITS, self.B, self.cols), generator=g,
                                                             device=DEV).float() * 2.0 ** -10
        self.ld_partial, self.split_stride = ld_p, (self.B + 1) * ld_p
        self.bias = (torch.randint(-128, 128, (self.cols,), generator=g, device=DEV).float() * 2.0 ** -10).to(torch.bfloat16)
        from kserve_b200.engine import hf_rope_tables
        cos, sin = hf_rope_tables(500000.0, 128, max(ctxs) + 64)
        self.cos, self.sin = cos.to(DEV).contiguous(), sin.to(DEV).contiguous()
        self.pos = torch.tensor([c - 1 for c in ctxs], dtype=torch.int32, device=DEV)

    def raw(self, bias):
        s = self.partial[:, :self.B, :self.cols].double().sum(0)
        if bias:
            s = s + self.bias.double()
        return s.to(torch.bfloat16)                                # [B][cols]

    def roped(self, raw):
        """HF apply_rotary_pos_emb in bf16 arithmetic (every op rounds) -> q [B][nh][128], k [B][nkv][128], v"""
        nh, nkv, B = self.nh, self.nkv, self.B
        c = torch.cat([self.cos, self.cos], -1)[self.pos.long()][:, None, :]
        s = torch.cat([self.sin, self.sin], -1)[self.pos.long()][:, None, :]

        def rot(x):
            return torch.cat((-x[..., 64:], x[..., :64]), -1)
        qh = raw[:, :nh * 128].view(B, nh, 128)
        kh = raw[:, nh * 128:(nh + nkv) * 128].view(B, nkv, 128)
        vh = raw[:, (nh + nkv) * 128:].view(B, nkv, 128)
        return qh * c + rot(qh) * s, kh * c + rot(kh) * s, vh

    def run(self, lib, paged, mode, splits, fold, part_fill="zero", reps=1):
        """mode: 'bf16' (q|k|v rows, no bias: the GEMM epilogue adds it), 'partial', 'partial+bias'"""
        B, nh, nkv, G = self.B, self.nh, self.nkv, self.G
        out = torch.full((B, nh * 128), float("nan"), dtype=torch.bfloat16, device=DEV)
        cnt = torch.zeros(B * nkv, dtype=torch.int32, device=DEV) if fold else None
        if mode == "bf16":
            qkv = torch.zeros((B, self.cols + 64), dtype=torch.bfloat16, device=DEV)
            qkv[:, :self.cols] = self.raw(False)
            args = (_ptr(qkv), qkv.shape[1], None, 0, 0, 0, None)
        else:
            args = (None, 0, _ptr(self.partial), QKV_SPLITS, self.split_stride, self.ld_partial,
                    _ptr(self.bias) if mode == "partial+bias" else None)
        slot = torch.arange(B, dtype=torch.int32, device=DEV)
        outs = []
        for _ in range(reps):
            po = _fill(part_fill, (B * nkv * splits * G * 128,), torch.float32)
            pml = _fill(part_fill, (B * nkv * splits * G * 2,), torch.float32)
            _check(lib, lib.b200_op_attn_decode_fused(*args, _ptr(self.cos), _ptr(self.sin), _ptr(out), nh * 128,
                                                      _ptr(paged.kc), _ptr(paged.vc), _ptr(paged.pt), paged.max_pages,
                                                      _ptr(slot), _ptr(self.pos), B, nh, nkv, splits, _ptr(po), _ptr(pml),
                                                      _ptr(cnt), None), "attn_decode_fused")
            torch.cuda.synchronize()
            outs.append(out.clone())
            if cnt is not None:
                assert int(cnt.abs().sum()) == 0, "split arrival counters must be back to zero after the launch"
        return outs

    def paged(self, stale, seed=11):
        return Paged(self.ks, self.vs, stale, seed, alloc=self.ctxs)

    def check(self, name, paged, out, raw):
        q, k, v = self.roped(raw)
        for b, c in enumerate(self.ctxs):
            page, s = paged.slot(b, c - 1)
            assert torch.equal(paged.kc[page, :, s], k[b]), f"{name}: appended k of sequence {b} is not HF RoPE in bf16"
            assert torch.equal(paged.vc[page, :, s], v[b]), f"{name}: appended v of sequence {b}"
            kk = torch.cat([self.ks[b], k[b][:, None]], 1)
            vv = torch.cat([self.vs[b], v[b][:, None]], 1)
            ref, pv = _ref(q[b][:, None], kk, vv, torch.tensor([c - 1], device=DEV))
            _close(f"{name} seq {b} ctx {c}", out[b:b + 1], ref, pv)


MODES = ["bf16", "partial", "partial+bias"]


def _merges(splits):
    return [True, False] if splits > 1 else [True]


@pytest.mark.parametrize("splits", [1, 2, 5, 8])
@pytest.mark.parametrize("nh,nkv", HEADS)
def test_decode_fused_vs_fp32(lib, nh, nkv, splits):
    """Every input mode and both merges at every context of DEC_CTX in one ragged batch (8 splits over a 1-tile context
    leaves 7 splits empty); NaN or 0x7F7F in the KV slots outside the contexts, or in the split partials, instead of
    zeros: bit-identical; a second launch
    gives the same bits (the merge is deterministic)."""
    dc = DecodeCase(nh, nkv, DEC_CTX, seed=nh * 13 + nkv + splits)
    for mode in MODES:
        for fold in _merges(splits):
            name = f"decode G{dc.G} splits {splits} {mode} {'folded' if fold else 'combine kernel'}"
            paged = dc.paged("zero")
            base, again = dc.run(lib, paged, mode, splits, fold, reps=2)
            _same(f"{name}: second launch", again, base)
            dc.check(name, paged, base, dc.raw(mode == "partial+bias"))
            for kind in STALE:     # the KV slots outside the contexts, and separately the split partials
                got, = dc.run(lib, dc.paged(kind), mode, splits, fold)
                _same(f"{name} stale KV={kind}", got, base)
                got, = dc.run(lib, dc.paged("zero"), mode, splits, fold, part_fill=kind)
                _same(f"{name} split partials={kind}", got, base)


def test_decode_current_token_and_position_zero_are_visible(lib):
    """Exactness of the decode mask from the visible side (keys past the context are the stale tests): changing the
    current token's k / v (it comes through the q|k|v row, not the cache) or key 0 changes the output."""
    dc = DecodeCase(28, 4, [1, 64, 65, 1000], seed=5)
    base, = dc.run(lib, dc.paged("zero"), "partial", 5, True)
    for what in ("k", "v"):
        col = (dc.nh + (0 if what == "k" else dc.nkv)) * 128
        dc.partial[0, :dc.B, col:col + dc.nkv * 128] += 1.0
        got, = dc.run(lib, dc.paged("zero"), "partial", 5, True)
        dc.partial[0, :dc.B, col:col + dc.nkv * 128] -= 1.0
        for b in range(0 if what == "v" else 1, dc.B):   # (a softmax over one key does not depend on that key)
            assert not torch.equal(got[b], base[b]), f"current token's {what} is not visible to sequence {b}"
    for b in range(1, dc.B):
        dc.ks[b][:, 0] += 4.0
        dc.vs[b][:, 0] += 16.0
    got, = dc.run(lib, dc.paged("zero"), "partial", 5, True)
    for b in range(1, dc.B):
        assert not torch.equal(got[b], base[b]), f"key 0 is not visible to sequence {b}"
    _same("sequence 0 (context 1: key 0 is the current token)", got[:1], base[:1])


@pytest.mark.parametrize("hot", ["first", "last"])
@pytest.mark.parametrize("splits,fold", [(1, True), (5, True), (5, False)])
def test_decode_peaked_softmax(lib, hot, splits, fold):
    """Scores spanning about +-40 (see test_prefill_peaked_softmax): the +40 key sits in the first KV tile, or in the last
    tile just before the current token — after the other splits' and warps' maxima settled near 10."""
    nh, nkv = 32, 8
    dc = DecodeCase(nh, nkv, [1000, 4097], seed=8, kscale=2.5)
    G = dc.G
    for s in range(QKV_SPLITS):      # the G query heads of a group share one raw row, so one key is hot for all of them
        qv = dc.partial[s, :dc.B, :nh * 128].view(dc.B, nkv, G, 128)
        qv[:] = qv[:, :, :1].clone()
    q, _, _ = dc.roped(dc.raw(False))
    for b, c in enumerate(dc.ctxs):
        u = q[b].view(nkv, G, 128)[:, 0].float()
        hot_pos = 3 if hot == "first" else c - 3
        for pos, target in ((hot_pos, 40.0), (c // 2, -40.0)):
            dc.ks[b][:, pos] = (u * (target / SCALE / (u * u).sum(-1, keepdim=True))).to(torch.bfloat16)
    paged = dc.paged("zero")
    base, = dc.run(lib, paged, "bf16", splits, fold)
    dc.check(f"peaked decode ({hot})", paged, base, dc.raw(False))
    for kind in STALE:
        got, = dc.run(lib, dc.paged(kind), "bf16", splits, fold, part_fill=kind)
        _same(f"peaked decode stale={kind}", got, base)
