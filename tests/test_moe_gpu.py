"""The sparse MoE block (Mixtral) as the engine launches it, through b200_op_moe_block, against a plain fp32 torch
reference with the rounding points of transformers' MixtralTopKRouter / MixtralExperts.forward:

  router : logits = bf16(xn wr^T), p = softmax(logits) in fp32, top-2 (the lowest index wins ties), w = p / (p_a + p_b)
  experts: g, u = bf16(x gate^T), bf16(x up^T);  h = bf16(bf16(silu(g)) u);  y = bf16(h down^T)
  combine: c = bf16(bf16(y_a w_a) + bf16(y_b w_b)) in ascending expert order;  x' = bf16(x + c);  xn' = RMSNorm(x')

Every stage is checked against the reference applied to the kernels' own output of the stage before, so each tolerance
covers one rounding step (RTOL = 2^-7 as in test_kernels_gpu.py; fp32 split-K partial sums at 1e-3).  SwiGLU's h has
three roundings, so it is held to the bracket of those roundings instead (see swiglu_bracket) and must equal the
reference itself almost everywhere.  The rest is exact:
- routing: with wr[e] = one-hot(e) the logits are xn[:, :E] exactly, so any routing (ties included) is chosen by setting
  those bf16 values; the tables must equal the reference (weights within 2 fp32 ulps), and prefill and decode routers
  must produce bit-identical tables;
- x and ysum are bit-exact given the kernels' expert outputs and weights, and split-K partials are summed in split order
  exactly as the combine does;
- every row of xg / hg / yg (and of the partials) outside the expert segments is NaN before the call: the outputs must be
  finite and bit-identical to a run on zero-filled buffers, and those rows must still hold their NaN afterwards;
- a second call on the same buffers with different routing equals a call on fresh buffers.

Shapes (H, I, E): the two fixture models, Mixtral-8x7B's shard at TP = 4 (4096, 3584, 8), the whole of Mixtral on one GPU
(4096, 14336, 8; slow: there the per-expert gate/up runs stream-K), and E = 16 and E = 2.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

torch.backends.cuda.matmul.allow_tf32 = False

DEV = "cuda"
RTOL = 2.0 ** -7
EPS = 1e-5
PREFILL, GROUPED, PER_EXPERT = 0, 1, 2
NAN16 = 0x7FC0   # torch's bf16 NaN

# (H, I, E), named by their role in the test ids
SHAPES = {"small": (512, 1024, 4), "moe8": (1024, 1536, 8), "mixtral_tp4": (4096, 3584, 8), "e16": (1024, 512, 16),
          "e2": (1024, 512, 2), "mixtral": (4096, 14336, 8)}
SMALL, MOE8, TP4, E16, E2, FULL = SHAPES


# ---------------------------------------------------------------------------------------------- reference
def interleave16(gate, up):
    """[.., I, H] gate and up -> [.., 2I, H] in the engine's 16-row interleave (rows 32j.. gate, 32j+16.. up)"""
    *lead, I, H = gate.shape
    return torch.stack([gate.reshape(*lead, I // 16, 16, H), up.reshape(*lead, I // 16, 16, H)], -3).reshape(*lead, 2 * I, H)


def bf(t):
    return t.to(torch.bfloat16).float()


def route_ref(logits):
    """fp32 softmax of bf16 logits [T][E], top-2 with the lowest index winning ties, renormalised fp32 weights.
    The softmax is exp(l - max) / sum with the sum taken in expert order: torch.softmax sums in another order, and its
    weights differ from these by up to 3 fp32 ulps (a bf16 rounding of y * w hardly ever sees that; the CPU test below
    holds this reference to HF's block)."""
    lf = logits.float()
    ex = torch.exp(lf - lf.max(-1, keepdim=True).values)
    tot = torch.zeros_like(ex[:, 0])
    for e in range(ex.shape[1]):
        tot = tot + ex[:, e]
    p = ex / tot[:, None]
    i0 = torch.argmax(logits, -1)                            # first maximum
    masked = logits.float().clone()
    masked.scatter_(1, i0[:, None], float("-inf"))
    i1 = torch.argmax(masked, -1)
    idx = torch.stack([i0, i1], 1)
    top = p.gather(1, idx)
    return idx.to(torch.int32), top / (top[:, 0] + top[:, 1])[:, None]


def tables_ref(tok_expert, E):
    """count [E], off [E + 1] (8-row aligned exclusive scan) and tok_row [T][2] (token order within a segment)"""
    flat = tok_expert.flatten().long()
    count = torch.bincount(flat, minlength=E)
    off = torch.zeros(E + 1, dtype=torch.long, device=flat.device)
    off[1:] = torch.cumsum((count + 7) // 8 * 8, 0)
    order = torch.sort(flat, stable=True).indices
    start = torch.zeros(E, dtype=torch.long, device=flat.device)
    start[1:] = torch.cumsum(count, 0)[:-1]
    rank = torch.arange(flat.numel(), device=flat.device) - start[flat[order]]
    tok_row = torch.empty_like(flat)
    tok_row[order] = off[flat[order]] + rank
    return count.to(torch.int32), off.to(torch.int32), tok_row.view(-1, 2).to(torch.int32)


def swiglu_ref(x, gate, up):
    g, u = bf(x.float() @ gate.float().T), bf(x.float() @ up.float().T)
    return bf(bf(F.silu(g)) * u)


def bf16_floor_ceil(v):
    """the bf16 values just below and just above each finite fp32 value (both v when v is a bf16): a bf16 is an fp32
    whose low 16 bits are zero, so truncating them rounds the magnitude down and adding 1 << 16 to that rounds it up"""
    vi = v.contiguous().view(torch.int32)
    t = vi & -65536
    tf, mf = t.view(torch.float32), (t + 65536).view(torch.float32)
    exact, pos = (vi & 65535) == 0, v > 0
    return torch.where(exact, v, torch.where(pos, tf, mf)), torch.where(exact, v, torch.where(pos, mf, tf))


def swiglu_bracket(x, gate, up):
    """[lo, hi] of h = bf16(bf16(silu(g)) u) over the values fp32 sums in another order can give: g and u anywhere within
    2^-18 of their terms' absolute sum (the accumulation-order error, which near a cancellation is several bf16 ulps of a
    small g), each rounded either way, and silu(g) within 2^-18 of itself (the kernels' fast SiLU) rounded either way.
    Two flipped roundings already move h by 2 - 3 ulps, more than a tolerance of one rounding step allows."""
    xf = x.float()

    def ends(w):
        v, d = xf @ w.float().T, (xf.abs() @ w.float().abs().T) * 2.0 ** -18
        return bf16_floor_ceil(v - d)[0], bf16_floor_ceil(v + d)[1]

    gs, us = ends(gate), ends(up)
    lo = hi = None
    for g in gs:
        sl = F.silu(g)
        for sv in (bf16_floor_ceil(sl - sl.abs() * 2.0 ** -18)[0], bf16_floor_ceil(sl + sl.abs() * 2.0 ** -18)[1]):
            for u in us:
                h = bf(sv * u)
                lo = h if lo is None else torch.minimum(lo, h)
                hi = h if hi is None else torch.maximum(hi, h)
    return lo, hi


def combine_ref(ya, yb, wa, wb):
    """ya / yb: bf16 expert outputs of the lower / higher expert index, wa / wb their fp32 weights -> bf16 c"""
    return bf(bf(ya.float() * wa[:, None]) + bf(yb.float() * wb[:, None]))


def rmsnorm_ref(x, w, eps):
    xf = x.float()
    var = xf.pow(2).mean(-1, keepdim=True)
    return w.float() * bf(xf * torch.rsqrt(var + eps))


def moe_ref(xn, wr, gate, up, down):
    """The whole block's reference, everything computed from the inputs: (tok_expert, tok_weight, c)"""
    te, tw = route_ref(bf(xn.float() @ wr.float().T))
    T, H = xn.shape
    y = torch.zeros(T, 2, H, dtype=torch.float32, device=xn.device)
    for e in range(wr.shape[0]):
        t, k = torch.nonzero(te == e, as_tuple=True)
        if t.numel():
            y[t, k] = bf(swiglu_ref(xn[t], gate[e], up[e]) @ down[e].float().T)
    return te, tw, _combine_sorted(te, tw, y)


def _combine_sorted(te, tw, y):
    swap = te[:, 1] < te[:, 0]                                  # combine in ascending expert index
    ya = torch.where(swap[:, None], y[:, 1], y[:, 0])
    yb = torch.where(swap[:, None], y[:, 0], y[:, 1])
    wa = torch.where(swap, tw[:, 1], tw[:, 0])
    wb = torch.where(swap, tw[:, 0], tw[:, 1])
    return combine_ref(ya, yb, wa, wb)


# ---------------------------------------------------------------------------------------------- helpers
def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _cmp(name, got, ref, atol, rtol):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    bad = ~(err <= atol + rtol * ref.abs())
    assert not bad.any(), (f"{name}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {float(err.nan_to_num(1e30).max()):.5g}"
                           f" at {tuple(int(i) for i in torch.nonzero(bad)[0])}; nan={bool(torch.isnan(got).any())}")


def _same(name, got, want):
    a, b = got.contiguous().view(torch.uint8), want.contiguous().view(torch.uint8)
    assert torch.equal(a, b), f"{name}: {int((a != b).sum())} bytes differ"


def eff_splits(I, want):
    kb = (I + 63) // 64
    s = max(1, min(want, kb))
    per = (kb + s - 1) // s
    return (kb + per - 1) // per


_WEIGHTS = {}


def weights(shape, seed=0):
    """router, gate, up, down, norm weight of one MoE layer (bf16, on the GPU), outputs O(1) for O(1) inputs"""
    key = (shape, seed)
    if key not in _WEIGHTS:
        _WEIGHTS.clear()
        H, I, E = SHAPES[shape]
        g = torch.Generator(device=DEV).manual_seed(1000 + seed)
        r = lambda *s, sc: (torch.randn(*s, generator=g, device=DEV) * sc).to(torch.bfloat16)   # noqa: E731
        w = dict(wr=r(E, H, sc=H ** -0.5), gate=r(E, I, H, sc=H ** -0.5), up=r(E, I, H, sc=H ** -0.5),
                 down=r(E, H, I, sc=I ** -0.5), norm=(1 + 0.1 * torch.randn(H, generator=g, device=DEV)).to(torch.bfloat16))
        w["onehot"] = torch.eye(E, H, device=DEV).to(torch.bfloat16)
        w["wgu"] = interleave16(w["gate"], w["up"]).contiguous()
        _WEIGHTS[key] = w
    return _WEIGHTS[key]


def forced_inputs(T, H, E, pairs, seed):
    """xn, x with xn[t, :E] chosen so that the one-hot router sends token t to pairs[t] = (first, second) with random
    margins: the first pick's logit in [1, 2), the second's in [0, 1), the rest in [-2, -0.25)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    xn = torch.randn(T, H, generator=g, device=DEV)
    x = torch.randn(T, H, generator=g, device=DEV) * 2
    lg = -2 + 1.75 * torch.rand(T, E, generator=g, device=DEV)
    ar = torch.arange(T, device=DEV)
    lg[ar, pairs[:, 0]] = 1 + torch.rand(T, generator=g, device=DEV)
    lg[ar, pairs[:, 1]] = torch.rand(T, generator=g, device=DEV)
    xn[:, :E] = lg
    return xn.to(torch.bfloat16), x.to(torch.bfloat16)


def tie_inputs(T, H, E, seed):
    """logit rows with exact ties: between the first and second pick, between the second and third, and three-way"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    xn = torch.randn(T, H, generator=g, device=DEV)
    x = torch.randn(T, H, generator=g, device=DEV) * 2
    lg = -2 + 1.75 * torch.rand(T, E, generator=g, device=DEV)
    for t in range(T):
        perm = torch.randperm(E, generator=torch.Generator().manual_seed(seed * 7919 + t))
        kind = t % 3
        if kind == 0 or E == 2:                                # top two equal
            lg[t, perm[0]] = lg[t, perm[1]] = 1.0
        elif kind == 1:                                        # second and third equal
            lg[t, perm[0]] = 1.5
            lg[t, perm[1]] = lg[t, perm[2]] = 0.5
        else:                                                  # three equal
            lg[t, perm[:3]] = 0.75
    xn[:, :E] = lg
    return xn.to(torch.bfloat16), x.to(torch.bfloat16)


def make_pairs(T, E, pattern, seed):
    """expert pairs [T][2] (first pick, second pick) of a routing pattern"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    if pattern == "random":
        a = torch.randint(0, E, (T,), generator=g, device=DEV)
        b = (a + torch.randint(1, E, (T,), generator=g, device=DEV)) % E
        return torch.stack([a, b], 1)
    if pattern == "pair01":                                    # experts 2.. get nothing
        flip = torch.rand(T, generator=g, device=DEV) < 0.5
        a = flip.long()
        return torch.stack([a, 1 - a], 1)
    if pattern == "all_to_one":                                # expert E // 2 gets every token
        j = E // 2
        b = (j + torch.randint(1, E, (T,), generator=g, device=DEV)) % E
        a = torch.full((T,), j, device=DEV)
        flip = torch.rand(T, generator=g, device=DEV) < 0.5
        return torch.stack([torch.where(flip, b, a), torch.where(flip, a, b)], 1)
    if pattern.startswith("count"):                            # expert 2 gets exactly n tokens behind segments of 37 and
        n = int(pattern[5:])                                   # 50 rows (row_off 96: not a multiple of 128)
        counts = [37, 50, n]
        rest = 2 * T - sum(counts)
        assert rest >= 0 and E >= 4 and n <= T
        per = [rest // (E - 3) + (1 if i < rest % (E - 3) else 0) for i in range(E - 3)]
        counts += per
        assert max(counts) <= T
        seq = torch.cat([torch.full((c,), e, device=DEV) for e, c in enumerate(counts)])
        pairs = torch.stack([seq[:T], seq[T:]], 1)              # a run of <= T equal ids never pairs with itself
        pairs = pairs[torch.randperm(T, generator=g, device=DEV)]
        flip = torch.rand(T, generator=g, device=DEV) < 0.5
        return torch.where(flip[:, None], pairs.flip(1), pairs)
    raise ValueError(pattern)


class Bufs:
    """Every buffer b200_op_moe_block writes, filled with zeros or NaN (int tables: 0x7F7F7F7F)"""

    def __init__(self, T, H, I, E, splits, fill):
        self.g_rows = 2 * T + 8 * E + 256      # as the engine sizes them
        f = 0.0 if fill == "zero" else float("nan")
        bfl = lambda *s: torch.full(s, f, dtype=torch.bfloat16, device=DEV)   # noqa: E731
        ints = lambda *s: torch.full(s, 0 if fill == "zero" else 0x7F7F7F7F, dtype=torch.int32, device=DEV)  # noqa: E731
        self.tok_expert, self.tok_row, self.count, self.off = ints(T, 2), ints(T, 2), ints(E), ints(E + 1)
        self.tok_weight = torch.full((T, 2), f, dtype=torch.float32, device=DEV)
        self.xg, self.hg, self.yg = bfl(self.g_rows, H), bfl(self.g_rows, I), bfl(self.g_rows, H)
        self.part = torch.full((E, splits, T, H), f, dtype=torch.float32, device=DEV) if splits > 1 else None
        self.ysum = None


def run(lib, mode, w, xn, x, splits=1, fill="nan", bufs=None, ysum=False, router="onehot"):
    """One b200_op_moe_block call; returns the buffers with x_out / xn_out (the inputs are not modified)"""
    T, H = xn.shape
    E, I = w["gate"].shape[0], w["gate"].shape[1]
    b = bufs or Bufs(T, H, I, E, splits, fill)
    b.x_out, b.xn_out = x.clone(), xn.clone()
    if ysum:
        b.ysum = torch.full((T, H), float("nan"), dtype=torch.bfloat16, device=DEV)
    rc = lib.b200_op_moe_block(mode, _ptr(w[router]), _ptr(w["wgu"]), _ptr(w["down"]), _ptr(w["norm"]), _ptr(b.x_out),
                               _ptr(b.xn_out), T, H, I, E, EPS, _ptr(b.tok_expert), _ptr(b.tok_weight), _ptr(b.count),
                               _ptr(b.off), _ptr(b.tok_row), _ptr(b.xg), _ptr(b.hg), _ptr(b.yg), b.g_rows, _ptr(b.part),
                               splits, _ptr(b.ysum), None)
    assert rc == 0, f"b200_op_moe_block: {lib.b200_last_error().decode()}"
    torch.cuda.synchronize()
    return b


def segment_rows(count, off):
    """(rows, expert of each row) of every expert segment, in row order"""
    rows, ex = [], []
    for e in range(count.numel()):
        c, o = int(count[e]), int(off[e])
        rows.append(torch.arange(o, o + c, device=DEV))
        ex.append(torch.full((c,), e, device=DEV))
    return torch.cat(rows), torch.cat(ex)


def expert_outputs(b, T, H):
    """y [T][2][H] fp32: each (token, k)'s expert output as the combine reads it (bf16 rows, or bf16 of the summed
    partials), plus the summed partials themselves (or None)"""
    tr = b.tok_row.long()
    if b.part is None:
        return b.yg[tr].float(), None
    E, S = b.part.shape[:2]
    acc = torch.zeros_like(b.part[:, 0])
    for s in range(S):                                         # sum_partials8: 0 + p0 + p1 + ... in split order
        acc = acc + b.part[:, s]
    te = b.tok_expert.long()
    n = tr - b.off.long()[te]
    ysum = acc[te, n]                                          # [T][2][H]
    return bf(ysum), ysum


def check_block(lib, name, b, w, xn, x, want_te=None):
    """Every stage of one call against the reference applied to the previous stage's kernel output"""
    T, H = xn.shape
    E, I = w["gate"].shape[0], w["gate"].shape[1]
    te, tw = b.tok_expert, b.tok_weight
    # routing
    if want_te is not None:
        ref_te, ref_tw = want_te
        assert torch.equal(te, ref_te), f"{name}: tok_expert differs at {torch.nonzero((te != ref_te).any(1))[:8].flatten().tolist()}"
        ulp = torch.exp2(torch.floor(torch.log2(ref_tw.abs().clamp_min(2.0 ** -126))) - 23)   # fp32 ulp of each weight
        err = (tw - ref_tw).abs()
        assert bool((err <= 2 * ulp).all()), f"{name}: tok_weight off by {float((err / ulp).max()):.1f} ulp"
    assert bool(((te >= 0) & (te < E)).all()) and bool((te[:, 0] != te[:, 1]).all()), f"{name}: tok_expert out of range"
    assert torch.allclose(tw.sum(1), torch.ones(T, device=DEV), atol=1e-6), f"{name}: weights do not sum to 1"
    count, off, tok_row = tables_ref(te, E)
    _same(f"{name}: count", b.count, count)
    _same(f"{name}: off", b.off, off)
    _same(f"{name}: tok_row", b.tok_row, tok_row)
    # gather
    _same(f"{name}: xg rows", b.xg[tok_row.long()], xn[:, None, :].expand(T, 2, H))
    rows, ex = segment_rows(count, off)
    # gate/up + SwiGLU, down projection (per expert, on the kernels' own xg / hg)
    # hg: within the bracket of every rounding flip, and equal to the reference itself but for the few elements whose
    # fp32 g, u or silu(g) lies next to a bf16 rounding midpoint (up to ~0.4 % at K = 4096; a kernel that skipped the
    # rounding of silu(g) would differ in about a quarter of them)
    y_ref = torch.empty(rows.numel(), H, device=DEV)
    differ = 0
    for e in range(E):
        sel = ex == e
        if sel.any():
            r = rows[sel]
            lo, hi = swiglu_bracket(b.xg[r], w["gate"][e], w["up"][e])
            h = b.hg[r].float()
            bad = ~((h >= lo) & (h <= hi))
            assert not bad.any(), (f"{name}: hg of expert {e}: {int(bad.sum())}/{bad.numel()} outside the reference's rounding "
                                   f"bracket, first at {tuple(int(i) for i in torch.nonzero(bad)[0])}")
            differ += int((h != swiglu_ref(b.xg[r], w["gate"][e], w["up"][e])).sum())
            y_ref[sel] = h @ w["down"][e].float().T
    assert differ <= 16 + rows.numel() * I // 50, f"{name}: hg differs from the reference in {differ}/{rows.numel() * I}"
    y, ysum_part = expert_outputs(b, T, H)
    if ysum_part is None:
        _cmp(f"{name}: yg", b.yg[rows], y_ref, 2e-3, RTOL)
    else:
        idx = torch.empty(off[E], dtype=torch.long, device=DEV)
        idx[tok_row.flatten().long()] = torch.arange(2 * T, device=DEV)
        _cmp(f"{name}: summed split-K partials", ysum_part.reshape(2 * T, H)[idx[rows]], y_ref, 1e-3, 1e-3)
    # combine: bit-exact from the kernels' expert outputs and weights
    c = _combine_sorted(te, tw, y)
    if b.ysum is not None:
        _same(f"{name}: ysum", b.ysum, c.to(torch.bfloat16))
        _same(f"{name}: x untouched with ysum", b.x_out, x)
        _same(f"{name}: xn untouched with ysum", b.xn_out, xn)
        return
    x_ref = (x.float() + c).to(torch.bfloat16)
    _same(f"{name}: x", b.x_out, x_ref)
    xn_ref = rmsnorm_ref(b.x_out, w["norm"], EPS)
    _cmp(f"{name}: xn", b.xn_out, xn_ref, 1e-3, 2 * RTOL)
    tight = (b.xn_out.float() - xn_ref).abs() <= 1e-3 + RTOL * xn_ref.abs()
    assert float(tight.float().mean()) >= 0.9999, f"{name}: xn"


def check_poison(name, bp, bz):
    """bp: run on NaN-filled buffers, bz: the same call on zero-filled ones"""
    for f in ("tok_expert", "tok_weight", "count", "off", "tok_row", "x_out", "xn_out"):
        _same(f"{name}: {f} (NaN-filled vs zero-filled buffers)", getattr(bp, f), getattr(bz, f))
    assert bool(torch.isfinite(bp.x_out.float()).all()) and bool(torch.isfinite(bp.xn_out.float()).all()), f"{name}: non-finite x / xn"
    count, off = bz.count, bz.off
    rows, ex = segment_rows(count, off)
    inside = torch.zeros(bp.g_rows, dtype=torch.bool, device=DEV)
    inside[rows] = True
    for f in ("xg", "hg", "yg"):
        got, ref = getattr(bp, f), getattr(bz, f)
        if f == "yg" and bp.part is not None:
            continue
        _same(f"{name}: {f} segment rows (NaN-filled vs zero-filled buffers)", got[inside], ref[inside])
        assert bool(torch.isfinite(got[inside].float()).all()), f"{name}: non-finite {f} rows"
        out = got[~inside].view(torch.int16)
        assert bool((out == NAN16).all()), f"{name}: {f}: {int(((out != NAN16).any(1)).sum())} rows outside the segments were written"
    if bp.part is not None:
        E, S, T, H = bp.part.shape
        for e in range(E):
            c = int(count[e])
            _same(f"{name}: partials of expert {e}", bp.part[e, :, :c], bz.part[e, :, :c])
            assert bool(torch.isnan(bp.part[e, :, c:]).all()), f"{name}: partials of expert {e} written past its count"
        assert bool(torch.isnan(bp.yg).all()), f"{name}: yg written by the split-K path"


def block_case(lib, shape, T, mode, pattern, splits=1, seed=0):
    H, I, E = SHAPES[shape]
    w = weights(shape)
    name = f"{'prefill grouped per-expert'.split()[mode]} H{H} I{I} E{E} T{T} {pattern} splits {splits}"
    if pattern == "ties":
        xn, x = tie_inputs(T, H, E, seed)
    else:
        xn, x = forced_inputs(T, H, E, make_pairs(T, E, pattern, seed), seed)
    want = route_ref(xn[:, :E].float())                        # the one-hot router's logits are xn[:, :E] exactly
    bp = run(lib, mode, w, xn, x, splits, "nan")
    check_block(lib, name, bp, w, xn, x, want)
    bz = run(lib, mode, w, xn, x, splits, "zero")
    check_poison(name, bp, bz)
    return bp


# ---------------------------------------------------------------------------------------------- GPU tests
ALL_T = [1, 7, 65, 129, 1000, 1024, 1025, 3000, 8192]
PREFILL_CASES = ([(s, T, "random") for s in (SMALL, TP4) for T in ALL_T] +
                 [(s, T, "random") for s in (MOE8, E16, E2) for T in (7, 129, 1025, 3000)] +
                 [(MOE8, 1025, "pair01"), (E16, 3000, "pair01"), (SMALL, 1000, "all_to_one"), (E16, 1025, "all_to_one"),
                  (E2, 8192, "all_to_one"), (SMALL, 129, "ties"), (E16, 1025, "ties"), (E2, 65, "ties")] +
                 [(s, 1000, f"count{n}") for s in (MOE8, TP4) for n in (127, 128, 129)] +
                 [(E16, 3000, "count129"), (MOE8, 8192, "count128")])


@pytest.mark.gpu
@pytest.mark.parametrize("shape,T,pattern", PREFILL_CASES)
def test_moe_prefill(lib, shape, T, pattern):
    block_case(lib, shape, T, PREFILL, pattern)


DECODE_T = [1, 2, 16, 17, 33, 64]
GROUPED_CASES = ([(s, T, "random") for s in (SMALL, MOE8, TP4, E16, E2) for T in DECODE_T] +
                 [(s, T, "all_to_one") for s in (MOE8, E16) for T in (16, 64)] +     # a group of exactly block_n tokens
                 [(SMALL, 32, "all_to_one"), (MOE8, 33, "pair01"), (E16, 17, "ties"), (TP4, 64, "pair01"), (E2, 64, "ties")])


@pytest.mark.gpu
@pytest.mark.parametrize("shape,T,pattern", GROUPED_CASES)
def test_moe_decode_grouped(lib, shape, T, pattern):
    block_case(lib, shape, T, GROUPED, pattern)


PER_EXPERT_CASES = ([(s, T, "random", sp) for s in (SMALL, TP4) for T in (1, 17, 64) for sp in (1, 2)] +
                    [(s, T, "random", 5) for s in (MOE8, TP4) for T in (2, 33, 64)] +
                    [(E16, 16, "all_to_one", 2), (E2, 33, "random", 1), (MOE8, 64, "all_to_one", 5), (SMALL, 17, "ties", 2),
                     (E16, 64, "pair01", 1)])


@pytest.mark.gpu
@pytest.mark.parametrize("shape,T,pattern,splits", PER_EXPERT_CASES)
def test_moe_decode_per_expert(lib, shape, T, pattern, splits):
    assert eff_splits(SHAPES[shape][1], splits) == splits
    block_case(lib, shape, T, PER_EXPERT, pattern, splits)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("T,mode,splits", [(1025, PREFILL, 1), (8192, PREFILL, 1), (64, GROUPED, 1), (1, PER_EXPERT, 1),
                                           (17, PER_EXPERT, 1), (64, PER_EXPERT, 1), (33, PER_EXPERT, 4)])
def test_moe_mixtral_one_gpu(lib, T, mode, splits):
    """Mixtral-8x7B's whole expert width on one GPU: the per-expert gate/up GEMM (224 tiles) runs stream-K"""
    block_case(lib, FULL, T, mode, "random", splits)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,T", [(MOE8, 1), (MOE8, 7), (MOE8, 33), (E16, 64), (E2, 17), (SMALL, 64), (TP4, 16)])
def test_moe_prefill_and_decode_routers_agree(lib, shape, T):
    """Random router weights: the prefill router (warp per token) and the decode router (CTA per token) must give
    bit-identical tables on the same rows, and agree with the reference wherever the top-2 choice is decisive"""
    H, I, E = SHAPES[shape]
    w = weights(shape)
    g = torch.Generator(device=DEV).manual_seed(T)
    xn = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    x = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    runs = [run(lib, m, w, xn, x, router="wr") for m in (PREFILL, GROUPED, PER_EXPERT)]
    for m, b in zip(("grouped", "per-expert"), runs[1:]):
        for f in ("tok_expert", "tok_weight", "count", "off", "tok_row", "xg"):
            _same(f"{m} vs prefill: {f}", getattr(b, f), getattr(runs[0], f))
    for b in runs:
        check_block(lib, f"random router T{T}", b, w, xn, x)
    logits = bf(xn.float() @ w["wr"].float().T)
    te, tw = route_ref(logits)
    srt = logits.sort(-1, descending=True).values
    ulp = lambda v: torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -126))) - 7)   # noqa: E731
    # one bf16 ulp of either logit can move a comparison: decisive when both gaps exceed the two ulps
    margin = lambda a, b: (a - b) > 2 * (ulp(a) + ulp(b))                                      # noqa: E731
    dec = margin(srt[:, 0], srt[:, 1]) & margin(srt[:, 1], srt[:, 2]) if E > 2 else margin(srt[:, 0], srt[:, 1])
    assert float(dec.float().mean()) >= 0.5, "too few decisive tokens"
    assert torch.equal(runs[0].tok_expert[dec], te[dec]), "random router: top-2 differs on decisive tokens"
    _cmp("random router: weights", runs[0].tok_weight[dec], tw[dec], 0.0, 2.0 ** -6)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,T,mode,splits", [(MOE8, 1025, PREFILL, 1), (SMALL, 8192, PREFILL, 1), (E16, 64, GROUPED, 1),
                                                 (TP4, 33, GROUPED, 1), (MOE8, 17, PER_EXPERT, 5), (SMALL, 64, PER_EXPERT, 1)])
def test_moe_buffers_reused(lib, shape, T, mode, splits):
    """A second call with other routing on the same (dirty) buffers equals a call on fresh NaN-filled buffers"""
    H, I, E = SHAPES[shape]
    w = weights(shape)
    xn1, x1 = forced_inputs(T, H, E, make_pairs(T, E, "all_to_one", 1), 1)
    xn2, x2 = forced_inputs(T, H, E, make_pairs(T, E, "random", 2), 2)
    b = run(lib, mode, w, xn1, x1, splits)
    b = run(lib, mode, w, xn2, x2, splits, bufs=b)
    fresh = run(lib, mode, w, xn2, x2, splits)
    for f in ("tok_expert", "tok_weight", "count", "off", "tok_row", "x_out", "xn_out"):
        _same(f"second call vs fresh buffers: {f}", getattr(b, f), getattr(fresh, f))
    rows, _ = segment_rows(fresh.count, fresh.off)
    for f in ("xg", "hg") + (("yg",) if splits == 1 else ()):
        _same(f"second call vs fresh buffers: {f}", getattr(b, f)[rows], getattr(fresh, f)[rows])
    check_block(lib, "second call", b, w, xn2, x2, route_ref(xn2[:, :E].float()))


@pytest.mark.gpu
@pytest.mark.parametrize("shape,T,mode,splits", [(SMALL, 1000, PREFILL, 1), (TP4, 65, PREFILL, 1), (MOE8, 33, GROUPED, 1),
                                                 (E16, 64, GROUPED, 1), (MOE8, 17, PER_EXPERT, 5), (TP4, 1, PER_EXPERT, 2)])
def test_moe_ysum(lib, shape, T, mode, splits):
    """Tensor parallelism's output: ysum = the combined expert outputs, x and xn left alone"""
    H, I, E = SHAPES[shape]
    w = weights(shape)
    xn, x = forced_inputs(T, H, E, make_pairs(T, E, "random", 3), 3)
    b = run(lib, mode, w, xn, x, splits, ysum=True)
    check_block(lib, "ysum", b, w, xn, x, route_ref(xn[:, :E].float()))
    full = run(lib, mode, w, xn, x, splits)
    _same("ysum run vs full run: yg / x", (x.float() + b.ysum.float()).to(torch.bfloat16), full.x_out)


# ---------------------------------------------------------------------------------------------- HF parity
def _hf_block(shape, wr, gate, up, down):
    from transformers import MixtralConfig
    from transformers.models.mixtral.modeling_mixtral import MixtralSparseMoeBlock
    H, I, E = shape
    cfg = MixtralConfig(hidden_size=H, intermediate_size=I, num_local_experts=E, num_experts_per_tok=2,
                        router_jitter_noise=0.0)
    blk = MixtralSparseMoeBlock(cfg).to(torch.bfloat16).eval()
    with torch.no_grad():
        blk.gate.weight.copy_(wr)
        blk.experts.gate_up_proj.copy_(torch.cat([gate, up], 1))
        blk.experts.down_proj.copy_(down)
    return blk


def _decisive(logits, E):
    srt = logits.float().sort(-1, descending=True).values
    return (srt[:, 0] - srt[:, 1] > 0.05) & ((srt[:, 1] - srt[:, 2] > 0.05) if E > 2 else True)


def test_reference_matches_hf_mixtral_block():
    """The reference of this file (and interleave16) against transformers' MixtralSparseMoeBlock in bf16 on the CPU"""
    shape = H, I, E = (256, 128, 4)
    g = torch.Generator().manual_seed(5)
    wr = (torch.randn(E, H, generator=g) * H ** -0.5).to(torch.bfloat16)
    gate, up = [(torch.randn(E, I, H, generator=g) * H ** -0.5).to(torch.bfloat16) for _ in range(2)]
    down = (torch.randn(E, H, I, generator=g) * I ** -0.5).to(torch.bfloat16)
    xn = torch.randn(1, 48, H, generator=g).to(torch.bfloat16)
    blk = _hf_block(shape, wr, gate, up, down)
    with torch.no_grad():
        hf = blk(xn)
        hf = hf[0] if isinstance(hf, tuple) else hf
        hf = hf[0].float()
    te, tw, c = moe_ref(xn[0], wr, gate, up, down)
    dec = _decisive(bf(xn[0].float() @ wr.float().T), E)
    assert int(dec.sum()) >= 24
    _cmp("reference vs HF MixtralSparseMoeBlock", c[dec], hf[dec], 1e-2, 2 * RTOL)
    # the 16-row interleave holds the same rows as HF's [gate; up] layout
    wgu = interleave16(gate, up)
    assert torch.equal(wgu[:, 0:16], gate[:, 0:16]) and torch.equal(wgu[:, 16:32], up[:, 0:16])
    assert torch.equal(wgu[:, 2 * I - 16:], up[:, I - 16:])


@pytest.mark.gpu
def test_op_matches_hf_mixtral_block(lib):
    """b200_op_moe_block against transformers' MixtralSparseMoeBlock (bf16, CPU) + residual add + RMSNorm, same weights"""
    shape = SMALL
    H, I, E = SHAPES[shape]
    w = weights(shape)
    T = 64
    g = torch.Generator(device=DEV).manual_seed(11)
    xn = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    x = (torch.randn(T, H, generator=g, device=DEV) * 2).to(torch.bfloat16)
    blk = _hf_block(SHAPES[shape], w["wr"].cpu(), w["gate"].cpu(), w["up"].cpu(), w["down"].cpu())
    with torch.no_grad():
        hf = blk(xn.cpu()[None])
        hf = (hf[0] if isinstance(hf, tuple) else hf)[0].to(DEV)
    hf_x = (x.float() + hf.float()).to(torch.bfloat16)
    hf_xn = rmsnorm_ref(hf_x, w["norm"], EPS)
    dec = _decisive(bf(xn.float() @ w["wr"].float().T), E)
    assert int(dec.sum()) >= T // 2
    for mode in (PREFILL, GROUPED, PER_EXPERT):
        b = run(lib, mode, w, xn, x, router="wr", ysum=True)
        _cmp(f"mode {mode}: ysum vs HF", b.ysum[dec], hf[dec], 1e-2, 2 * RTOL)
        b = run(lib, mode, w, xn, x, router="wr")
        _cmp(f"mode {mode}: x vs HF", b.x_out[dec], hf_x[dec], 2e-2, 2 * RTOL)
        _cmp(f"mode {mode}: xn vs HF", b.xn_out[dec], hf_xn[dec], 2e-2, 4 * RTOL)
