"""Reference for sample_kernel (sampling.cuh): Philox4x32-10, transformers' processor chain, and the token a draw must give.

The chain is the one `_sample` runs: logits.float() -> RepetitionPenaltyLogitsProcessor -> TemperatureLogitsWarper ->
TopKLogitsWarper (every tie with the k-th value kept) -> TopPLogitsWarper.  The kept set is ordered as the kernel orders it,
score descending then index ascending; where a top-p cut falls inside a run of equal scores the lowest indices are kept.

The draw is deterministic: u = ((philox(ctr, key = seed).x >> 8) + 0.5) / 2^24 with ctr = (step, row, 0x5eed5eed, 0), or
(n_gen[slot], 0, 0x5eed5eed, 0) in continuous batching.  Two independent checks decide which tokens are acceptable:
  * fp64: the token whose interval of the fp64 CDF holds u.  A draw within n * 2^-24 of a boundary (n = kept tokens of
    non-zero weight, which bounds the error of an fp32 serial sum) may give either neighbour.
  * fp32 bracket: the kernel's own serial fp32 sums, run with every weight rounded down and with every weight rounded up
    by more than expf's error.  fp32 addition, multiplication and division are monotone, so the kernel's keep count and
    pick lie between the two runs; outside that bracket the kernel is wrong whatever its rounding.
The kernel's token must be acceptable to both.  A draw is exact when the fp32 bracket admits one token; otherwise it is
in the band, and the tests bound how often that happens (the fp64 band is far wider: it covers any order of summation)."""
import numpy as np
import torch

M32 = 0xFFFFFFFF
MAX_TOP_K = 1024          # kSampleMaxCand: b200_gen_params_t.top_k is capped here (0 selects 50)


def philox4x32_10(ctr, key):
    c0, c1, c2, c3 = (int(x) & M32 for x in ctr)
    k0, k1 = (int(x) & M32 for x in key)
    for _ in range(10):
        p0 = 0xD2511F53 * c0
        p1 = 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & M32, p1 & M32, ((p0 >> 32) ^ c3 ^ k1) & M32, p0 & M32
        k0 = (k0 + 0x9E3779B9) & M32
        k1 = (k1 + 0xBB67AE85) & M32
    return c0, c1, c2, c3


def uniform(seed, c0, c1):
    """the kernel's u for counter (c0, c1): exact in fp64 (24 bits plus one half)"""
    x = philox4x32_10((c0, c1, 0x5EED5EED, 0), (seed & M32, (seed >> 32) & M32))[0]
    return ((x >> 8) + 0.5) / 2.0 ** 24


def config(repetition_penalty=0.0, do_sample=0, temperature=0.0, top_p=0.0, top_k=0, seed=0):
    """b200_gen_params_t's sampling fields -> the effective values, with the engine's defaults (0 = default) and cap"""
    f32 = lambda v: float(np.float32(v))
    return dict(pen=f32(repetition_penalty) if repetition_penalty > 0 else 1.0, do_sample=bool(do_sample),
                temp=f32(temperature) if temperature > 0 else 1.0, top_p=f32(top_p) if 0 < top_p < 1 else 1.0,
                top_k=min(top_k, MAX_TOP_K) if top_k > 0 else 50, seed=int(seed) & 0xFFFFFFFFFFFFFFFF)


def process(logits, seen, c):
    """fp32 scores after the penalty and (when sampling) the temperature; logits: one row (bf16 or float),
    seen: bool [V] or None.  numpy float32 arithmetic is IEEE, as torch's and the kernel's are"""
    x = logits.float().numpy().copy()
    if c["pen"] != 1.0 and seen is not None:
        p, s = np.float32(c["pen"]), np.asarray(seen, dtype=bool)
        neg = s & (x < 0)
        pos = s & ~(x < 0)
        x[neg] *= p
        x[pos] /= p
    if c["do_sample"]:
        x /= np.float32(c["temp"])
    return torch.from_numpy(x)


def kept_order(x, top_k):
    """indices kept by TopKLogitsWarper (x >= k-th value: all ties kept), in the kernel's order"""
    k = min(top_k, x.numel())
    kth = float(torch.topk(x, k).values[-1])
    xn = x.numpy()
    idx = np.flatnonzero(xn >= kth)
    v = xn[idx]
    o = np.lexsort((idx, -v))            # score descending, index ascending (-0.0 and +0.0 compare equal)
    return idx[o], v[o]


def topp_keep_fp64(p, top_p, band):
    """possible keep counts under TopPLogitsWarper on fp64 probabilities p (kernel order); the threshold is 1 - top_p in
    fp32 (the kernel) or in fp64 (torch against a double), and a tail within `band` of it may go either way"""
    n = len(p)
    if top_p >= 1.0 or n == 1:
        return n, n
    tails = np.cumsum(p[::-1])[::-1][1:]               # tail from position j = 1 .. n-1
    thr = [float(np.float32(1.0) - np.float32(top_p)), 1.0 - top_p]
    lo = min(1 + int(np.count_nonzero(tails > t + band)) for t in thr)
    hi = max(1 + int(np.count_nonzero(tails > t - band)) for t in thr)
    return lo, hi


def _picks_fp64(w, keep_range, u, band):
    out = set()
    for keep in range(keep_range[0], keep_range[1] + 1):
        q = w[:keep] / w[:keep].sum()
        hi = np.cumsum(q)
        lo = np.concatenate([[0.0], hi[:-1]])
        ok = (q > 0) & (lo - band <= u) & (u <= hi + band)
        out |= set(np.nonzero(ok)[0].tolist())
    return out


def _wbounds(v):
    """fp32 weights expf(v - m) bracketed: below and above anything expf (<= 2 ulp) can return; exp(0) = 1 and
    exp(-inf) = 0 are exact"""
    d = (v.astype(np.float32) - v[0].astype(np.float32)).astype(np.float32)
    e = np.exp(d.astype(np.float64))
    lo = np.float32(e * (1 - 2.0 ** -20) - 2.0 ** -140).clip(0)
    hi = np.float32(e * (1 + 2.0 ** -20) + 2.0 ** -140)
    exact = (d == 0) | np.isneginf(d)
    lo[exact] = np.float32(e[exact])
    hi[exact] = np.float32(e[exact])
    return lo.astype(np.float32), hi.astype(np.float32)


def _serial(w):
    return np.cumsum(w, dtype=np.float32)            # np.cumsum adds left to right, like the kernel's thread 0


def _picks_fp32(v, top_p, u):
    """every (keep, pick) the kernel's fp32 arithmetic can reach with expf anywhere in its error bound"""
    wl, wh = _wbounds(v)
    n = len(v)
    Zl, Zh = _serial(wl)[-1], _serial(wh)[-1]
    if top_p < 1.0 and n > 1:
        thr = np.float32(1.0) - np.float32(top_p)
        tl = _serial((wl / Zh).astype(np.float32)[::-1])[:-1]       # tail over j = n-1 .. 1
        th = _serial((wh / Zl).astype(np.float32)[::-1])[:-1]
        first = lambda t: (n - 1 - int(np.argmax(t > thr))) + 1 if np.any(t > thr) else 1
        keeps = range(first(tl), first(th) + 1)
    else:
        keeps = range(n, n + 1)
    out = set()
    u32 = np.float32(u)
    for keep in keeps:
        al, ah = _serial(wl[:keep]), _serial(wh[:keep])
        tlo, thi = u32 * al[-1], u32 * ah[-1]
        # pick j: acc_j >= target and acc_{j-1} < target, for some target in [tlo, thi]
        prev_l = np.concatenate([[np.float32(0)], al[:-1]])
        ok = (ah >= tlo) & (prev_l < thi)
        ok[0] = ah[0] >= tlo
        out |= set(np.nonzero(ok)[0].tolist())
    return out


def expected(logits, seen, c, c0, c1):
    """(greedy) -> (token, score); (sampling) -> (acceptable tokens, exact?, {token: score}); c0, c1: the RNG counter"""
    x = process(logits, seen, c)
    if not c["do_sample"]:
        i = int(torch.argmax(x))                       # first maximum, as the kernel breaks ties
        return {i}, True, {i: float(x[i])}
    idx, v = kept_order(x, c["top_k"])
    u = uniform(c["seed"], c0, c1)
    w = np.exp(v.astype(np.float64) - float(v[0]))
    n_eff = int(np.count_nonzero(w > 0))
    band = (n_eff + 2) * 2.0 ** -24
    p = w / w.sum()
    keep = topp_keep_fp64(p, c["top_p"], band)
    f64 = _picks_fp64(w, keep, u, band)
    f32 = _picks_fp32(v, c["top_p"], u)
    both = f64 & f32
    return {int(idx[j]) for j in both}, len(f32) == 1 and f32 <= f64, {int(idx[j]): float(v[j]) for j in both}


def bits_to_mask(words, V):
    """uint32 [(V + 31) / 32] bitmap -> bool [V]"""
    w = np.asarray(words, dtype=np.uint32)
    b = np.unpackbits(w.view(np.uint8), bitorder="little")[:V]
    return torch.from_numpy(b.astype(bool))


def mask_to_bits(mask):
    """bool [V] -> uint32 [(V + 31) / 32] (token t is bit t & 31 of word t >> 5)"""
    m = np.asarray(mask, dtype=bool)
    V = len(m)
    pad = np.zeros(((V + 31) // 32) * 32, dtype=bool)
    pad[:V] = m
    return np.packbits(pad, bitorder="little").view(np.uint32)
