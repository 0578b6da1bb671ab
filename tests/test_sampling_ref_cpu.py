"""The sampling reference (tests/sampling_ref.py) pinned on the CPU: Philox4x32-10 against the Random123 known-answer
vectors, and the processor chain against transformers' own LogitsProcessor classes."""
import numpy as np
import pytest
import torch

import sampling_ref as R


@pytest.mark.parametrize("ctr,key,out", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, out):
    assert R.philox4x32_10(ctr, key) == out


def test_uniform_is_in_the_open_interval_and_keyed_by_all_64_seed_bits():
    us = [R.uniform(s, t, r) for s in (0, 1, 1 << 32, (1 << 64) - 1) for t in (0, 7) for r in (0, 3)]
    assert all(0 < u < 1 for u in us) and len(set(us)) == len(us)


def _transformers_chain(x, ids, c):
    from transformers.generation.logits_process import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)
    s = x.float().unsqueeze(0)
    if c["pen"] != 1.0:
        s = RepetitionPenaltyLogitsProcessor(c["pen"])(ids.unsqueeze(0), s)
    processed = s.clone()
    s = TemperatureLogitsWarper(c["temp"])(None, s)
    tempered = s.clone()
    s = TopKLogitsWarper(c["top_k"])(None, s)
    topk = s.clone()
    if c["top_p"] < 1.0:
        s = TopPLogitsWarper(c["top_p"])(None, s)
    return processed[0], tempered[0], topk[0], s[0]


def _rows(V, n, seed):
    g = torch.Generator().manual_seed(seed)
    for r in range(n):
        x = (torch.randn(V, generator=g) * (1.5 + 2.5 * r / n)).bfloat16()
        if r % 3 == 1:                                  # coarse values: long runs of ties everywhere
            x = (x.float() * 2).round().div(2).bfloat16()
        if r % 3 == 2:
            x[torch.randperm(V, generator=g)[:V // 4]] = 0.0
            x[torch.randperm(V, generator=g)[:V // 8]] = -0.0
        yield x


@pytest.mark.parametrize("V", [1031, 4099])
@pytest.mark.parametrize("pen,temp,top_k,top_p", [(1.0, 1.0, 50, 1.0), (1.05, 0.7, 20, 0.8), (1.0, 0.6, 50, 0.9),
                                                  (1.8, 1.3, 1024, 1.0), (0.7, 5.0, 200, 0.999), (1.0, 1e-3, 50, 0.01),
                                                  (1.0, 1.0, 1, 1.0), (1.2, 1.0, 64, 0.5)])
def test_reference_matches_transformers_warpers(V, pen, temp, top_k, top_p):
    c = R.config(repetition_penalty=pen, do_sample=1, temperature=temp, top_k=top_k, top_p=top_p)
    for r, x in enumerate(_rows(V, 12, 1000 * V + top_k)):
        g = torch.Generator().manual_seed(r)
        ids = torch.randint(0, V, (64,), generator=g)
        seen = torch.zeros(V, dtype=torch.bool)
        seen[ids] = True
        p_ref = R.process(x, seen, dict(c, do_sample=False))
        processed, tempered, topk, final = _transformers_chain(x, ids, c)
        assert torch.equal(p_ref.view(torch.int32), processed.view(torch.int32))
        s_ref = R.process(x, seen, c)
        assert torch.equal(s_ref, tempered)
        idx, v = R.kept_order(s_ref, c["top_k"])
        assert set(idx.tolist()) == set(torch.isfinite(topk).nonzero().flatten().tolist())
        if c["top_p"] < 1.0:
            w = np.exp(v.astype(np.float64) - float(v[0]))
            lo, hi = R.topp_keep_fp64(w / w.sum(), c["top_p"], (len(v) + 2) * 2.0 ** -24)
            kept = torch.isfinite(final).nonzero().flatten()
            assert lo <= len(kept) <= hi
            # same count -> the same multiset of scores: transformers keeps some of a tie run, the reference its lowest indices
            k = len(kept)
            assert sorted(v[:k].tolist()) == sorted(s_ref[kept].tolist())


def test_kept_order_is_score_descending_then_index_with_signed_zeros_equal():
    x = torch.tensor([0.0, -0.0, 1.0, -0.0, 0.0, -1.0, 1.0])
    idx, v = R.kept_order(x, 3)
    assert idx.tolist() == [2, 6, 0, 1, 3, 4]


def test_bitmap_round_trip():
    m = torch.rand(1031, generator=torch.Generator().manual_seed(0)) < 0.3
    w = R.mask_to_bits(m.numpy())
    assert w.dtype == np.uint32 and len(w) == 33
    assert bool(((w[5] >> 7) & 1) == int(m[5 * 32 + 7]))
    assert torch.equal(R.bits_to_mask(w, 1031), m)


def test_expected_draw_follows_the_cdf():
    """a row of four equal scores: the draw is the token whose quarter holds u, exactly"""
    x = torch.full((8,), -float("inf"))
    x[[1, 3, 4, 6]] = 2.0
    c = R.config(do_sample=1, top_k=50, seed=12345)
    for step in range(64):
        u = R.uniform(c["seed"], step, 0)
        toks, exact, _ = R.expected(x.bfloat16(), None, c, step, 0)
        if exact:
            assert toks == {[1, 3, 4, 6][int(u * 4)]}
    c = R.config(do_sample=1, top_k=50, top_p=0.5, seed=7)     # tails 0.25, 0.5, 0.75: the cut keeps exactly 2
    for step in range(32):
        toks, exact, _ = R.expected(x.bfloat16(), None, c, step, 0)
        assert exact and toks <= {1, 3}
