"""The schedules of tests/test_cb_parity_gpu.py (tests/cb_parity.py) keep covering what they are written for: decode
row counts 1, 5, 16, 17, 32, 33, 64 and a rotating window over more than 64 sequences, reused slots, and the prefix
hits, prefill passes and chunk boundaries of the chunked scenario, including the fully cached block-aligned prompt."""
import pytest

import cb_parity as CB
import layer_parity as LP

SEED = 2
VOCAB = 1024


def _join_plan():
    return CB.plan_join_leave(LP.prompt_pool(200, VOCAB, SEED), SEED)


def test_join_leave_plan_covers_the_row_counts_and_reuses_slots():
    plan = _join_plan()
    counts = [s.resident for s in plan.steps]
    assert counts[:len(CB.JOIN_TARGETS)] == CB.JOIN_TARGETS
    for r in (1, 5, 16, 17, 32, 33, 64):
        assert r in counts, r
    assert max(counts) == 90 and sum(c > CB.MAX_ROWS for c in counts) >= 4, counts
    slots = [r.slot for r in plan.rows]
    assert len(slots) > len(set(slots)) and max(slots) < CB.A_MAX_BATCH, "later admits must land in released slots"
    assert {r.prompt.__len__() for r in plan.rows[:7]} == {1, 63, 64, 65, 127, 128, 129}
    assert all(CB.JOIN_MAX_NEW[0] <= r.max_new <= CB.JOIN_MAX_NEW[1] for r in plan.rows)
    # every row runs to its max_new, and each is released the step after it finishes
    released = [i for s in plan.steps for i in s.release]
    assert sorted(released) == list(range(len(plan.rows)))
    last = {}
    for s in plan.steps:
        for i, n in s.n_gen.items():
            assert n >= last.get(i, 0)
            last[i] = n
    assert all(last[i] == r.max_new for i, r in enumerate(plan.rows))


def test_join_leave_plan_rotates_the_window_over_every_sequence():
    """while more than 64 sequences are resident, every one of them advances"""
    plan = _join_plan()
    rot = [k for k, s in enumerate(plan.steps) if s.resident > CB.MAX_ROWS]
    assert len(rot) >= 4 and rot == list(range(rot[0], rot[-1] + 1)), rot
    start, end = plan.steps[rot[0] - 1].n_gen, plan.steps[rot[-1]].n_gen
    for k in rot:
        for i in plan.steps[k].n_gen:      # (a row released before the end had run to max_new)
            assert end.get(i, plan.rows[i].max_new) > start.get(i, 0), f"row {i} did not advance while the window rotated"


def _chunked(chunk, swap=True):
    shorts = LP.prompt_pool(8, VOCAB, SEED + 2)
    longs = LP.prompt_pool(2, VOCAB, SEED + 1, fixed=CB.LONG)
    P = LP.prompt_pool(1, VOCAB, SEED + 3, fixed=(CB.P_LEN,))[0]
    return CB.plan_chunked(shorts, longs, P, VOCAB, SEED, chunk, swap)


@pytest.mark.parametrize("chunk", [512, 1024])
def test_chunked_plan_prefix_hits_and_passes(chunk):
    plan = _chunked(chunk)
    fam = [plan.rows[i] for i in plan.family]
    # P[:256]+37, P[:896]+1, P, P[:640] (5 blocks cached, the last recomputed), the chain broken inside block 1
    assert [r.hit for r in fam] == [256, 896, 896, 512, 128]
    assert [len(r.prompt) for r in fam] == [293, 897, 1000, 640, 300]
    assert plan.hit_tokens == 2688
    total = sum(len(r.prompt) for r in plan.rows)
    assert plan.prefilled == total - plan.hit_tokens
    # the family's tails (37 + 1 + 104 + 128 + 172 tokens) share one pass
    assert all(len(r.chunks) == 1 for r in fam) and sum(c for r in fam for _, c in r.chunks) == 442
    P = plan.rows[plan.p_row]
    assert len(P.chunks) >= 2 and P.chunks[1][0] > 0, "P must be prefilled in more than one pass"
    for r in plan.rows:      # chunks tile each prompt after its cached prefix, each starting on a 128-token boundary
        pos = r.hit
        for start, count in r.chunks:
            assert start == pos and start % CB.BLOCK == 0
            pos += count
        assert pos == len(r.prompt)
    longs = plan.rows[8:10]
    assert all(len(r.chunks) >= 4000 // chunk for r in longs)
    want_passes = {512: 21, 1024: 11}[chunk]
    assert plan.passes == want_passes, plan.passes


def test_chunked_plan_swaps_running_sequences_with_shared_pages():
    plan = _chunked(512)
    outs = [s for s in plan.steps if s.swap_out]
    ins = [s for s in plan.steps if s.swap_in]
    assert len(outs) == 1 and len(ins) == 1 and sorted(outs[0].swap_out) == sorted(ins[0].swap_in)
    sw = outs[0].swap_out
    assert plan.family[1] in sw and plan.p_row in sw          # leading pages shared with the prefix cache
    k = plan.steps.index(outs[0])
    assert all(plan.steps[k].n_gen[i] == plan.steps[k - 1].n_gen[i] for i in sw), "swapped sequences do not advance"
    assert all(plan.steps[-1].n_gen.get(i, plan.rows[i].max_new) == plan.rows[i].max_new for i in sw)
    # short rows were decoding while the long prompts were prefilled
    first_long_done = min(t for t, s in enumerate(plan.steps) if 8 in s.n_gen and s.n_gen[8] > 0)
    assert any(plan.steps[t].resident > 0 for t in range(1, first_long_done))
