"""Schedules of the continuous-batching parity test (helper of tests/test_cb_parity_cpu.py and _gpu.py).

A plan is the list of what a driver does before each b200_cb_step(1) — release the sequences that finished, swap
sequences out to host memory and back, admit new prompts — and what b200_cb_poll must report afterwards.  The plan is
made by a model of the engine's host-side bookkeeping (engine.cu: cb_admit, cb_prefill_pending, cb_decode_step):

  slots          an admit takes the lowest free slots, in prompt order
  prefix reuse   a prompt's leading 128-token blocks are served from the cache while the chain of blocks matches and at
                 least one token is left to compute (128 * (k + 1) < len); a prompt's full blocks enter the cache when
                 its last chunk has been prefilled
  prefill        one pass per step (every pass of the admit itself when chunking is off) over a prefix of the FIFO of
                 pending prompts: at most 64 rows and `budget` tokens, a prompt the budget ends inside cut at a
                 multiple of 128 tokens; the rows that end their prompt get their first token and join the decode list, last row first
  decode         one pass over the running slots; with more than 64 a 64-row window rotates over them (round robin)

Every step of the GPU test compares the polled n_gen of every slot with the plan, so the plan is also a check of the
engine's slot-indexed state.  The CPU test holds the plans to the coverage they are written for (decode row counts 1, 5,
16, 17, 32, 33, 64 and more than 64, reused slots, the prefix hits and passes of the chunked scenario).
"""
from __future__ import annotations

from collections import deque
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple

import torch

MAX_ROWS = 64          # engine.cu kMaxRows: rows of one prefill or decode pass
BLOCK = 128            # prefix-cache block / chunk granule (tokens)

# scenario A: the number of resident sequences each step is driven to (admitting the difference), then drained
JOIN_TARGETS = [1, 5, 16, 17, 32, 33, 64, 64, 80, 90, 90]
JOIN_MAX_NEW = (3, 10)
A_MAX_BATCH = 96
MAX_PREFILL_TOKENS = 8192
LONG = (4001, 3968)   # tokens of the two long prompts of scenario B (as in the static parity test)
P_LEN = 1000


@dataclass
class Row:
    prompt: List[int]
    max_new: int
    slot: int = -1
    chunks: List[Tuple[int, int]] = field(default_factory=list)   # (start, count) of each prefill pass over the prompt
    hit: int = 0                                                    # prompt tokens served from cached blocks


@dataclass
class Step:
    release: List[int]
    swap_out: List[int]
    swap_in: List[int]
    admit: List[int]
    resident: int                 # sequences in the decode list when the step runs (the decode pass covers min(., 64))
    n_gen: Dict[int, int]         # row -> tokens generated after the step, every admitted, unreleased row
    run: bool = True              # False: the last entry, which only releases


@dataclass
class Plan:
    rows: List[Row]
    steps: List[Step]
    chunk: int
    prefix: bool
    max_batch: int
    hit_tokens: int = 0
    passes: int = 0
    prefilled: int = 0


class EngineModel:
    def __init__(self, rows: List[Row], max_batch: int, chunk: int, prefix: bool, cap_t: int = MAX_PREFILL_TOKENS):
        self.rows, self.chunk, self.prefix, self.cap_t = rows, chunk, prefix, cap_t
        self.slot_row: List[Optional[int]] = [None] * max_batch
        self.active: List[int] = []            # running slots, in the engine's row order
        self.dec_rows: List[int] = []          # slots of the last decode pass
        self.dirty = True
        self.window = 0
        self.pending: deque = deque()          # [row, done]
        self.cache = set()                     # cached blocks, keyed by the tokens up to the block's end
        self.n_gen: Dict[int, int] = {}
        self.finished: Dict[int, bool] = {}
        self.hit_tokens = self.passes = self.prefilled = 0

    def admit(self, rids: List[int]) -> None:
        free = [s for s, r in enumerate(self.slot_row) if r is None]
        assert len(rids) <= len(free), "not enough free slots"
        total = sum(len(self.rows[i].prompt) for i in rids)
        assert self.chunk > 0 or total <= self.cap_t, "an unchunked admit must fit max_prefill_tokens"
        for i, s in zip(rids, free):
            row = self.rows[i]
            row.slot = s
            self.slot_row[s] = i
            p, hit = row.prompt, 0
            if self.prefix:
                for k in range(len(p) // BLOCK):
                    if BLOCK * (k + 1) < len(p) and tuple(p[:BLOCK * (k + 1)]) in self.cache:
                        hit = k + 1
                    else:
                        break
            row.hit = hit * BLOCK
            self.hit_tokens += row.hit
            self.n_gen[i], self.finished[i] = 0, False
            self.pending.append([i, row.hit])
        if self.chunk == 0:
            while self.pending:
                self.prefill_pass(self.cap_t)

    def prefill_pass(self, budget: int) -> None:
        budget, parts = min(budget, self.cap_t), []
        for ent in self.pending:
            if len(parts) == MAX_ROWS:
                break
            i, done = ent
            rem = len(self.rows[i].prompt) - done
            c = rem if rem <= budget else (budget // BLOCK) * BLOCK
            if c <= 0:
                break
            parts.append((ent, c, c == rem))
            budget -= c
            if c < rem:
                break
        if not parts:
            return
        self.passes += 1
        for ent, c, last in parts:
            i = ent[0]
            self.rows[i].chunks.append((ent[1], c))
            self.prefilled += c
            if last:
                self._gen(i)
        for ent, c, last in reversed(parts):
            ent[1] += c
            if not last:
                continue
            p = self.rows[ent[0]].prompt
            if self.prefix:
                self.cache.update(tuple(p[:BLOCK * (k + 1)]) for k in range(len(p) // BLOCK))
            self.active.append(self.rows[ent[0]].slot)
            self.dirty = True
            self.pending.remove(ent)

    def _gen(self, i: int) -> None:
        if not self.finished[i]:
            self.n_gen[i] += 1
            self.finished[i] = self.n_gen[i] >= self.rows[i].max_new

    def decode(self) -> None:
        rt = len(self.active)
        if rt == 0:
            return
        r = min(rt, MAX_ROWS)
        if self.dirty or rt > MAX_ROWS:
            start = self.window % rt if rt > MAX_ROWS else 0
            self.dec_rows = [self.active[(start + k) % rt] for k in range(r)]
            if rt > MAX_ROWS:
                self.window += r
            self.dirty = False
        for s in self.dec_rows:
            self._gen(self.slot_row[s])

    def release(self, i: int) -> None:
        s = self.rows[i].slot
        self.slot_row[s] = None
        if s in self.active:
            self.active.remove(s)
            self.dirty = True
        self.pending = deque(e for e in self.pending if e[0] != i)
        del self.n_gen[i], self.finished[i]

    def swap_out(self, i: int) -> None:
        self.active.remove(self.rows[i].slot)
        self.dirty = True

    def swap_in(self, i: int) -> None:
        self.active.append(self.rows[i].slot)
        self.dirty = True

    def step(self) -> None:
        if self.pending:
            self.prefill_pass(self.chunk if self.chunk > 0 else self.cap_t)
        self.decode()


Actions = Callable[[int, EngineModel], Tuple[List[int], List[int], List[int]]]


def make_plan(rows: List[Row], max_batch: int, chunk: int, prefix: bool, actions: Actions, max_steps: int = 400) -> Plan:
    """actions(t, model) -> (swap_out, swap_in, admit) row indices for step t, after that step's releases"""
    m = EngineModel(rows, max_batch, chunk, prefix)
    steps: List[Step] = []
    for t in range(max_steps):
        rel = sorted(i for i, f in m.finished.items() if f)
        for i in rel:
            m.release(i)
        out, back, adm = actions(t, m)
        if not m.n_gen and not (out or back or adm):
            steps.append(Step(rel, [], [], [], 0, {}, run=False))
            break
        for i in out:
            m.swap_out(i)
        for i in back:
            m.swap_in(i)
        if adm:
            m.admit(adm)
        resident = len(m.active)
        m.step()
        steps.append(Step(rel, out, back, adm, resident, dict(m.n_gen)))
    else:
        raise AssertionError("plan did not finish")
    return Plan(rows, steps, chunk, prefix, max_batch, m.hit_tokens, m.passes, m.prefilled)


# ---- scenario A: sequences join and leave, the window rotates ----------------------------------------------------------
def join_leave_rows(prompts: List[List[int]], seed: int) -> List[Row]:
    g = torch.Generator().manual_seed(seed + 11)
    mx = torch.randint(JOIN_MAX_NEW[0], JOIN_MAX_NEW[1] + 1, (len(prompts),), generator=g).tolist()
    return [Row(list(p), m) for p, m in zip(prompts, mx)]


def plan_join_leave(prompts: List[List[int]], seed: int) -> Plan:
    """drive the resident count through JOIN_TARGETS (admitting the difference each step, releasing every sequence as it
    finishes), then run the rest to completion"""
    rows = join_leave_rows(prompts, seed)
    nxt = [0]

    def actions(t, m):
        if t >= len(JOIN_TARGETS):
            return [], [], []
        k = JOIN_TARGETS[t] - sum(r is not None for r in m.slot_row)
        assert nxt[0] + k <= len(rows), "prompt pool too small for the plan"
        adm = list(range(nxt[0], nxt[0] + k))
        nxt[0] += k
        return [], [], adm

    plan = make_plan(rows, A_MAX_BATCH, 0, False, actions)
    return Plan(rows[:nxt[0]], plan.steps, 0, False, A_MAX_BATCH, plan.hit_tokens, plan.passes, plan.prefilled)


# ---- scenario B / C: chunked prefill, prefix reuse, host swap ----------------------------------------------------------
SHORT_MAX_NEW = 12
LONG_MAX_NEW = (4, 3)
P_MAX_NEW = 8
FAMILY_MAX_NEW = [6, 8, 5, 7, 6]
SWAP_STEPS = 2          # steps the swapped sequences stay in host memory


def family_prompts(P: List[int], vocab: int, seed: int) -> List[List[int]]:
    """the prompts admitted once P is cached: a partial-block tail, a one-token tail, P itself, a block-aligned prefix
    of P (every block cached, the last one recomputed) and a prompt whose chain breaks inside block 1"""
    g = torch.Generator().manual_seed(seed + 23)
    suffix = torch.randint(0, vocab, (38,), generator=g).tolist()
    broken = list(P[:300])
    broken[BLOCK + 50] = (broken[BLOCK + 50] + 1) % vocab
    return [P[:256] + suffix[:37], P[:896] + suffix[37:], list(P), P[:640], broken]


def plan_chunked(shorts: List[List[int]], longs: List[List[int]], P: List[int], vocab: int, seed: int, chunk: int,
                 swap: bool = True) -> Plan:
    """short rows decoding while two ~4000-token prompts and P (1000 tokens) are prefilled in chunks; once P is cached
    the five family prompts arrive in one admit; with `swap`, three running sequences — the P[:896] row (its leading
    pages are shared cache pages), P itself and the broken-chain row — go to host memory for SWAP_STEPS steps"""
    fam = family_prompts(P, vocab, seed)
    rows = [Row(list(p), SHORT_MAX_NEW) for p in shorts]
    rows += [Row(list(p), m) for p, m in zip(longs, LONG_MAX_NEW)]
    ip = len(rows)
    rows.append(Row(list(P), P_MAX_NEW))
    jf = len(rows)
    rows += [Row(p, m) for p, m in zip(fam, FAMILY_MAX_NEW)]
    swapped = [jf + 1, ip, jf + 4] if swap else []
    state = {"fam_at": None, "out_at": None}

    def actions(t, m):
        if t == 0:
            return [], [], list(range(len(shorts)))
        if t == 1:
            return [], [], list(range(len(shorts), jf))
        if state["fam_at"] is None and m.rows[ip].slot in m.active:
            state["fam_at"] = t
            return [], [], list(range(jf, len(rows)))
        if swapped and state["fam_at"] is not None and state["out_at"] is None and \
                all(m.rows[i].slot in m.active for i in range(jf, len(rows))):
            assert all(not m.finished[i] for i in swapped), "a sequence to swap finished first"
            state["out_at"] = t
            return swapped, [], []
        if state["out_at"] is not None and t == state["out_at"] + SWAP_STEPS:
            return [], swapped, []
        return [], [], []

    plan = make_plan(rows, A_MAX_BATCH, chunk, True, actions)
    plan.family, plan.p_row, plan.swapped = list(range(jf, len(rows))), ip, swapped
    return plan


# ---- references -----------------------------------------------------------------------------------------------------
def reference_sequence(row: Row, gen: List[int]) -> List[int]:
    """the tokens whose causal pass gives the row's n_gen tapped steps as its last n_gen positions"""
    return list(row.prompt) + list(gen[:-1])


@torch.no_grad()
def hidden_at(model, ids: List[int], n_steps: int, pos: Optional[List[int]] = None) -> torch.Tensor:
    """layer_parity.final_hidden with explicit position ids (default 0 .. len - 1): [n_steps, H] float64 on the CPU"""
    dev = next(model.parameters()).device
    x = torch.tensor(ids, dtype=torch.int64, device=dev)[None]
    p = torch.arange(len(ids), device=dev) if pos is None else torch.tensor(pos, dtype=torch.int64, device=dev)
    h = model.model(input_ids=x, position_ids=p[None]).last_hidden_state[0]
    return h[-n_steps:].double().cpu()
