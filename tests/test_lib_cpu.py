"""No-GPU checks of the C ABI library: it loads, exports every symbol include/*.h declares, fails loudly
without a device, and its batcher state machine agrees with the Go-batcher oracle on random traces."""
import ctypes as C
import glob
import os
import random
import re

import pytest

from conftest import ROOT


def _declared_symbols():
    syms = set()
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        txt = open(h).read()
        txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
        syms |= set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", txt))
    return sorted(syms)


def test_library_exports_every_declared_symbol(lib):
    syms = _declared_symbols()
    assert len(syms) >= 25, syms
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, f"declared in include/*.h but not exported: {missing}"
    assert b"sm_90a" in lib.b200_version()


def test_no_cpu_fallback(lib):
    """Without a CUDA device the engine refuses to exist (no CPU / oracle fallback in the product path)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from kserve_b200 import _lib
    mc = _lib.ModelConfig()
    mc.vocab_size, mc.hidden_size, mc.intermediate_size, mc.num_layers = 1000, 512, 1024, 1
    mc.num_heads, mc.num_kv_heads, mc.head_dim, mc.max_position = 4, 2, 128, 256
    mc.max_batch, mc.max_seq_len, mc.max_prefill_tokens, mc.tp_size = 2, 128, 256, 1
    h = C.c_void_p()
    rc = lib.b200_engine_create(C.byref(mc), None, C.byref(h))
    assert rc != 0 and lib.b200_last_error()
    from kserve_b200.engine import B200Engine
    with pytest.raises(_lib.B200Error):
        B200Engine(dict(vocab_size=1000, hidden_size=512, intermediate_size=1024, num_hidden_layers=1,
                        num_attention_heads=4, num_key_value_heads=2, head_dim=128))


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under kserve_b200/ may reference it."""
    bad = []
    for root, _, files in os.walk(os.path.join(ROOT, "kserve_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(root, f), errors="ignore").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M) or "oracle/" in txt.replace("oracle/__init__", ""):
                    bad.append(os.path.join(root, f))
    assert not bad, bad


def _run_core(lib, trace, mbs, ml):
    h = C.c_void_p()
    assert lib.b200_batcher_create(mbs, ml, C.byref(h)) == 0
    fired = []
    tickets, first, count = (C.c_int64 * 4096)(), (C.c_int32 * 4096)(), (C.c_int32 * 4096)()
    n, total = C.c_int32(), C.c_int32()
    tk2rid = {}

    def tick(t):
        assert lib.b200_batcher_tick(h, t, 4096, tickets, first, count, C.byref(n), C.byref(total)) == 0
        if n.value:
            fired.append((t, total.value, {tk2rid[tickets[i]]: list(range(first[i], first[i] + count[i])) for i in range(n.value)}))
    for kind, t, rid, k in trace:
        if kind == "req":
            tk = C.c_int64()
            assert lib.b200_batcher_add(h, t, k, C.byref(tk)) == 0
            tk2rid[tk.value] = rid
        tick(t)
    lib.b200_batcher_destroy(h)
    return fired


@pytest.mark.parametrize("seed", range(6))
def test_batcher_core_matches_go_oracle(lib, seed):
    from oracle.batcher_oracle import GoBatcherOracle
    rng = random.Random(seed)
    mbs, ml = rng.choice([(32, 50), (64, 50), (4, 7), (-1, -1), (1, 1)])
    t, trace = 0, []
    for rid in range(300):
        gap = rng.choice([0, 10, 100, 100, 500, 3000, 20000]) if ml > 0 else rng.choice([0, 100, 2_000_000])
        # the goroutine wakes every 100 us while idle: emit those polls too
        for _ in range(min(gap // 100, 400)):
            t += 100
            trace.append(("poll", t, None, 0))
        t += gap % 100 if gap >= 100 else gap
        trace.append(("req", t, rid, rng.choice([1, 1, 1, 2, 5, 40])))
    for _ in range(60000 if ml < 0 else 600):
        t += 100
        trace.append(("poll", t, None, 0))
    o = GoBatcherOracle(mbs, ml)
    want = []
    for kind, tt, rid, k in trace:
        f = o.on_request(tt, rid, [None] * k) if kind == "req" else o.check(tt)
        if f:
            want.append((f.at_us, len(f.instances), f.index))
    got = _run_core(lib, trace, mbs, ml)
    assert got == want
    assert sum(len(ix) for _, _, ix in got) == 300, "every request must be answered exactly once"


def test_batcher_defaults(lib):
    """handler_test.go:133-174 — New(-1, -1) -> MaxBatchSize 32, MaxLatency 5000."""
    h = C.c_void_p()
    assert lib.b200_batcher_create(-1, -1, C.byref(h)) == 0
    a, b = C.c_int32(), C.c_int32()
    assert lib.b200_batcher_config(h, C.byref(a), C.byref(b)) == 0
    assert (a.value, b.value) == (32, 5000)
    lib.b200_batcher_destroy(h)
