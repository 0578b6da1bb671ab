"""Engine lifetime: b200_engine_destroy, and a b200_engine_create that fails after it has allocated, give back every byte
of device memory the engine took, including the buffers that are allocated on first use (sampling config, repetition
penalty bitmaps, continuous-batching state, captured graphs, host-DRAM KV buffers)."""
import pytest
import torch

from helpers import make_engine
from kserve_b200 import _lib
from kserve_b200.engine import B200Engine

pytestmark = pytest.mark.gpu

SLACK = 2 << 20   # bytes of free-memory noise tolerated between two readings


def _free_bytes() -> int:
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def _cycle():
    eng = make_engine("tiny_g2", 0, max_batch=256, max_seq_len=2048)
    try:
        ids = torch.randint(3, 1000, (4, 48), generator=torch.Generator().manual_seed(0))
        r = eng.generate(ids, None, max_new_tokens=8, pad_token_id=0, repetition_penalty=1.3)
        assert r.num_generated == 8
        for b in range(ids.shape[0]):
            eng.kv_swap_out(b, scrub=True)
        for b in range(ids.shape[0]):
            eng.kv_swap_in(b)
        eng.cb_begin(0, [])
        slots = eng.cb_admit([ids[0].tolist(), ids[1].tolist()], [8, 8],
                             sampling=[dict(repetition_penalty=1.3), dict(do_sample=True, top_k=20, seed=1)])
        eng.cb_step(3)
        for s in slots:
            eng.cb_release(s)
        eng.cb_end()
    finally:
        eng.close()


def test_destroy_returns_every_byte():
    _cycle()   # lazy module loading keeps device memory on the first use of each kernel
    base = _free_bytes()
    for i in range(3):
        _cycle()
        lost = base - _free_bytes()
        assert abs(lost) <= SLACK, f"cycle {i}: {lost / 2**20:.1f} MiB of device memory not returned"


def test_failed_create_frees_what_it_took():
    from oracle import weights as W
    cfg = W.CONFIGS["tiny_g2"]

    def create():
        # tp_size 2 passes the shape checks and allocates the whole engine, then is refused for want of an NCCL id
        with pytest.raises(_lib.B200Error):
            B200Engine(cfg, max_batch=256, max_seq_len=2048, tp_size=2, tp_rank=0, nccl_id=None)

    create()
    base = _free_bytes()
    create()
    lost = base - _free_bytes()
    assert abs(lost) <= SLACK, f"a failed create kept {lost / 2**20:.1f} MiB of device memory"
