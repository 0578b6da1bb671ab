"""Prefill GEMM (gemm_prefill_kernel) edge cases through the C ABI: rows past M are never written (sentinel rows
after M must survive), odd m-tile counts and grids, the residual epilogue in place, SwiGLU with out_cols tails, and
outputs TMA cannot address (row pitch not a multiple of 16 bytes).  Partial last tiles take the same masked
per-thread store as the device-side extents (m_rt / row_off) of the MoE expert GEMMs."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENTINEL_ROWS = 67
RTOL = 2.0 ** -7


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def _gemm(lib, A, W, out, res, M, N, K, epi, ocols):
    rc = lib.b200_op_gemm(_ptr(A), _ptr(W), _ptr(out), _ptr(res), M, N, K, epi, 256, 1, ocols, None)
    assert rc == 0, lib.b200_last_error().decode()
    torch.cuda.synchronize()


def _close(name, got, ref, atol, rtol):
    err = (got.float() - ref).abs()
    bad = err > atol + rtol * ref.abs()
    assert not bad.any(), f"{name}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {float(err.max()):.5f}"


def _sentinel(ocols, seed):
    return _rand(SENTINEL_ROWS, ocols, seed=seed)


# M: one row, one row short of / past a tile, odd tile counts; N: 1031 has an odd row pitch (no TMA store), 520 a
# column tail inside the last tile; the grids (m_tiles * n_tiles) are odd for several of them
@pytest.mark.parametrize("M", [1, 127, 129, 300, 1000, 4100])
@pytest.mark.parametrize("N,K", [(520, 512), (1031, 256), (768, 1024)])
def test_prefill_store_sentinel_rows(lib, M, N, K):
    A, W = _rand(M, K, seed=1), _rand(N, K, scale=1 / math.sqrt(K), seed=2)
    out = torch.full((M + SENTINEL_ROWS, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    sent = _sentinel(N, 3)
    out[M:] = sent
    _gemm(lib, A, W, out, None, M, N, K, 0, N)
    assert torch.equal(out[M:].view(torch.int16), sent.view(torch.int16)), "rows past M were written"
    _close(f"store {M}x{N}x{K}", out[:M], A.float() @ W.float().T, 2e-3, RTOL)


@pytest.mark.parametrize("M", [129, 300, 4100])
@pytest.mark.parametrize("N", [512, 520])
def test_prefill_residual_in_place(lib, M, N):
    K = 1024
    A, W, R = _rand(M, K, seed=4), _rand(N, K, scale=1 / math.sqrt(K), seed=5), _rand(M, N, seed=6)
    x = torch.empty((M + SENTINEL_ROWS, N), dtype=torch.bfloat16, device=DEV)
    x[:M] = R
    sent = _sentinel(N, 7)
    x[M:] = sent
    _gemm(lib, A, W, x, x, M, N, K, 1, N)   # out == residual
    assert torch.equal(x[M:].view(torch.int16), sent.view(torch.int16)), "rows past M were written"
    acc = (A.float() @ W.float().T).to(torch.bfloat16).float()
    ref = acc + R.float()
    # bf16(acc) may differ by one ulp of acc (summation order) before the add, then the sum is rounded once more
    err = (x[:M].float() - ref).abs()
    bad = err > 4e-3 + RTOL * (acc.abs() + ref.abs())
    assert not bad.any(), f"residual in place {M}x{N}: {int(bad.sum())} out of tolerance, max err {float(err.max()):.5f}"


def _interleave16(gate, up):
    I, K = gate.shape
    w = torch.empty((2 * I, K), dtype=gate.dtype, device=gate.device)
    w.view(I // 16, 2, 16, K)[:, 0] = gate.view(I // 16, 16, K)
    w.view(I // 16, 2, 16, K)[:, 1] = up.view(I // 16, 16, K)
    return w


# I = out_cols: 528 and 1040 end 16 columns into a 128-column output tile, 1008 inside its second 64-column box
@pytest.mark.parametrize("M", [1, 129, 300])
@pytest.mark.parametrize("I", [528, 1040, 1008])
def test_prefill_swiglu_out_cols_tail(lib, M, I):
    K = 512
    x = _rand(M, K, seed=8)
    gate, up = _rand(I, K, scale=1 / math.sqrt(K), seed=9), _rand(I, K, scale=1 / math.sqrt(K), seed=10)
    w = _interleave16(gate, up)
    out = torch.full((M + SENTINEL_ROWS, I), float("nan"), dtype=torch.bfloat16, device=DEV)
    sent = _sentinel(I, 11)
    out[M:] = sent
    _gemm(lib, x, w, out, None, M, 2 * I, K, 2, I)
    assert torch.equal(out[M:].view(torch.int16), sent.view(torch.int16)), "rows past M were written"
    g = (x.float() @ gate.float().T).to(torch.bfloat16)
    u = (x.float() @ up.float().T).to(torch.bfloat16)
    ref = torch.nn.functional.silu(g.float()).to(torch.bfloat16).float() * u.float()
    _close(f"swiglu {M}x{I}", out[:M], ref, 1e-2, 2 * RTOL)


def test_prefill_store_deterministic(lib):
    """Two launches of a many-tile problem give the same bits (no race between a tile's TMA store and the next
    tile's epilogue writing the shared output tile)."""
    M, N, K = 4096, 2048, 512
    A, W = _rand(M, K, seed=12), _rand(N, K, scale=1 / math.sqrt(K), seed=13)
    outs = []
    for _ in range(2):
        o = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
        _gemm(lib, A, W, o, None, M, N, K, 0, N)
        outs.append(o)
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    _close("store 4096x2048", outs[0], A.float() @ W.float().T, 2e-3, RTOL)
