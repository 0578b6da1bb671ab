"""The FP8 KV cache without a GPU: the quantization rule (kserve_b200.fp8.quantize_kv, what the kernels' cvt.rn.satfinite
computes) on every bf16 value, the exact expansion the kernels apply to every code, the oracle fixtures of
tools/kv8_oracle.py, the --kv_cache_dtype flag, load()'s hand-over and refusals, and the memory plan."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import load_case, logits_tol, logits_tol_elementwise
from oracle import weights as W

TWINS = ["tiny_g4_ids", "tiny_g4_peaked", "tiny_qwen2_ids", "tiny_qwen2_peaked", "tiny_moe_ids"]
PEAKED = {"tiny_g4_peaked", "tiny_qwen2_peaked"}


def _e4m3_table():
    """(value, code) of the 127 non-negative finite e4m3fn codes from the format's definition (bias 7, no infinities,
    S.1111.111 is NaN)"""
    vals = []
    for code in range(0x7F):
        e, m = code >> 3, code & 7
        vals.append((m / 8) * 2.0 ** -6 if e == 0 else (1 + m / 8) * 2.0 ** (e - 7))
    return np.array(vals), np.arange(0x7F)


def _reference_codes(x):
    """round to nearest even onto e4m3fn after clamping to +-448; x float64 without NaN"""
    vals, codes = _e4m3_table()
    a = np.minimum(np.abs(x), 448.0)
    hi = np.clip(np.searchsorted(vals, a), 0, len(vals) - 1)       # first value >= a
    lo = np.maximum(hi - 1, 0)
    dlo, dhi = a - vals[lo], vals[hi] - a
    pick = np.where(dlo < dhi, lo, np.where(dhi < dlo, hi, np.where(codes[lo] % 2 == 0, lo, hi)))
    pick = np.where(vals[hi] == a, hi, pick)
    return (codes[pick] | np.where(np.signbit(x), 0x80, 0)).astype(np.uint8)


def test_quantization_rule_on_every_bf16_value():
    from kserve_b200.fp8 import quantize_kv
    x = torch.arange(1 << 16, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)   # every bit pattern
    got = quantize_kv(x)
    nan = torch.isnan(x)
    assert bool(torch.isnan(got.float()[nan]).all()), "NaN must stay NaN"
    xf = x.double().numpy()
    ref = _reference_codes(xf[~nan.numpy()])
    g = got.view(torch.uint8).numpy()[~nan.numpy()]
    bad = np.nonzero(g != ref)[0]
    assert len(bad) == 0, f"{len(bad)} values differ, first x={xf[~nan.numpy()][bad[0]]}: {g[bad[0]]:#x} vs {ref[bad[0]]:#x}"
    # the edges named by the rule
    q = lambda v: int(quantize_kv(torch.tensor([v], dtype=torch.bfloat16)).view(torch.uint8))
    assert q(0.0) == 0x00 and q(-0.0) == 0x80
    assert q(float("inf")) == 0x7E and q(float("-inf")) == 0xFE           # +-448
    assert q(464.0) == 0x7E and q(-500.0) == 0xFE and q(448.0) == 0x7E
    assert q(2.0 ** -9) == 0x01 and q(2.0 ** -10) == 0x00                # smallest subnormal; a tie rounds to even (0)
    # torch's plain cast turns |x| past 464 into NaN: the clamp is what keeps them finite
    assert torch.isnan(torch.tensor([480.0]).to(torch.float8_e4m3fn).float()).all()


def test_expansion_of_every_finite_code_is_exact():
    """bf16(code) is exact, and it is what the kernels' fp8x16_dequant computes with a unit scale: the code's sign, exponent
    and mantissa placed in a bf16 (sign << 15 | bits << 4), then one bf16 multiply by 2^120"""
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    f8 = codes.view(torch.float8_e4m3fn)
    finite = ~torch.isnan(f8.float())
    assert int(finite.sum()) == 254
    vals, _ = _e4m3_table()
    want = np.concatenate([vals, [np.nan], -vals, [np.nan]])
    assert np.array_equal(f8.double().numpy()[finite.numpy()], want[finite.numpy()])
    assert torch.equal(f8.to(torch.bfloat16).double()[finite], f8.double()[finite])
    c = codes.int()
    placed = ((c & 0x80) << 8) | ((c & 0x7F) << 4)
    placed = placed.to(torch.int16).view(torch.bfloat16)
    expanded = (placed * torch.tensor(2.0 ** 120, dtype=torch.bfloat16))
    assert torch.equal(expanded[finite].view(torch.int16), f8.to(torch.bfloat16)[finite].view(torch.int16))


# ---- fixtures ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("twin", TWINS)
def test_fixture_differs_from_its_bf16_twin(twin):
    """the FP8-KV fixture and the bf16 one share config, seed and prompts; their logits differ by more than the parity
    tolerance, so a GPU run that ignored the FP8 cache (or quantized nothing) fails"""
    a, b = load_case(twin), load_case(twin + "_kv8")
    assert a["meta"]["cfg"] == b["meta"]["cfg"] and a["meta"]["seed"] == b["meta"]["seed"]
    assert torch.equal(a["input_ids"], b["input_ids"]) and a["T"] == b["T"]
    tol = logits_tol_elementwise(b["step_logits"]) if twin in PEAKED else logits_tol(b["step_logits"])
    assert bool(((a["step_logits"] - b["step_logits"]).abs() > tol).any())


def test_big_fixture_differs_from_its_bf16_twin():
    a, b = load_case("llama3_8b_2l_b4"), load_case("llama3_8b_2l_b4_kv8")
    assert torch.equal(a["input_ids"], b["input_ids"]) and torch.equal(a["sub_cols"], b["sub_cols"])
    assert float((a["sub_logits"] - b["sub_logits"]).abs().max()) > logits_tol(b["sub_logits"])


@pytest.mark.parametrize("twin", TWINS)
def test_oracle_reproduces_fixture(twin):
    from tools.kv8_oracle import run
    _, res, _, _ = run(twin)
    c = load_case(twin + "_kv8")
    got = torch.stack(res.step_logits, 1)
    tol = logits_tol(c["step_logits"])
    assert float((got - c["step_logits"]).abs().max()) <= tol
    gen = res.output_ids[:, c["S"]:]
    decisive = c["margin"] > 2 * tol
    assert bool((gen == c["gen"])[decisive.cumprod(1).bool()].all())


def test_oracle_cache_rounds_what_attention_sees():
    """Fp8KVCache.update hands attention the quantized states (and stores them)"""
    from kserve_b200.fp8 import quantize_kv
    from tools.kv8_oracle import Fp8KVCache
    k = torch.randn(1, 2, 5, 128, dtype=torch.bfloat16) * 300
    v = torch.randn(1, 2, 5, 128, dtype=torch.bfloat16)
    kc, vc = Fp8KVCache().update(k, v, 0)
    assert torch.equal(kc, quantize_kv(k).to(torch.bfloat16)) and torch.equal(vc, quantize_kv(v).to(torch.bfloat16))
    assert float(kc.abs().max()) == 448.0


# ---- flag, load() ------------------------------------------------------------------------------------------------
def test_kv_cache_dtype_names():
    from kserve_b200.fp8 import UnsupportedQuantization, kv_cache_format
    assert [kv_cache_format(n) for n in ("auto", "bfloat16", "fp8", "fp8_e4m3")] == [0, 0, 1, 1]
    assert kv_cache_format("auto", tp_size=2) == 0
    with pytest.raises(UnsupportedQuantization, match="fp8_e5m2"):
        kv_cache_format("fp8_e5m2")
    with pytest.raises(UnsupportedQuantization, match="tensor parallelism"):
        kv_cache_format("fp8", tp_size=2)
    with pytest.raises(UnsupportedQuantization):
        kv_cache_format("int8")


def _main(monkeypatch, argv):
    import kserve_b200.__main__ as entry
    import kserve_b200.generative_model as gm
    seen = {}

    class FakeModel:
        def __init__(self, *a, **kw):
            seen.update(kw)

        def load(self):
            return True

    class FakeServer:
        def __init__(self, **kw):
            pass

        def start(self, models):
            pass
    monkeypatch.setattr(gm, "B200GenerativeModel", FakeModel)
    monkeypatch.setattr(entry, "ModelServer", FakeServer)
    entry.main(argv)
    return seen


@pytest.mark.parametrize("flag, want", [(None, "auto"), ("auto", "auto"), ("bfloat16", "bfloat16"), ("fp8", "fp8"),
                                        ("fp8_e4m3", "fp8_e4m3")])
def test_cli_flag_reaches_the_model(monkeypatch, flag, want):
    argv = ["--model_dir", "/nonexistent"] + (["--kv_cache_dtype", flag] if flag else [])
    assert _main(monkeypatch, argv)["kv_cache_dtype"] == want


@pytest.mark.parametrize("flag", ["fp8_e5m2", "int8"])
def test_cli_refuses(monkeypatch, capsys, flag):
    with pytest.raises(SystemExit):
        _main(monkeypatch, ["--model_dir", "/nonexistent", "--kv_cache_dtype", flag])
    assert "kv_cache_dtype" in capsys.readouterr().err


def _tiny_cfg():
    return dict(W.hf_config_dict(W.CONFIGS["tiny_g2"]), architectures=["LlamaForCausalLM"], model_type="llama")


@pytest.mark.parametrize("name, fmt", [("auto", 0), ("bfloat16", 0), ("fp8", 1), ("fp8_e4m3", 1)])
def test_load_hands_kv_cache_dtype_to_the_engine(monkeypatch, name, fmt):
    from test_fp8_cpu import _load
    _, eng = _load(monkeypatch, _tiny_cfg(), iter(()), kv_cache_dtype=name)
    assert eng.kw["kv_cache_dtype"] == fmt and eng.kw["weight_format"] == 0


def test_load_combines_fp8_weights_and_kv(monkeypatch):
    from test_fp8_cpu import _load, _qconfig
    _, eng = _load(monkeypatch, dict(_tiny_cfg(), quantization_config=_qconfig()), iter(()), kv_cache_dtype="fp8")
    assert eng.kw["kv_cache_dtype"] == 1 and eng.kw["weight_format"] == 1


def test_tensor_parallel_is_refused(monkeypatch, lib):
    """load() and b200_engine_create refuse an FP8 KV cache with tensor_parallel_size > 1"""
    from test_fp8_cpu import _load
    from kserve_b200 import _lib
    from kserve_b200.kserve_api.protocol.rest.openai.errors import OpenAIError
    with pytest.raises(OpenAIError, match="tensor parallelism"):
        _load(monkeypatch, _tiny_cfg(), iter(()), kv_cache_dtype="fp8", tensor_parallel_size=2)
    mc = _lib.ModelConfig()
    mc.vocab_size, mc.hidden_size, mc.intermediate_size, mc.num_layers = 1031, 512, 1024, 2
    mc.num_heads, mc.num_kv_heads, mc.head_dim, mc.max_position = 4, 2, 128, 256
    mc.max_batch, mc.max_seq_len, mc.max_prefill_tokens, mc.tp_rank, mc.tp_size = 2, 128, 256, 0, 2
    mc.kv_cache_dtype = 1
    h = C.c_void_p()
    assert lib.b200_engine_create(C.byref(mc), None, C.byref(h)) != 0
    assert b"FP8 KV cache is supported on one GPU only" in lib.b200_last_error()
    mc.tp_size, mc.kv_cache_dtype = 1, 2
    assert lib.b200_engine_create(C.byref(mc), None, C.byref(h)) != 0
    assert b"kv_cache_dtype must be" in lib.b200_last_error()


def test_kv_cache_scheme_checkpoints_stay_refused(monkeypatch):
    from test_fp8_cpu import _load, _qconfig
    from kserve_b200.kserve_api.protocol.rest.openai.errors import OpenAIError
    cfg = dict(_tiny_cfg(), quantization_config=_qconfig(kv_cache_scheme=dict(num_bits=8, type="float", strategy="tensor")))
    with pytest.raises(OpenAIError, match="kv_cache_scheme"):
        _load(monkeypatch, cfg, iter(()), kv_cache_dtype="fp8")


# ---- memory plan -------------------------------------------------------------------------------------------------
def test_plan_memory_gives_fp8_kv_twice_the_pages():
    """Llama-3-8B at max_batch 32, max_model_len 131072, 60 GB free is memory-bound (65,536 pages wanted)"""
    from kserve_b200.utils import plan_memory
    from tools.synth_weights import CONFIGS
    cfg = CONFIGS["llama3_8b"]
    args = (cfg, cfg["vocab_size"], 32, 131072, 1, 60 << 30)
    cap16, bf16_pages = plan_memory(*args)
    cap8, fp8_pages = plan_memory(*args, kv_bytes=1)
    assert bf16_pages == plan_memory(*args, kv_bytes=2)[1] == 4212 and cap8 == cap16
    assert fp8_pages >= 1.9 * bf16_pages and fp8_pages < 32 * 2048
