"""FP8 checkpoints without a GPU: the dequantization rule the engine computes is what transformers computes for a
compressed-tensors checkpoint, load() accepts the FP8 checkpoints the runtime serves and hands their tensors over
unconverted, it refuses the rest with a clear message, and the memory plan gives FP8 weights' savings to the KV pool."""
import json
import os

import pytest
import torch

from helpers import load_case, logits_tol
from oracle import weights as W
from oracle.hf_oracle import OracleGenerativeModel
from tools.fp8_oracle import TINY_CASES, load_oracle, write_checkpoint

E4M3_MAX = 448.0


def _qconfig(strategy="channel", input_activations=None, **over):
    qc = dict(quant_method="compressed-tensors", format="float-quantized", quantization_status="compressed",
              ignore=["lm_head"], kv_cache_scheme=None,
              config_groups={"group_0": dict(targets=["Linear"], input_activations=input_activations, output_activations=None,
                                             weights=dict(num_bits=8, type="float", symmetric=True, strategy=strategy,
                                                          dynamic=False))})
    qc.update(over)
    return qc


DYNAMIC = dict(num_bits=8, type="float", symmetric=True, strategy="token", dynamic=True)


# ---- the dequantization rule -----------------------------------------------------------------------------------
def _codes():
    c = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn)
    return c[~c.float().isnan()].reshape(-1, 1)          # 254 codes: zeros, subnormals, +-448


SCALES = [1e-30, 3e-39, 1e-8, 3.7e-3, 0.0173, 1.0, 2.5, 255.0, 1e5, 3e38]


@pytest.mark.parametrize("scale_dtype", [torch.bfloat16, torch.float32])
def test_rule_equals_compressed_tensors_dequantize(scale_dtype):
    """compressed_tensors' dequantize on the scale as transformers holds it (the bf16 model's parameter dtype)"""
    from compressed_tensors.quantization.lifecycle.forward import dequantize
    from kserve_b200.fp8 import dequantize_reference
    codes = _codes()
    for sc in SCALES:
        s = torch.full((codes.shape[0], 1), sc, dtype=scale_dtype)
        ref = dequantize(codes, s.to(torch.bfloat16), dtype=torch.bfloat16)
        got = dequantize_reference(codes, s)
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), sc


def test_transformers_decompresses_to_the_rule(tmp_path):
    """AutoModelForCausalLM.from_pretrained on a compressed-tensors checkpoint with fp32 channel scales: the weights the
    model multiplies are the rule's W' — and not the fp32 product rounded to bf16, which differs by an ulp"""
    from transformers import AutoModelForCausalLM
    from kserve_b200.fp8 import dequantize_reference
    d = write_checkpoint(str(tmp_path), "tiny_g2_fp8_tensor", 0)      # fp32 scales
    from safetensors.torch import load_file
    sd = load_file(os.path.join(d, "model.safetensors"))
    m = AutoModelForCausalLM.from_pretrained(d, dtype=torch.bfloat16)
    with torch.no_grad():
        m(torch.tensor([[5, 6, 7]]))                      # the first forward decompresses the weights
    naive_differs = False
    for name, p in m.named_parameters():
        if name.endswith("_proj.weight"):
            assert p.dtype == torch.bfloat16
            w, s = sd[name], sd[name + "_scale"]
            assert torch.equal(dequantize_reference(w, s).view(torch.int16), p.detach().view(torch.int16)), name
            naive_differs |= not torch.equal((w.float() * s.float()).bfloat16(), p.detach())
    assert naive_differs


# ---- quantization_config --------------------------------------------------------------------------------------
@pytest.mark.parametrize("qc, want", [
    (_qconfig("channel"), dict(strategy="channel", activations=None)),
    (_qconfig("tensor"), dict(strategy="tensor", activations=None)),
    (_qconfig("channel", DYNAMIC), dict(strategy="channel", activations="dynamic")),
    (_qconfig("channel", ignore=["re:.*lm_head"]), dict(strategy="channel", activations=None)),
])
def test_accepted_quantization_configs(qc, want):
    from kserve_b200.fp8 import parse_quantization_config
    assert parse_quantization_config(dict(model_type="llama", quantization_config=qc)) == want
    assert parse_quantization_config(dict(model_type="llama")) is None


def _group(**w):
    return {"group_0": dict(targets=["Linear"], input_activations=None,
                            weights=dict(dict(num_bits=8, type="float", symmetric=True, strategy="channel"), **w))}


REFUSED = [
    (dict(quantization_config=_qconfig(config_groups=_group(strategy="block", block_structure=[128, 128]))), "block"),
    (dict(quantization_config=_qconfig(config_groups=_group(strategy="group", group_size=128))), "group"),
    (dict(quantization_config=dict(quant_method="fp8", fmt="e4m3", weight_block_size=[128, 128])), "quant_method='fp8'"),
    (dict(quantization_config=_qconfig(config_groups=_group(type="int", num_bits=8))), "8-bit int weights"),
    (dict(quantization_config=_qconfig(config_groups=_group(type="int", num_bits=4))), "4-bit int weights"),
    (dict(quantization_config=_qconfig(ignore=[])), "FP8 lm_head"),
    (dict(quantization_config=_qconfig(config_groups={"g": dict(targets=["Linear", "Embedding"],
                                                               weights=_group()["group_0"]["weights"])})), "targets"),
    (dict(quantization_config=_qconfig(kv_cache_scheme=dict(num_bits=8, type="float", strategy="tensor"))), "KV cache"),
    (dict(model_type="mixtral", num_local_experts=8, quantization_config=_qconfig()), "Mixtral"),
    (dict(quantization_config=_qconfig("channel", dict(DYNAMIC, dynamic=False, strategy="tensor"))), "static input"),
    (dict(quantization_config=dict(quant_method="gptq", bits=4)), "quant_method='gptq'"),
    (dict(quantization_config=dict(quant_method="awq", bits=4)), "quant_method='awq'"),
    (dict(quantization_config=_qconfig(ignore=["lm_head", "model.layers.0.mlp.down_proj"])), "unquantized"),
    (dict(quantization_config=_qconfig(ignore=["lm_head", "re:.*down_proj"])), "unquantized"),
]


@pytest.mark.parametrize("over, match", REFUSED)
def test_refused_quantization_configs(over, match):
    from kserve_b200.fp8 import UnsupportedQuantization, parse_quantization_config
    with pytest.raises(UnsupportedQuantization, match=match):
        parse_quantization_config(dict(dict(model_type="llama"), **over))


# ---- load() -----------------------------------------------------------------------------------------------------
class RecordingEngine:
    """stands in for the CUDA engine: records the configuration and the tensors load() hands over"""
    last = None

    def __init__(self, cfg, **kw):
        self.cfg, self.kw, self.tensors = cfg, kw, []
        RecordingEngine.last = self

    def load_weights(self, named):
        self.tensors = [(n, t.dtype, tuple(t.shape)) for n, t in named]

    def close(self):
        pass


def _load(monkeypatch, cfg, state_dict=None, model_dir=None, **kw):
    import kserve_b200.generative_model as gm
    monkeypatch.setattr(gm, "B200Engine", RecordingEngine)
    model = gm.B200GenerativeModel("fp8", model_dir, model_config=cfg, state_dict=state_dict, pad_token_id=0, **kw)
    try:
        model.load()
    finally:
        model.stop()
    return model, RecordingEngine.last


@pytest.mark.parametrize("cfg_name, strategy, scale_dtype", [("tiny_qwen2_fp8", "channel", torch.bfloat16),
                                                              ("tiny_g2_fp8_tensor", "tensor", torch.float32),
                                                              ("tiny_qwen2_g6_tied_fp8", "channel", torch.float32)])
def test_load_hands_fp8_tensors_over_unconverted(monkeypatch, tmp_path, cfg_name, strategy, scale_dtype):
    d = write_checkpoint(str(tmp_path), cfg_name, 0)
    _, eng = _load(monkeypatch, None, model_dir=d)
    assert eng.kw["weight_format"] == 1
    cfg = W.CONFIGS[cfg_name]
    L = cfg["num_hidden_layers"]
    got = {n: (dt, s) for n, dt, s in eng.tensors}
    from kserve_b200.fp8 import PROJECTIONS
    for i in range(L):
        for p in PROJECTIONS:
            n = f"model.layers.{i}.{p}.weight"
            assert got[n][0] == torch.float8_e4m3fn
            assert got[n + "_scale"] == (scale_dtype, (got[n][1][0], 1) if strategy == "channel" else (1,))
    assert got["model.embed_tokens.weight"][0] == torch.bfloat16 and got["lm_head.weight"][0] == torch.bfloat16
    assert len(eng.tensors) == 3 + (9 + 7) * L + (3 * L if cfg.get("model_type") == "qwen2" else 0)


def test_load_accepts_fp8_dynamic_as_w8a16_and_says_so(monkeypatch, caplog):
    cfg = dict(W.hf_config_dict(W.CONFIGS["tiny_g2"]), architectures=["LlamaForCausalLM"], model_type="llama",
               quantization_config=_qconfig("channel", DYNAMIC))
    with caplog.at_level("WARNING", logger="kserve_b200"):
        _, eng = _load(monkeypatch, cfg, iter(()))
    assert eng.kw["weight_format"] == 1
    assert any("W8A16" in r.getMessage() for r in caplog.records)


def test_bf16_checkpoint_still_loads_with_weight_format_0(monkeypatch):
    cfg = dict(W.hf_config_dict(W.CONFIGS["tiny_g2"]), architectures=["LlamaForCausalLM"], model_type="llama")
    _, eng = _load(monkeypatch, cfg, iter(()))
    assert eng.kw["weight_format"] == 0


@pytest.mark.parametrize("over, match", REFUSED)
def test_load_refuses(monkeypatch, over, match):
    from kserve_b200.kserve_api.protocol.rest.openai.errors import OpenAIError
    cfg = dict(W.hf_config_dict(W.CONFIGS["tiny_g2"]), architectures=["LlamaForCausalLM"], model_type="llama")
    cfg.update(over)
    if cfg.get("model_type") == "mixtral":
        cfg.update(architectures=["MixtralForCausalLM"], num_experts_per_tok=2)
    with pytest.raises(OpenAIError, match=match):
        _load(monkeypatch, cfg, iter(()))


# ---- memory plan ------------------------------------------------------------------------------------------------
def test_plan_memory_gives_fp8_more_kv_pages():
    tp = 1
    from kserve_b200.utils import plan_memory
    from tools.synth_weights import CONFIGS
    cfg = CONFIGS["llama3_8b"]
    free = 60 << 30
    _, bf16_pages = plan_memory(cfg, cfg["vocab_size"], 512, 8192, tp, free)
    _, fp8_pages = plan_memory(dict(cfg, quantization_config=_qconfig()), cfg["vocab_size"], 512, 8192, tp, free)
    page = cfg["num_hidden_layers"] * 2 * (cfg["num_key_value_heads"] // tp) * 64 * 128 * 2
    assert fp8_pages > bf16_pages
    # Llama-3-8B: 6.98 GB of projections at one byte instead of two, less the bf16 prefill scratch of one layer
    assert (fp8_pages - bf16_pages) * page > 6.0e9


def test_tensor_parallel_is_refused(monkeypatch, lib):
    """FP8 engines run on one GPU: load() and b200_engine_create refuse tensor_parallel_size > 1"""
    import ctypes as C
    from kserve_b200 import _lib
    from kserve_b200.kserve_api.protocol.rest.openai.errors import OpenAIError
    cfg = dict(W.hf_config_dict(W.CONFIGS["tiny_g2"]), architectures=["LlamaForCausalLM"], model_type="llama",
               quantization_config=_qconfig())
    with pytest.raises(OpenAIError, match="tensor parallelism"):
        _load(monkeypatch, cfg, iter(()), tensor_parallel_size=2)
    mc = _lib.ModelConfig()
    mc.vocab_size, mc.hidden_size, mc.intermediate_size, mc.num_layers = 1031, 512, 1024, 2
    mc.num_heads, mc.num_kv_heads, mc.head_dim, mc.max_position = 4, 2, 128, 256
    mc.max_batch, mc.max_seq_len, mc.max_prefill_tokens, mc.tp_rank, mc.tp_size, mc.weight_format = 2, 128, 256, 0, 2, 1
    h = C.c_void_p()
    assert lib.b200_engine_create(C.byref(mc), None, C.byref(h)) != 0
    assert b"one GPU only" in lib.b200_last_error()


def test_nan_codes_are_refused():
    """0x7F / 0xFF are float8_e4m3fn's NaNs; the engine does not propagate them, so the loader refuses them"""
    from kserve_b200 import _lib
    from kserve_b200.engine import B200Engine
    w = torch.zeros(16, 32, dtype=torch.uint8)
    w[3, 5] = 0xFF
    with pytest.raises(_lib.B200Error, match="NaN codes"):
        B200Engine.set_weight_fp8(None, "model.layers.0.self_attn.q_proj.weight", w.view(torch.float8_e4m3fn),
                                  torch.ones(16, 1))


# ---- the oracle fixtures ------------------------------------------------------------------------------------------
FIXTURES = list(TINY_CASES)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_fp8_fixture(name):
    """transformers, loading the FP8 checkpoint directory with from_pretrained, regenerates the fixture"""
    c = load_case(name)
    m = c["meta"]
    torch.set_num_threads(m.get("threads", 8))
    assert abs(W.checksum(W.synth_state_dict(W.CONFIGS[m["cfg"]], m["seed"])) - m["weights_checksum"]) < 1e-3
    orc = OracleGenerativeModel(load_oracle(m["cfg"], m["seed"]), pad_token_id=m["pad_token_id"])
    r = orc.create_completion(c["input_ids"].tolist(), max_tokens=m["max_tokens"], want_logits=True)
    assert r.prompt_tokens == m["prompt_tokens"] and r.completion_tokens == m["completion_tokens"]
    tol = logits_tol(c["step_logits"])
    assert float((torch.stack(r.step_logits, 1) - c["step_logits"]).abs().max()) <= tol
    gen_same = (r.output_ids == c["output_ids"])[:, c["S"]:]
    for b in range(gen_same.shape[0]):
        bad = (~gen_same[b]).nonzero()
        if len(bad):
            assert float(c["margin"][b, int(bad[0])]) <= 2 * tol


@pytest.mark.parametrize("name", FIXTURES)
@pytest.mark.parametrize("control", ["per_tensor", "no_scale"])
def test_fixture_logits_depend_on_the_channel_scales(name, control):
    """negative control: with the scales dropped (1.0), or one per-tensor scale (the largest row's) substituted for the
    per-row ones, the oracle's teacher-forced logits miss the fixture by more than the GPU tests' tolerance"""
    c = load_case(name)
    m = c["meta"]
    if control == "per_tensor" and W.CONFIGS[m["cfg"]]["_fp8"] == "tensor":
        pytest.skip("the fixture already has per-tensor scales")
    override = (lambda n, s: torch.ones_like(s)) if control == "no_scale" else (lambda n, s: s.max().expand_as(s).clone())
    orc = OracleGenerativeModel(load_oracle(m["cfg"], m["seed"], override), pad_token_id=m["pad_token_id"])
    with torch.no_grad():
        got = orc.forward_logits(c["output_ids"][:, :-1])[:, c["S"] - 1:]
    assert float((got - c["step_logits"]).abs().max()) > logits_tol(c["step_logits"])
