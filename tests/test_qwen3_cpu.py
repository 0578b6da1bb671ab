"""Dense Qwen3 support without a GPU: the oracle reproduces the Qwen3 fixtures, and those fixtures tell a dropped, a
post-RoPE and a swapped q / k norm apart; the tensor table matches transformers' Qwen3ForCausalLM; and
B200GenerativeModel.load() accepts Qwen3 checkpoints (bf16 and compressed-tensors FP8) while it keeps refusing Qwen3-MoE,
attention_bias, yarn and block-scaled FP8, with the Llama / Qwen2 / Mixtral decisions unchanged."""
import types

import pytest
import torch

from helpers import load_case, logits_tol
from oracle import weights as W
from oracle.hf_oracle import OracleGenerativeModel
from tools.qwen3_oracle import build_model

FIXTURES = ["tiny_qwen3_ids", "tiny_qwen3_peaked", "tiny_qwen3_g4_ids", "tiny_qwen3_g5_ids", "tiny_qwen3_wide_ids"]


def _oracle(c):
    m = c["meta"]
    torch.set_num_threads(m.get("threads", 8))
    cfg = W.CONFIGS[m["cfg"]]
    sd = W.synth_state_dict(cfg, m["seed"])
    assert abs(W.checksum(sd) - m["weights_checksum"]) < 1e-3
    return build_model(cfg, sd)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_qwen3_fixture(name):
    c = load_case(name)
    m = c["meta"]
    model = _oracle(c)
    assert type(model).__name__ == "Qwen3ForCausalLM"
    orc = OracleGenerativeModel(model, pad_token_id=m["pad_token_id"])
    r = orc.create_completion(c["input_ids"].tolist(), max_tokens=m["max_tokens"], want_logits=True)
    assert r.finish_reason == m["finish_reason"]
    assert r.prompt_tokens == m["prompt_tokens"] and r.completion_tokens == m["completion_tokens"]
    tol = logits_tol(c["step_logits"])
    gen_same = (r.output_ids == c["output_ids"])[:, c["S"]:]
    for b in range(gen_same.shape[0]):
        bad = (~gen_same[b]).nonzero()
        if len(bad):
            assert float(c["margin"][b, int(bad[0])]) <= 2 * tol


def _norm_after_rope(self, hidden_states, position_embeddings, attention_mask, past_key_values=None, **kwargs):
    """Qwen3Attention.forward with q_norm / k_norm moved after RoPE (the mistake the control stands for)"""
    import transformers.models.qwen3.modeling_qwen3 as q3
    input_shape = hidden_states.shape[:-1]
    hidden_shape = (*input_shape, -1, self.head_dim)
    q = self.q_proj(hidden_states).view(hidden_shape).transpose(1, 2)
    k = self.k_proj(hidden_states).view(hidden_shape).transpose(1, 2)
    v = self.v_proj(hidden_states).view(hidden_shape).transpose(1, 2)
    cos, sin = position_embeddings
    q, k = q3.apply_rotary_pos_emb(q, k, cos, sin)
    q, k = self.q_norm(q), self.k_norm(k)
    if past_key_values is not None:
        k, v = past_key_values.update(k, v, self.layer_idx)
    attn = q3.ALL_ATTENTION_FUNCTIONS.get_interface(self.config._attn_implementation, q3.eager_attention_forward)
    out, w = attn(self, q, k, v, attention_mask, dropout=0.0, scaling=self.scaling, sliding_window=self.sliding_window, **kwargs)
    return self.o_proj(out.reshape(*input_shape, -1).contiguous()), w


def _drop(attn):
    attn.q_norm, attn.k_norm = torch.nn.Identity(), torch.nn.Identity()


def _after_rope(attn):
    attn.forward = types.MethodType(_norm_after_rope, attn)


def _swap(attn):
    wq = attn.q_norm.weight.data.clone()
    attn.q_norm.weight.data.copy_(attn.k_norm.weight.data)
    attn.k_norm.weight.data.copy_(wq)


@pytest.mark.parametrize("name", FIXTURES)
@pytest.mark.parametrize("mistake", [_drop, _after_rope, _swap], ids=["dropped", "after_rope", "swapped"])
def test_fixture_logits_tell_each_norm_mistake_apart(name, mistake):
    """negative controls: an oracle without the q / k norms, with them after RoPE, or with q_norm and k_norm swapped
    misses the fixture's teacher-forced logits by more than the tolerance the GPU tests apply"""
    c = load_case(name)
    model = _oracle(c)
    for layer in model.model.layers:
        mistake(layer.self_attn)
    orc = OracleGenerativeModel(model, pad_token_id=c["meta"]["pad_token_id"])
    with torch.no_grad():
        got = orc.forward_logits(c["output_ids"][:, :-1])[:, c["S"] - 1:]
    ref = c["step_logits"]
    assert float((got - ref).abs().max()) > logits_tol(ref)


@pytest.mark.parametrize("cfg_name", ["tiny_qwen3", "tiny_qwen3_g4", "tiny_qwen3_peaked", "qwen3_8b_2l"])
def test_tensor_table_matches_transformers_qwen3(cfg_name):
    from transformers import Qwen3Config, Qwen3ForCausalLM
    from kserve_b200.model_spec import llama_tensor_specs
    cfg = W.CONFIGS[cfg_name]
    hf = Qwen3Config(**{k: v for k, v in W.hf_config_dict(cfg).items() if k != "model_type"})
    with torch.device("meta"):
        model = Qwen3ForCausalLM(hf)
    sd = model.state_dict()
    tied = set(getattr(model, "_tied_weights_keys", None) or {}) if hf.tie_word_embeddings else set()
    want = [(k, tuple(v.shape)) for k, v in sd.items() if k not in tied]
    spec = [(n, s) for n, s, _ in llama_tensor_specs(cfg)]
    assert sorted(spec) == sorted(want)
    assert ("lm_head.weight" in dict(spec)) == (not cfg.get("tie_word_embeddings"))
    assert [n for n, _, k in llama_tensor_specs(cfg) if "_norm." in n] == [
        f"model.layers.{i}.self_attn.{p}_norm.weight" for i in range(cfg["num_hidden_layers"]) for p in "qk"]
    assert not any(k == "bias" for _, _, k in llama_tensor_specs(cfg))
    # the synthetic checkpoint has the same tensors in the same order
    assert [(n, s) for n, s, _ in W.tensor_specs(cfg)] == spec


def test_synthetic_qk_norms_and_projections_are_far_from_identity():
    sd = W.synth_state_dict(W.CONFIGS["tiny_qwen3"], 0)
    qn, kn = sd["model.layers.0.self_attn.q_norm.weight"].float(), sd["model.layers.0.self_attn.k_norm.weight"].float()
    assert qn.min() < 0.3 and qn.max() > 3.0 and bool((qn > 0).all())
    assert kn.abs().max() >= 10.0
    H = W.CONFIGS["tiny_qwen3"]["hidden_size"]
    rms = lambda t: float(t.float().pow(2).mean().sqrt()) * H ** 0.5    # RMS of a projection of a unit-RMS input
    assert rms(sd["model.layers.0.self_attn.q_proj.weight"]) > 2.0
    assert rms(sd["model.layers.0.self_attn.k_proj.weight"]) < 0.5


def test_llama_and_qwen2_tensor_tables_are_unchanged():
    from kserve_b200.model_spec import llama_tensor_specs
    names = [n for n, _, _ in llama_tensor_specs(W.CONFIGS["llama3_8b_2l"])]
    assert len(names) == 3 + 9 * 2 and not any("_norm." in n and "self_attn" in n for n in names)
    names = [n for n, _, _ in llama_tensor_specs(W.CONFIGS["tiny_qwen2"])]
    assert len(names) == 3 + 12 * 2 and not any("self_attn.q_norm" in n for n in names)


# ---- B200GenerativeModel.load() ---------------------------------------------------------------------------------
class RecordingEngine:
    """stands in for the CUDA engine: records the configuration and the tensors load() hands over"""
    last = None

    def __init__(self, cfg, **kw):
        self.cfg, self.kw, self.tensors = cfg, kw, []
        RecordingEngine.last = self

    def load_weights(self, named):
        self.tensors = [(n, tuple(t.shape), t.dtype) for n, t in named]

    def close(self):
        pass


def _qwen3_hf_config(base="tiny_qwen3", **over):
    """what a Qwen3 config.json carries (Qwen3-0.6B / 8B keys) at a synthetic config's shapes"""
    cfg = dict(W.hf_config_dict(W.CONFIGS[base]), architectures=["Qwen3ForCausalLM"], model_type="qwen3",
               use_sliding_window=False, sliding_window=None, max_window_layers=28, max_position_embeddings=40960,
               attention_bias=False, attention_dropout=0.0, torch_dtype="bfloat16", hidden_act="silu", rope_scaling=None,
               layer_types=["full_attention"] * W.CONFIGS[base]["num_hidden_layers"])
    cfg.update(over)
    return cfg


def _load(monkeypatch, cfg, state_dict=None, **kw):
    import kserve_b200.generative_model as gm
    monkeypatch.setattr(gm, "B200Engine", RecordingEngine)
    model = gm.B200GenerativeModel("qwen3", model_config=cfg, state_dict=state_dict, pad_token_id=0, **kw)
    try:
        model.load()
    finally:
        model.stop()
    return model, RecordingEngine.last


def test_load_accepts_a_qwen3_0p6b_like_config_and_ties_the_head(monkeypatch):
    """tiny_qwen3: q dim = 2 H as in Qwen3-0.6B (2048 vs 1024), tied embeddings"""
    cfg = _qwen3_hf_config(tie_word_embeddings=True)
    assert cfg["num_attention_heads"] * 128 == 2 * cfg["hidden_size"]
    model, eng = _load(monkeypatch, cfg, W.iter_state_dict(W.CONFIGS["tiny_qwen3"], 0))
    assert model.max_length == 40960
    names = [n for n, _, _ in eng.tensors]
    assert names.count("lm_head.weight") == 1 and names[-1] == "lm_head.weight"
    assert sum(n.endswith(("q_norm.weight", "k_norm.weight")) for n in names) == 2 * cfg["num_hidden_layers"]
    assert len(names) == 3 + 11 * cfg["num_hidden_layers"]


def _qk_norms(cfg, drop=()):
    """just the per-head q / k norm tensors of a config (load() requires them of a Qwen3 checkpoint)"""
    for i in range(cfg["num_hidden_layers"]):
        for p in "qk":
            name = f"model.layers.{i}.self_attn.{p}_norm.weight"
            if name not in drop:
                yield name, torch.ones(128, dtype=torch.bfloat16)


def test_load_accepts_a_qwen3_8b_like_config(monkeypatch):
    cfg = _qwen3_hf_config("qwen3_8b_2l", tie_word_embeddings=False)
    model, eng = _load(monkeypatch, cfg, _qk_norms(cfg), max_model_len=4096)
    assert model.max_length == 4096 and eng.cfg["model_type"] == "qwen3"


@pytest.mark.parametrize("drop", [
    None,                                                                        # no q / k norms at all
    ("model.layers.1.self_attn.k_norm.weight",),
])
def test_load_refuses_a_qwen3_checkpoint_without_its_qk_norms(monkeypatch, drop):
    """the engine applies the norms when their weights arrive: a Qwen3 checkpoint without them would run as Llama"""
    from kserve_b200.kserve_api.protocol.rest.openai.errors import OpenAIError
    cfg = _qwen3_hf_config("qwen3_8b_2l", tie_word_embeddings=False)
    sd = iter(()) if drop is None else _qk_norms(cfg, drop)
    want = "model.layers.0.self_attn.k_norm.weight" if drop is None else drop[0]
    with pytest.raises(OpenAIError, match=want.replace(".", r"\.") + ".*not supported"):
        _load(monkeypatch, cfg, sd, max_model_len=4096)


def test_load_accepts_an_fp8_qwen3_checkpoint(monkeypatch):
    """compressed-tensors FP8 (channel scales, lm_head ignored): the projections arrive as e4m3 codes with their scales,
    the q / k norms stay bf16"""
    cfg = _qwen3_hf_config(tie_word_embeddings=True, quantization_config=W.fp8_quantization_config("channel"))
    model, eng = _load(monkeypatch, cfg, W.iter_state_dict(W.CONFIGS["tiny_qwen3_fp8"], 0))
    assert eng.kw["weight_format"] == 1
    dt = {n: d for n, _, d in eng.tensors}
    assert dt["model.layers.0.self_attn.q_proj.weight"] == torch.float8_e4m3fn
    assert dt["model.layers.0.self_attn.q_norm.weight"] == torch.bfloat16
    assert dt["model.layers.1.self_attn.k_norm.weight"] == torch.bfloat16


@pytest.mark.parametrize("over, match", [
    (dict(model_type="qwen3_moe", architectures=["Qwen3MoeForCausalLM"], num_experts=128, num_experts_per_tok=8),
     "not supported"),
    (dict(model_type="qwen3_next", architectures=["Qwen3NextForCausalLM"]), "not supported"),
    (dict(attention_bias=True), "attention_bias"),
    (dict(rope_scaling=dict(rope_type="yarn", factor=4.0, original_max_position_embeddings=32768)), "yarn"),
    (dict(hidden_size=1024, num_attention_heads=16, head_dim=64), "head_dim=64"),
    (dict(quantization_config=dict(quant_method="fp8", fmt="e4m3", activation_scheme="dynamic",
                                   weight_block_size=[128, 128])), "block"),
    (dict(quantization_config=dict(W.fp8_quantization_config("channel"), config_groups={"group_0": dict(
        targets=["Linear"], weights=dict(num_bits=8, type="float", symmetric=True, strategy="block", dynamic=False,
                                         block_structure=[128, 128]))})), "block"),
])
def test_load_refuses_what_the_engine_cannot_run(monkeypatch, over, match):
    from kserve_b200.kserve_api.protocol.rest.openai.errors import OpenAIError
    # (rope_inv_freq's refusal of yarn is a ValueError, as it is for every family)
    with pytest.raises(ValueError if match == "yarn" else OpenAIError, match=match):
        _load(monkeypatch, _qwen3_hf_config(**over), iter(()))


@pytest.mark.parametrize("cfg_name, over, match", [
    ("tiny_g2", dict(architectures=["LlamaForCausalLM"], model_type="llama"), None),
    ("tiny_qwen2", dict(architectures=["Qwen2ForCausalLM"], use_sliding_window=False), None),
    ("tiny_moe", dict(architectures=["MixtralForCausalLM"], model_type="mixtral"), None),
    ("tiny_g2", dict(architectures=["LlamaForCausalLM"], model_type="llama", attention_bias=True), "attention_bias"),
    ("tiny_qwen2", dict(architectures=["Qwen2MoeForCausalLM"], model_type="qwen2_moe"), "not supported"),
])
def test_other_families_are_decided_as_before(monkeypatch, cfg_name, over, match):
    from kserve_b200.kserve_api.protocol.rest.openai.errors import OpenAIError
    cfg = dict(W.hf_config_dict(W.CONFIGS[cfg_name]), hidden_act="silu", **over)
    if match is None:
        model, eng = _load(monkeypatch, cfg, iter(()))
        assert model.ready is False and eng.cfg is cfg            # (stop() after load)
    else:
        with pytest.raises(OpenAIError, match=match):
            _load(monkeypatch, cfg, iter(()))
