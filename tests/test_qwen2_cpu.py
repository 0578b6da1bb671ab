"""Qwen2 / Qwen2.5 support without a GPU: the oracle reproduces the Qwen2 fixtures and those fixtures depend on the q / k / v
projection biases, the tensor table matches transformers' Qwen2ForCausalLM, and B200GenerativeModel.load() accepts Qwen2
checkpoints (full attention, tied embeddings) while it keeps refusing what the engine cannot run."""
import pytest
import torch

from helpers import load_case, logits_tol
from oracle import weights as W
from oracle.hf_oracle import OracleGenerativeModel
from tools.qwen2_oracle import build_model

FIXTURES = ["tiny_qwen2_ids", "tiny_qwen2_peaked", "tiny_qwen2_g6_tied_ids", "tiny_qwen2_g5_ids", "tiny_qwen2_wide_ids"]


def _oracle(c):
    m = c["meta"]
    torch.set_num_threads(m.get("threads", 8))
    cfg = W.CONFIGS[m["cfg"]]
    sd = W.synth_state_dict(cfg, m["seed"])
    assert abs(W.checksum(sd) - m["weights_checksum"]) < 1e-3
    return build_model(cfg, sd)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_qwen2_fixture(name):
    c = load_case(name)
    m = c["meta"]
    model = _oracle(c)
    assert type(model).__name__ == "Qwen2ForCausalLM"
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


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_logits_depend_on_the_projection_biases(name):
    """negative control: with the biases zeroed the oracle's teacher-forced logits miss the fixture by more than the
    tolerance the GPU tests apply, so an engine that dropped the biases could not pass them"""
    c = load_case(name)
    model = _oracle(c)
    for layer in model.model.layers:
        for proj in (layer.self_attn.q_proj, layer.self_attn.k_proj, layer.self_attn.v_proj):
            proj.bias.data.zero_()
    orc = OracleGenerativeModel(model, pad_token_id=c["meta"]["pad_token_id"])
    ids = c["output_ids"][:, :-1]
    with torch.no_grad():
        got = orc.forward_logits(ids)[:, c["S"] - 1:]          # the logits of every generated step, teacher forced
    ref = c["step_logits"]
    assert float((got - ref).abs().max()) > logits_tol(ref)


@pytest.mark.parametrize("cfg_name", ["tiny_qwen2", "tiny_qwen2_g6_tied", "qwen2_7b_2l"])
def test_tensor_table_matches_transformers_qwen2(cfg_name):
    from transformers import Qwen2Config, Qwen2ForCausalLM
    from kserve_b200.model_spec import llama_tensor_specs
    cfg = W.CONFIGS[cfg_name]
    hf = Qwen2Config(**{k: v for k, v in W.hf_config_dict(cfg).items() if k != "model_type"})
    with torch.device("meta"):
        model = Qwen2ForCausalLM(hf)
    sd = model.state_dict()
    tied = set(getattr(model, "_tied_weights_keys", None) or {}) if hf.tie_word_embeddings else set()
    want = [(k, tuple(v.shape)) for k, v in sd.items() if k not in tied]
    spec = [(n, s) for n, s, _ in llama_tensor_specs(cfg)]
    assert sorted(spec) == sorted(want)
    assert [n for n, _, k in llama_tensor_specs(cfg) if k == "bias"] == [
        f"model.layers.{i}.self_attn.{p}_proj.bias" for i in range(cfg["num_hidden_layers"]) for p in "qkv"]
    # the synthetic checkpoint has the same tensors (biases right after their weights)
    assert [(n, s) for n, s, _ in W.tensor_specs(cfg)] == spec


def test_llama_tensor_table_is_unchanged():
    from kserve_b200.model_spec import llama_tensor_specs
    names = [n for n, _, _ in llama_tensor_specs(W.CONFIGS["llama3_8b_2l"])]
    assert len(names) == 3 + 9 * 2 and names[-1] == "lm_head.weight"
    assert not any(n.endswith(".bias") for n in names)


# ---- B200GenerativeModel.load() ---------------------------------------------------------------------------------
class RecordingEngine:
    """stands in for the CUDA engine: records the configuration and the tensors load() hands over"""
    last = None

    def __init__(self, cfg, **kw):
        self.cfg, self.kw, self.tensors = cfg, kw, []
        RecordingEngine.last = self

    def load_weights(self, named):
        self.tensors = [(n, tuple(t.shape)) for n, t in named]

    def close(self):
        pass


def _qwen2_hf_config(**over):
    """what a Qwen2 / Qwen2.5 config.json carries (Qwen2.5-3B-like keys) at tiny_qwen2_g6_tied's shapes"""
    cfg = dict(W.hf_config_dict(W.CONFIGS["tiny_qwen2_g6_tied"]), architectures=["Qwen2ForCausalLM"], model_type="qwen2",
               use_sliding_window=False, sliding_window=131072, max_window_layers=28, max_position_embeddings=32768,
               tie_word_embeddings=True, torch_dtype="bfloat16", hidden_act="silu")
    cfg.update(over)
    return cfg


def _load(monkeypatch, cfg, state_dict=None, **kw):
    import kserve_b200.generative_model as gm
    monkeypatch.setattr(gm, "B200Engine", RecordingEngine)
    model = gm.B200GenerativeModel("qwen", model_config=cfg, state_dict=state_dict, pad_token_id=0, **kw)
    try:
        model.load()
    finally:
        model.stop()
    return model, RecordingEngine.last


def test_load_accepts_qwen2_full_attention_and_ties_the_head(monkeypatch):
    cfg = _qwen2_hf_config()
    sd = W.iter_state_dict(W.CONFIGS["tiny_qwen2_g6_tied"], 0)
    model, eng = _load(monkeypatch, cfg, sd)
    assert model.max_length == 32768                 # sliding_window 131072 with use_sliding_window false: full attention
    names = [n for n, _ in eng.tensors]
    assert names.count("lm_head.weight") == 1 and names[-1] == "lm_head.weight"       # the embedding, handed over as the head
    assert sum(n.endswith("_proj.bias") for n in names) == 3 * cfg["num_hidden_layers"]
    assert len(names) == 3 + 12 * cfg["num_hidden_layers"]


def test_qwen2_window_fields_never_shorten_the_context(monkeypatch):
    """use_sliding_window false: a sliding_window shorter than the context (and max_window_layers) is not a window"""
    model, _ = _load(monkeypatch, _qwen2_hf_config(sliding_window=4096), W.iter_state_dict(W.CONFIGS["tiny_qwen2_g6_tied"], 0),
                     max_model_len=8192)
    assert model.max_length == 8192


@pytest.mark.parametrize("over, match", [
    (dict(model_type="qwen2_moe", architectures=["Qwen2MoeForCausalLM"], num_experts=60), "not supported"),
    (dict(model_type="qwen3", architectures=["Qwen3ForCausalLM"]), "not supported"),
    (dict(model_type="llama", architectures=["LlamaForCausalLM"], attention_bias=True), "attention_bias"),
    (dict(hidden_size=896, num_attention_heads=14, head_dim=None), "head_dim=64"),     # Qwen2-0.5B / Qwen2.5-0.5B
])
def test_load_still_refuses(monkeypatch, over, match):
    from kserve_b200.kserve_api.protocol.rest.openai.errors import OpenAIError
    cfg = _qwen2_hf_config(**over)
    if cfg.get("head_dim") is None:
        cfg.pop("head_dim")
    with pytest.raises(OpenAIError, match=match):
        _load(monkeypatch, cfg, iter(()))
