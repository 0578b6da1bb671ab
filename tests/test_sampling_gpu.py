"""Logits processors + sampling (sampling.cuh) through the C ABI.

Deterministic parts are pinned by the oracle (repetition penalty under greedy decoding: fixture tiny_g2_reppen made by
the reference's own call path with presence_penalty=1.8) or by identities (temperature -> 0 and top_k = 1 are greedy,
same seed -> same tokens).  The stochastic part cannot be bit-equal to torch's generator stream; it is checked against
the warper chain of transformers applied in fp32 to the engine's own logits: the support must be exactly the kept set
and the empirical frequencies must match the renormalised probabilities (total-variation bound)."""
import pytest
import torch

from helpers import load_case, logits_tol, make_engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    c = load_case("tiny_g2_reppen")
    m = c["meta"]
    e = make_engine(m["cfg"], m["seed"], vocab_rows=m["vocab_rows"], max_batch=8, max_seq_len=512)
    yield e, c
    e.close()


def test_repetition_penalty_greedy_matches_oracle(eng):
    e, c = eng
    m = c["meta"]
    r = e.generate(c["input_ids"], None, max_new_tokens=c["T"], pad_token_id=m["pad_token_id"],
                   repetition_penalty=m["presence_penalty"])
    gen = r.output_ids[:, c["S"]:]
    tol = logits_tol(c["step_logits"])
    changed = (c["step_logits"].argmax(-1) != c["gen"])           # steps where the processor changed the oracle's argmax
    covered = 0
    for b in range(gen.shape[0]):
        neq = (gen[b] != c["gen"][b]).nonzero()
        upto = int(neq[0]) if len(neq) else gen.shape[1]
        if len(neq):
            assert float(c["margin"][b, upto]) <= 2 * tol * m["presence_penalty"], f"row {b} diverges at decisive step {upto}"
        covered += int(changed[b, :upto].sum())
    assert covered >= 1, "no penalised decision was exercised before the first near-tie"
    # and without the penalty the engine follows the raw argmax there instead
    r0 = e.generate(c["input_ids"], None, max_new_tokens=c["T"], pad_token_id=m["pad_token_id"])
    assert not torch.equal(r0.output_ids, r.output_ids)


def test_sampling_identities(eng):
    e, c = eng
    kw = dict(max_new_tokens=8, pad_token_id=c["meta"]["pad_token_id"])
    greedy = e.generate(c["input_ids"], None, **kw).output_ids
    cold = e.generate(c["input_ids"], None, do_sample=True, temperature=1e-4, top_k=50, seed=1, **kw).output_ids
    k1 = e.generate(c["input_ids"], None, do_sample=True, temperature=1.7, top_k=1, seed=2, **kw).output_ids
    # top_k = 1 keeps every token tied at the maximum and draws among them: the argmax unless two logits tie exactly
    assert int((k1 == greedy).all(dim=1).sum()) >= k1.shape[0] - 1
    S = c["S"]            # T -> 0 picks the argmax unless two logits tie exactly (then either is a legal draw)
    assert int((cold[:, S] == greedy[:, S]).sum()) >= cold.shape[0] - 1
    a = e.generate(c["input_ids"], None, do_sample=True, temperature=1.5, top_p=0.9, seed=1234, **kw).output_ids
    b = e.generate(c["input_ids"], None, do_sample=True, temperature=1.5, top_p=0.9, seed=1234, **kw).output_ids
    d = e.generate(c["input_ids"], None, do_sample=True, temperature=1.5, top_p=0.9, seed=99, **kw).output_ids
    assert torch.equal(a, b) and not torch.equal(a, d)


@pytest.mark.parametrize("temperature,top_k,top_p", [(1.0, 50, 1.0), (0.7, 50, 0.9), (1.3, 8, 0.75)])
def test_first_token_distribution_matches_the_warper_chain(eng, temperature, top_k, top_p):
    e, c = eng
    ids = c["input_ids"][:1]
    pad = c["meta"]["pad_token_id"]
    ref = e.generate(ids, None, max_new_tokens=1, pad_token_id=pad, want_logits=True)
    logits = ref.logits[0, 0].float()                                # what `logits[:, -1].float()` holds
    # transformers warpers, in their order: temperature, top-k (ties with the k-th value kept), top-p
    s = logits / temperature
    kth = torch.topk(s, top_k).values[-1]
    s = s.masked_fill(s < kth, float("-inf"))
    if top_p < 1.0:
        sl, si = torch.sort(s, descending=False)
        cum = sl.softmax(-1).cumsum(-1)
        rm = cum <= (1 - top_p)
        rm[-1:] = False
        s = s.masked_fill(torch.zeros_like(rm).scatter(0, si, rm), float("-inf"))
    probs = s.softmax(-1)
    support = set(probs.nonzero().flatten().tolist())
    N = 1500
    counts = torch.zeros_like(probs)
    for seed in range(N):
        t = int(e.generate(ids, None, max_new_tokens=1, pad_token_id=pad, do_sample=True, temperature=temperature,
                           top_k=top_k, top_p=top_p, seed=seed).output_ids[0, -1])
        assert t in support, f"sampled token {t} is outside the kept set"
        counts[t] += 1
    tv = 0.5 * float((counts / N - probs).abs().sum())
    # E[TV] of an N-sample empirical distribution over K cells is about sqrt(K / (2 pi N)); allow 2.5x
    bound = 2.5 * (len(support) / (2 * 3.14159 * N)) ** 0.5 + 0.01
    assert tv < bound, f"total variation {tv:.3f} over {len(support)} tokens exceeds {bound:.3f}"
    assert len(set(counts.nonzero().flatten().tolist())) >= min(3, len(support))


def test_openai_route_presence_penalty_and_checkpoint_sampling_defaults():
    """presence_penalty through /openai/v1/completions equals the oracle's strings-as-ids; a checkpoint whose
    generation_config turns sampling on (q9) samples reproducibly per `seed` and falls back to greedy at temperature 0."""
    from fastapi.testclient import TestClient
    from kserve_b200.generative_model import B200GenerativeModel
    from kserve_b200.kserve_api import ModelServer
    from oracle import weights as W
    c = load_case("tiny_g2_reppen")
    m = c["meta"]
    cfg = dict(W.CONFIGS["tiny_g2"], architectures=["LlamaForCausalLM"], model_type="llama")
    model = B200GenerativeModel("tiny", model_config=cfg, state_dict=W.iter_state_dict(W.CONFIGS["tiny_g2"], 0), pad_token_id=m["pad_token_id"],
                                max_model_len=512, max_batch=8, generation_defaults={"do_sample": True, "temperature": 0.8, "top_p": 0.9})
    assert model.load()
    try:
        with TestClient(ModelServer().create_application([model])) as client:
            prompt = c["input_ids"][0].tolist()
            post = lambda **kw: client.post("/openai/v1/completions", json={"model": "tiny", "prompt": prompt, "max_tokens": 12, **kw})
            g = post(temperature=0, presence_penalty=m["presence_penalty"])
            assert g.status_code == 200, g.text
            toks = [int(x) for x in g.json()["choices"][0]["text"].split()]
            ref = c["gen"][0].tolist()[:12]
            tol = logits_tol(c["step_logits"])
            for t, (a, b) in enumerate(zip(toks, ref)):
                if a != b:
                    assert float(c["margin"][0, t]) <= 2 * tol * m["presence_penalty"]
                    break
            s1 = post(seed=7).json()["choices"][0]["text"]
            s2 = post(seed=7).json()["choices"][0]["text"]
            s3 = post(seed=8).json()["choices"][0]["text"]
            assert s1 == s2 and s1 != s3
            # logit_bias: the reference's sequence_bias keyed by tuple(str) is rejected by transformers inside generate (q8)
            bad = TestClient(client.app, raise_server_exceptions=False).post(
                "/openai/v1/completions", json={"model": "tiny", "prompt": prompt, "max_tokens": 12, "logit_bias": {"5": 1.0}})
            assert bad.status_code == 500 and "sequence_bias" in bad.text
    finally:
        model.stop()
