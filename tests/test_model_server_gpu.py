"""The drop-in surface on a real GPU: B200GenerativeModel registered with ModelServer and driven through the
REST routes the reference exposes (/openai/v1/completions, chat, SSE), the V1/V2 predict legs the north star
adds, and the batcher in front of :predict.  Expected strings / usage come from the oracle fixtures."""
import asyncio
import json
import os

import numpy as np
import pytest
import torch
from fastapi.testclient import TestClient

from helpers import GOLDEN, load_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def served():
    from transformers import AutoTokenizer
    from kserve_b200.generative_model import B200GenerativeModel
    from kserve_b200.kserve_api import ModelServer
    from oracle import weights as W
    c = load_case("tiny_g2_text")
    cfg = dict(W.CONFIGS["tiny_g2"], architectures=["LlamaForCausalLM"], model_type="llama")
    tok = AutoTokenizer.from_pretrained(os.path.join(GOLDEN, "byte_tokenizer"))
    model = B200GenerativeModel("tiny", model_config=cfg, state_dict=W.iter_state_dict(W.CONFIGS["tiny_g2"], 0), tokenizer=tok,
                                max_model_len=512, max_batch=8)
    assert model.load() and model.ready and model.vocab_rows == 257
    app = ModelServer().create_application([model])
    with TestClient(app) as client:
        yield client, model, tok, c
    model.stop()


def test_completions_text_prompts_match_oracle(served):
    client, model, tok, c = served
    m = c["meta"]
    r = client.post("/openai/v1/completions", json={"model": "tiny", "prompt": m["prompt"], "max_tokens": m["max_tokens"], "temperature": 0})
    assert r.status_code == 200, r.text
    j = r.json()
    assert [ch["text"] for ch in j["choices"]] == m["texts"]
    assert all(ch["finish_reason"] == "length" for ch in j["choices"])
    assert j["usage"] == {"prompt_tokens": m["prompt_tokens"], "completion_tokens": m["completion_tokens"],
                          "total_tokens": m["prompt_tokens"] + m["completion_tokens"]}
    # echo: the output slice starts at 0 (generative_model.py:324-327)
    e = client.post("/openai/v1/completions", json={"model": "tiny", "prompt": m["prompt"][1], "max_tokens": 4, "echo": True}).json()
    assert e["choices"][0]["text"].startswith(m["prompt"][1])


def test_token_id_prompts_and_default_max_tokens(served):
    client, model, tok, c = served
    ids = load_case("tiny_g2_text")["input_ids"][1].tolist()          # no pads in row 1
    j = client.post("/openai/v1/completions", json={"model": "tiny", "prompt": ids}).json()
    assert j["usage"]["completion_tokens"] == 16                       # vLLM type default max_tokens=16 (q1)
    j2 = client.post("/openai/v1/completions", json={"model": "tiny", "prompt": [ids], "max_tokens": 16}).json()
    assert j2["choices"][0]["text"] == j["choices"][0]["text"]


def test_context_length_error_text(served):
    client, *_ = served
    r = client.post("/openai/v1/completions", json={"model": "tiny", "prompt": "hello", "max_tokens": 600})
    assert r.status_code == 500
    assert r.json()["error"]["message"] == (
        "This model's maximum context length is 512 tokens. However, you requested 605 tokens "
        "(5 in the messages, 600 in the completion). Please reduce the length of the messages or completion.")
    for bad in ({"frequency_penalty": 0.5}, {"n": 2}):
        assert client.post("/openai/v1/completions", json={"model": "tiny", "prompt": "x", **bad}).status_code == 500


def test_stop_string_sets_finish_reason_stop(served):
    client, model, tok, c = served
    prompt = "KServe on B200!"
    ids = client.post("/v1/models/tiny:predict", json={"instances": [tok.encode(prompt)], "parameters": {"max_tokens": 12}}).json()["predictions"][0]
    full = client.post("/openai/v1/completions", json={"model": "tiny", "prompt": prompt, "max_tokens": 12}).json()
    # a stop string must survive decode -> encode (random weights emit arbitrary bytes): find such a token pair
    pos = next((i for i in range(1, 10) if tok.encode(tok.decode(ids[i:i + 2]), add_special_tokens=False) == ids[i:i + 2]
                and ids[i:i + 2] not in [ids[k:k + 2] for k in range(i)]), None)
    if pos is None:
        pytest.skip("no round-trippable token pair in this sample")
    stop = tok.decode(ids[pos:pos + 2])
    j = client.post("/openai/v1/completions", json={"model": "tiny", "prompt": prompt, "max_tokens": 12, "stop": stop}).json()
    assert j["choices"][0]["finish_reason"] == "stop"
    assert j["usage"]["completion_tokens"] == pos + 2 < full["usage"]["completion_tokens"]
    assert j["choices"][0]["text"] == tok.decode(ids[:pos + 2], skip_special_tokens=True)


def test_streaming_and_chat(served):
    client, model, tok, c = served
    body = {"model": "tiny", "prompt": "The quick brown fox", "max_tokens": 24}
    whole = client.post("/openai/v1/completions", json=body).json()["choices"][0]["text"]
    with client.stream("POST", "/openai/v1/completions", json={**body, "stream": True}) as r:
        lines = [l for l in r.iter_lines() if l]
    assert lines[-1] == "data: [DONE]"
    chunks = [json.loads(l[6:]) for l in lines[:-1]]
    assert "".join(ch["choices"][0]["text"] for ch in chunks) == whole
    assert len({ch["id"] for ch in chunks}) == 1
    chat = {"model": "tiny", "messages": [{"role": "user", "content": "hi"}], "max_tokens": 8}
    j = client.post("/openai/v1/chat/completions", json=chat).json()
    assert j["object"] == "chat.completion" and j["choices"][0]["message"]["role"] == "assistant"
    direct = client.post("/openai/v1/completions", json={"model": "tiny", "prompt": "<|user|>hi\n<|assistant|>", "max_tokens": 8}).json()
    assert j["choices"][0]["message"]["content"] == direct["choices"][0]["text"]


def test_v1_predict_and_v2_infer(served):
    client, model, tok, c = served
    m = c["meta"]
    r = client.post("/v1/models/tiny:predict", json={"instances": m["prompt"], "parameters": {"max_tokens": m["max_tokens"]}})
    assert r.status_code == 200 and r.json()["predictions"] == m["texts"]
    rows = [tok.encode(p) for p in m["prompt"]]                      # ragged token-id instances -> left padded on device
    r = client.post("/v1/models/tiny:predict", json={"instances": rows, "parameters": {"max_tokens": m["max_tokens"]}})
    assert r.json()["predictions"] == c["gen"].tolist()
    ids = c["input_ids"].numpy()
    mask = c["mask"].numpy()
    hdr = json.dumps({"inputs": [{"name": "input_ids", "shape": list(ids.shape), "datatype": "INT64", "parameters": {"binary_data_size": ids.nbytes}},
                                 {"name": "attention_mask", "shape": list(mask.shape), "datatype": "INT64", "parameters": {"binary_data_size": mask.nbytes}}],
                      "parameters": {"max_tokens": m["max_tokens"], "binary_data_output": True}}).encode()
    r = client.post("/v2/models/tiny/infer", content=hdr + ids.tobytes() + mask.tobytes(),
                    headers={"Inference-Header-Content-Length": str(len(hdr))})
    assert r.status_code == 200, r.text
    n = int(r.headers["inference-header-content-length"])
    meta = json.loads(r.content[:n])
    out = meta["outputs"][0]
    got = np.frombuffer(r.content[n:n + out["parameters"]["binary_data_size"]], dtype=np.int64).reshape(out["shape"])
    assert np.array_equal(got, c["gen"].numpy())


def test_batcher_in_front_of_predict(served):
    """BASELINE config 5 in miniature: concurrent single-instance clients, one device batch, one batchId."""
    client, model, tok, c = served
    from kserve_b200.batcher import BatchHandler
    m = c["meta"]

    async def next_handler(path, body):
        body["parameters"] = {"max_tokens": m["max_tokens"]}
        return 200, await model.predict(body)

    async def main():
        h = BatchHandler(4, 200, next_handler)
        return await asyncio.gather(*[h.serve("/v1/models/tiny:predict", json.dumps({"instances": [p]}).encode()) for p in m["prompt"]])
    outs = asyncio.run(main())
    assert len({o[1]["batchId"] for o in outs}) == 1
    assert [o[1]["predictions"][0] for o in outs] == m["texts"]


def test_batch_predict_ragged_rows_equal_padded_generate(served):
    client, model, tok, c = served
    rows = [c["input_ids"][b][c["mask"][b].bool()].tolist() for b in range(c["input_ids"].shape[0])]
    pred, stop = model._engine.batch_predict(rows, max_new_tokens=c["T"], pad_token_id=256)
    ref = model._engine.generate(c["input_ids"], c["mask"], max_new_tokens=c["T"], pad_token_id=256)
    assert torch.equal(pred, ref.output_ids[:, c["S"]:]) and not stop


@pytest.mark.parametrize("ends", ["eos", "stop"])
def test_batch_predict_rows_ended_early_equal_padded_generate(served, ends):
    """As above when an EOS id or a stop sequence ends rows before max_new_tokens: the unpadded rows through
    b200_batch_predict give b200_generate's tokens on the left-padded batch, number of steps and stop flag included
    (a row that is done is filled with the pad id)."""
    client, model, tok, c = served
    eng, S, T, pad = model._engine, c["S"], c["T"], 256
    rows = [c["input_ids"][b][c["mask"][b].bool()].tolist() for b in range(c["input_ids"].shape[0])]
    free = eng.generate(c["input_ids"], c["mask"], max_new_tokens=T, pad_token_id=pad).output_ids[:, S:]
    kw = {"eos_token_ids": [int(free[1, 2])]} if ends == "eos" else {"stop_sequences": [free[0, 3:5].tolist()]}
    pred, stop = eng.batch_predict(rows, max_new_tokens=T, pad_token_id=pad, **kw)
    ref = eng.generate(c["input_ids"], c["mask"], max_new_tokens=T, pad_token_id=pad, **kw)
    if ends == "eos":        # row 1 emits the EOS id by step 2, then pads
        row = ref.output_ids[1, S:].tolist()
        first = row.index(kw["eos_token_ids"][0])
        assert first <= 2 and all(t == pad for t in row[first + 1:])
    else:
        assert ref.stop_triggered and ref.num_generated < T
    assert pred.shape[1] == ref.num_generated and stop == ref.stop_triggered == (ends == "stop")
    assert torch.equal(pred, ref.output_ids[:, S:])


def test_enable_batcher_served_over_http(served):
    """--enable_batcher on the served path (VERDICT r01 #7): the batcher sits in front of /v1/models/{m}:predict
    (cmd/agent/main.go:431-433), concurrent requests are merged and run as ONE b200_batch_predict call over
    their ragged rows, every caller gets its own slice under a shared batchId
    (test/e2e/batcher/test_batcher.py:33-85)."""
    import concurrent.futures
    from kserve_b200.kserve_api import ModelServer
    _, model, tok, c = served
    rows = [c["input_ids"][b][c["mask"][b].bool()].tolist() for b in range(c["input_ids"].shape[0])]
    want = model._engine.generate(c["input_ids"], c["mask"], max_new_tokens=16, pad_token_id=256).output_ids[:, c["S"]:]
    calls = []
    orig = model._engine.batch_predict
    model._engine.batch_predict = lambda r, **kw: (calls.append(len(r)), orig(r, **kw))[1]
    try:
        with TestClient(ModelServer(batcher=(len(rows), 2000)).create_application([model])) as client:
            with concurrent.futures.ThreadPoolExecutor(len(rows)) as ex:
                rs = list(ex.map(lambda row: client.post("/v1/models/tiny:predict", json={"instances": [row]}), rows))
            assert all(r.status_code == 200 for r in rs), [r.text for r in rs]
            js = [r.json() for r in rs]
            assert len({j["batchId"] for j in js}) == 1 and all(j["message"] == "" for j in js)
            assert calls == [len(rows)]                                   # one engine call for the formed batch
            for b, j in enumerate(js):                                    # the batcher forwards instances only: 16 = default max_tokens
                assert j["predictions"] == [want[b].tolist()]
    finally:
        model._engine.batch_predict = orig


def test_grpc_model_infer_on_the_cuda_engine(served):
    """Open Inference Protocol gRPC `ModelInfer` (python/kserve/kserve/protocol/grpc/servicer.py:109-127) against the real
    engine: INT64 token ids in as raw bytes, generated ids out as raw bytes — the same tensors as the V2 REST leg."""
    import grpc
    from kserve_b200.kserve_api.protocol.grpc import GRPCServer, pb
    from kserve_b200.kserve_api.protocol.rest.openai.dataplane import OpenAIDataPlane
    from kserve_b200.kserve_api.model_repository import ModelRepository
    _, model, tok, c = served
    ids, mask = c["input_ids"].numpy(), c["mask"].numpy()

    async def main():
        repo = ModelRepository()
        repo.update(model)
        srv = await GRPCServer(0, OpenAIDataPlane(model_registry=repo), host="127.0.0.1").start()
        try:
            async with grpc.aio.insecure_channel(f"127.0.0.1:{srv.bound_port}") as ch:
                infer = ch.unary_unary(f"/{pb.SERVICE_NAME}/ModelInfer", request_serializer=pb.ModelInferRequest.SerializeToString,
                                       response_deserializer=pb.ModelInferResponse.FromString)
                req = pb.ModelInferRequest(model_name="tiny", id="g1", inputs=[
                    {"name": "input_ids", "shape": list(ids.shape), "datatype": "INT64"},
                    {"name": "attention_mask", "shape": list(mask.shape), "datatype": "INT64"}],
                    raw_input_contents=[ids.tobytes(), mask.tobytes()])
                req.parameters["max_tokens"].int64_param = c["meta"]["max_tokens"]
                return await infer(req)
        finally:
            await srv.stop(0)
    res = asyncio.run(main())
    assert res.model_name == "tiny" and res.id == "g1"
    out = res.outputs[0]
    assert out.name == "output_ids" and out.datatype == "INT64"
    got = np.frombuffer(res.raw_output_contents[0], dtype=np.int64).reshape(list(out.shape))
    assert np.array_equal(got, c["gen"].numpy())
