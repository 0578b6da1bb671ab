"""The whole host path of the runtime model without a GPU: B200GenerativeModel wired to a scripted engine
(`generate()` returns prompt + a deterministic continuation), driven through the REST routes, the V2 binary leg and gRPC.
What the CUDA engine computes is covered by the `-m gpu` tests; this pins everything around it: tokenisation and left
padding, usage accounting (q3), echo, stop -> finish_reason, SSE framing, chat re-wrap, V1 / V2 / gRPC envelopes."""
import asyncio
import json
import os
from threading import Thread

import numpy as np
import pytest
import torch
from fastapi.testclient import TestClient

from helpers import GOLDEN
from kserve_b200.engine import GenerateResult
from kserve_b200.generative_model import B200GenerativeModel
from kserve_b200.kserve_api import ModelServer


class ScriptedEngine:
    """continuation token k of a row = (last prompt token + 1 + k) mod 250 + 3: printable-ish bytes for the byte tokenizer"""
    max_batch, max_seq_len = 8, 512

    def __init__(self):
        self.calls = []

    def generate(self, ids, mask=None, *, max_new_tokens, pad_token_id=0, eos_token_ids=(), stop_sequences=(), streamer=None, **kw):
        self.calls.append(dict(shape=tuple(ids.shape), mask=None if mask is None else mask.sum(1).tolist(), max_new=max_new_tokens,
                               stops=[list(s) for s in stop_sequences], extra=kw))
        last = ids[:, -1]
        gen = torch.stack([(last + 1 + k) % 250 + 3 for k in range(max_new_tokens)], 1)
        n, stopped = max_new_tokens, False
        for k in range(1, max_new_tokens + 1):            # batch-wide stop sequences, like the device kernel
            for s in stop_sequences:
                if len(s) and k >= len(s) and any(gen[b, k - len(s):k].tolist() == list(s) for b in range(gen.shape[0])):
                    n, stopped = k, True
            if stopped:
                break
        gen = gen[:, :n]
        if streamer is not None:
            for k in range(n):
                streamer(k, gen[:, k].tolist())
        return GenerateResult(output_ids=torch.cat([ids, gen], 1), stop_triggered=stopped, num_generated=n, logits=None,
                              prefill_ms=1.0, decode_ms=1.0, decode_steps=max(0, n - 1), kernel_launches=0)

    def batch_predict(self, rows, *, max_new_tokens, pad_token_id=0, eos_token_ids=(), stop_sequences=()):
        """ragged rows in, predictions [n_rows, T] out (b200_batch_predict): same script as generate, no padding involved"""
        self.calls.append(dict(batch_predict=[len(r) for r in rows], max_new=max_new_tokens))
        last = torch.tensor([r[-1] for r in rows])
        return torch.stack([(last + 1 + k) % 250 + 3 for k in range(max_new_tokens)], 1), False

    def last_timing(self):
        from kserve_b200._lib import Timing
        return Timing(prefill_ms=1.0, decode_ms=1.0, decode_steps=1, kernel_launches=0)

    def close(self):
        pass


@pytest.fixture(scope="module")
def served():
    from transformers import AutoTokenizer
    tok = AutoTokenizer.from_pretrained(os.path.join(GOLDEN, "byte_tokenizer"), padding_side="left")
    m = B200GenerativeModel("stub", model_config={"vocab_size": 257}, tokenizer=tok, max_model_len=512, max_batch=8)
    # what load() sets up, minus the CUDA engine
    if not tok.pad_token:
        tok.add_special_tokens({"pad_token": "[PAD]"})
    m._pad_token_id, m.eos_token_ids, m.generation_defaults, m.vocab_rows = tok.pad_token_id, [], {}, len(tok)
    m._engine = ScriptedEngine()
    m._thread = Thread(target=m._process_requests, daemon=True)
    m._thread.start()
    m.ready = True
    with TestClient(ModelServer().create_application([m])) as client:
        yield client, m, tok
    m._request_queue.put(None)


def _continuation(tok, prompt, n):
    last = tok.encode(prompt)[-1]
    return [(last + 1 + k) % 250 + 3 for k in range(n)]


def test_completion_usage_echo_and_ragged_batch(served):
    client, m, tok = served
    prompts = ["Hello world", "a"]
    r = client.post("/openai/v1/completions", json={"model": "stub", "prompt": prompts, "max_tokens": 5})
    assert r.status_code == 200, r.text
    j = r.json()
    S = max(len(tok.encode(p)) for p in prompts)
    assert j["usage"] == {"prompt_tokens": S * 2, "completion_tokens": 10, "total_tokens": S * 2 + 10}      # q3: pads are counted
    assert [c["text"] for c in j["choices"]] == [tok.decode(_continuation(tok, p, 5), skip_special_tokens=True) for p in prompts]
    assert all(c["finish_reason"] == "length" and "logprobs" not in c for c in j["choices"])
    call = m._engine.calls[-1]
    assert call["shape"] == (2, S) and call["mask"] == [len(tok.encode(p)) for p in prompts]              # left padded
    e = client.post("/openai/v1/completions", json={"model": "stub", "prompt": "Hello", "max_tokens": 3, "echo": True}).json()
    assert e["choices"][0]["text"].startswith("Hello")


def test_stop_string_finish_reason_and_default_max_tokens(served):
    client, m, tok = served
    # a prompt whose continuation bytes survive decode -> encode (the byte tokenizer does not round-trip invalid UTF-8)
    prompt = next(p for p in ("xy" + chr(c) for c in range(33, 100))
                  if tok.encode(tok.decode(_continuation(tok, p, 16)[3:5]), add_special_tokens=False) == _continuation(tok, p, 16)[3:5])
    cont = _continuation(tok, prompt, 16)
    stop = tok.decode(cont[3:5])
    j = client.post("/openai/v1/completions", json={"model": "stub", "prompt": prompt, "stop": stop}).json()
    assert j["choices"][0]["finish_reason"] == "stop" and j["usage"]["completion_tokens"] == 5
    assert m._engine.calls[-1]["stops"] == [tok.encode(stop, add_special_tokens=False)] and m._engine.calls[-1]["max_new"] == 16   # q1
    j = client.post("/openai/v1/completions", json={"model": "stub", "prompt": "xyz", "max_tokens": None}).json()
    assert j["usage"]["completion_tokens"] == 512 - 3                                                       # max_length - S (:563-564)


def test_sse_stream_and_chat(served):
    client, m, tok = served
    whole = client.post("/openai/v1/completions", json={"model": "stub", "prompt": "abc", "max_tokens": 12}).json()["choices"][0]["text"]
    with client.stream("POST", "/openai/v1/completions", json={"model": "stub", "prompt": "abc", "max_tokens": 12, "stream": True}) as r:
        assert r.headers["content-type"].startswith("text/event-stream")
        lines = [l for l in r.iter_lines() if l]
    assert lines[-1] == "data: [DONE]"
    chunks = [json.loads(l[6:]) for l in lines[:-1]]
    assert "".join(c["choices"][0]["text"] for c in chunks) == whole and len({c["id"] for c in chunks}) == 1
    chat = {"model": "stub", "messages": [{"role": "user", "content": "hi"}], "max_tokens": 4}
    j = client.post("/openai/v1/chat/completions", json=chat).json()
    assert j["object"] == "chat.completion" and j["choices"][0]["message"]["role"] == "assistant"
    direct = client.post("/openai/v1/completions", json={"model": "stub", "prompt": "<|user|>hi\n<|assistant|>", "max_tokens": 4}).json()
    assert j["choices"][0]["message"]["content"] == direct["choices"][0]["text"]


def test_v1_v2_binary_and_grpc_envelopes(served):
    client, m, tok = served
    ids = np.array([[5, 6, 7], [8, 9, 10]], dtype=np.int64)
    want = [[(int(r[-1]) + 1 + k) % 250 + 3 for k in range(4)] for r in ids]
    r = client.post("/v1/models/stub:predict", json={"instances": ids.tolist(), "parameters": {"max_tokens": 4}})
    assert r.status_code == 200 and r.json()["predictions"] == want
    hdr = json.dumps({"inputs": [{"name": "input_ids", "shape": [2, 3], "datatype": "INT64", "parameters": {"binary_data_size": ids.nbytes}}],
                      "parameters": {"max_tokens": 4, "binary_data_output": True}}).encode()
    r = client.post("/v2/models/stub/infer", content=hdr + ids.tobytes(), headers={"Inference-Header-Content-Length": str(len(hdr))})
    assert r.status_code == 200, r.text
    n = int(r.headers["inference-header-content-length"])
    out = json.loads(r.content[:n])["outputs"][0]
    assert np.frombuffer(r.content[n:n + out["parameters"]["binary_data_size"]], dtype=np.int64).reshape(out["shape"]).tolist() == want

    import grpc
    from kserve_b200.kserve_api.model_repository import ModelRepository
    from kserve_b200.kserve_api.protocol.grpc import GRPCServer, pb
    from kserve_b200.kserve_api.protocol.rest.openai.dataplane import OpenAIDataPlane

    async def call():
        repo = ModelRepository()
        repo.update(m)
        srv = await GRPCServer(0, OpenAIDataPlane(model_registry=repo), host="127.0.0.1").start()
        try:
            async with grpc.aio.insecure_channel(f"127.0.0.1:{srv.bound_port}") as ch:
                infer = ch.unary_unary(f"/{pb.SERVICE_NAME}/ModelInfer", request_serializer=pb.ModelInferRequest.SerializeToString,
                                       response_deserializer=pb.ModelInferResponse.FromString)
                return await infer(pb.ModelInferRequest(model_name="stub", id="9", parameters={"max_tokens": {"int64_param": 4}},
                                                        inputs=[{"name": "input_ids", "shape": [2, 3], "datatype": "INT64"}],
                                                        raw_input_contents=[ids.tobytes()]))
        finally:
            await srv.stop(0)
    res = asyncio.run(call())
    by = {o.name: i for i, o in enumerate(res.outputs)}
    assert np.frombuffer(res.raw_output_contents[by["output_ids"]], dtype=np.int64).reshape(2, 4).tolist() == want
    assert res.id == "9" and "text" in by


class ScriptedCbEngine(ScriptedEngine):
    """the b200_cb_* surface with the same continuation rule, for the --continuous_batching wiring"""
    def __init__(self):
        super().__init__()
        self.slots, self.released = {}, []

    def cb_begin(self, pad, eos):
        pass

    def cb_end(self):
        pass

    def cb_admit(self, prompts, max_new, stops, sampling=None):
        out = []
        self.last_sampling = sampling
        for p, m_, ss in zip(prompts, max_new, stops):
            s = next(i for i in range(self.max_batch) if i not in self.slots)
            self.slots[s] = dict(last=p[-1], out=[], max_new=m_, fin=False)
            out.append(s)
        self.cb_step(1)
        return out

    def cb_step(self, n):
        import time
        time.sleep(0.002 * n)
        for _ in range(n):
            for st in self.slots.values():
                if not st["fin"]:
                    st["out"].append((st["last"] + 1 + len(st["out"])) % 250 + 3)
                    st["fin"] = len(st["out"]) >= st["max_new"]

    def cb_poll(self):
        get = lambda k, d: [self.slots[s][k] if s in self.slots else d for s in range(self.max_batch)]
        return [len(x) if isinstance(x, list) else 0 for x in get("out", [])], [int(x) for x in get("fin", 0)], [0] * self.max_batch

    def cb_read(self, slot, first=0, cap=4096):
        return self.slots[slot]["out"][first:first + cap]

    def cb_release(self, slot):
        self.released.append(slot)
        del self.slots[slot]


def test_continuous_batching_wiring_and_stream_disconnect(served):
    """--continuous_batching: completions and SSE streams go through the scheduler; a client that disconnects mid-stream
    frees its slot (the reference cannot abort a running generate, q10)."""
    from kserve_b200.continuous import ContinuousBatcher
    client, m, tok = served
    eng = ScriptedCbEngine()
    cb = ContinuousBatcher(eng, pad_token_id=m._pad_token_id, steps_per_poll=2)
    cb.start()
    m._cb = cb
    try:
        j = client.post("/openai/v1/completions", json={"model": "stub", "prompt": ["Hello world", "a"], "max_tokens": 5}).json()
        assert [c["text"] for c in j["choices"]] == [tok.decode(_continuation(tok, p, 5), skip_special_tokens=True) for p in ("Hello world", "a")]
        assert j["usage"]["completion_tokens"] == 10
        with client.stream("POST", "/openai/v1/completions", json={"model": "stub", "prompt": "abc", "max_tokens": 9, "stream": True}) as r:
            lines = [l for l in r.iter_lines() if l]
        assert lines[-1] == "data: [DONE]"
        assert "".join(json.loads(l[6:])["choices"][0]["text"] for l in lines[:-1]) == tok.decode(_continuation(tok, "abc", 9), skip_special_tokens=True)
        # logits processors ride along per sequence (round 2: b200_cb_admit takes per-sequence sampling parameters)
        assert client.post("/openai/v1/completions", json={"model": "stub", "prompt": "x", "presence_penalty": 1.5}).status_code == 200
        assert eng.last_sampling == [{"repetition_penalty": 1.5}]

        async def abandon():          # start a long stream, read one chunk, close the generator
            from kserve_b200.kserve_api.protocol.rest.openai.types import CompletionRequest
            gen = await m.create_completion(CompletionRequest(model="stub", prompt="abc", max_tokens=400, stream=True))
            first = await gen.__anext__()
            assert first.startswith("data: ")
            await gen.aclose()
            await asyncio.sleep(0.1)
        asyncio.run(abandon())
        assert cb.stats["cancelled"] == 1 and cb.free_slots == eng.max_batch and not eng.slots
    finally:
        m._cb = None
        cb.stop()


def test_enable_batcher_installs_batch_handler_in_front_of_predict(served):
    """--enable_batcher: concurrent V1 :predict requests are merged into ONE engine call (over all their
    ragged instances) and each caller gets {"message", "batchId", "predictions"} with its own slice — the wiring of
    cmd/agent/main.go:431-433 + pkg/batcher/handler.go:222-266; scenario of test/e2e/batcher/test_batcher.py:33-85
    (same batchId for requests that were batched together)."""
    import concurrent.futures
    _, m, tok = served
    app = ModelServer(batcher=(4, 200)).create_application([m])     # maxBatchSize 4 instances, maxLatency 200 ms
    with TestClient(app) as client:
        n0 = len(m._engine.calls)
        bodies = [{"instances": [[5, 6, 7]]}, {"instances": [[8, 9]]}, {"instances": [[1, 2, 3, 4], [9]]}]
        with concurrent.futures.ThreadPoolExecutor(3) as ex:
            rs = list(ex.map(lambda b: client.post("/v1/models/stub:predict", json=b), bodies))
        assert all(r.status_code == 200 for r in rs), [r.text for r in rs]
        js = [r.json() for r in rs]
        assert len({j["batchId"] for j in js}) == 1 and all(j["message"] == "" for j in js)          # one formed batch
        calls = m._engine.calls[n0:]
        assert len(calls) == 1 and sorted(calls[0]["batch_predict"]) == [1, 2, 3, 4]                # ONE engine call, ragged rows
        for b, j in zip(bodies, js):                                                                 # each caller gets its own rows back
            assert j["predictions"] == [[(row[-1] + 1 + k) % 250 + 3 for k in range(16)] for row in b["instances"]]
        # below the size trigger the latency trigger fires
        r = client.post("/v1/models/stub:predict", json={"instances": [[3, 4]]})
        assert r.status_code == 200 and len(r.json()["predictions"]) == 1 and r.json()["batchId"] != js[0]["batchId"]
        # handler.go:233-243
        assert client.post("/v1/models/stub:predict", content=b"{not json").status_code == 400
        r = client.post("/v1/models/stub:predict", json={"instances": []})
        assert r.status_code == 400 and "no instances in the request" in r.text
        # a failing downstream answers 200 with the message set and predictions null (handler.go:108-117)
        r = client.post("/v1/models/stub:predict", json={"instances": [["not", "ids", 1]]})
        assert r.status_code == 200 and r.json()["predictions"] is None and r.json()["message"]


def test_logit_bias_reproduces_the_reference_error(served):
    """q8: the reference turns logit_bias into sequence_bias keyed by tuple(str) (generative_model.py:396-401), which
    transformers' SequenceBiasLogitsProcessor rejects inside generate(): the request fails with that ValueError."""
    _, m, tok = served
    client = TestClient(served[0].app, raise_server_exceptions=False)     # the 500 itself is what is being asserted
    n0 = len(m._engine.calls)
    r = client.post("/openai/v1/completions", json={"model": "stub", "prompt": "abc", "max_tokens": 3, "logit_bias": {"123": 5.0}})
    assert r.status_code == 500
    assert "Each key in `sequence_bias` has to be a non-empty tuple of positive integers, but is {('1', '2', '3'): 5.0}." in r.text
    r = client.post("/openai/v1/completions", json={"model": "stub", "prompt": "abc", "max_tokens": 3, "logit_bias": {}})
    assert r.status_code == 500 and "`sequence_bias` has to be a non-empty dictionary" in r.text
    assert len(m._engine.calls) == n0          # nothing reached the engine, as nothing is generated in the reference


def test_predict_rejects_bad_user_parameters_with_400(served):
    """ADVICE r01 (low): user errors of the V1 / V2 predict legs are 400s, not 500s from inside the engine."""
    client, m, tok = served
    r = client.post("/v1/models/stub:predict", json={"instances": [[5, 6, 7]], "parameters": {"max_tokens": 0}})
    assert r.status_code == 400 and "max_tokens" in r.text
    r = client.post("/v1/models/stub:predict", json={"instances": [[5, 6, 7]], "parameters": {"max_tokens": "many"}})
    assert r.status_code == 400
    r = client.post("/v1/models/stub:predict", json={"instances": [[5] * 10], "parameters": {"max_tokens": 510}})
    assert r.status_code == 400 and "maximum context length" in r.text
    ids = {"name": "input_ids", "shape": [2, 3], "datatype": "INT64", "data": [1, 2, 3, 4, 5, 6]}
    bad_mask = {"name": "attention_mask", "shape": [2, 2], "datatype": "INT64", "data": [1, 1, 1, 1]}
    r = client.post("/v2/models/stub/infer", json={"inputs": [ids, bad_mask]})
    assert r.status_code == 400 and "attention_mask shape" in r.text
    holes = {"name": "attention_mask", "shape": [2, 3], "datatype": "INT64", "data": [1, 0, 1, 0, 1, 1]}
    r = client.post("/v2/models/stub/infer", json={"inputs": [ids, holes]})
    assert r.status_code == 400 and "left padding" in r.text
