"""BASELINE.json configs[4] over HTTP: 512 concurrent closed-loop clients against the real model server (uvicorn +
FastAPI routes of kserve_b200.kserve_api) fronting Llama-3-8B dims (random init) on one H100.

    MODE=continuous  POST /openai/v1/completions (token-id prompts) served by the iteration-level scheduler
                     (--continuous_batching, chunked prefill, up to SLOTS resident sequences)
    MODE=batcher     POST /v1/models/llama:predict behind --enable_batcher (maxBatchSize 64, maxLatency 50 ms): formed
                     batches run as one b200_batch_predict call, like the Go agent + predictor

Every request carries one ragged prompt of U[512,1024] token ids and asks for 128 new tokens.  Latency is measured at the
client (aiohttp); TTFT is taken where the first token becomes available to the server (scheduler: submit -> first token;
batcher: arrival -> end of the prefill of the device batch that served the request), i.e. without the response framing."""
import asyncio
import json
import os
import random
import sys
import threading
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import LLAMA3_8B, gpu_weights  # noqa: E402


def main():
    import aiohttp
    import uvicorn
    from kserve_b200.generative_model import B200GenerativeModel
    from kserve_b200.kserve_api import ModelServer
    clients = int(os.environ.get("CLIENTS", "512"))
    duration = float(os.environ.get("DURATION", "40"))
    max_new = int(os.environ.get("MAX_TOKENS", "128"))
    mode = os.environ.get("MODE", "continuous")
    slots = int(os.environ.get("SLOTS", "512" if mode == "continuous" else "64"))
    chunk = int(os.environ.get("CHUNK", "8192"))
    port = int(os.environ.get("PORT", "18080"))
    cfg = dict(LLAMA3_8B, architectures=["LlamaForCausalLM"], model_type="llama")
    model = B200GenerativeModel("llama", model_config=cfg, state_dict=gpu_weights(LLAMA3_8B, torch.device("cuda")), tokenizer=None,
                                pad_token_id=cfg["vocab_size"] - 1, max_model_len=1024 + max_new, max_batch=slots,
                                continuous_batching=(mode == "continuous"))
    model.prefill_chunk_tokens = chunk
    if os.environ.get("KV_PAGES"):      # over-subscribe the pool: admissions preempt running requests to the host-DRAM KV tier
        model.kv_pages_limit = int(os.environ["KV_PAGES"])
    model.load()
    server = ModelServer(http_port=port, batcher=(64, 50) if mode == "batcher" else None)
    app = server.create_application([model])
    uv = uvicorn.Server(uvicorn.Config(app, host="127.0.0.1", port=port, log_level="warning", access_log=False))
    th = threading.Thread(target=uv.run, daemon=True)
    th.start()
    while not uv.started:
        time.sleep(0.05)
    ttft_batches = []
    if mode == "batcher":       # TTFT of a batched request = arrival -> end of the prefill of its device batch
        orig = model._engine.batch_predict

        def timed(rows, **kw):
            t0 = time.perf_counter()
            out = orig(rows, **kw)
            ttft_batches.append((t0, model._engine.last_timing().prefill_ms / 1e3, time.perf_counter()))
            return out
        model._engine.batch_predict = timed
    lat, ttft = [], []
    done = [0]

    async def run():
        conn = aiohttp.TCPConnector(limit=0)
        async with aiohttp.ClientSession(connector=conn, timeout=aiohttp.ClientTimeout(total=600)) as sess:
            async def one(rng):
                n = rng.randint(512, 1024)
                row = [rng.randint(3, 127999) for _ in range(n)]
                t0 = time.perf_counter()
                if mode == "continuous":
                    async with sess.post(f"http://127.0.0.1:{port}/openai/v1/completions",
                                         json={"model": "llama", "prompt": row, "max_tokens": max_new}) as r:
                        j = await r.json()
                        assert r.status == 200, j
                        assert j["usage"]["completion_tokens"] == max_new
                else:
                    async with sess.post(f"http://127.0.0.1:{port}/v1/models/llama:predict", json={"instances": [row]}) as r:
                        j = await r.json()
                        assert r.status == 200 and j["message"] == "" and len(j["predictions"][0]) == 16, j
                t1 = time.perf_counter()
                return t0, t1
            # warm-up: graphs for the row counts that will occur
            await asyncio.gather(*[one(random.Random(1000 + i)) for i in range(64)])
            if model._cb is not None:
                model._cb.ttft_samples.clear()
            ttft_batches.clear()
            t_start = time.perf_counter()
            stop_at = t_start + duration

            async def client(i):
                rng = random.Random(i)
                while time.perf_counter() < stop_at:
                    t0, t1 = await one(rng)
                    lat.append(t1 - t0)
                    done[0] += max_new if mode == "continuous" else 16
                    if mode == "batcher":
                        b = max((b for b in ttft_batches if b[0] <= t1), key=lambda b: b[0])
                        ttft.append(b[0] + b[1] - t0)
            await asyncio.gather(*[client(i) for i in range(clients)])
            return time.perf_counter() - t_start
    elapsed = asyncio.run(run())
    if model._cb is not None:
        ttft = list(model._cb.ttft_samples)
    q = lambda xs, p: round(sorted(xs)[min(len(xs) - 1, int(p * len(xs)))], 3) if xs else None
    res = dict(config=f"HTTP, mode={mode}, {clients} closed-loop clients, 1 prompt U[512,1024] token ids, "
                      f"{max_new if mode == 'continuous' else 16} new tokens, slots={slots}" + (f", KV pool limited to {os.environ['KV_PAGES']} pages" if os.environ.get("KV_PAGES") else "") + (f", prefill chunks {chunk}" if mode == "continuous" else ", maxBatchSize 64 / maxLatency 50 ms"),
               seconds=round(elapsed, 2), requests=len(lat), output_tokens_per_s=round(done[0] / elapsed, 1),
               request_latency_s=dict(p50=q(lat, .5), p99=q(lat, .99)), ttft_s=dict(p50=q(ttft, .5), p99=q(ttft, .99)),
               scheduler=dict(model._cb.stats) if model._cb is not None else None,
               engine=model._engine.cb_stats() if model._cb is not None else None)
    print(json.dumps(res))
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(res, open(f"gpurun_out/r02_http_load_{mode}.json", "w"), indent=1)
    uv.should_exit = True
    th.join(timeout=10)
    model.stop()


if __name__ == "__main__":
    main()
