"""BASELINE.json configs[4]: batcher maxBatchSize=64 maxLatency=50ms fronting Llama-3-8B on 1xH100, 512 concurrent
closed-loop clients, one instance (one ragged token-id prompt, U[512,1024] tokens) per request.

The Go sidecar cannot be built here (no Go toolchain): the same trigger state machine (C ABI b200_batcher_*) is
driven by the Python BatchHandler; the downstream call is one b200_batch_predict per formed batch.
Reports tokens/s, request latency and TTFT percentiles and the mean formed batch size."""
import asyncio
import json
import os
import random
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import LLAMA3_8B, gpu_weights  # noqa: E402
from kserve_b200.batcher import BatchHandler  # noqa: E402
from kserve_b200.engine import B200Engine  # noqa: E402


def main():
    clients = int(os.environ.get("CLIENTS", "512"))
    duration = float(os.environ.get("DURATION", "30"))
    max_new = int(os.environ.get("MAX_TOKENS", "128"))
    cfg = LLAMA3_8B
    eng = B200Engine(cfg, max_batch=64, max_seq_len=1024 + max_new, max_prefill_tokens=64 * 1024)
    eng.load_weights(gpu_weights(cfg, torch.device("cuda")))
    pool = ThreadPoolExecutor(max_workers=1)       # the engine is serial, like the reference's worker thread
    batches = []

    def run_batch(rows):
        t0 = time.perf_counter()
        pred, _ = eng.batch_predict(rows, max_new_tokens=max_new, pad_token_id=cfg["vocab_size"] - 1)
        tm = eng.lib  # timing of this call
        from kserve_b200 import _lib
        import ctypes as C
        t = _lib.Timing()
        eng.lib.b200_engine_last_timing(eng.h, C.byref(t))
        batches.append(dict(start=t0, size=len(rows), prefill_ms=t.prefill_ms, decode_ms=t.decode_ms, wall=time.perf_counter() - t0))
        return pred.tolist()

    async def next_handler(path, body):
        loop = asyncio.get_running_loop()
        # a fired batch may exceed 64 instances (handler.go appends whole requests): the engine takes <= 64 per call
        inst = body["instances"]
        out = []
        for i in range(0, len(inst), 64):
            out += await loop.run_in_executor(pool, run_batch, inst[i:i + 64])
        return 200, {"predictions": out}

    lat, ttft = [], []
    done_tokens = 0
    stop_at = None
    mode = os.environ.get("MODE", "batcher")
    if mode == "continuous":
        # SURVEY.md §8(f) rank 1: the same 512 closed-loop clients, served by the iteration-level scheduler
        from kserve_b200.continuous import ContinuousBatcher
        cb = ContinuousBatcher(eng, pad_token_id=cfg["vocab_size"] - 1, eos_token_ids=[], steps_per_poll=int(os.environ.get("STEPS_PER_POLL", "4")))
        cb.start()

        async def cclient(i):
            nonlocal done_tokens
            rng = random.Random(i)
            while time.perf_counter() < stop_at:
                n = rng.randint(512, 1024)
                row = [rng.randint(3, 127999) for _ in range(n)]
                first = []
                t0 = time.perf_counter()
                r = await cb.submit([row], torch.tensor([row]), max_new, on_tokens=lambda s, t: first.append(time.perf_counter()) if s == 0 else None)
                t1 = time.perf_counter()
                assert r.num_generated == max_new
                lat.append(t1 - t0)
                ttft.append(first[0] - t0)
                done_tokens += max_new

        async def cmain():
            nonlocal stop_at
            await cb.submit([[5] * 600] * 64, torch.full((64, 600), 5), 8)      # warm-up (graphs for 64 rows)
            t0 = time.perf_counter()
            stop_at = t0 + duration
            await asyncio.gather(*[cclient(i) for i in range(clients)])
            return time.perf_counter() - t0
        elapsed = asyncio.run(cmain())
        cb.stop()
        q = lambda xs, p: sorted(xs)[min(len(xs) - 1, int(p * len(xs)))]
        st = cb.stats
        res = dict(config="continuous batching, 64 slots, %d closed-loop clients, 1 prompt U[512,1024] tokens, %d new tokens" % (clients, max_new),
                   seconds=round(elapsed, 2), requests=len(lat), output_tokens_per_s=round(done_tokens / elapsed, 1),
                   request_latency_s=dict(p50=round(q(lat, .5), 3), p99=round(q(lat, .99), 3)),
                   ttft_s=dict(p50=round(q(ttft, .5), 3), p99=round(q(ttft, .99), 3)),
                   prefill_calls=int(st["prefill_calls"]), decode_steps=int(st["decode_steps"]),
                   mean_rows_per_step=round(st["row_steps"] / max(1, st["decode_steps"]), 2))
        print(json.dumps(res))
        os.makedirs("gpurun_out", exist_ok=True)
        json.dump(res, open("gpurun_out/continuous_load.json", "w"), indent=1)
        return

    async def client(i, handler):
        nonlocal done_tokens
        rng = random.Random(i)
        while time.perf_counter() < stop_at:
            n = rng.randint(512, 1024)
            row = [rng.randint(3, 127999) for _ in range(n)]
            t0 = time.perf_counter()
            code, resp = await handler.serve("/v1/models/llama:predict", json.dumps({"instances": [row]}).encode())
            t1 = time.perf_counter()
            assert code == 200 and resp["message"] == "" and len(resp["predictions"][0]) == max_new
            lat.append(t1 - t0)
            # first token of this request = end of the prefill of the device batch that served it
            b = max((b for b in batches if b["start"] <= t1), key=lambda b: b["start"])
            ttft.append(b["start"] + b["prefill_ms"] / 1e3 - t0)
            done_tokens += max_new

    async def main_async():
        nonlocal stop_at
        handler = BatchHandler(64, 50, next_handler)
        # warm-up batch (graph capture etc.)
        await handler.serve("/v1/models/llama:predict", json.dumps({"instances": [[5] * 600] * 64}).encode())
        batches.clear()
        t0 = time.perf_counter()
        stop_at = t0 + duration
        await asyncio.gather(*[client(i, handler) for i in range(clients)])
        return time.perf_counter() - t0

    elapsed = asyncio.run(main_async())
    q = lambda xs, p: sorted(xs)[min(len(xs) - 1, int(p * len(xs)))]
    res = dict(config="batcher maxBatchSize=64 maxLatency=50ms, %d closed-loop clients, 1 instance U[512,1024] tokens, %d new tokens" % (clients, max_new),
               seconds=round(elapsed, 2), requests=len(lat), output_tokens_per_s=round(done_tokens / elapsed, 1),
               request_latency_s=dict(p50=round(q(lat, .5), 3), p99=round(q(lat, .99), 3)),
               ttft_s=dict(p50=round(q(ttft, .5), 3), p99=round(q(ttft, .99), 3)),
               device_batches=len(batches), mean_batch_size=round(statistics.mean(b["size"] for b in batches), 2),
               mean_prefill_ms=round(statistics.mean(b["prefill_ms"] for b in batches), 1),
               mean_decode_ms=round(statistics.mean(b["decode_ms"] for b in batches), 1))
    print(json.dumps(res))
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(res, open("gpurun_out/batcher_load.json", "w"), indent=1)


if __name__ == "__main__":
    main()
