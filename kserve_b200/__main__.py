"""`python -m kserve_b200 --model_dir /mnt/models --model_name llama` — the entrypoint that replaces
`python -m huggingfaceserver --backend huggingface` (python/huggingfaceserver/huggingfaceserver/__main__.py:60-345)
for Llama-family decoders: same --model_id/--model_dir/--model_name/--max_model_len/--dtype flags, backend fixed to
the H100 engine (no vLLM / transformers dispatch), plus --tensor_parallel_size (one process per GPU under torchrun)."""
import argparse
import os
import sys

from .kserve_api import model_server
from .kserve_api.model_server import ModelServer


def main(argv=None):
    parser = argparse.ArgumentParser(parents=[model_server.parser])
    parser.add_argument("--model_dir", default="/mnt/models", help="HF checkpoint directory (config.json, *.safetensors, tokenizer)")
    parser.add_argument("--model_id", default=None, help="alias of --model_dir (no Hub access in this runtime)")
    parser.add_argument("--max_model_len", "--max_length", type=int, default=None)
    parser.add_argument("--dtype", default="auto", choices=["auto", "float16", "float32", "bfloat16", "float", "half"],
                        help="the reference's choices (__main__.py:195-210); the H100 engine computes in bfloat16, which is what "
                             "'auto' and 'bfloat16' select — the other values are refused at start-up rather than silently "
                             "served at a different precision")
    parser.add_argument("--backend", default="b200", choices=["b200"])
    parser.add_argument("--max_batch", type=int, default=32)
    parser.add_argument("--continuous_batching", action="store_true",
                        help="iteration-level batching: requests join / leave the running decode batch between steps")
    parser.add_argument("--prefill_chunk_tokens", type=int, default=8192,
                        help="with --continuous_batching: prompts are prefilled in chunks of this many tokens between decode steps (0 = whole prompts at admit)")
    parser.add_argument("--enable_prefix_caching", action="store_true",
                        help="with --continuous_batching: share the KV pages of common 128-token prompt prefixes between requests")
    parser.add_argument("--kv_cache_dtype", default="auto", choices=["auto", "bfloat16", "fp8", "fp8_e4m3", "fp8_e5m2"],
                        help="KV cache element type: auto / bfloat16 = bf16 pages; fp8 / fp8_e4m3 = float8_e4m3fn codes (per-tensor "
                             "scale 1), half the bytes per cached token (fp8_e5m2 is refused)")
    parser.add_argument("--tensor_parallel_size", type=int, default=int(os.environ.get("WORLD_SIZE", "1")))
    # the agent's flags (cmd/agent/main.go:66-68 --enable-batcher / --max-batchsize / --max-latency), same defaults
    parser.add_argument("--enable_batcher", "--enable-batcher", dest="enable_batcher", action="store_true",
                        help="install the request batcher in front of V1 :predict (pkg/batcher), formed batches run as one engine call")
    parser.add_argument("--max-batchsize", "--max_batchsize", dest="max_batchsize", type=int, default=32)
    parser.add_argument("--max-latency", "--max_latency", dest="max_latency", type=int, default=5000)
    args, _ = parser.parse_known_args(argv)
    if args.dtype not in ("auto", "bfloat16"):
        parser.error(f"--dtype {args.dtype}: the H100 runtime computes in bfloat16 only (use --dtype auto or bfloat16)")
    if args.kv_cache_dtype == "fp8_e5m2":
        parser.error("--kv_cache_dtype fp8_e5m2 is not supported: the FP8 KV cache is float8_e4m3fn (use fp8 or fp8_e4m3)")
    if args.enable_batcher and (args.max_batchsize <= 0 or args.max_latency <= 0):
        parser.error("Invalid max batch size / max latency")        # cmd/agent/main.go:256-273
    from .generative_model import B200GenerativeModel
    path = args.model_id or args.model_dir
    nccl_id, rank = None, int(os.environ.get("RANK", "0"))
    if args.tensor_parallel_size > 1:
        import torch
        import torch.distributed as dist
        from .tp import broadcast_nccl_id
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("gloo")
        nccl_id = broadcast_nccl_id(rank)
    if args.enable_batcher:
        args.max_batch = max(args.max_batch, min(args.max_batchsize, 64))     # a formed batch must fit one engine call
    model = B200GenerativeModel(args.model_name, path, max_model_len=args.max_model_len, max_batch=args.max_batch,
                                device=int(os.environ.get("LOCAL_RANK", "0")), tensor_parallel_size=args.tensor_parallel_size,
                                tp_rank=rank, nccl_id=nccl_id, continuous_batching=args.continuous_batching,
                                kv_cache_dtype=args.kv_cache_dtype)
    model.prefill_chunk_tokens, model.prefix_cache = max(0, args.prefill_chunk_tokens), args.enable_prefix_caching
    model.load()
    if rank != 0:
        from .tp import follower_loop
        return follower_loop(model)
    ModelServer(http_port=args.http_port, enable_latency_logging=args.enable_latency_logging, grpc_port=args.grpc_port,
                enable_grpc=args.enable_grpc,
                batcher=(args.max_batchsize, args.max_latency) if args.enable_batcher else None).start([model])


if __name__ == "__main__":
    sys.exit(main())
