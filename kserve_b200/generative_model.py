"""B200GenerativeModel — drop-in for the reference's ``HuggingfaceGenerativeModel``
(python/huggingfaceserver/huggingfaceserver/generative_model.py:143-646) behind the same
``OpenAIChatAdapterModel`` plug-in API, plus the ``kserve.Model.predict()`` leg the north star adds for
V1 ``:predict`` (what the Go batcher fronts) and V2 ``/infer``.

Request semantics follow the reference line by line (cited inline, SURVEY.md §8a' q1-q13); the one call that
differs is the compute: where the reference runs ``self._model.generate(**kwargs)`` (:314, :328) on
transformers, this model calls the CUDA engine through the C ABI.  There is no CPU / transformers fallback.
"""
from __future__ import annotations

import asyncio
import json
import os
import queue
import time
import uuid
from threading import Thread
from typing import Any, AsyncGenerator, Dict, Iterable, List, Optional, Tuple, Union

import numpy as np
import torch

from .engine import B200Engine, GenerateResult
from .fp8 import UnsupportedQuantization, kv_cache_format, log_activation_scheme, parse_quantization_config
from .utils import get_and_verify_max_len, logger, plan_memory, rope_inv_freq
from .kserve_api.errors import InvalidInput
from .kserve_api.metrics import DECODE_TOKENS_PER_S, LLM_STATS_KEY, TTFT_HIST, LLMStats, get_labels
from .kserve_api.model import Model
from .kserve_api.protocol.infer_type import InferOutput, InferRequest, InferResponse
from .kserve_api.protocol.rest.openai.errors import OpenAIError
from .kserve_api.protocol.rest.openai.openai_chat_adapter_model import OpenAIChatAdapterModel
from .kserve_api.protocol.rest.openai.openai_model import ChatPrompt
from .kserve_api.protocol.rest.openai.types import (ChatCompletionRequest, Completion, CompletionChoice,
                                                    CompletionChunk, CompletionChunkChoice, CompletionRequest,
                                                    ErrorResponse, UsageInfo, generate_uuid)


class IncrementalDetokenizer:
    """Text pieces exactly as transformers' TextIteratorStreamer emits them (what the reference streams,
    generative_model.py:307-322): decode the token cache, flush on newline, otherwise hold back the last
    partial word; batch size 1 only (TextStreamer raises for more)."""

    def __init__(self, tokenizer, skip_special_tokens: bool = True):
        self.tok, self.kw = tokenizer, dict(skip_special_tokens=skip_special_tokens)
        self.cache: List[int] = []
        self.print_len = 0

    @staticmethod
    def _is_cjk(cp: int) -> bool:
        return (0x4E00 <= cp <= 0x9FFF or 0x3400 <= cp <= 0x4DBF or 0x20000 <= cp <= 0x2A6DF or 0x2A700 <= cp <= 0x2B73F
                or 0x2B740 <= cp <= 0x2B81F or 0x2B820 <= cp <= 0x2CEAF or 0xF900 <= cp <= 0xFAFF or 0x2F800 <= cp <= 0x2FA1F)

    def put(self, tokens: List[int]) -> str:
        self.cache.extend(tokens)
        text = self.tok.decode(self.cache, **self.kw)
        if text.endswith("\n"):
            out = text[self.print_len:]
            self.cache, self.print_len = [], 0
        elif len(text) > 0 and self._is_cjk(ord(text[-1])):
            out = text[self.print_len:]
            self.print_len += len(out)
        else:
            out = text[self.print_len: text.rfind(" ") + 1]
            self.print_len += len(out)
        return out

    def end(self) -> str:
        if self.cache:
            text = self.tok.decode(self.cache, **self.kw)
            out = text[self.print_len:]
            self.cache, self.print_len = [], 0
            return out
        return ""


class CompletionStreamer:
    """generative_model.py:99-140 — one id per stream, finish_reason on every chunk."""

    def __init__(self, request: CompletionRequest, generate_queue: asyncio.Queue, stop_state: Dict[str, bool],
                 system_fingerprint: Optional[str] = None):
        self.request, self.generate_queue, self.stop_state = request, generate_queue, stop_state
        self.index = 0
        self.id = generate_uuid()
        self.system_fingerprint = system_fingerprint

    def __aiter__(self):
        return self

    async def __anext__(self):
        text = await self.generate_queue.get()
        if text is None:
            raise StopAsyncIteration()
        if isinstance(text, Exception):
            raise text
        finish_reason = "stop" if self.stop_state.get("triggered") else "length"
        return CompletionChunk(
            id=self.id, created=int(time.time()), model=self.request.model, object="text_completion",
            choices=[CompletionChunkChoice(finish_reason=finish_reason, index=self.index, text=text, logprobs=None)],
            system_fingerprint=self.system_fingerprint)


def load_safetensors_dir(model_dir: str) -> Iterable[Tuple[str, torch.Tensor]]:
    """Yield (hf_name, tensor) from every *.safetensors file of an HF checkpoint directory."""
    from safetensors import safe_open
    files = sorted(f for f in os.listdir(model_dir) if f.endswith(".safetensors"))
    if not files:
        raise FileNotFoundError(f"no *.safetensors under {model_dir}")
    for f in files:
        with safe_open(os.path.join(model_dir, f), framework="pt", device="cpu") as sf:
            for name in sf.keys():
                yield name, sf.get_tensor(name)


class B200GenerativeModel(OpenAIChatAdapterModel, Model):
    def __init__(self, model_name: str, model_id_or_path: Optional[str] = None, *,
                 model_config: Optional[dict] = None, state_dict: Optional[Iterable[Tuple[str, torch.Tensor]]] = None,
                 tokenizer=None, pad_token_id: Optional[int] = None, max_model_len: Optional[int] = None,
                 max_batch: int = 32, device: int = 0, tensor_parallel_size: int = 1, tp_rank: int = 0,
                 nccl_id: Optional[bytes] = None, system_fingerprint: Optional[str] = None,
                 request_logger=None, continuous_batching: bool = False, generation_defaults: Optional[dict] = None,
                 kv_cache_dtype: str = "auto"):
        Model.__init__(self, model_name)
        self.ready = False
        self.model_id_or_path = model_id_or_path
        self.model_config = model_config
        self._state_dict = state_dict
        self._tokenizer = tokenizer
        self._pad_token_id = pad_token_id
        self.max_length = max_model_len
        self._user_max_len = max_model_len
        self.max_batch = max_batch
        self.device_index = device
        self.tp_size, self.tp_rank, self.nccl_id = tensor_parallel_size, tp_rank, nccl_id
        self.kv_cache_dtype = kv_cache_dtype      # "auto" / "bfloat16" = bf16 KV pages; "fp8" / "fp8_e4m3" = e4m3 codes
        self.system_fingerprint = system_fingerprint
        self.request_logger = request_logger
        self.is_encoder_decoder = False
        self._engine: Optional[B200Engine] = None
        self._request_queue: "queue.Queue" = queue.Queue()
        self._thread: Optional[Thread] = None
        self.eos_token_ids: List[int] = []
        # iteration-level batching instead of the reference's one-request-at-a-time loop (continuous.py)
        self._generation_defaults = generation_defaults
        self._seed_counter = 0
        self.continuous_batching = bool(continuous_batching)
        self.prefill_chunk_tokens, self.prefix_cache = 0, False     # set before load(): see kserve_b200/__main__.py
        self._cb = None

    # ------------------------------------------------------------------ load / stop (generative_model.py:203-285)
    def load(self) -> bool:
        if self.model_config is None:
            with open(os.path.join(self.model_id_or_path, "config.json")) as f:
                self.model_config = json.load(f)
        cfg = self.model_config
        arch = (cfg.get("architectures") or ["LlamaForCausalLM"])[0]
        model_type = cfg.get("model_type", "llama")
        # (Qwen3 = the dense decoders; qwen3_moe and the other qwen3_* types are different models)
        if not arch.endswith("ForCausalLM") or model_type not in ("llama", "mistral", "mixtral", "qwen2", "qwen3"):
            raise OpenAIError(f"architecture {arch} (model_type {model_type}) is not supported by the H100 runtime "
                              "(Llama / Mistral / Mixtral / Qwen2 / dense Qwen3 decoders only)")
        head_dim = cfg.get("head_dim") or cfg["hidden_size"] // cfg["num_attention_heads"]
        if head_dim != 128:
            # (Qwen2-0.5B, Qwen2.5-0.5B, Llama-3.2-1B: the KV page layout and both attention kernels are built for 128)
            raise OpenAIError(f"head_dim={head_dim} is not supported by the H100 runtime (head_dim 128 only)")
        if self._tokenizer is None and self.model_id_or_path and os.path.exists(
                os.path.join(self.model_id_or_path, "tokenizer.json")):
            from transformers import AutoTokenizer
            self._tokenizer = AutoTokenizer.from_pretrained(self.model_id_or_path, padding_side="left")  # :225-245
        vocab_rows = cfg["vocab_size"]
        if self._tokenizer is not None:
            self._tokenizer.padding_side = "left"
            if not self._tokenizer.pad_token:                       # :256-265 fallback [PAD] + embedding resize
                self._tokenizer.add_special_tokens({"pad_token": "[PAD]"})
                vocab_rows = len(self._tokenizer)
            self._pad_token_id = self._tokenizer.pad_token_id
        try:
            self.max_length = get_and_verify_max_len(cfg, self.max_length)    # :206 -> utils.py:28-159
        except (ValueError, NotImplementedError) as e:
            raise OpenAIError(str(e))
        # What this runtime cannot execute must not load (a silently ignored field generates fluent, wrong tokens):
        rope_inv_freq(cfg, cfg.get("head_dim") or cfg["hidden_size"] // cfg["num_attention_heads"])   # raises on yarn / dynamic / longrope
        window = cfg.get("sliding_window")
        layer_types = cfg.get("layer_types")
        uses_window = window is not None and cfg.get("use_sliding_window", True) and (
            layer_types is None or any(t == "sliding_attention" for t in layer_types))
        if uses_window and window < self.max_length:
            # inside the window sliding-window attention IS full attention, so serving at most `window` tokens is exact
            if self._user_max_len is not None:
                raise OpenAIError(f"max_model_len ({self.max_length}) exceeds the checkpoint's sliding_window ({window}); "
                                  "the H100 runtime implements full attention only")
            logger.warning("sliding_window=%d < max length %d: serving at most %d tokens (full attention == sliding "
                           "window inside the window)", window, self.max_length, window)
            self.max_length = int(window)
        # Qwen2's q / k / v biases and Qwen3's q / k norms are implied by the architecture (they come with the
        # checkpoint); attention_bias (Llama, Qwen3) would also put a bias on o_proj, which the engine does not have
        for key in ("attention_bias", "mlp_bias"):
            if cfg.get(key):
                raise OpenAIError(f"config.{key}=true is not supported by the H100 runtime")
        if cfg.get("hidden_act", "silu") != "silu":
            raise OpenAIError(f"hidden_act={cfg.get('hidden_act')} is not supported by the H100 runtime (silu only)")
        try:
            quant = parse_quantization_config(cfg, self.tp_size)     # None = bf16 checkpoint; FP8: kserve_b200/fp8.py
        except UnsupportedQuantization as e:
            raise OpenAIError(str(e))
        if quant is not None:
            log_activation_scheme(quant)
        try:
            kv_format = kv_cache_format(self.kv_cache_dtype, self.tp_size)
        except UnsupportedQuantization as e:
            raise OpenAIError(str(e))
        # checkpoint generation defaults: transformers merges the None fields of the request's GenerationConfig from
        # model.generation_config (generation/utils.py:1693-1701) — this is how instruct checkpoints turn sampling on (q9)
        self.generation_defaults = dict(self._generation_defaults or {})
        gpath = os.path.join(self.model_id_or_path, "generation_config.json") if self.model_id_or_path else None
        if gpath and os.path.exists(gpath):
            with open(gpath) as f:
                self.generation_defaults = {**json.load(f), **self.generation_defaults}
        ck_dtype = cfg.get("torch_dtype") or cfg.get("dtype")
        if ck_dtype not in (None, "bfloat16"):
            # the reference's `--dtype auto` would compute in the checkpoint's type (__main__.py:249-259); this runtime's
            # only arithmetic type is bfloat16 (fp32 accumulation), so other checkpoints are converted at load
            logger.warning("checkpoint dtype %s: weights are converted to bfloat16, the only compute type of the H100 runtime",
                           ck_dtype)
        eos = cfg.get("eos_token_id")
        self.eos_token_ids = [] if eos is None else ([int(e) for e in eos] if isinstance(eos, list) else [int(eos)])
        try:
            if torch.cuda.is_available():
                cap_t, pages = plan_memory(cfg, vocab_rows, self.max_batch, self.max_length, self.tp_size,
                                           torch.cuda.mem_get_info(self.device_index)[0], kv_bytes=1 if kv_format else 2)
            else:       # B200Engine raises below (no CPU fallback); nothing to plan
                cap_t, pages = None, self.max_batch * -(-self.max_length // 64)
        except ValueError as e:
            raise OpenAIError(str(e))
        if getattr(self, "kv_pages_limit", None):       # tests / load experiments: a deliberately small KV page pool
            pages = min(pages, int(self.kv_pages_limit))
        # (continuous batching draws pages from the pool per request; an exhausted pool defers or preempts, it never fails load)
        self.max_prefill_tokens = cap_t
        self._engine = B200Engine(cfg, max_batch=self.max_batch, max_seq_len=self.max_length, device=self.device_index,
                                  max_prefill_tokens=cap_t, num_kv_pages=pages,
                                  tp_rank=self.tp_rank, tp_size=self.tp_size, nccl_id=self.nccl_id, vocab_rows=vocab_rows,
                                  weight_format=0 if quant is None else 1, kv_cache_dtype=kv_format)
        weights = self._state_dict if self._state_dict is not None else load_safetensors_dir(self.model_id_or_path)
        V0 = cfg["vocab_size"]

        tied: List[Optional[torch.Tensor]] = [None]
        seen_head = [False]
        # Qwen3: the engine applies the per-head q / k norms when their weights arrive, so a checkpoint without them would
        # run as a plain Llama decoder and generate wrong tokens; they must be there for every layer
        qk_norms = {f"model.layers.{i}.self_attn.{p}_norm.weight" for i in range(cfg["num_hidden_layers"]) for p in "qk"} \
            if model_type == "qwen3" else set()

        def resized():
            for name, t in weights:
                qk_norms.discard(name)
                if name in ("model.embed_tokens.weight", "lm_head.weight") and t.shape[0] != vocab_rows:
                    # resize_token_embeddings: keep the first rows, new rows = mean of the old ones (HF default)
                    if t.shape[0] > vocab_rows:
                        t = t[:vocab_rows]
                    else:
                        extra = t.float().mean(0, keepdim=True).to(t.dtype).expand(vocab_rows - t.shape[0], -1)
                        t = torch.cat([t, extra], 0)
                if name == "model.embed_tokens.weight" and cfg.get("tie_word_embeddings"):
                    tied[0] = t
                if name == "lm_head.weight":
                    seen_head[0] = True
                yield name, t
            if qk_norms:
                raise OpenAIError(f"the qwen3 checkpoint has no {min(qk_norms)}: a Qwen3 decoder without its per-head q / k "
                                  "norms is not supported by the H100 runtime")
            # tie_word_embeddings: the checkpoint has no lm_head.weight; the head IS the (resized) embedding matrix
            if cfg.get("tie_word_embeddings") and not seen_head[0]:
                if tied[0] is None:
                    raise OpenAIError("tie_word_embeddings is set but the checkpoint has no model.embed_tokens.weight")
                yield "lm_head.weight", tied[0]
        self._engine.load_weights(resized())
        self._state_dict = None
        self.vocab_rows = vocab_rows
        self._thread = Thread(target=self._process_requests, daemon=True)   # :267-269
        self._thread.start()
        if self.continuous_batching and self.tp_rank == 0:     # followers replay the scheduler's engine calls (tp.follower_loop)
            from .continuous import ContinuousBatcher
            self._cb = ContinuousBatcher(self._engine, self._pad_token_id or 0, self.eos_token_ids,
                                         prefill_chunk_tokens=self.prefill_chunk_tokens, prefix_cache=self.prefix_cache)

            def _cb_down(err):           # a dead scheduler thread must not leave the model advertised as ready
                self.ready = False
            self._cb.on_fatal = _cb_down
            self._cb.start()
        self.ready = True
        return self.ready

    def stop(self):
        if self.tp_size > 1 and self.tp_rank == 0 and self._engine is not None:
            from .tp import leader_call
            leader_call("stop", (), {})
        if self._cb is not None:
            self._cb.stop()
            self._cb = None
        self._request_queue.put(None)    # :273-277
        if self._thread is not None:
            self._thread.join(timeout=5)
        if self._engine is not None:
            self._engine.close()
            self._engine = None
        self.ready = False

    # ------------------------------------------------------------------ worker thread (:286-354)
    def _process_requests(self):
        while True:
            req = self._request_queue.get()
            if not req:
                break
            fn, done = req
            try:
                done(fn(), None)
            except Exception as e:  # delivered to the awaiting coroutine
                from ._lib import EngineFault
                if isinstance(e, EngineFault):      # a tensor-parallel peer is gone: stop advertising the model as ready
                    self.ready = False
                done(None, e)

    async def _submit(self, fn):
        """Run fn on the generation thread; results come back with loop.call_soon_threadsafe (:299-300, :356-374)."""
        loop = asyncio.get_running_loop()
        fut: asyncio.Future = loop.create_future()

        def done(result, err):
            def _set():
                if fut.cancelled():
                    return
                if err is not None:
                    fut.set_exception(err)
                else:
                    fut.set_result(result)
            loop.call_soon_threadsafe(_set)
        self._request_queue.put((fn, done))
        return await fut

    def _generate(self, ids, mask, streamer=None, **kw) -> GenerateResult:
        """The call that replaces `self._model.generate(**kwargs)` (:314, :328).  Under TP the leader first
        replicates the call to the follower ranks (they run it without the streamer)."""
        if self.tp_size > 1:
            from .tp import leader_call
            leader_call("generate", (ids, mask), kw)
        return self._engine.generate(ids, mask, streamer=streamer, **kw)

    def _batch_predict(self, rows, **kw):
        """engine.batch_predict (b200_batch_predict) with the tensor-parallel call replication of `_generate`"""
        if self.tp_size > 1:
            from .tp import leader_call
            leader_call("batch_predict", (rows,), kw)
        t0 = time.perf_counter()
        out = self._engine.batch_predict(rows, **kw)
        labels = get_labels(self.name)
        tm = self._engine.last_timing()
        TTFT_HIST.labels(**labels).observe(tm.prefill_ms / 1e3)
        if tm.decode_ms > 0 and tm.decode_steps > 0:
            DECODE_TOKENS_PER_S.labels(**labels).observe(len(rows) * tm.decode_steps / (tm.decode_ms / 1e3))
        return out

    @staticmethod
    def _unpadded_rows(ids: torch.Tensor, mask: Optional[torch.Tensor]) -> List[List[int]]:
        """left-padded [B, S] (+ mask) -> the real token rows (what the packed engine layout holds)"""
        if mask is None:
            return [row.tolist() for row in ids]
        rows = []
        for b in range(ids.shape[0]):
            nz = mask[b].nonzero()
            first = int(nz[0]) if len(nz) else ids.shape[1] - 1
            rows.append(ids[b, first:].tolist())
        return rows

    def build_generation_config(self, request: CompletionRequest) -> Dict[str, Any]:
        """generative_model.py:388-402: `top_p`, `temperature` pass through; `presence_penalty > 0` becomes
        `repetition_penalty` (q8); nothing sets do_sample, so sampling is on only if the checkpoint's own
        generation_config.json says so (q9), whose temperature / top_p / top_k then fill the request's None fields.
        `seed` (:302-303 calls set_seed) keys this runtime's Philox stream instead."""
        d = self.generation_defaults
        out: Dict[str, Any] = {}
        rp = request.presence_penalty if (request.presence_penalty and request.presence_penalty > 0) else d.get("repetition_penalty")
        if rp and float(rp) != 1.0:
            out["repetition_penalty"] = float(rp)
        if d.get("do_sample"):
            temperature = request.temperature if request.temperature is not None else d.get("temperature", 1.0)
            if temperature is not None and float(temperature) > 0:      # temperature == 0: greedy, as vLLM's type documents it
                out["do_sample"] = True
                out["temperature"] = float(temperature)
                top_p = request.top_p if request.top_p is not None else d.get("top_p", 1.0)
                out["top_p"] = float(top_p if top_p is not None else 1.0)
                out["top_k"] = int(d.get("top_k", 50) or 0) or 1024      # GenerationConfig default 50; 0 / None = "off" -> widest supported
                seed = getattr(request, "seed", None)
                if seed is None:
                    self._seed_counter += 1
                    seed = (int(time.time_ns()) ^ (self._seed_counter * 0x9E3779B97F4A7C15)) & 0xFFFFFFFFFFFFFFFF
                out["seed"] = int(seed)
        return out

    async def _agenerate(self, ids, mask, *, max_new_tokens, pad_token_id, eos_token_ids, stop_sequences=(), **sampling) -> GenerateResult:
        """One request through the engine: the continuous batcher when enabled, else the serial generation thread."""
        if self._cb is not None:
            try:
                return await self._cb.submit(self._unpadded_rows(ids, mask), ids, max_new_tokens, stop_sequences, sampling=sampling or None)
            except (ValueError, RuntimeError) as e:
                raise OpenAIError(str(e))
        return await self._submit(lambda: self._generate(ids, mask, max_new_tokens=max_new_tokens, pad_token_id=pad_token_id,
                                                         eos_token_ids=eos_token_ids, stop_sequences=stop_sequences, **sampling))

    # ------------------------------------------------------------------ request validation (:376-402)
    def validate_supported_completion_params(self, request: CompletionRequest):
        if request.frequency_penalty is not None and request.frequency_penalty > 0:
            raise OpenAIError("'frequency_penalty' is not supported")
        if request.n is not None and request.n > 1:
            raise OpenAIError("'n' > 1 is not supported")
        if request.echo and self.is_encoder_decoder:
            raise OpenAIError("'echo' is not supported by encoder-decoder models")
        # presence_penalty / temperature / top_p are handled by build_generation_config (device-side processors).
        # logit_bias (q8): the reference maps it to `sequence_bias = {tuple(token): bias}` (:396-401).  The keys of an
        # OpenAI logit_bias are token-id STRINGS, so tuple("123") is ('1', '2', '3') and transformers'
        # SequenceBiasLogitsProcessor._validate_arguments rejects every such request inside generate() — an empty dict
        # is rejected too.  The observable behaviour of the reference is therefore this error, reproduced verbatim.
        if request.logit_bias is not None:
            sequence_bias = {tuple(token): bias for token, bias in request.logit_bias.items()}
            if len(sequence_bias) == 0:
                raise ValueError(f"`sequence_bias` has to be a non-empty dictionary, or non-empty list of lists but is {sequence_bias}.")
            raise ValueError(f"Each key in `sequence_bias` has to be a non-empty tuple of positive integers, but is {sequence_bias}.")

    # ------------------------------------------------------------------ tokenisation (:546-562)
    def _encode_prompts(self, prompt) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        prompts = prompt if isinstance(prompt, list) and not isinstance(prompt[0], int) else [prompt]
        if isinstance(prompts[0][0], int):
            ids = torch.tensor(prompts, dtype=torch.int64)     # :552-555, NO attention mask is sent
            # transformers then infers one iff pad_token_id occurs in the ids (utils.py:731-763, q4)
            mask = None
            if self._pad_token_id is not None and bool((ids == self._pad_token_id).any()) and \
                    self._pad_token_id not in self.eos_token_ids:
                mask = (ids != self._pad_token_id).long()
            return ids, mask
        if self._tokenizer is None:
            raise OpenAIError("this model was loaded without a tokenizer: send token-id prompts")
        enc = self._tokenizer(prompts, padding=True, return_tensors="pt")   # :557-559
        return enc["input_ids"].to(torch.int64), enc["attention_mask"].to(torch.int64)

    # ------------------------------------------------------------------ OpenAI completions (:535-646)
    async def create_completion(self, request: CompletionRequest, raw_request=None,
                                context: Optional[Dict[str, Any]] = None
                                ) -> Union[AsyncGenerator[str, None], Completion, ErrorResponse]:
        self._log_request(request, raw_request)
        if request.prompt is None:
            raise OpenAIError("prompt is required")
        stats = LLMStats()
        context = {LLM_STATS_KEY: stats}
        ids, mask = self._encode_prompts(request.prompt)
        B, S = ids.shape
        stats.num_prompt_tokens = S * B                       # :560-562 (counts pad tokens, q3)
        if request.max_tokens is None:
            request.max_tokens = self.max_length - S           # :563-564
        if S + request.max_tokens > self.max_length:           # :565-572
            raise OpenAIError(
                f"This model's maximum context length is {self.max_length} tokens. "
                f"However, you requested {request.max_tokens + S} tokens "
                f"({S} in the messages, "
                f"{request.max_tokens} in the completion). "
                f"Please reduce the length of the messages or completion.")
        self.validate_supported_completion_params(request)
        if B > min(self.max_batch, 64):
            raise OpenAIError(f"batch of {B} prompts exceeds this engine's max batch {min(self.max_batch, 64)}")
        stop_sequences: List[List[int]] = []
        if request.stop is not None:                            # :578-593 (stop defaults to [], q2)
            stop = request.stop if isinstance(request.stop, list) else [request.stop]
            for seq in stop:
                if self._tokenizer is None:
                    raise OpenAIError("stop strings need a tokenizer")
                stop_sequences.append(self._tokenizer.encode(seq, add_special_tokens=False))
        echo = bool(request.echo)
        stop_state: Dict[str, bool] = {"triggered": False}
        common = dict(max_new_tokens=request.max_tokens, pad_token_id=self._pad_token_id,
                      eos_token_ids=self.eos_token_ids, stop_sequences=stop_sequences, **self.build_generation_config(request))

        if request.stream:
            if B != 1:
                raise OpenAIError("TextStreamer only supports batch size 1")   # what transformers raises
            out_q: asyncio.Queue = asyncio.Queue()
            loop = asyncio.get_running_loop()

            def put(x):
                loop.call_soon_threadsafe(out_q.put_nowait, x)

            def run_stream():
                detok = IncrementalDetokenizer(self._tokenizer)
                try:
                    if echo:                                   # skip_prompt = not echo (:305-311)
                        piece = detok.put(ids[0][mask[0].bool()].tolist() if mask is not None else ids[0].tolist())
                        if piece != "":
                            put(piece)

                    def on_step(step, toks):
                        piece = detok.put([int(toks[0])])
                        if piece != "":                         # empty pieces are dropped (:317-319)
                            put(piece)
                        return False
                    r = self._generate(ids, mask, streamer=on_step, **common)
                    stop_state["triggered"] = r.stop_triggered
                    self._observe(r, B)
                    piece = detok.end()
                    if piece != "":
                        put(piece)
                except Exception as e:
                    put(e)
                put(None)
                return None
            if self._cb is not None:
                detok = IncrementalDetokenizer(self._tokenizer)
                if echo:
                    piece = detok.put(self._unpadded_rows(ids, mask)[0])
                    if piece != "":
                        put(piece)

                def on_tokens(step, toks):
                    piece = detok.put([int(toks[0])])
                    if piece != "":
                        put(piece)

                def cb_done(res, err):
                    if err is not None:
                        put(err)
                    else:
                        stop_state["triggered"] = res.stop_triggered
                        self._observe(res, B)
                        piece = detok.end()
                        if piece != "":
                            put(piece)
                    put(None)
                try:
                    cb_req = self._cb.submit_nowait(self._unpadded_rows(ids, mask), ids, request.max_tokens, stop_sequences, cb_done, on_tokens,
                                                    sampling=self.build_generation_config(request) or None)
                except (ValueError, RuntimeError) as e:
                    raise OpenAIError(str(e))
            else:
                cb_req = None
                self._request_queue.put((run_stream, lambda r, e: None))
            completion = CompletionStreamer(request=request, generate_queue=out_q, stop_state=stop_state,
                                            system_fingerprint=self.system_fingerprint)

            async def stream_results() -> AsyncGenerator[str, None]:   # :612-617 SSE framing
                finished = False
                try:
                    async for partial in completion:
                        yield f"data: {partial.model_dump_json()}\n\n"
                    finished = True
                    yield "data: [DONE]\n\n"
                finally:
                    if not finished and cb_req is not None:     # the client went away mid-stream: free the slot
                        self._cb.cancel(cb_req)
            return stream_results()

        r: GenerateResult = await self._agenerate(ids, mask, **common)
        self._observe(r, B)
        output_start = 0 if echo else S                        # :324-327
        stats.num_generation_tokens = r.num_generated * B      # :329-335 (every row counts the same length)
        out = r.output_ids[:, output_start:]
        if self._tokenizer is not None:
            texts = self._tokenizer.batch_decode(out, skip_special_tokens=True)   # :336-338
        else:
            texts = [" ".join(str(int(t)) for t in row) for row in out]           # tokenizer-less synthetic runs
        finish_reason = "stop" if r.stop_triggered else "length"                 # :621-627
        choices = [CompletionChoice(finish_reason=finish_reason, index=i, text=o, logprobs=None)
                   for i, o in enumerate(texts)]
        return Completion(
            id=generate_uuid(), choices=choices, created=int(time.time()), object="text_completion",
            model=request.model, system_fingerprint=self.system_fingerprint,
            usage=UsageInfo(prompt_tokens=stats.num_prompt_tokens, completion_tokens=stats.num_generation_tokens,
                            total_tokens=stats.num_prompt_tokens + stats.num_generation_tokens))

    def _observe(self, r: GenerateResult, B: int):
        labels = get_labels(self.name)
        TTFT_HIST.labels(**labels).observe(r.prefill_ms / 1e3)
        if r.decode_ms > 0 and r.decode_steps > 0:
            DECODE_TOKENS_PER_S.labels(**labels).observe(B * r.decode_steps / (r.decode_ms / 1e3))

    def _log_request(self, request: CompletionRequest, raw_request=None) -> None:
        if self.request_logger:   # :648-666
            is_ids = isinstance(request.prompt, list) and (isinstance(request.prompt[0], int) or (
                isinstance(request.prompt[0], list) and isinstance(request.prompt[0][0], int)))
            rid = raw_request.headers.get("x-request-id", None) if raw_request else None
            self.request_logger.log_inputs(rid, prompt=None if is_ids else request.prompt,
                                           prompt_token_ids=request.prompt if is_ids else None,
                                           params=request.model_dump(exclude={"prompt"}))

    # ------------------------------------------------------------------ chat (:509-533)
    def apply_chat_template(self, request: ChatCompletionRequest) -> ChatPrompt:
        if self._tokenizer is None:
            raise OpenAIError("chat completions need a tokenizer with a chat template")
        conversation = [{"role": m.role, "content": m.content if isinstance(m.content, str) else
                         "".join(p.get("text", "") for p in (m.content or []))} for m in request.messages]
        if request.chat_template is None and getattr(self._tokenizer, "chat_template", None) is None:    # :495-500
            raise OpenAIError("As of transformers v4.44, default chat template is no longer allowed, so you must provide a chat "
                              "template if the tokenizer does not define one.")
        kwargs = dict(request.chat_template_kwargs or {})
        prompt = self._tokenizer.apply_chat_template(
            conversation=conversation, chat_template=request.chat_template, tokenize=False,
            add_generation_prompt=request.add_generation_prompt,
            continue_final_message=request.continue_final_message, tools=request.tools, documents=request.documents,
            **kwargs)
        return ChatPrompt(prompt=prompt)

    # ------------------------------------------------------------------ kserve.Model.predict: V1 / V2 (extension)
    def get_input_types(self) -> List[Dict]:
        return [{"name": "input_ids", "datatype": "INT64", "shape": [-1, -1]},
                {"name": "attention_mask", "datatype": "INT64", "shape": [-1, -1]}]

    def get_output_types(self) -> List[Dict]:
        return [{"name": "output_ids", "datatype": "INT64", "shape": [-1, -1]},
                {"name": "text", "datatype": "BYTES", "shape": [-1]}]

    def _batch_from_instances(self, instances: List[Any]) -> Tuple[torch.Tensor, Optional[torch.Tensor], bool]:
        """V1 instances: token-id lists (ragged allowed -> left padded, as the tokenizer would) or strings."""
        if len(instances) == 0:
            raise InvalidInput("no instances in the request")
        if all(isinstance(i, str) for i in instances):
            ids, mask = self._encode_prompts(list(instances))
            return ids, mask, True
        rows = []
        for i in instances:
            if isinstance(i, dict):
                i = i.get("input_ids", i.get("prompt"))
            if not isinstance(i, (list, tuple)) or not all(isinstance(t, int) for t in i) or len(i) == 0:
                raise InvalidInput("each instance must be a string, a non-empty list of token ids or {'input_ids': [...]}")
            rows.append(list(i))
        S = max(len(r) for r in rows)
        pad = self._pad_token_id if self._pad_token_id is not None else 0
        ids = torch.full((len(rows), S), pad, dtype=torch.int64)
        mask = torch.zeros((len(rows), S), dtype=torch.int64)
        for b, r in enumerate(rows):
            ids[b, S - len(r):] = torch.tensor(r, dtype=torch.int64)
            mask[b, S - len(r):] = 1
        return ids, (None if bool(mask.all()) else mask), False

    async def predict(self, payload: Union[Dict, InferRequest], headers: Dict[str, str] = None,
                      response_headers: Dict[str, str] = None) -> Union[Dict, InferResponse]:
        if isinstance(payload, InferRequest):
            params = payload.parameters or {}
            inp = payload.get_input_by_name("input_ids")
            text_in = payload.get_input_by_name("text")
            if inp is not None:
                try:
                    arr = inp.as_numpy()
                except InvalidInput:
                    raise
                except Exception as e:       # byte count / shape mismatch of a binary tensor is the client's error
                    raise InvalidInput(f"malformed 'input_ids' tensor: {e}")
                if arr.ndim != 2:
                    raise InvalidInput("input_ids must be [batch, seq]")
                ids = torch.from_numpy(np.ascontiguousarray(arr.astype(np.int64, copy=False)))
                m = payload.get_input_by_name("attention_mask")
                mask = None if m is None else torch.from_numpy(np.ascontiguousarray(m.as_numpy().astype(np.int64, copy=False)))
                as_text = False
            elif text_in is not None:
                ids, mask = self._encode_prompts(text_in.as_string())
                as_text = True
            else:
                raise InvalidInput("expected an 'input_ids' INT64 [B,S] or a 'text' BYTES [B] input")
        else:
            if not isinstance(payload, dict):
                raise InvalidInput("expected a JSON object with 'instances'")
            params = payload.get("parameters") or {}
            ids, mask, as_text = self._batch_from_instances(payload.get("instances", []))
        try:
            max_tokens = int(params.get("max_tokens", params.get("max_new_tokens", 16)))
        except (TypeError, ValueError):
            raise InvalidInput("'max_tokens' must be an integer")
        if max_tokens < 1:
            raise InvalidInput("'max_tokens' must be >= 1")
        B, S = ids.shape
        if mask is not None and tuple(mask.shape) != (B, S):
            raise InvalidInput(f"attention_mask shape {list(mask.shape)} differs from input_ids shape {[B, S]}")
        if B > min(self.max_batch, 64):
            raise InvalidInput(f"batch of {B} exceeds this engine's max batch {min(self.max_batch, 64)}")
        if S + max_tokens > self.max_length:
            raise InvalidInput(f"prompt ({S}) + max_tokens ({max_tokens}) exceeds the model's maximum context length {self.max_length}")
        if mask is not None:
            lead = mask.cumsum(1) > 0                  # left padding only: once a row starts it may not contain zeros
            if bool(((mask == 0) & lead).any()) or not bool(lead[:, -1].all()):
                raise InvalidInput("attention_mask must be left padding (zeros, then ones) with at least one token per row")
        if not isinstance(payload, InferRequest) and not as_text and self._cb is None:
            # the V1 `:predict` leg the batcher fronts: the instances (ragged token rows, one per instance of every merged
            # request) run as one batch and the predictions come back as one matrix in instance order —
            # the body of BatchHandler.batchPredict (pkg/batcher/handler.go:99-155) as one C-ABI call
            rows = self._unpadded_rows(ids, mask)
            pred, _ = await self._submit(lambda: self._batch_predict(rows, max_new_tokens=max_tokens, pad_token_id=self._pad_token_id,
                                                                     eos_token_ids=self.eos_token_ids))
            return {"predictions": [row.tolist() for row in pred]}
        r: GenerateResult = await self._agenerate(ids, mask, max_new_tokens=max_tokens, pad_token_id=self._pad_token_id,
                                                  eos_token_ids=self.eos_token_ids)
        self._observe(r, B)
        gen = r.output_ids[:, S:]
        texts = self._tokenizer.batch_decode(gen, skip_special_tokens=True) if self._tokenizer is not None else None
        if isinstance(payload, InferRequest):
            o = InferOutput("output_ids", list(gen.shape), "INT64")
            o.data = gen.numpy()
            outs = [o]
            if texts is not None:
                t = InferOutput("text", [len(texts)], "BYTES")
                t.data = np.array([x.encode("utf-8") for x in texts], dtype=np.object_)
                outs.append(t)
            return InferResponse(response_id=payload.id or str(uuid.uuid4()), model_name=self.name, infer_outputs=outs,
                                 use_binary_outputs=payload.use_binary_outputs, requested_outputs=payload.request_outputs)
        if as_text and texts is not None:
            return {"predictions": texts}
        return {"predictions": [row.tolist() for row in gen]}
