"""Python handle over the C ABI engine (include/kserve_b200.h).

This is the object `B200GenerativeModel` calls where the reference calls
``self._model.generate(**kwargs)`` (python/huggingfaceserver/huggingfaceserver/generative_model.py:314,328).
PyTorch is used only to hold host/device buffers; all compute is in libkserve_b200.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Callable, Iterable, List, Optional, Sequence, Tuple

import torch

from . import _lib


@dataclass
class GenerateResult:
    output_ids: torch.Tensor          # int64 [B, S + T]  (prompt echoed, like transformers.generate)
    stop_triggered: bool
    num_generated: int
    logits: Optional[torch.Tensor]    # bf16 [T, B, V] when requested
    prefill_ms: float
    decode_ms: float
    decode_steps: int
    kernel_launches: int


def hf_rope_tables(rope_theta_or_cfg, head_dim: int, max_pos: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """cos/sin exactly as LlamaRotaryEmbedding computes them (see utils.hf_rope_tables); accepts a bare rope_theta
    (default rope) or a config dict (rope_scaling / rope_parameters: default, linear, llama3)."""
    from .utils import hf_rope_tables as _tables
    cfg = rope_theta_or_cfg if isinstance(rope_theta_or_cfg, dict) else {"rope_theta": float(rope_theta_or_cfg)}
    return _tables(cfg, head_dim, max_pos)


class PoolExhausted(_lib.B200Error):
    """b200_cb_admit could not obtain KV pages (rc -7): nothing was admitted, retry after a release"""


class B200Engine:
    def __init__(self, cfg: dict, *, max_batch: int = 8, max_seq_len: int = 2048,
                 max_prefill_tokens: Optional[int] = None, num_kv_pages: int = 0, device: int = 0,
                 tp_rank: int = 0, tp_size: int = 1, nccl_id: Optional[bytes] = None,
                 vocab_rows: Optional[int] = None, weight_format: int = 0, kv_cache_dtype: int = 0):
        """weight_format 1: the seven projection weights are FP8 (float8_e4m3fn + a scale per row, kserve_b200/fp8.py);
        kv_cache_dtype 1: the KV pages hold float8_e4m3fn codes (fp8.quantize_kv) instead of bf16"""
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.B200Error("no CUDA device: kserve_b200 has no CPU fallback")
        self.cfg = dict(cfg)
        self.vocab = int(vocab_rows or cfg["vocab_size"])
        self.max_batch, self.max_seq_len = max_batch, max_seq_len
        mc = _lib.ModelConfig()
        mc.vocab_size = self.vocab
        mc.hidden_size = cfg["hidden_size"]
        mc.intermediate_size = cfg["intermediate_size"]
        mc.num_layers = cfg["num_hidden_layers"]
        mc.num_heads = cfg["num_attention_heads"]
        mc.num_kv_heads = cfg["num_key_value_heads"]
        mc.head_dim = cfg.get("head_dim") or cfg["hidden_size"] // cfg["num_attention_heads"]
        mc.max_position = max(max_seq_len, 64)
        mc.rms_eps = cfg.get("rms_norm_eps", 1e-5)
        from .utils import rope_parameters
        mc.rope_theta = float(rope_parameters(cfg)["rope_theta"])
        mc.max_batch = max_batch
        mc.max_seq_len = max_seq_len
        mc.max_prefill_tokens = max_prefill_tokens or min(max_batch, 64) * max_seq_len     # one pass covers at most 64 sequences
        mc.num_kv_pages = num_kv_pages
        mc.tp_rank, mc.tp_size, mc.device = tp_rank, tp_size, device
        mc.num_experts = int(cfg.get("num_local_experts", 0) or 0)
        mc.num_experts_per_tok = int(cfg.get("num_experts_per_tok", 0) or 0) if mc.num_experts else 0
        mc.weight_format = int(weight_format)
        self.weight_format = int(weight_format)
        mc.kv_cache_dtype = int(kv_cache_dtype)
        self.kv_cache_dtype = int(kv_cache_dtype)
        self.device = device
        self.tp_size, self.tp_rank = tp_size, tp_rank
        # rope tables first: an unsupported rope_scaling type must fail before any device memory is taken
        cos, sin = hf_rope_tables(self.cfg, mc.head_dim, mc.max_position)
        h = C.c_void_p()
        idbuf = C.create_string_buffer(nccl_id, 128) if nccl_id is not None else None
        _lib.check(self.lib.b200_engine_create(C.byref(mc), idbuf, C.byref(h)), "b200_engine_create")
        self.h = h
        _lib.check(self.lib.b200_engine_set_rope_table(self.h, cos.data_ptr(), sin.data_ptr(), mc.max_position),
                   "b200_engine_set_rope_table")
        self._cb_keepalive = None
        if tp_size > 1:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized():
                self.setup_p2p()      # collective: every rank constructs its engine at the same point

    def vocab_shard(self) -> Tuple[int, int]:
        """(first column, columns) of the LM-head shard this rank owns (the whole vocabulary on one GPU)"""
        per = -(-self.vocab // self.tp_size)
        v0 = per * self.tp_rank
        return v0, max(0, min(per, self.vocab - v0))

    def setup_p2p(self) -> None:
        """Exchange the IPC handles of the peer-memory blocks (torch.distributed is only the courier)."""
        if self.tp_size == 1:
            return
        import torch.distributed as dist
        raw = C.create_string_buffer(64)
        _lib.check(self.lib.b200_engine_ipc_export(self.h, raw), "b200_engine_ipc_export")
        gathered = [None] * self.tp_size
        dist.all_gather_object(gathered, bytes(raw.raw))
        blob = C.create_string_buffer(b"".join(gathered), 64 * self.tp_size)
        _lib.check(self.lib.b200_engine_ipc_import(self.h, blob, self.tp_size), "b200_engine_ipc_import")

    # ------------------------------------------------------------------ weights
    def set_weight(self, name: str, t: torch.Tensor) -> None:
        if "inv_freq" in name:
            return
        if t.dtype != torch.bfloat16:
            t = t.to(torch.bfloat16)
        t = t.contiguous()
        on_dev = 1 if t.is_cuda else 0
        shape = (C.c_int64 * t.dim())(*t.shape)
        _lib.check(self.lib.b200_engine_set_weight(self.h, name.encode(), t.data_ptr(), on_dev, t.dim(), shape),
                   f"set_weight({name})")

    def set_weight_fp8(self, name: str, w: torch.Tensor, scale: torch.Tensor) -> None:
        """an FP8 projection weight: e4m3 codes [out, in] and its checkpoint weight_scale (channel or tensor)"""
        from .fp8 import row_scales
        if w.dtype != torch.float8_e4m3fn:
            raise _lib.B200Error(f"set_weight_fp8({name}): expected float8_e4m3fn codes, got {w.dtype}")
        w = w.contiguous()
        if bool(((w.view(torch.uint8) & 0x7F) == 0x7F).any()):
            # (e4m3fn has no infinities; 0x7F / 0xFF are its NaNs, which no quantizer writes for a finite weight)
            raise _lib.B200Error(f"set_weight_fp8({name}): the weight holds NaN codes")
        s = row_scales(scale, w.shape[0]).to(w.device)
        if s.dtype != torch.bfloat16:
            s = s.to(torch.float32)             # (exact for fp16 / fp32; the engine rounds it to bf16 as transformers does)
        s = s.contiguous()
        shape = (C.c_int64 * 2)(*w.shape)
        _lib.check(self.lib.b200_engine_set_weight_fp8(self.h, name.encode(), w.data_ptr(), s.data_ptr(),
                                                       0 if s.dtype == torch.bfloat16 else 1, 1 if w.is_cuda else 0, 2, shape),
                   f"set_weight_fp8({name})")

    def load_weights(self, named_tensors: Iterable[Tuple[str, torch.Tensor]]) -> None:
        """HF state_dict tensors; FP8 `<proj>.weight` codes are paired with their `<proj>.weight_scale` in any order"""
        pending = {}
        for name, t in named_tensors:
            if name.endswith(".input_scale"):
                raise _lib.B200Error(f"{name}: static FP8 activation scales are not supported (activations stay bf16)")
            if name.endswith(".weight_scale") or (name.endswith(".weight") and t.dtype == torch.float8_e4m3fn):
                base = name[:-len("_scale")] if name.endswith("_scale") else name
                pair = pending.setdefault(base, {})
                pair["scale" if name.endswith("_scale") else "w"] = t
                if len(pair) == 2:
                    self.set_weight_fp8(base, pair["w"], pair["scale"])
                    del pending[base]
                continue
            self.set_weight(name, t)
        if pending:
            raise _lib.B200Error("FP8 weights and scales must come in pairs; unpaired: " + ", ".join(sorted(pending)))
        _lib.check(self.lib.b200_engine_finalize_weights(self.h), "finalize_weights")

    # ------------------------------------------------------------------ generate
    def _params(self, max_new_tokens, pad_token_id, eos_token_ids, stop_sequences, forced_tokens, sampling=None):
        gp = _lib.GenParams()
        sp = sampling or {}
        gp.repetition_penalty = float(sp.get("repetition_penalty") or 0.0)
        gp.do_sample = 1 if sp.get("do_sample") else 0
        gp.temperature = float(sp.get("temperature") or 0.0)
        gp.top_p = float(sp.get("top_p") or 0.0)
        gp.top_k = int(sp.get("top_k") or 0)
        gp.seed = int(sp.get("seed") or 0) & 0xFFFFFFFFFFFFFFFF
        keep = []
        gp.max_new_tokens = int(max_new_tokens)
        gp.pad_token_id = int(pad_token_id if pad_token_id is not None else 0)
        eos = [int(x) for x in (eos_token_ids or [])]
        if eos:
            arr = (C.c_int64 * len(eos))(*eos)
            keep.append(arr)
            gp.eos_token_ids = arr
        gp.num_eos = len(eos)
        stops = [list(map(int, s)) for s in (stop_sequences or []) if len(s) > 0]
        if stops:
            flat = [t for s in stops for t in s]
            offs = [0]
            for s in stops:
                offs.append(offs[-1] + len(s))
            a1 = (C.c_int64 * len(flat))(*flat)
            a2 = (C.c_int32 * len(offs))(*offs)
            keep += [a1, a2]
            gp.stop_tokens, gp.stop_offsets = a1, a2
        gp.num_stop = len(stops)
        if forced_tokens is not None:
            ft = torch.as_tensor(forced_tokens, dtype=torch.int64).contiguous()
            if ft.dim() != 2 or ft.shape[1] != max_new_tokens:
                raise ValueError("forced_tokens must be [B, max_new_tokens]")
            keep.append(ft)
            gp.forced_tokens = C.cast(ft.data_ptr(), C.POINTER(C.c_int64))
        return gp, keep

    def generate(self, input_ids, attention_mask=None, *, max_new_tokens: int, pad_token_id: Optional[int] = 0,
                 eos_token_ids: Sequence[int] = (), stop_sequences: Sequence[Sequence[int]] = (),
                 forced_tokens=None, want_logits: bool = False,
                 streamer: Optional[Callable[[int, List[int]], bool]] = None,
                 repetition_penalty: Optional[float] = None, do_sample: bool = False, temperature: Optional[float] = None,
                 top_p: Optional[float] = None, top_k: Optional[int] = None, seed: Optional[int] = None) -> GenerateResult:
        """`repetition_penalty` / `do_sample` / `temperature` / `top_p` / `top_k` / `seed`: the GenerationConfig fields the
        reference sets (generative_model.py:388-402) plus the checkpoint defaults transformers merges in; greedy when
        do_sample is false (the penalty still applies, as a logits processor does under greedy decoding)."""
        ids = torch.as_tensor(input_ids, dtype=torch.int64).contiguous()
        if ids.dim() != 2 or ids.is_cuda:
            raise ValueError("input_ids must be a host int64 [B, S] tensor")
        B, S = ids.shape
        if int(max_new_tokens) < 1:
            raise ValueError("max_new_tokens must be >= 1")
        mask = None
        if attention_mask is not None:
            mask = torch.as_tensor(attention_mask, dtype=torch.int64).contiguous()
            if mask.shape != ids.shape:          # the C side reads B*S mask words: never let a short buffer through
                raise ValueError(f"attention_mask shape {tuple(mask.shape)} differs from input_ids shape {tuple(ids.shape)}")
        gp, keep = self._params(max_new_tokens, pad_token_id, eos_token_ids, stop_sequences, forced_tokens,
                                dict(repetition_penalty=repetition_penalty, do_sample=do_sample, temperature=temperature,
                                     top_p=top_p, top_k=top_k, seed=seed))
        out = torch.empty((B, S + max_new_tokens), dtype=torch.int64).pin_memory()
        out_len, stop = C.c_int32(0), C.c_int32(0)
        logits = None
        if want_logits:      # tensor parallel: this rank's vocabulary shard (see include/kserve_b200.h)
            logits = torch.empty((max_new_tokens, B, self.vocab_shard()[1]), dtype=torch.bfloat16).pin_memory()
        if streamer is not None:
            def _cb(user, step, toks, batch):
                return 1 if streamer(step, [toks[i] for i in range(batch)]) else 0
            cb = _lib.TOKEN_CALLBACK(_cb)
        else:
            cb = _lib.TOKEN_CALLBACK()
        self._cb_keepalive = cb
        rc = self.lib.b200_generate(self.h, ids.data_ptr(), mask.data_ptr() if mask is not None else None, B, S,
                                    C.byref(gp), out.data_ptr(), C.byref(out_len), C.byref(stop),
                                    logits.data_ptr() if logits is not None else None, cb, None)
        if rc not in (0, 1):
            _lib.check(rc, "b200_generate")
        tm = _lib.Timing()
        self.lib.b200_engine_last_timing(self.h, C.byref(tm))
        T = out_len.value - S
        return GenerateResult(output_ids=out[:, :out_len.value].clone(), stop_triggered=bool(stop.value),
                              num_generated=T, logits=logits[:T].clone() if logits is not None else None,
                              prefill_ms=tm.prefill_ms, decode_ms=tm.decode_ms, decode_steps=tm.decode_steps,
                              kernel_launches=tm.kernel_launches)

    # ------------------------------------------------------------------ batcher leg (ragged rows, no padding)
    def batch_predict(self, rows: Sequence[Sequence[int]], *, max_new_tokens: int, pad_token_id: Optional[int] = 0,
                      eos_token_ids: Sequence[int] = (), stop_sequences: Sequence[Sequence[int]] = ()):
        """-> (predictions int64 [n_rows, T], stop_triggered). The rows run as one batch, without padding."""
        n = len(rows)
        arrs = [(C.c_int64 * len(r))(*[int(t) for t in r]) for r in rows]
        ptrs = (C.c_void_p * n)(*[C.cast(a, C.c_void_p) for a in arrs])
        lens = (C.c_int32 * n)(*[len(r) for r in rows])
        gp, keep = self._params(max_new_tokens, pad_token_id, eos_token_ids, stop_sequences, None)
        pred = torch.empty((n, max_new_tokens), dtype=torch.int64)
        ngen, stop = C.c_int32(0), C.c_int32(0)
        _lib.check(self.lib.b200_batch_predict(self.h, ptrs, lens, n, C.byref(gp), pred.data_ptr(), C.byref(ngen),
                                               C.byref(stop)), "b200_batch_predict")
        return pred[:, :ngen.value].clone(), bool(stop.value)

    # ------------------------------------------------------------------ device-resident replay (bench)
    def stage(self, input_ids, attention_mask=None, *, max_new_tokens: int, pad_token_id: int = 0):
        ids = torch.as_tensor(input_ids, dtype=torch.int64).contiguous()
        mask = None if attention_mask is None else torch.as_tensor(attention_mask, dtype=torch.int64).contiguous()
        gp, keep = self._params(max_new_tokens, pad_token_id, (), (), None)
        B, S = ids.shape
        self._staged_shape = (B, S, max_new_tokens)
        _lib.check(self.lib.b200_stage_prompt(self.h, ids.data_ptr(), mask.data_ptr() if mask is not None else None,
                                              B, S, C.byref(gp)), "b200_stage_prompt")

    def run_staged(self, do_prefill: bool, decode_steps: int) -> None:
        _lib.check(self.lib.b200_run_staged(self.h, 1 if do_prefill else 0, decode_steps), "b200_run_staged")

    def run_staged_timed(self, decode_steps: int):
        """-> (prefill_ms, decode_ms) from CUDA events on the engine stream."""
        a, b = C.c_float(0), C.c_float(0)
        _lib.check(self.lib.b200_run_staged_timed(self.h, decode_steps, C.byref(a), C.byref(b)), "b200_run_staged_timed")
        return a.value, b.value

    def last_timing(self) -> "_lib.Timing":
        tm = _lib.Timing()
        self.lib.b200_engine_last_timing(self.h, C.byref(tm))
        return tm

    def last_launches(self) -> int:
        tm = _lib.Timing()
        self.lib.b200_engine_last_timing(self.h, C.byref(tm))
        return tm.kernel_launches

    def kv_swap_out(self, slot: int, scrub: bool = False) -> None:
        _lib.check(self.lib.b200_kv_swap_out(self.h, slot, 1 if scrub else 0), "b200_kv_swap_out")

    def kv_swap_in(self, slot: int) -> None:
        _lib.check(self.lib.b200_kv_swap_in(self.h, slot), "b200_kv_swap_in")

    # ------------------------------------------------------------------ continuous batching (b200_cb_*)
    def cb_begin(self, pad_token_id: int = 0, eos_token_ids: Sequence[int] = ()) -> None:
        eos = [int(x) for x in eos_token_ids]
        arr = (C.c_int64 * max(1, len(eos)))(*eos)
        _lib.check(self.lib.b200_cb_begin(self.h, int(pad_token_id or 0), arr, len(eos)), "b200_cb_begin")
        self._cb_slots = self.max_batch

    def cb_config(self, prefill_chunk_tokens: int = 0, prefix_cache: bool = False) -> None:
        """chunked prefill (one chunk pass before every decode step) / prefix KV reuse across requests"""
        _lib.check(self.lib.b200_cb_config(self.h, int(prefill_chunk_tokens), 1 if prefix_cache else 0), "b200_cb_config")

    def cb_stats(self) -> dict:
        out = (C.c_int64 * 10)()
        _lib.check(self.lib.b200_cb_stats(self.h, out), "b200_cb_stats")
        keys = ("prompt_tokens", "prefix_hit_tokens", "prefilled_tokens", "evictions", "prefill_passes", "available_pages",
                "cached_blocks", "pending_prompts", "swap_outs", "swap_ins")
        return dict(zip(keys, [int(v) for v in out]))

    def cb_admit(self, prompts: Sequence[Sequence[int]], max_new_tokens: Sequence[int],
                 stop_sequences: Optional[Sequence[Sequence[Sequence[int]]]] = None,
                 sampling: Optional[Sequence[Optional[dict]]] = None) -> List[int]:
        """Admit `prompts` into free slots (prefilled here, or chunk by chunk during the following cb_step calls when
        chunked prefill is configured); returns the slot of each prompt.  `sampling[i]`: None (greedy) or a dict with
        repetition_penalty / do_sample / temperature / top_p / top_k / seed.  Raises PoolExhausted when the KV page
        pool cannot supply the pages: nothing was admitted."""
        n = len(prompts)
        rows = [(C.c_int64 * len(p))(*[int(t) for t in p]) for p in prompts]
        ptrs = (C.POINTER(C.c_int64) * n)(*[C.cast(r, C.POINTER(C.c_int64)) for r in rows])
        lens = (C.c_int32 * n)(*[len(p) for p in prompts])
        mx = (C.c_int32 * n)(*[int(m) for m in max_new_tokens])
        stops = [[list(map(int, q)) for q in (ss or []) if len(q)] for ss in (stop_sequences or [[]] * n)]
        cnt = (C.c_int32 * n)(*[len(ss) for ss in stops])
        flat, offs = [], [0]
        for ss in stops:
            for q in ss:
                flat += q
                offs.append(len(flat))
        offs_a = (C.c_int32 * len(offs))(*offs)
        flat_a = (C.c_int64 * max(1, len(flat)))(*flat)
        samp = None
        if sampling is not None and any(sp for sp in sampling):
            samp = (_lib.GenParams * n)()
            for i, sp in enumerate(sampling):
                sp = sp or {}
                samp[i].repetition_penalty = float(sp.get("repetition_penalty") or 0.0)
                samp[i].do_sample = 1 if sp.get("do_sample") else 0
                samp[i].temperature = float(sp.get("temperature") or 0.0)
                samp[i].top_p = float(sp.get("top_p") or 0.0)
                samp[i].top_k = int(sp.get("top_k") or 0)
                samp[i].seed = int(sp.get("seed") or 0) & 0xFFFFFFFFFFFFFFFF
        slots = (C.c_int32 * n)()
        rc = self.lib.b200_cb_admit(self.h, n, ptrs, lens, mx, cnt, offs_a, flat_a, samp, slots)
        if rc == -7:
            raise PoolExhausted(self.lib.b200_last_error().decode("utf-8", "replace"))
        _lib.check(rc, "b200_cb_admit")
        return list(slots)

    def cb_swap_out(self, slot: int) -> None:
        """preempt a running sequence: its KV pages go to pinned host memory and back to the pool (host-DRAM KV tier)"""
        _lib.check(self.lib.b200_cb_swap_out(self.h, int(slot)), "b200_cb_swap_out")

    def cb_swap_in(self, slot: int) -> None:
        """resume a swapped-out sequence (raises PoolExhausted while the pool cannot supply its pages)"""
        rc = self.lib.b200_cb_swap_in(self.h, int(slot))
        if rc == -7:
            raise PoolExhausted(self.lib.b200_last_error().decode("utf-8", "replace"))
        _lib.check(rc, "b200_cb_swap_in")

    def cb_step(self, n_steps: int = 1) -> None:
        _lib.check(self.lib.b200_cb_step(self.h, n_steps), "b200_cb_step")

    def cb_poll(self):
        """-> (n_gen, finished, stop_hit), each a list over the slots."""
        nb = self.max_batch
        a, b, c = (C.c_int32 * nb)(), (C.c_int32 * nb)(), (C.c_int32 * nb)()
        _lib.check(self.lib.b200_cb_poll(self.h, a, b, c), "b200_cb_poll")
        return list(a), list(b), list(c)

    def cb_read(self, slot: int, first: int = 0, cap: int = 4096) -> List[int]:
        out = (C.c_int64 * cap)()
        n = C.c_int32(0)
        _lib.check(self.lib.b200_cb_read(self.h, slot, first, out, cap, C.byref(n)), "b200_cb_read")
        return list(out[: n.value])

    def cb_release(self, slot: int) -> None:
        _lib.check(self.lib.b200_cb_release(self.h, slot), "b200_cb_release")

    def cb_end(self) -> None:
        _lib.check(self.lib.b200_cb_end(self.h), "b200_cb_end")

    def cb_logits_tap(self, max_steps: int) -> Optional[torch.Tensor]:
        """Turn on the batcher's logits tap (include/kserve_b200.h: b200_cb_logits_tap) and return its device buffer,
        bf16 [max_batch, max_steps, vocab] filled with NaN: row [s, n] receives the logits from which slot s's n-th
        generated token was chosen.  max_steps 0 turns the tap off and returns None."""
        buf = None
        if max_steps > 0:
            buf = torch.full((self.max_batch, int(max_steps), self.vocab), float("nan"), dtype=torch.bfloat16,
                             device=torch.device("cuda", self.device))
            torch.cuda.synchronize(buf.device)
        _lib.check(self.lib.b200_cb_logits_tap(self.h, buf.data_ptr() if buf is not None else None, int(max_steps)),
                   "b200_cb_logits_tap")
        self._cb_tap = buf         # the engine writes into it until the tap is turned off or replaced
        return buf

    def fetch_staged(self) -> torch.Tensor:
        B, S, T = self._staged_shape
        out = torch.empty((B, S + T), dtype=torch.int64)
        out_len, stop = C.c_int32(0), C.c_int32(0)
        _lib.check(self.lib.b200_fetch_staged(self.h, out.data_ptr(), C.byref(out_len), C.byref(stop)),
                   "b200_fetch_staged")
        return out[:, :out_len.value]

    def close(self) -> None:
        if getattr(self, "h", None):
            self.lib.b200_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
