// Continuous (iteration-level) batching — SURVEY.md §8(f) rank 1: replaces the strictly serial request loop of
// the reference (generative_model.py:341-354, one `generate` at a time, q10) and subsumes what the Go batcher does
// for throughput (handler.go:157-188): sequences join and leave the running batch between decode steps.
//
// State is kept per SLOT (a slot owns a fixed run of KV pages: slot s -> pages [s * max_pages, (s+1) * max_pages)).
// A decode step runs over the compact list of active slots `row_slot[R]`; the three per-row arrays the forward pass
// reads (next token, sequence slot, position) are gathered from the slot state at the start of every step, so the
// forward kernels are exactly the ones of the static-batch path (same CUDA graph structure, keyed by R).
#pragma once
#include "common.cuh"
#include "ops.cuh"
#include "p2p_base.cuh"

namespace b200 {

constexpr int kCbMaxStop = 4;       // stop sequences per sequence
constexpr int kCbMaxStopLen = 8;    // tokens per stop sequence
constexpr int kCbInitInts = 4 + kCbMaxStop + kCbMaxStop * kCbMaxStopLen;   // host -> device init record per sequence

struct CbState {
  int32_t* len;        // [slots] tokens in the KV cache
  int32_t* n_gen;      // [slots] tokens generated so far
  int32_t* max_new;    // [slots]
  int32_t* finished;   // [slots] 1 once EOS / length / stop ended the sequence
  int32_t* stop_hit;   // [slots] 1 iff a stop sequence matched (finish_reason == "stop")
  int32_t* next_tok;   // [slots] input token of the next decode step
  int32_t* out;        // [slots][out_ld] generated tokens
  int32_t* stop_len;   // [slots][kCbMaxStop]
  int32_t* stop_tok;   // [slots][kCbMaxStop][kCbMaxStopLen]
  int out_ld;
};

// record i: {slot, prompt_len, max_new, num_stop, stop_len[4], stop_tok[4][8]}
__global__ void cb_init_kernel(const int32_t* __restrict__ rec, int n, CbState st) {
  const int i = blockIdx.x;
  if (i >= n) return;
  const int32_t* r = rec + (long long)i * kCbInitInts;
  const int slot = r[0];
  if (threadIdx.x == 0) {
    st.len[slot] = r[1] - 1;     // the step kernel's len++ after the prefill pass makes it prompt_len
    st.n_gen[slot] = 0;
    st.max_new[slot] = r[2];
    st.finished[slot] = 0;
    st.stop_hit[slot] = 0;
    st.next_tok[slot] = 0;
  }
  for (int j = threadIdx.x; j < kCbMaxStop; j += blockDim.x) st.stop_len[slot * kCbMaxStop + j] = j < r[3] ? r[4 + j] : 0;
  for (int j = threadIdx.x; j < kCbMaxStop * kCbMaxStopLen; j += blockDim.x)
    st.stop_tok[slot * kCbMaxStop * kCbMaxStopLen + j] = r[4 + kCbMaxStop + j];
}

// row arrays of the decode forward pass from the slot state
__global__ void cb_gather_kernel(const int32_t* __restrict__ row_slot, int R, CbState st, int32_t* __restrict__ next_tok,
                                 int32_t* __restrict__ seq_slot, int32_t* __restrict__ dec_pos) {
  TraceScope _ts(TK_OTHER);
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int slot = row_slot[r];
  next_tok[r] = st.next_tok[slot];
  seq_slot[r] = slot;
  dec_pos[r] = st.len[slot];     // a finished slot keeps rewriting the same cache position: harmless, never read
}

// logits tap (b200_cb_logits_tap): one CTA per row copies the row's logits to buf[slot][n_gen[slot]], the step whose
// token the step kernel is about to append, while that is below max_steps.  Runs between the LM-head GEMM and the
// argmax / sample kernel, so n_gen has not advanced yet; finished slots (frozen rows of the decode pass) are skipped.
__global__ void cb_tap_kernel(const bf16* __restrict__ logits, long long ld, int V, const int32_t* __restrict__ row_slot,
                              CbState st, bf16* __restrict__ buf, int max_steps) {
  TraceScope _ts(TK_OTHER);
  pdl_launch_dependents();
  pdl_wait();
  const int slot = row_slot[blockIdx.x];
  const int g = st.n_gen[slot];
  if (st.finished[slot] || g >= max_steps) return;
  const bf16* src = logits + (long long)blockIdx.x * ld;
  bf16* dst = buf + ((long long)slot * max_steps + g) * V;
  for (int i = threadIdx.x; i < V; i += blockDim.x) dst[i] = src[i];
}

// one thread per row: merge the argmax candidates, append the token, EOS / max_new / stop sequences per sequence.
// use_p2p: tensor parallel — the vocab-parallel candidates of every rank arrive through peer memory (argmax_kernel
// pushes them); every row merges them even when its slot is finished, so the exchange epochs stay in step on all ranks.
// seen: per-SLOT token-presence bitmaps of the repetition penalty (null when no running sequence uses one).
__global__ void __launch_bounds__(128)
cb_step_kernel(const float* __restrict__ cand_val, const int32_t* __restrict__ cand_idx, int ranks, int R,
               const int32_t* __restrict__ row_slot, CbState st, const int32_t* __restrict__ eos, int num_eos,
               P2P pp, int use_p2p, uint32_t* __restrict__ seen, int seen_words, int V) {
  TraceScope _ts(TK_STEP);
  pdl_launch_dependents();
  pdl_wait();
  _ts.mark();
  if (use_p2p && threadIdx.x == 0) pp.row_epoch[0] += 1;   // epoch base of the next forward pass's peer all-reduces
  for (int r = threadIdx.x; r < R; r += blockDim.x) {
    const int slot = row_slot[r];
    float best = cand_val[r];
    int tok = cand_idx[r];
    if (use_p2p) merge_candidates(pp, r, best, tok);
    for (int k = 1; k < ranks && !use_p2p; ++k) {
      const float v = cand_val[k * R + r];
      const int i = cand_idx[k * R + r];
      if (v > best || (v == best && i < tok)) { best = v; tok = i; }
    }
    if (st.finished[slot]) continue;
    const int g = st.n_gen[slot];
    int32_t* out = st.out + (long long)slot * st.out_ld;
    out[g] = tok;
    st.n_gen[slot] = g + 1;
    st.len[slot] += 1;
    st.next_tok[slot] = tok;
    if (seen && tok >= 0 && tok < V) atomicOr(seen + (long long)slot * seen_words + (tok >> 5), 1u << (tok & 31));
    int fin = 0;
    for (int e = 0; e < num_eos; ++e) fin |= (tok == eos[e]);
    if (g + 1 >= st.max_new[slot]) fin = 1;
    for (int s = 0; s < kCbMaxStop; ++s) {
      const int n = st.stop_len[slot * kCbMaxStop + s];
      if (n == 0 || n > g + 1) continue;
      const int32_t* sq = st.stop_tok + (slot * kCbMaxStop + s) * kCbMaxStopLen;
      bool eq = true;
      for (int i = 0; i < n && eq; ++i) eq = out[g + 1 - n + i] == sq[i];
      if (eq) { fin = 1; st.stop_hit[slot] = 1; }
    }
    if (fin) st.finished[slot] = 1;
  }
}

}  // namespace b200
