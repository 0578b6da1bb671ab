// Logits processors + sampling on the device — SURVEY.md §8(f) rank 4 / §8a row 4:
// what `build_generation_config` (huggingfaceserver/generative_model.py:388-402) hands to transformers' `_sample`
// (generation/utils.py:2762-2800): logits[:, -1].float() -> RepetitionPenaltyLogitsProcessor (presence_penalty > 0 is
// mapped to repetition_penalty, q8) -> [do_sample only] TemperatureLogitsWarper -> TopKLogitsWarper (GenerationConfig
// default top_k = 50) -> TopPLogitsWarper -> softmax -> multinomial; argmax when do_sample is off (q9).
//
//   * repetition penalty: score = score > 0 ? score / p : score * p for every token id present in input_ids (prompt,
//     pads included, + generated so far) — a bitmap [row][V/32] maintained by seen_init_kernel / step_update_kernel
//   * top-k by an exact 4-pass radix select on the order-preserving uint32 image of the fp32 scores; every tie with the
//     k-th value is kept, as `scores < topk[..., -1]` does, however many there are (candidates above the k-th value and
//     the ties that fit are sorted in shared memory; a draw among the rest counts the ties in index order)
//   * top_k = 1 with do_sample draws among the tokens tied at the maximum; only do_sample = 0 is greedy
//   * top-p exactly as TopPLogitsWarper: ascending cumulative probability <= 1 - top_p is removed, at least one kept
//   * multinomial by inverse CDF with a Philox4x32-10 uniform keyed by (seed, step, row): reproducible per seed, but
//     NOT torch's generator stream — sampled ids are distribution-equal, not bit-equal, to the reference
#pragma once
#include "common.cuh"
#include "ops.cuh"

namespace b200 {

struct SampleCfg {             // device-resident (constant pointer inside CUDA graphs, rewritten per request)
  float rep_penalty;           // 1 = off
  int do_sample;
  float temperature;
  float top_p;
  int top_k;                   // 1..kSampleMaxCand
  unsigned long long seed;
};

constexpr int kSampleMaxCand = 1024;

// -0.0 maps to the key of +0.0: they compare equal, so top-k keeps both or neither
__device__ __forceinline__ uint32_t f32_order_key(float f) {
  const uint32_t u = (f == 0.0f) ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Philox4x32-10 (Salmon et al.), one block
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned long long p0 = (unsigned long long)0xD2511F53u * ctr.x;
    const unsigned long long p1 = (unsigned long long)0xCD9E8D57u * ctr.z;
    uint4 n;
    n.x = (uint32_t)(p1 >> 32) ^ ctr.y ^ key.x;
    n.y = (uint32_t)p1;
    n.z = (uint32_t)(p0 >> 32) ^ ctr.w ^ key.y;
    n.w = (uint32_t)p0;
    ctr = n;
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}

// seen[row][tok] for every prompt token (+ the pad id for left-padded rows: the reference's input_ids holds the pads);
// the bitmap is zeroed with cudaMemsetAsync first
__global__ void seen_set_kernel(uint32_t* __restrict__ seen, int words, const int32_t* __restrict__ tok,
                                const int32_t* __restrict__ tok_seq, int T, const int32_t* __restrict__ cur_len, int B, int S,
                                int pad_token, int V) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < T; i += gridDim.x * blockDim.x) {
    const int t = tok[i];
    if (t >= 0 && t < V) atomicOr(seen + (long long)tok_seq[i] * words + (t >> 5), 1u << (t & 31));
  }
  if (blockIdx.x == 0)
    for (int b = threadIdx.x; b < B; b += blockDim.x)
      if (cur_len[b] < S && pad_token >= 0 && pad_token < V) atomicOr(seen + (long long)b * words + (pad_token >> 5), 1u << (pad_token & 31));
}

struct SampleParams {
  const bf16* logits; long long ld; int V;
  const uint32_t* seen; int words;       // null when the penalty is off
  const SampleCfg* cfg;
  const StepState* st;                   // step counter -> RNG counter
  float* out_val; int32_t* out_idx;      // [B]
  // continuous batching: row b belongs to slot row_slot[b]; cfg[] and the seen bitmaps are per SLOT and the RNG counter
  // of a sequence is its own generated-token count, so a request's stream does not depend on who shares its batch
  const int32_t* row_slot;               // null: static batch (one cfg for all rows, bitmap row == batch row)
  const int32_t* n_gen;                  // [slots]
};

// one CTA of 1024 threads per row
// minimum 1 CTA per SM: ptxas otherwise plans two 1024-thread CTAs per SM, caps the kernel at 32 registers and spills
__global__ void __launch_bounds__(1024, 1) sample_kernel(const SampleParams p) {
  TraceScope _ts(TK_ARGMAX);
  pdl_launch_dependents();
  pdl_wait();
  _ts.mark();
  __shared__ uint32_t hist[256];
  __shared__ float c_key[kSampleMaxCand];
  __shared__ int c_idx[kSampleMaxCand];
  __shared__ uint32_t s_prefix, s_remaining;
  __shared__ int s_count, s_ties, s_pick;
  __shared__ float sv[32];
  __shared__ int si[32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int srow = p.row_slot ? p.row_slot[b] : b;        // row of the per-sequence state
  const SampleCfg cfg = p.cfg[p.row_slot ? srow : 0];
  const bf16* row = p.logits + (long long)b * p.ld;
  const float pen = cfg.rep_penalty;
  const uint32_t* seen = (p.seen && pen != 1.0f) ? p.seen + (long long)srow * p.words : nullptr;
  const bool sampling = cfg.do_sample != 0;
  const float temp = sampling ? cfg.temperature : 1.0f;
  auto score = [&](int i) -> float {
    float x = __bfloat162float(row[i]);                 // logits[:, -1].float()
    if (seen && ((seen[i >> 5] >> (i & 31)) & 1u)) x = (x < 0.f) ? x * pen : x / pen;
    if (sampling) x = x / temp;
    return x;
  };
  if (!sampling) {
    // ---- greedy over the processed scores (ties -> lowest index, like torch.argmax)
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < p.V; i += blockDim.x) {
      const float v = score(i);
      if (v > best || (v == best && i < bi)) { best = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    const int w = tid >> 5, l = tid & 31;
    if (l == 0) { sv[w] = best; si[w] = bi; }
    __syncthreads();
    if (w == 0) {
      best = sv[l]; bi = si[l];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      }
      if (l == 0) { p.out_val[b] = best; p.out_idx[b] = bi; }
    }
    return;
  }
  // ---- top-k: radix select of the k-th largest order key
  const int k = min(min(cfg.top_k, kSampleMaxCand), p.V);
  if (tid == 0) { s_prefix = 0; s_remaining = (uint32_t)k; s_count = 0; s_ties = 0; }
  for (int pass = 3; pass >= 0; --pass) {
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    const uint32_t hi_mask = (pass == 3) ? 0u : (0xFFFFFFFFu << ((pass + 1) * 8));
    for (int i = tid; i < p.V; i += blockDim.x) {
      const uint32_t u = f32_order_key(score(i));
      if ((u & hi_mask) == (prefix & hi_mask)) atomicAdd(&hist[(u >> (pass * 8)) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      uint32_t rem = s_remaining;
      int bin = 255;
      for (; bin > 0; --bin) {
        if (hist[bin] >= rem) break;
        rem -= hist[bin];
      }
      s_remaining = rem;
      s_prefix = prefix | ((uint32_t)bin << (pass * 8));
    }
    __syncthreads();
  }
  // ---- kept set: the G = k - s_remaining tokens above the k-th key, then every tie at the k-th key (transformers keeps
  // them all, `scores < kth` removes none of them).  Order: score descending, index ascending, so the ties come last and
  // share one weight.  The G tokens go to c_[0, G); the ties follow from slot G while they fit.
  const uint32_t kth = s_prefix;
  const int G = k - (int)s_remaining;
  for (int i = tid; i < p.V; i += blockDim.x) {
    const float x = score(i);
    const uint32_t key = f32_order_key(x);
    if (key > kth) {
      const int slot = atomicAdd(&s_count, 1);
      c_key[slot] = x; c_idx[slot] = i;
    } else if (key == kth) {
      const int slot = G + atomicAdd(&s_ties, 1);
      if (slot < kSampleMaxCand) { c_key[slot] = x; c_idx[slot] = i; }
    }
  }
  __syncthreads();
  const int n = G + s_ties;                    // kept tokens; candidate j >= G is a tie
  const int nb = min(n, kSampleMaxCand);
  for (int i = nb + tid; i < kSampleMaxCand; i += blockDim.x) { c_key[i] = -INFINITY; c_idx[i] = 0x7fffffff; }
  __syncthreads();
  // bitonic sort, descending by score, ascending index on ties
  for (int size = 2; size <= kSampleMaxCand; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const int i = tid, j = i ^ stride;
      if (j > i) {
        const bool desc = ((i & size) == 0);
        const float ki = c_key[i], kj = c_key[j];
        const int ii = c_idx[i], ij = c_idx[j];
        const bool i_first = (ki > kj) || (ki == kj && ii < ij);   // i should precede j in descending order
        if (desc ? !i_first : i_first) { c_key[i] = kj; c_key[j] = ki; c_idx[i] = ij; c_idx[j] = ii; }
      }
      __syncthreads();
    }
  }
  if (tid == 0) {
    // softmax over the kept tokens, TopPLogitsWarper, renormalise, inverse-CDF draw
    const float m = c_key[0];
    const float e_tie = expf(c_key[G] - m);
    auto wt = [&](int j) { return j < G ? expf(c_key[j] - m) : e_tie; };
    float Z = 0.f;
    for (int j = 0; j < n; ++j) Z += wt(j);
    int keep = n;
    if (cfg.top_p < 1.0f) {
      // ascending cumulative prob (tail sum from the smallest up to j) <= 1 - top_p  =>  removed
      float tail = 0.f;
      keep = 1;
      for (int j = n - 1; j >= 1; --j) {
        tail += wt(j) / Z;
        if (tail > 1.0f - cfg.top_p) { keep = j + 1; break; }
      }
    }
    float Zk = 0.f;
    for (int j = 0; j < keep; ++j) Zk += wt(j);
    const uint4 r = philox4x32_10(make_uint4(p.row_slot ? (uint32_t)p.n_gen[srow] : (uint32_t)p.st->step, p.row_slot ? 0u : (uint32_t)b, 0x5eed5eedu, 0u),
                                  make_uint2((uint32_t)cfg.seed, (uint32_t)(cfg.seed >> 32)));
    const float u = ((float)(r.x >> 8) + 0.5f) * (1.0f / 16777216.0f);   // (0, 1)
    const float target = u * Zk;
    float acc = 0.f;
    int pick = keep - 1;
    for (int j = 0; j < keep; ++j) {
      acc += wt(j);
      if (acc >= target) { pick = j; break; }
    }
    s_pick = pick;
  }
  __syncthreads();
  const int pick = s_pick;
  if (pick < G || n <= kSampleMaxCand) {       // the candidate buffer holds the pick
    if (tid == 0) { p.out_val[b] = c_key[pick]; p.out_idx[b] = c_idx[pick]; }
    return;
  }
  // more ties than the buffer holds: the pick is tie number pick - G in index order, found by an ordered block-wide count
  const int want = pick - G, w = tid >> 5, l = tid & 31;
  for (int t0 = 0, before = 0; t0 < p.V && before <= want; t0 += blockDim.x) {   // before: ties at indices < t0
    const int i = t0 + tid;
    const bool tie = i < p.V && f32_order_key(score(i)) == kth;
    const uint32_t bal = __ballot_sync(0xffffffffu, tie);
    if (l == 0) si[w] = __popc(bal);
    __syncthreads();
    int below = before + __popc(bal & ((1u << l) - 1u)), total = before;
    for (int q = 0; q < 32; ++q) { total += si[q]; if (q < w) below += si[q]; }
    if (tie && below == want) { p.out_val[b] = score(i); p.out_idx[b] = i; }
    before = total;
    __syncthreads();
  }
}

}  // namespace b200
