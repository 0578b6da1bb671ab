// Persistent, warp-specialised bf16 GEMM for sm_90a:  D[M,N] = A[M,K] * B[N,K]^T  (both K-major).
//
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx)
//   warpgroups 1-2 : wgmma consumers, one 64-row half of the 128-row tile each (m64nBLOCK_Nk16, fp32 accumulators in
//                    registers); the accumulators are staged through shared memory so that the fused epilogue sees
//                    one tile row per thread, 32 consecutive columns at a time
//
// The same kernel serves both phases of the LLM path (SURVEY.md §8a rows 13-17):
//   * prefill  : A = activations [T,K], B = weight [N_out,K]           -> row-major epilogues
//   * decode   : A = weight [N_out,K] (M = N_out), B = activations [batch,K] ("swap-AB": the 128-row MMA
//                M dimension is filled by weight rows, the small batch rides in the MMA N dimension, so no
//                tensor-core work is wasted on padding and each CTA streams a contiguous weight slab)
//                -> transposed epilogues, optional split-K with fp32 partials.
#pragma once
#include "common.cuh"

namespace b200 {

enum GemmEpi : int {
  EPI_STORE = 0,      // out[m][n] = bf16(acc)
  EPI_STORE_RES = 1,  // out[m][n] = bf16(bf16(acc) + residual[m][n])           (o_proj / down_proj + residual)
  EPI_SWIGLU = 2,     // B rows interleaved {16 gate,16 up}: out[m][n/2] = bf16(bf16(silu(g)) * u)
  EPI_T_STORE = 3,    // out[n][m] = bf16(acc)                                    (swap-AB)
  EPI_T_SWIGLU = 4,   // A rows interleaved {16 gate,16 up}: out[n][m/2] = ...    (swap-AB)
  EPI_T_PARTIAL = 5,  // ws[split][n][m] = acc (fp32)                             (swap-AB split-K)
  EPI_ROPE_KV = 6,    // prefill QKV projection (BLOCK_N 256): columns are [q heads | k heads | v heads] x 128;
                      // q <- RoPE(q) in place in `out`, RoPE(k) and v go straight to the paged KV cache
};

struct GemmParams {
  int M, N, K;
  int m_tiles, n_tiles, splits;
  int kb_total;       // ceil(K / 64)
  int kb_per_split;   // ceil(kb_total / splits)
  void* out;
  const bf16* residual;
  long long ldo;           // leading dimension of out (elements)
  long long split_stride;  // EPI_T_PARTIAL: elements between split slices
  int out_cols;            // logical number of output columns (bounds for SWIGLU modes = N/2 resp. M/2)
  unsigned long long hint_a, hint_b;
  int prefetch_a;          // A (weights) does not depend on the previous kernel: stream it before griddepcontrol.wait
  int l2_prefetch_kb;      // additional k-blocks of A to pull into L2 (beyond the smem stages) before the wait
  // sched == 1: "stream-K" — the m_tiles * kb_total k-block iterations are cut into gridDim.x equal contiguous
  // ranges, so every SM streams the same number of weight bytes whatever the tile count (few tiles under tensor
  // parallelism, 224 tiles on 132 SMs, ...).  A tile covered by several CTAs is finished by the CTA that owns
  // its last k-block: the others park fp32 partials in sk_ws[tile][piece] and bump sk_flags[tile]; the owner
  // waits for the count, adds the pieces in piece order (deterministic) and runs the normal epilogue.
  // Each CTA processes its non-final piece first and its tile-finishing piece last, so nobody waits on a CTA
  // that is itself waiting.  Requires n_tiles == 1 and splits == 1.
  // runtime extents (device counters, e.g. tokens routed to one MoE expert): when set they replace M (row-major
  // kernels) / N (swap-AB kernels) and the kernel first waits for its predecessor to read them; 0 => nothing to do
  const int* m_rt;
  const int* n_rt;
  const int* row_off;      // device row offset of the activation / output rows inside a grouped (per-expert) buffer
  int swap_ab;             // 1: A is the weight (decode kernels) -> row_off applies to B and to the output rows n
  // grouped (per-expert) swap-AB problem in ONE launch: A = [groups][M][K] stacked weights, m_tiles = groups * group_m_tiles;
  // tile m_t belongs to group g = m_t / group_m_tiles whose activation rows are row_off[g] .. + n_rt[g] (tiles of
  // empty groups are skipped: their weights are never streamed) and whose outputs start at out + g * group_out_stride
  int group_m_tiles;
  long long group_out_stride;
  // EPI_ROPE_KV: one output row = one prompt token (HF bf16 rounding points of apply_rotary_pos_emb; bit-identical to rope_kv_kernel)
  const int32_t* rope_tok_seq; const int32_t* rope_tok_pos;   // [M] page-table row / position of each token
  const int32_t* rope_page_table; int rope_max_pages;
  bf16* rope_kcache; bf16* rope_vcache;                      // this layer's [page][kv_head][64][128]
  const bf16* rope_cos; const bf16* rope_sin;                // [max_pos][64]
  int rope_nh, rope_nkv;
  int stream_out;          // row-major epilogues: cache-streaming output stores
  int sched;
  int sk_slots;            // partial slots per tile
  float* sk_ws;            // [m_tiles][sk_slots][BLOCK_N][128] fp32
  int* sk_flags;           // [m_tiles] arrival counters, 0 between launches
};

constexpr int kGemmBlockM = 128;
constexpr int kGemmBlockK = 64;
constexpr int kGemmThreads = 384;
constexpr int kGemmGroupM = 16;
constexpr int kStgStride = 132;   // floats between two staged accumulator columns: 128 rows + 4 (conflict-free fragment stores)

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kABytes = kGemmBlockM * kGemmBlockK * 2;  // 16 KB
  static constexpr int kBBytes = BLOCK_N * kGemmBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (BLOCK_N >= 256) ? 3 : 8;
  static constexpr int kChunk = (BLOCK_N >= 32) ? 32 : 16;             // columns one epilogue thread takes at a time
  static constexpr int kRoundCols = (BLOCK_N < 128) ? BLOCK_N : 128;   // columns staged per epilogue round (one head)
  static constexpr int kChunks = kRoundCols / kChunk;
  static constexpr int kStgBytes = kRoundCols * kStgStride * 4;
  static constexpr int kSmemBytes = kStages * kStageBytes + kStgBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 227 * 1024, "GEMM shared memory exceeds the 227 KB a block may use");
};

template <int N>
__device__ __forceinline__ void wgmma_tile(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  if constexpr (N == 16) wgmma_ss_n16(d, adesc, bdesc, scale_d);
  else if constexpr (N == 32) wgmma_ss_n32(d, adesc, bdesc, scale_d);
  else if constexpr (N == 64) wgmma_ss_n64(d, adesc, bdesc, scale_d);
  else wgmma_ss_n256(d, adesc, bdesc, scale_d);
}

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }   // both MMA warpgroups

// output tiles are written once and read by a LATER kernel: with stream_out they go out as cache-streaming stores so that
// the (up to 940 MB per GEMM) output stream does not push the A / B tiles the other CTAs are about to re-read out of L2
__device__ __forceinline__ void st_out_v4(bf16* p, const uint4& o, int stream_out) {
  if (stream_out) asm volatile("st.global.cs.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(o.x), "r"(o.y), "r"(o.z), "r"(o.w) : "memory");
  else *reinterpret_cast<uint4*>(p) = o;
}

// SiLU on an already bf16-rounded input whose result is rounded to bf16 again: the fast exp / divide intrinsics
// (rel. error ~1e-6) cannot change the bf16 result except on exact rounding ties, and keep the epilogue short.
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }


struct GemmSeg { int m_t, n_t, kb0, kb1, split, type, slot; };  // type: 0 full tile, 1 partial piece -> workspace slot, 2 tile-finishing piece (adds `slot` parked pieces)

__device__ __forceinline__ int sk_owner(long long it, long long W, int P) {   // CTA whose range contains iteration `it`
  int c = (int)((it * P) / W);
  while (W * (c + 1) / P <= it) ++c;
  while (W * c / P > it) --c;
  return c;
}

// The work list of CTA `cta` of `ncta`: shared by the GEMM kernel (cta = blockIdx.x) and by the weight-stream
// prefetcher, which walks the same list ahead of it.
struct GemmSched { int m_tiles, n_tiles, splits, kb_total, kb_per_split, sched; };

__device__ __forceinline__ bool gemm_get_seg(const GemmSched& p, int idx, GemmSeg& g, int m_tiles_rt, int cta, int ncta) {
  g.slot = 0;
  if (m_tiles_rt <= 0) return false;
  if (p.sched == 0) {
    const int u = cta + idx * ncta;
    if (u >= m_tiles_rt * p.n_tiles * p.splits) return false;
    const int tile = u / p.splits;
    g.split = u - tile * p.splits;
    const int per_group = kGemmGroupM * p.n_tiles;
    const int grp = tile / per_group;
    const int first_m = grp * kGemmGroupM;
    const int gsize = min(m_tiles_rt - first_m, kGemmGroupM);
    const int r = tile - grp * per_group;
    g.m_t = first_m + r % gsize;
    g.n_t = r / gsize;
    g.kb0 = g.split * p.kb_per_split;
    g.kb1 = min(g.kb0 + p.kb_per_split, p.kb_total);
    g.type = 0;
    return true;
  }
  const int P = ncta, c = cta, KB = p.kb_total;
  const long long W = (long long)p.m_tiles * KB;
  const long long lo = W * c / P, hi = W * (c + 1) / P;
  if (lo >= hi) return false;
  const int t0 = (int)(lo / KB), k_lo = (int)(lo % KB);
  const int t1 = (int)((hi - 1) / KB), k_hi = (int)((hi - 1) % KB) + 1;
  const int has_piece = (k_hi < KB) ? 1 : 0;                                   // last tile of the range is finished by a later CTA
  const int has_tail = (k_lo > 0 && !(t0 == t1 && has_piece)) ? 1 : 0;          // first tile was started by an earlier CTA, we finish it
  const int f0 = t0 + ((k_lo > 0) ? 1 : 0), f1 = t1 - has_piece;
  const int n_full = max(0, f1 - f0 + 1);
  g.n_t = 0; g.split = 0;
  if (idx < has_piece) {
    g.m_t = t1; g.kb0 = (t0 == t1) ? k_lo : 0; g.kb1 = k_hi; g.type = 1;
    g.slot = c - sk_owner((long long)t1 * KB, W, P);
    return true;
  }
  idx -= has_piece;
  if (idx < n_full) { g.m_t = f0 + idx; g.kb0 = 0; g.kb1 = KB; g.type = 0; return true; }
  idx -= n_full;
  if (idx < has_tail) {
    g.m_t = t0; g.kb0 = k_lo; g.kb1 = KB; g.type = 2;
    g.slot = c - sk_owner((long long)t0 * KB, W, P);   // number of parked pieces to wait for
    return true;
  }
  return false;
}

__device__ __forceinline__ bool gemm_get_seg(const GemmParams& p, int idx, GemmSeg& g, int m_tiles_rt) {
  const GemmSched sc{p.m_tiles, p.n_tiles, p.splits, p.kb_total, p.kb_per_split, p.sched};
  return gemm_get_seg(sc, idx, g, m_tiles_rt, (int)blockIdx.x, (int)gridDim.x);
}

template <int BLOCK_N, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmParams p) {
  TraceScope _ts(TK_GEMM + 100 * EPI + 1000 * (p.M >> 7));
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int STAGES = Cfg::kStages;
  constexpr int CH = Cfg::kChunk;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* stg = reinterpret_cast<float*>(smem + STAGES * Cfg::kStageBytes);   // [kRoundCols][kStgStride] fp32
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::kStageBytes + Cfg::kStgBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrival per MMA warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  int M_rt = p.M, N_rt = p.N;
  const int gmt = p.group_m_tiles;
  if (p.m_rt != nullptr || p.n_rt != nullptr) {   // extents produced by the previous kernel
    pdl_wait();
    if (p.m_rt) M_rt = min(p.M, *p.m_rt);
    if (p.n_rt && !gmt) N_rt = min(p.N, *p.n_rt);
  }
  const int m_tiles_rt = gmt ? p.m_tiles : ((M_rt <= 0 || N_rt <= 0) ? 0 : (M_rt + kGemmBlockM - 1) / kGemmBlockM);
  const int roff = (p.row_off && !gmt) ? *p.row_off : 0;   // (read after the wait above: set together with m_rt / n_rt)
  const int roff_a = p.swap_ab ? 0 : roff;
  int roff_b = p.swap_ab ? roff : 0;

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      bool first = true;
      GemmSeg sg;
      for (int idx = 0; gemm_get_seg(p, idx, sg, m_tiles_rt); ++idx) {
        const int m_t = sg.m_t, n_t = sg.n_t, kb0 = sg.kb0, kb1 = sg.kb1;
        int a_row = m_t * kGemmBlockM + roff_a, b_off = roff_b;
        if (gmt) {
          const int g = m_t / gmt;
          if (p.n_rt[g] <= 0) continue;
          a_row = g * p.M + (m_t - g * gmt) * kGemmBlockM;
          b_off = p.row_off[g];
        }
        int kb = kb0;
        if (first) {
          first = false;
          if (p.prefetch_a) {
            // Weight tiles of the first k-blocks are requested before the previous kernel has finished; only the
            // activation tiles wait for it.  (All stages are free at this point: no empty-barrier wait needed.)
            const int npre = min(STAGES, kb1 - kb0);
            for (int i = 0; i < npre; ++i) {
              mbar_arrive_expect_tx(&full_bar[i], Cfg::kStageBytes);
              tma_load_2d(smem + i * Cfg::kStageBytes, &tmap_a, &full_bar[i], (kb0 + i) * kGemmBlockK, a_row, p.hint_a);
            }
            const int npf = min(npre + p.l2_prefetch_kb, kb1 - kb0);
            for (int i = npre; i < npf; ++i) tma_prefetch_l2_2d(&tmap_a, (kb0 + i) * kGemmBlockK, m_t * kGemmBlockM);
            pdl_wait();
            _ts.mark();
            for (int i = 0; i < npre; ++i)
              tma_load_2d(smem + i * Cfg::kStageBytes + Cfg::kABytes, &tmap_b, &full_bar[i], (kb0 + i) * kGemmBlockK, n_t * BLOCK_N + b_off, p.hint_b);
            kb = kb0 + npre;
            if (npre == STAGES) { stage = 0; phase = 1; } else { stage = npre; }
          } else {
            pdl_wait();
          }
        }
        for (; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * kGemmBlockK, a_row, p.hint_a);
          tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * kGemmBlockK, n_t * BLOCK_N + b_off, p.hint_b);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA + epilogue (2 warpgroups)
    setmaxnreg_inc<232>();
    const int half = wg - 1;                 // accumulator rows 64 * half ... + 63 of the tile
    const int t = threadIdx.x - 128 * wg;    // thread of the warpgroup == tile row it owns in the epilogue
    const int et = threadIdx.x - 128;        // 0 .. 255
    const int q = t >> 5;                    // 32-row slab of the epilogue row (lane == t & 31)
    const int frag_row = 64 * half + 16 * (warp & 3) + (lane >> 2);   // accumulator rows frag_row, frag_row + 8
    pdl_wait();              // outputs / residual must not be touched before the previous kernel is complete
    int stage = 0;
    uint32_t phase = 0;
    float accum[BLOCK_N / 2];
    GemmSeg sg;
    for (int idx = 0; gemm_get_seg(p, idx, sg, m_tiles_rt); ++idx) {
      const int n_t = sg.n_t, s = sg.split, kb0 = sg.kb0, kb1 = sg.kb1;
      int m_t = sg.m_t;
      long long out_off = 0;   // elements
      if (gmt) {
        const int g = m_t / gmt;
        N_rt = min(p.N, p.n_rt[g]);
        if (N_rt <= 0) continue;
        roff_b = p.row_off[g];
        m_t -= g * gmt;         // tile index inside the group: output features are per expert
        out_off = (long long)g * p.group_out_stride;
      }
      // ---- main loop: one k-block in flight behind the one being issued
      wgmma_keep(accum);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
        const uint64_t adesc = make_smem_desc_sw128(sa + half * 64 * 128);
        const uint64_t bdesc = make_smem_desc_sw128(sa + Cfg::kABytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kGemmBlockK / 16; ++k)
          wgmma_tile<BLOCK_N>(accum, adesc + 2 * k, bdesc + 2 * k, (kb > kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);   // the k-block before this one has been consumed
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_keep(accum);
      if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);

      // ---- epilogue
      const int m = m_t * kGemmBlockM + t;  // accumulator row of this thread
      const int n0 = n_t * BLOCK_N;
      const long long sk_piece = (long long)BLOCK_N * kGemmBlockM;
      float* skw = (sg.type != 0) ? p.sk_ws + ((long long)sg.m_t * p.sk_slots) * sk_piece + t : nullptr;
      if (sg.type == 2 && et == 0) {   // wait until every other piece of this tile has been parked
        SpinGuard spins;
        while (*reinterpret_cast<volatile int*>(p.sk_flags + sg.m_t) != sg.slot)
          if (spin_give_up(spins, 4)) break;
        __threadfence();
      }
#pragma unroll
      for (int r0 = 0; r0 < BLOCK_N; r0 += Cfg::kRoundCols) {
        if (n0 + r0 >= N_rt) break;   // uniform: nothing valid from here on
        consumer_bar();               // the previous round's staged columns have been read
#pragma unroll
        for (int j = r0 / 8; j < (r0 + Cfg::kRoundCols) / 8; ++j) {
          float* s0 = stg + (8 * j + 2 * (lane & 3) - r0) * kStgStride + frag_row;
          s0[0] = accum[4 * j];
          s0[kStgStride] = accum[4 * j + 1];
          s0[8] = accum[4 * j + 2];
          s0[kStgStride + 8] = accum[4 * j + 3];
        }
        consumer_bar();
        if constexpr (EPI == EPI_ROPE_KV) {
          // the round's 128 columns are one whole head; this warpgroup takes dims [32 * half, 32 * half + 32) and their
          // rotate-half partners 64 further (V: the same two 32-column chunks)
          const int col0 = n0 + r0;
          const int head = col0 >> 7;
          if (m < M_rt) {
            const int pos = p.rope_tok_pos[m + roff_a];
            const int page = p.rope_page_table[(long long)p.rope_tok_seq[m + roff_a] * p.rope_max_pages + (pos >> 6)];
            const long long page_row = (long long)page * p.rope_nkv * 64 + (pos & 63);   // row of kv head 0 in [..][64][128]
            const int c = 32 * half;
            if (head >= p.rope_nh + p.rope_nkv) {           // ---- V head: copy to the cache
              bf16* vrow = p.rope_vcache + (page_row + (long long)(head - p.rope_nh - p.rope_nkv) * 64) * 128;
#pragma unroll
              for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int j = 0; j < 32; j += 8) {
                  const float* sv = stg + (hh * 64 + c + j) * kStgStride + t;
                  uint4 o;
                  o.x = pack_bf16x2(sv[0], sv[kStgStride]);
                  o.y = pack_bf16x2(sv[2 * kStgStride], sv[3 * kStgStride]);
                  o.z = pack_bf16x2(sv[4 * kStgStride], sv[5 * kStgStride]);
                  o.w = pack_bf16x2(sv[6 * kStgStride], sv[7 * kStgStride]);
                  *reinterpret_cast<uint4*>(vrow + hh * 64 + c + j) = o;
                }
            } else {                                         // ---- q or k head: rotate-half RoPE on the pairs (d, d + 64)
              bf16* dst = head < p.rope_nh ? reinterpret_cast<bf16*>(p.out) + (long long)(m + roff_a) * p.ldo + col0
                                           : p.rope_kcache + (page_row + (long long)(head - p.rope_nh) * 64) * 128;
#pragma unroll
              for (int j = 0; j < 32; j += 8) {
                const uint4 cu = *reinterpret_cast<const uint4*>(p.rope_cos + (long long)pos * 64 + c + j);
                const uint4 su = *reinterpret_cast<const uint4*>(p.rope_sin + (long long)pos * 64 + c + j);
                const uint32_t cw[4] = {cu.x, cu.y, cu.z, cu.w}, sw[4] = {su.x, su.y, su.z, su.w};
                const float* s1 = stg + (c + j) * kStgStride + t;
                const float* s2 = s1 + 64 * kStgStride;
                float o1[8], o2[8];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                  const float2 cs = unpack_bf16x2(cw[u]), sn = unpack_bf16x2(sw[u]);
                  const float a0 = bf16_round(s1[(2 * u) * kStgStride]), a1 = bf16_round(s1[(2 * u + 1) * kStgStride]);
                  const float b0 = bf16_round(s2[(2 * u) * kStgStride]), b1 = bf16_round(s2[(2 * u + 1) * kStgStride]);
                  o1[2 * u] = bf16_round(a0 * cs.x) + bf16_round(-b0 * sn.x);
                  o1[2 * u + 1] = bf16_round(a1 * cs.y) + bf16_round(-b1 * sn.y);
                  o2[2 * u] = bf16_round(b0 * cs.x) + bf16_round(a0 * sn.x);
                  o2[2 * u + 1] = bf16_round(b1 * cs.y) + bf16_round(a1 * sn.y);
                }
                uint4 w1, w2;
                w1.x = pack_bf16x2(o1[0], o1[1]); w1.y = pack_bf16x2(o1[2], o1[3]); w1.z = pack_bf16x2(o1[4], o1[5]); w1.w = pack_bf16x2(o1[6], o1[7]);
                w2.x = pack_bf16x2(o2[0], o2[1]); w2.y = pack_bf16x2(o2[2], o2[3]); w2.z = pack_bf16x2(o2[4], o2[5]); w2.w = pack_bf16x2(o2[6], o2[7]);
                *reinterpret_cast<uint4*>(dst + c + j) = w1;
                *reinterpret_cast<uint4*>(dst + 64 + c + j) = w2;
              }
            }
          }
          continue;
        }
        // this warpgroup's chunks of the round: half, half + 2
#pragma unroll
        for (int ch = half; ch < Cfg::kChunks; ch += 2) {
          const int c0 = r0 + ch * CH;
          if (n0 + c0 >= N_rt) break;  // warpgroup-uniform: nothing valid in this chunk
          float v[CH];
#pragma unroll
          for (int j = 0; j < CH; ++j) v[j] = stg[(ch * CH + j) * kStgStride + t];
          const int nvalid = min(CH, N_rt - (n0 + c0));
          if (sg.type == 1) {          // park the fp32 accumulators of this piece, the tile's owner finishes it
            float* w = skw + (long long)sg.slot * sk_piece;
#pragma unroll
            for (int j = 0; j < CH; ++j) w[(long long)(c0 + j) * kGemmBlockM] = v[j];
            continue;
          }
          if (sg.type == 2) {          // pieces are added in piece (= k) order, then this CTA's own tail
            float acc[CH];
#pragma unroll
            for (int j = 0; j < CH; ++j) acc[j] = 0.f;
            for (int sl = 0; sl < sg.slot; ++sl) {
              const float* w = skw + (long long)sl * sk_piece;
#pragma unroll
              for (int j = 0; j < CH; ++j) acc[j] += __ldcg(w + (long long)(c0 + j) * kGemmBlockM);
            }
#pragma unroll
            for (int j = 0; j < CH; ++j) v[j] += acc[j];
          }
          if constexpr (EPI == EPI_STORE || EPI == EPI_STORE_RES) {
            if (m < M_rt) {
              bf16* orow = reinterpret_cast<bf16*>(p.out) + (long long)(m + roff_a) * p.ldo + n0 + c0;
              const bf16* rrow = (EPI == EPI_STORE_RES) ? p.residual + (long long)(m + roff_a) * p.ldo + n0 + c0 : nullptr;
              const bool vec = (nvalid == CH) && ((p.ldo & 7) == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 15) == 0);
              if (vec) {
#pragma unroll
                for (int j = 0; j < CH; j += 8) {
                  float f[8];
#pragma unroll
                  for (int u = 0; u < 8; ++u) f[u] = v[j + u];
                  if constexpr (EPI == EPI_STORE_RES) {
                    uint4 rr = *reinterpret_cast<const uint4*>(rrow + j);
                    const uint32_t rw[4] = {rr.x, rr.y, rr.z, rr.w};
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                      float2 r2 = unpack_bf16x2(rw[u]);
                      f[2 * u] = bf16_round(f[2 * u]) + r2.x;
                      f[2 * u + 1] = bf16_round(f[2 * u + 1]) + r2.y;
                    }
                  }
                  uint4 o;
                  o.x = pack_bf16x2(f[0], f[1]);
                  o.y = pack_bf16x2(f[2], f[3]);
                  o.z = pack_bf16x2(f[4], f[5]);
                  o.w = pack_bf16x2(f[6], f[7]);
                  st_out_v4(orow + j, o, p.stream_out);
                }
              } else {
                for (int j = 0; j < nvalid; ++j) {
                  float f = v[j];
                  if constexpr (EPI == EPI_STORE_RES) f = bf16_round(f) + __bfloat162float(rrow[j]);
                  orow[j] = __float2bfloat16_rn(f);
                }
              }
            }
          } else if constexpr (EPI == EPI_SWIGLU) {
            // columns [c0, c0+16) = gate, [c0+16, c0+32) = up of output columns (n0+c0)/2 + j
            static_assert(EPI != EPI_SWIGLU || CH == 32, "SWIGLU needs 32-column chunks");
            if (m < M_rt) {
              const int oc = (n0 + c0) >> 1;
              bf16* orow = reinterpret_cast<bf16*>(p.out) + (long long)(m + roff_a) * p.ldo + oc;
              float h[16];
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const float g = bf16_round(v[j]);
                const float up = bf16_round(v[16 + j]);
                h[j] = bf16_round(silu_f(g)) * up;
              }
              if (oc + 16 <= p.out_cols && (p.ldo & 7) == 0) {
                uint4 o0, o1;
                o0.x = pack_bf16x2(h[0], h[1]);   o0.y = pack_bf16x2(h[2], h[3]);
                o0.z = pack_bf16x2(h[4], h[5]);   o0.w = pack_bf16x2(h[6], h[7]);
                o1.x = pack_bf16x2(h[8], h[9]);   o1.y = pack_bf16x2(h[10], h[11]);
                o1.z = pack_bf16x2(h[12], h[13]); o1.w = pack_bf16x2(h[14], h[15]);
                st_out_v4(orow, o0, p.stream_out);
                st_out_v4(orow + 8, o1, p.stream_out);
              } else {
                for (int j = 0; j < 16 && oc + j < p.out_cols; ++j) orow[j] = __float2bfloat16_rn(h[j]);
              }
            }
          } else if constexpr (EPI == EPI_T_STORE) {
            if (m < M_rt) {
              bf16* o = reinterpret_cast<bf16*>(p.out) + out_off + (long long)(n0 + c0 + roff_b) * p.ldo + m;
#pragma unroll
              for (int j = 0; j < CH; ++j)
                if (j < nvalid) o[(long long)j * p.ldo] = __float2bfloat16_rn(v[j]);
            }
          } else if constexpr (EPI == EPI_T_SWIGLU) {
            // rows of a 32-row warp slab: lanes 0-15 gate, lanes 16-31 up, for output feature (slab/2 + lane)
            const int f = ((m_t * kGemmBlockM + q * 32) >> 1) + (lane & 15);
            bf16* o = reinterpret_cast<bf16*>(p.out) + out_off + (long long)(n0 + c0 + roff_b) * p.ldo + f;
#pragma unroll
            for (int j = 0; j < CH; j += 2) {
              // lanes 16-31 hold `up`: hand two bf16 columns per shuffle to the gate lane 16 below
              const uint32_t mine = pack_bf16x2(v[j], v[j + 1]);
              const uint32_t other = __shfl_down_sync(0xffffffffu, mine, 16);
              if (lane < 16 && f < p.out_cols) {
                const float2 g2 = unpack_bf16x2(mine), u2 = unpack_bf16x2(other);
                if (j < nvalid) o[(long long)j * p.ldo] = __float2bfloat16_rn(bf16_round(silu_f(g2.x)) * u2.x);
                if (j + 1 < nvalid) o[(long long)(j + 1) * p.ldo] = __float2bfloat16_rn(bf16_round(silu_f(g2.y)) * u2.y);
              }
            }
          } else {  // EPI_T_PARTIAL
            if (m < M_rt) {
              float* o = reinterpret_cast<float*>(p.out) + out_off + (long long)s * p.split_stride +
                         (long long)(n0 + c0) * p.ldo + m;
#pragma unroll
              for (int j = 0; j < CH; ++j)
                if (j < nvalid) o[(long long)j * p.ldo] = v[j];
            }
          }
        }
      }
      if (sg.type == 1) {          // publish the partial
        __threadfence();
        consumer_bar();
        if (et == 0) atomicAdd(p.sk_flags + sg.m_t, 1);
      } else if (sg.type == 2) {   // consumed: leave the flag clean for the next launch / graph replay
        consumer_bar();
        if (et == 0) atomicExch(p.sk_flags + sg.m_t, 0);
      }
    }
  }
}

}  // namespace b200
