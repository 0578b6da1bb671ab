// Persistent, warp-specialised bf16 GEMM for sm_90a:  D[M,N] = A[M,K] * B[N,K]^T  (both K-major).
//
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx)
//   warpgroups 1-2 : wgmma consumers, one 64-row half of the 128-row tile each (m64nBLOCK_Nk16, fp32 accumulators in
//                    registers); the accumulators are staged through shared memory so that the fused epilogue sees
//                    one tile row per thread, 32 consecutive columns at a time
//
// This file holds the decode kernel (SURVEY.md §8a rows 13-17): A = weight [N_out,K] (M = N_out), B = activations
// [batch,K] ("swap-AB": the 128-row MMA M dimension is filled by weight rows, the small batch rides in the MMA N
// dimension, so no tensor-core work is wasted on padding and each CTA streams a contiguous weight slab) -> transposed
// epilogues, optional split-K with fp32 partials.  The prefill GEMMs (A = activations [T,K], B = weight [N_out,K],
// row-major epilogues) run gemm_prefill_kernel (gemm_prefill.cuh), which shares the parameters and the schedule.
#pragma once
#include "common.cuh"

namespace b200 {

enum GemmEpi : int {
  EPI_STORE = 0,      // out[m][n] = bf16(acc [+ bias[n]])
  EPI_STORE_RES = 1,  // out[m][n] = bf16(bf16(acc) + residual[m][n])           (o_proj / down_proj + residual)
  EPI_SWIGLU = 2,     // B rows interleaved {16 gate,16 up}: out[m][n/2] = bf16(bf16(silu(g)) * u)
  EPI_T_STORE = 3,    // out[n][m] = bf16(acc [+ bias[m]])                        (swap-AB)
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
  bf16* rope_kcache; bf16* rope_vcache;                      // this layer's [page][kv_head][64][128] (KV8: e4m3 codes)
  const bf16* rope_cos; const bf16* rope_sin;                // [max_pos][64]
  int rope_nh, rope_nkv;
  const bf16* rope_q_norm; const bf16* rope_k_norm; float rope_qk_eps;   // EPI_ROPE_KV<.., QKNORM>: Qwen3 q / k norm weights [128]
  int stream_out;          // row-major epilogues: cache-streaming output stores
  int out_tma;             // row-major epilogues: `out` is addressable by TMA (16-byte aligned base and row pitch)
  int sched;
  int sk_slots;            // partial slots per tile
  float* sk_ws;            // [m_tiles][sk_slots][BLOCK_N][128] fp32
  int* sk_flags;           // [m_tiles] arrival counters, 0 between launches
  // per-output-feature bias (EPI_STORE, EPI_ROPE_KV: column n; EPI_T_STORE: weight row m), nullptr = none.  It is added
  // in fp32 to the finished accumulator, so the output is ONE bf16 rounding of (acc + bias) as nn.Linear(bias=True) gives.
  const bf16* bias;
  // FP8 weights (gemm_tn_kernel<..., true>): A is e4m3 [M][K] and a_scale[m] the bf16 scale of weight row m
  const bf16* a_scale;
};

constexpr int kGemmBlockM = 128;
constexpr int kGemmBlockK = 64;
constexpr int kGemmThreads = 384;
constexpr int kGemmGroupM = 16;
constexpr int kStgStride = 132;   // floats between two staged accumulator columns: 128 rows + 4 (conflict-free fragment stores)

template <int BLOCK_N, bool FP8A = false>
struct GemmCfg {
  static_assert(BLOCK_N <= 64, "swap-AB tiles carry the batch in N");
  static constexpr int kABytes = kGemmBlockM * kGemmBlockK * (FP8A ? 1 : 2);  // 16 KB (8 KB of e4m3 codes)
  static constexpr int kBBytes = BLOCK_N * kGemmBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = 8;
  // FP8: every consumer warpgroup expands its 64-row half of the A tile into one of 3 bf16 buffers (8 KB each) that
  // wgmma reads; 3 because the k-block before the previous one may still be in flight when the next one is written
  static constexpr int kXBufs = FP8A ? 3 : 0;
  static constexpr int kXBytes = 2 * kXBufs * 64 * kGemmBlockK * 2;
  static constexpr int kChunk = (BLOCK_N >= 32) ? 32 : 16;             // columns one epilogue thread takes at a time
  static constexpr int kRoundCols = BLOCK_N;                           // columns staged per epilogue round
  static constexpr int kChunks = kRoundCols / kChunk;
  static constexpr int kStgBytes = kRoundCols * kStgStride * 4;
  static constexpr int kSmemBytes = kStages * kStageBytes + kXBytes + kStgBytes + 1024 /*align slack*/ + 256 /*barriers*/;
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


// ---- FP8 (e4m3) weights
// The engine multiplies exactly the bf16 operand compressed-tensors' decompression gives transformers:
// W' = bf16(code) * s in bf16 arithmetic (one round-to-nearest-even), s = the row's scale rounded to bf16.
// e4m3 -> bf16 is exact: the code's 7 exponent / mantissa bits are moved to their bf16 position, which gives a bf16 of
// 2^-120 times the code's value (subnormal codes become bf16 subnormals), and multiplied back by 2^120 (exact).
// The NaN codes 0x7F / 0xFF would come out as +-480 * s: the loader refuses checkpoints that contain them.
__device__ __forceinline__ uint32_t bf16x2_mul(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
// A row's scale as the pair the expansion multiplies by: {s * 2^120, s * 2^120} when |s| < 2^8 (exact and finite, and
// then ONE multiply gives bf16(code * s) with a single rounding), else {s, s} after an exact multiply by 2^120
struct Fp8Scale { uint32_t s2; bool folded; };
__device__ __forceinline__ uint32_t bf16_pair(bf16 s) {
  const uint32_t u = *reinterpret_cast<const unsigned short*>(&s);
  return u | (u << 16);
}
__device__ __forceinline__ Fp8Scale fp8_scale(bf16 s) {
  const float f = __bfloat162float(s);
  const bool folded = fabsf(f) < 256.f;
  return Fp8Scale{bf16_pair(folded ? __float2bfloat16_rn(f * 0x1p120f) : s), folded};
}
// 4 codes of `w` (byte order) -> bf16 pairs {code0, code1} in lo, {code2, code3} in hi, each times the row's scale
__device__ __forceinline__ void fp8x4_dequant(uint32_t w, const Fp8Scale& sc, uint32_t& lo, uint32_t& hi) {
  constexpr uint32_t kPow120 = 0x7B807B80u;   // {2^120, 2^120}
  const uint32_t a = __byte_perm(w, 0, 0x1404), b = __byte_perm(w, 0, 0x3424);   // each code in the high byte of a half
  lo = (a & 0x80008000u) | ((a >> 4) & 0x07F007F0u);
  hi = (b & 0x80008000u) | ((b >> 4) & 0x07F007F0u);
  if (!sc.folded) {
    lo = bf16x2_mul(lo, kPow120);
    hi = bf16x2_mul(hi, kPow120);
  }
  lo = bf16x2_mul(lo, sc.s2);
  hi = bf16x2_mul(hi, sc.s2);
}
// 16 codes -> 16 bf16 (two 16-byte chunks)
__device__ __forceinline__ void fp8x16_dequant(const uint4& v, const Fp8Scale& sc, uint4& o0, uint4& o1) {
  fp8x4_dequant(v.x, sc, o0.x, o0.y);
  fp8x4_dequant(v.y, sc, o0.z, o0.w);
  fp8x4_dequant(v.z, sc, o1.x, o1.y);
  fp8x4_dequant(v.w, sc, o1.z, o1.w);
}

// A layer's FP8 matrices -> bf16 (prefill feeds the unchanged bf16 GEMM from this scratch); K % 16 == 0
struct Fp8Seg { const uint8_t* q; const bf16* s; bf16* out; long long chunks; int K; };   // chunks = rows * K / 16
struct Fp8Segs { Fp8Seg seg[4]; int n; };

__global__ void __launch_bounds__(256) dequant_fp8_kernel(const Fp8Segs p) {
  long long total = 0;
  for (int i = 0; i < p.n; ++i) total += p.seg[i].chunks;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
    long long cc = c;
    int i = 0;
    while (cc >= p.seg[i].chunks) { cc -= p.seg[i].chunks; ++i; }
    const Fp8Seg& g = p.seg[i];
    const long long row = cc * 16 / g.K;
    const uint4 v = ld_nc_v4(g.q + cc * 16);
    uint4 o0, o1;
    fp8x16_dequant(v, fp8_scale(g.s[row]), o0, o1);
    uint4* o = reinterpret_cast<uint4*>(g.out + cc * 16);
    o[0] = o0;
    o[1] = o1;
  }
}

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

// FP8A: A is e4m3 (weights with a bf16 scale per row, p.a_scale); the consumers expand every k-block's A tile into the
// bf16 layout the bf16 kernel's TMA would have written (128B swizzle), so the MMAs, their k order, the schedule and the
// epilogues are those of the bf16 kernel on W' (bit-identical results), while HBM streams one byte per weight.
template <int BLOCK_N, int EPI, bool FP8A = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmParams p) {
  static_assert(EPI == EPI_T_STORE || EPI == EPI_T_SWIGLU || EPI == EPI_T_PARTIAL, "swap-AB epilogues only");
  TraceScope _ts(TK_GEMM + 100 * EPI + 1000 * (p.M >> 7));
  using Cfg = GemmCfg<BLOCK_N, FP8A>;
  constexpr int STAGES = Cfg::kStages;
  constexpr int CH = Cfg::kChunk;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* xbuf = smem + STAGES * Cfg::kStageBytes;   // FP8A: [2 warpgroups][kXBufs][64 rows][128 B] bf16, swizzled
  float* stg = reinterpret_cast<float*>(xbuf + Cfg::kXBytes);   // [kRoundCols][kStgStride] fp32
  uint64_t* bars = reinterpret_cast<uint64_t*>(xbuf + Cfg::kXBytes + Cfg::kStgBytes);
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
    int xk = 0;               // FP8A: k-blocks expanded so far (selects the bf16 buffer)
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
      // FP8A: this thread expands two 16-byte chunks of codes per k-block, rows t/4 and t/4 + 32 of the warpgroup's half
      Fp8Scale xsc[2] = {{0u, true}, {0u, true}};
      if constexpr (FP8A) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int row = m_t * kGemmBlockM + half * 64 + (t >> 2) + 32 * i;
          if (row < p.M) xsc[i] = fp8_scale(p.a_scale[row]);   // (rows past M: TMA zero-filled codes, scale 0)
        }
      }
      // ---- main loop: one k-block in flight behind the one being issued
      wgmma_keep(accum);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
        uint64_t adesc;
        if constexpr (FP8A) {
          // codes: [128 rows][64 B] unswizzled; bf16: [64 rows][128 B], 16-byte chunk c of row r at chunk c ^ (r & 7)
          const uint8_t* a8 = smem + stage * Cfg::kStageBytes + half * 64 * kGemmBlockK;
          uint8_t* xb = xbuf + (half * Cfg::kXBufs + xk % Cfg::kXBufs) * (64 * 128);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int j = t + 128 * i, r = j >> 2, c0 = (j & 3) * 2;
            uint4 o0, o1;
            fp8x16_dequant(*reinterpret_cast<const uint4*>(a8 + j * 16), xsc[i], o0, o1);
            *reinterpret_cast<uint4*>(xb + r * 128 + ((c0 ^ (r & 7)) << 4)) = o0;
            *reinterpret_cast<uint4*>(xb + r * 128 + (((c0 + 1) ^ (r & 7)) << 4)) = o1;
          }
          fence_proxy_async_shared();   // generic-proxy stores -> visible to wgmma
          asm volatile("bar.sync %0, 128;" ::"r"(2 + half) : "memory");
          adesc = make_smem_desc_sw128(smem_u32(xb));
          ++xk;
        } else {
          adesc = make_smem_desc_sw128(sa + half * 64 * 128);
        }
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
          if constexpr (EPI == EPI_T_STORE) {
            if (m < M_rt) {
              if (p.bias != nullptr) {   // after the stream-K pieces are in: one code point for plain and stream-K tiles
                const float bm = __bfloat162float(p.bias[m]);
#pragma unroll
                for (int j = 0; j < CH; ++j) v[j] += bm;
              }
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
