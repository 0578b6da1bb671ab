// Causal prefill attention on the Hopper tensor cores (wgmma), SURVEY.md §8a row 15.
//
// One CTA = 128 query rows of one (sequence, head); KV is consumed in tiles of 64 tokens (= one page).
//   warpgroup 0    : TMA producer — Q once, then K / V tiles into 2-stage 128B-swizzled rings straight from the paged
//                    cache (tensor map over [page*nkv*64 rows][128 dims], two 8 KB boxes per tile)
//   warpgroups 1-2 : 64 query rows each — S = Q K^T (wgmma m64n64k16, both operands K-major from shared memory, S in
//                    registers), online softmax in the log2 domain on the register fragment (a row is spread over the
//                    4 threads of a quad), then O += P V (wgmma m64n128k16 with P as the register A operand — the S
//                    fragment layout is the A fragment layout, so P never goes through shared memory — and V as an
//                    MN-major shared-memory operand), finally O / l stored as bf16.
// The two consumer warpgroups run independently, so one's softmax overlaps the other's tensor-core work.
//
// FP8 KV cache (attn_prefill_tc_kernel<true>): the cache holds e4m3 codes.  TMA brings each K / V tile as codes (an 8 KB
// [64 tokens][128 B] box) into a 2-stage code ring, and the 128 threads of warpgroup 0 expand it (exactly) into the same
// 128B-swizzled bf16 boxes the consumers read, writing the V rows past the end of the keys as zeros.  The consumers'
// code is the bf16 kernel's; the conversion stays off their critical path.
#pragma once
#include "common.cuh"
#include "gemm_wgmma.cuh"
#include "ops.cuh"

namespace b200 {

constexpr int kTcQ = 128;                    // query rows per CTA
constexpr int kTcKv = 64;                    // KV tokens per tile == one page
constexpr int kTcTile = 128 * 64 * 2;        // one [128 x 64] bf16 swizzled tile = 16 KB (a K or V stage: two [64 x 64] boxes)
// Q 2 tiles + K ring 2 stages + V ring 2 stages = 96 KB, + alignment slack and barriers; one CTA per SM
constexpr int kTcSmem = 2 * kTcTile /*Q*/ + 2 * kTcTile /*K ring*/ + 2 * kTcTile /*V ring*/ + 1024 + 256;
constexpr int kTcThreads = 384;
constexpr int kTcTile8 = 64 * 128;           // one K or V tile of e4m3 codes = 8 KB
constexpr int kTcSmem8 = kTcSmem + 2 * 2 * kTcTile8;   // + code ring[2] x {K, V}

// warpgroup 0 (128 threads): codes [64 tokens][128 B] -> the two 128B-swizzled [64 x 64] bf16 boxes of a K / V stage;
// rows >= valid_rows become zeros
__device__ __forceinline__ void expand_tc_tile8(uint8_t* dst, const uint8_t* codes, int valid_rows) {
  const Fp8Scale one = fp8_scale(__float2bfloat16(1.0f));
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int idx = threadIdx.x + it * 128;
    const int r = idx >> 3, c = idx & 7;            // codes of dims [16 c, 16 c + 16) of token r
    uint4 o0 = make_uint4(0u, 0u, 0u, 0u), o1 = o0;
    if (r < valid_rows) fp8x16_dequant(*reinterpret_cast<const uint4*>(codes + r * 128 + c * 16), one, o0, o1);
    uint8_t* row = dst + (c >> 2) * (kTcTile / 2) + r * 128;   // box (c >> 2), its 16-byte chunks 2 (c & 3) and + 1
    const int cc = 2 * (c & 3);
    *reinterpret_cast<uint4*>(row + ((cc ^ (r & 7)) << 4)) = o0;
    *reinterpret_cast<uint4*>(row + (((cc + 1) ^ (r & 7)) << 4)) = o1;
  }
}

struct AttnTcParams {
  bf16* out; long long ldo;
  const int32_t* page_table; int max_pages;
  const int32_t* cu_seqlens; const int32_t* seq_slot;
  int nh, nkv;
  float scale_log2;
  // Chunked prefill / prefix reuse: tokens [0, kv_off[b]) of sequence b are already in the paged cache (an earlier
  // chunk, or pages shared with a previous request) and the packed query rows are positions kv_off[b] ... of it.
  // Must be a multiple of 128 (query tiles stay aligned with KV tiles); nullptr == all zero.
  const int32_t* kv_off;
};

// KV8: tmap_k / tmap_v are maps over the e4m3 caches, box [64][128 B] (else bf16, box [64][64], 128B swizzle)
template <bool KV8>
__global__ void __launch_bounds__(kTcThreads, 1)
attn_prefill_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                       const __grid_constant__ CUtensorMap tmap_v, const AttnTcParams p) {
  TraceScope _ts(TK_ATTN_PREFILL);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                       // 2 tiles (dims 0-63 | 64-127), 128 rows each
  uint8_t* sK = sQ + 2 * kTcTile;           // ring[2] x {dims 0-63 | 64-127} x 64 tokens
  uint8_t* sV = sK + 2 * kTcTile;           // ring[2], same shape
  uint8_t* s8 = sV + 2 * kTcTile;           // KV8: code ring[2] x {K, V}
  uint64_t* bars = reinterpret_cast<uint64_t*>(s8 + (KV8 ? 2 * 2 * kTcTile8 : 0));
  uint64_t *q_full = bars, *k_full = bars + 1, *k_empty = bars + 3, *v_full = bars + 5, *v_empty = bars + 7;
  uint64_t* c_full = bars + 9;              // KV8: codes of stage st have landed

  const int b = blockIdx.z, h = blockIdx.y, qt = blockIdx.x;
  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_launch_dependents();
  pdl_wait();
  const int tok0 = p.cu_seqlens[b];
  const int len = p.cu_seqlens[b + 1] - tok0;
  const int q0 = qt * kTcQ;
  if (q0 >= len) return;
  const int kvh = h / (p.nh / p.nkv);
  const int32_t* pages = p.page_table + (long long)p.seq_slot[b] * p.max_pages;
  const int off_tiles = p.kv_off ? (p.kv_off[b] >> 7) : 0;    // 128-token blocks that precede this chunk's first query row
  const int ntiles_causal = 2 * (off_tiles + qt + 1);          // causal: 64-token KV tiles 0 .. 2 * (off_tiles + qt) + 1
  // Keys [0, kv_end) exist.  The last query tile's second KV tile can lie wholly past kv_end: it is neither loaded nor
  // multiplied (every p of it would be 0, so skipping it changes no bit).  The tile that straddles kv_end gets its V rows
  // past the end zeroed before P.V (below): the page's tail is stale memory and 0 * NaN is NaN.
  const int kv_end = off_tiles * 128 + len;
  const int ntiles = min(ntiles_causal, (kv_end + kTcKv - 1) / kTcKv);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&k_full[i], KV8 ? 128 : 1); mbar_init(&k_empty[i], 2);   // one arrival per consumer warpgroup
      mbar_init(&v_full[i], KV8 ? 128 : 1); mbar_init(&v_empty[i], 2);   // KV8: one per expanding producer thread
      if (KV8) mbar_init(&c_full[i], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (KV8 && wg == 0) {
    auto issue_codes = [&](int j) {   // thread 0: K and V codes of tile j into code stage j & 1
      const int st = j & 1;
      const int row0 = (pages[min(j, p.max_pages - 1)] * p.nkv + kvh) * kPageTokens;
      mbar_arrive_expect_tx(&c_full[st], 2 * kTcTile8);
      tma_load_2d(s8 + st * 2 * kTcTile8, &tmap_k, &c_full[st], 0, row0, kEvictLast);
      tma_load_2d(s8 + st * 2 * kTcTile8 + kTcTile8, &tmap_v, &c_full[st], 0, row0, kEvictLast);
    };
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, 2 * kTcTile);
      tma_load_2d(sQ, &tmap_q, q_full, h * kHeadDim, tok0 + q0, kEvictNormal);
      tma_load_2d(sQ + kTcTile, &tmap_q, q_full, h * kHeadDim + 64, tok0 + q0, kEvictNormal);
      for (int j = 0; j < min(2, ntiles); ++j) issue_codes(j);
    }
    for (int j = 0; j < ntiles; ++j) {
      const int st = j & 1;
      const uint32_t ph = (j >> 1) & 1;
      const uint8_t* codes = s8 + st * 2 * kTcTile8;
      mbar_wait(&c_full[st], ph);
      mbar_wait(&k_empty[st], ph ^ 1);
      expand_tc_tile8(sK + st * kTcTile, codes, kTcKv);   // K rows past kv_end are masked, whatever they hold
      fence_proxy_async_shared();                          // generic-proxy stores -> visible to wgmma
      mbar_arrive(&k_full[st]);
      mbar_wait(&v_empty[st], ph ^ 1);
      expand_tc_tile8(sV + st * kTcTile, codes + kTcTile8, kv_end - j * kTcKv);   // 0 * stale V row would be NaN
      fence_proxy_async_shared();
      mbar_arrive(&v_full[st]);
      if (j + 2 < ntiles) {
        asm volatile("bar.sync 2, 128;" ::: "memory");   // every producer thread is done reading code stage st
        if (threadIdx.x == 0) issue_codes(j + 2);
      }
    }
    return;
  }
  if (wg == 0) {
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, 2 * kTcTile);
      tma_load_2d(sQ, &tmap_q, q_full, h * kHeadDim, tok0 + q0, kEvictNormal);
      tma_load_2d(sQ + kTcTile, &tmap_q, q_full, h * kHeadDim + 64, tok0 + q0, kEvictNormal);
      for (int j = 0; j < ntiles; ++j) {
        const int st = j & 1;
        const uint32_t ph = (j >> 1) & 1;
        const int row0 = (pages[min(j, p.max_pages - 1)] * p.nkv + kvh) * kPageTokens;
        mbar_wait(&k_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&k_full[st], kTcTile);
        uint8_t* kd = sK + st * kTcTile;
        tma_load_2d(kd, &tmap_k, &k_full[st], 0, row0, kEvictLast);
        tma_load_2d(kd + kTcTile / 2, &tmap_k, &k_full[st], 64, row0, kEvictLast);
        mbar_wait(&v_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&v_full[st], kTcTile);
        uint8_t* vd = sV + st * kTcTile;
        tma_load_2d(vd, &tmap_v, &v_full[st], 0, row0, kEvictLast);
        tma_load_2d(vd + kTcTile / 2, &tmap_v, &v_full[st], 64, row0, kEvictLast);
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers: softmax + both MMAs
  const int half = wg - 1;                                        // query rows 64 * half ... + 63 of the tile
  const int t = threadIdx.x - 128 * wg;
  const int r_lo = 64 * half + 16 * (warp & 3) + (lane >> 2);     // this thread's fragment rows r_lo, r_lo + 8
  const int qpos_lo = off_tiles * 128 + q0 + r_lo;                // position of row r_lo in the sequence (causal mask)
  const int col_t = 2 * (lane & 3);                               // fragment column offset inside each 8-column group
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t sq = smem_u32(sQ) + half * 64 * 128;
  mbar_wait(q_full, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int st = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    // ---- S = Q K^T
    float s[32];
    mbar_wait(&k_full[st], ph);
    {
      const uint32_t kk = smem_u32(sK + st * kTcTile);
      wgmma_fence();
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss_n64(s, make_smem_desc_sw128(sq + hh * kTcTile) + 2 * k, make_smem_desc_sw128(kk + hh * (kTcTile / 2)) + 2 * k,
                       (hh | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_keep(s);
    }
    if (t == 0) mbar_arrive(&k_empty[st]);
    // ---- online softmax; the softmax scale is folded into the exponent (max on the raw scores — the scale is
    // positive — then p = exp2(fma(s, scale, -m)): one FFMA per element)
    if (j >= ntiles_causal - 2) {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int key = j * kTcKv + 8 * (i >> 2) + col_t + (i & 1);
        if (key > qpos_lo + 8 * ((i >> 1) & 1)) s[i] = -INFINITY;
      }
    }
    float corr[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (((i >> 1) & 1) == rr) mx = fmaxf(mx, s[i]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[rr], mx * p.scale_log2);   // finite from tile 0 on: key 0 is visible to every row
      corr[rr] = (m_run[rr] == -INFINITY) ? 0.f : exp2f(m_run[rr] - m_new);
      m_run[rr] = m_new;
      l_run[rr] *= corr[rr];
    }
    uint32_t pa[16];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int rr = (i >> 1) & 1;
      const float p0 = exp2f(fmaf(s[i], p.scale_log2, -m_run[rr]));
      const float p1 = exp2f(fmaf(s[i + 1], p.scale_log2, -m_run[rr]));
      l_run[rr] += p0 + p1;
      pa[i >> 1] = pack_bf16x2(p0, p1);
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] *= corr[(i >> 1) & 1];
    // ---- O += P V: 16 tokens per MMA; the S fragment of tokens [16k, 16k + 16) is the A fragment {pa[4k] .. pa[4k + 3]}
    mbar_wait(&v_full[st], ph);
    if (!KV8 && kv_end < (j + 1) * kTcKv) {   // the tile straddling kv_end (uniform per CTA): zero its V rows past the end
      // a 128B-swizzled row keeps its 128 bytes, so row r of each [64 x 64] box is bytes [128 r, 128 r + 128)
      uint8_t* vd = sV + st * kTcTile;
      const int r0 = kv_end - j * kTcKv;
      for (int i = threadIdx.x - 128; i < (kTcKv - r0) * 16; i += 256) {   // 16 B chunks: 8 per row in each of the 2 boxes
        const int row = r0 + (i >> 4), box = (i >> 3) & 1, c = i & 7;
        *reinterpret_cast<uint4*>(vd + box * (kTcTile / 2) + row * 128 + c * 16) = make_uint4(0u, 0u, 0u, 0u);
      }
      fence_proxy_async_shared();                      // generic-proxy stores -> visible to wgmma
      asm volatile("bar.sync 1, 256;" ::: "memory");   // both consumer warpgroups
    }
    {
      const uint32_t vb = smem_u32(sV + st * kTcTile);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t a[4] = {pa[4 * k], pa[4 * k + 1], pa[4 * k + 2], pa[4 * k + 3]};
        wgmma_rs_n128_tb(o, a, make_smem_desc_sw128_mn(vb + (k * 16) * 128, kTcTile / 2), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_keep(o);
    }
    if (t == 0) mbar_arrive(&v_empty[st]);
  }
  // epilogue: O / l -> bf16
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    l_run[rr] += __shfl_xor_sync(0xffffffffu, l_run[rr], 1);
    l_run[rr] += __shfl_xor_sync(0xffffffffu, l_run[rr], 2);
  }
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int qrow = q0 + r_lo + 8 * rr;
    if (qrow >= len) continue;
    const float inv = 1.0f / l_run[rr];
    bf16* orow = p.out + (long long)(tok0 + qrow) * p.ldo + h * kHeadDim + col_t;
#pragma unroll
    for (int g = 0; g < 16; ++g)
      *reinterpret_cast<uint32_t*>(orow + 8 * g) = pack_bf16x2(o[4 * g + 2 * rr] * inv, o[4 * g + 2 * rr + 1] * inv);
  }
}

}  // namespace b200
