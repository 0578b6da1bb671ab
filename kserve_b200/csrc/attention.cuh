// Attention over the paged KV cache (SURVEY.md §8a row 15: LlamaAttention.forward + SDPA with GQA).
//
//   attn_prefill_kernel : causal flash attention for the prompt tokens of ragged sequences.
//   attn_decode_kernel  : one query token per sequence, split over the KV length (flash-decoding),
//                         the G query heads that share a KV head are packed into the MMA M dimension.
//   attn_combine_kernel : merges the per-split partials.
//
// KV pages are [page][kv_head][64 tokens][128 dims] bf16, so one (page, kv_head) tile is a contiguous
// 16 KB block that is staged with 128-bit cp.async into XOR-swizzled shared memory and consumed with
// ldmatrix + mma.sync.m16n8k16 (fp32 softmax / accumulation).  This round's kernels use the legacy
// warp-level MMA path; they are HBM-bound in decode (the KV read) and 2% of prefill FLOPs.
//
// FP8 KV cache (attn_decode_kernel<true>): pages hold e4m3 codes, [page][kv_head][64][128] bytes, so a tile is 8 KB.  The
// codes go through a cp.async ring of their own and the CTA expands each tile (exactly: every e4m3 value is a bf16
// value) into the same swizzled bf16 tile as above, so the MMA loop and the merges are the bf16 kernel's.
#pragma once
#include "common.cuh"
#include "gemm_wgmma.cuh"
#include "ops.cuh"

namespace b200 {

constexpr int kAttnThreads = 128;
constexpr int kDecStages = 3;   // cp.async ring of the decode kernel: two KV tiles (64 KB) in flight per CTA
constexpr int kTileBytes = kPageTokens * kHeadDim * 2;  // 16 KB
constexpr int kDecStages8 = 4;  // FP8 KV: code ring of 4 (K, V) stages = 64 KB, + one bf16 K and V tile = the bf16 ring's 96 KB
constexpr int kTile8Bytes = kPageTokens * kHeadDim;     // 8 KB of e4m3 codes

// byte offset of 16-byte chunk `c` (0..15) of row `r` in a [rows][128] bf16 tile with XOR swizzle
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * 256 + ((c ^ (r & 7)) << 4)); }

// stage one 64x128 bf16 tile (contiguous in global memory) into swizzled smem; 128 threads.  Rows >= valid_rows are
// zero-filled instead of copied: a page's slots past the context hold whatever an earlier owner of the page left there
// (possibly Inf / NaN), and a masked key's p = 0 times a NaN V row is still NaN inside the P.V MMA.
__device__ __forceinline__ void load_kv_tile(uint32_t sdst, const bf16* gsrc, int valid_rows = kPageTokens) {
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int idx = threadIdx.x + it * kAttnThreads;
    const int r = idx >> 4, c = idx & 15;
    cp_async_16(sdst + swz(r, c), gsrc + r * kHeadDim + c * 8, r < valid_rows);
  }
}

// stage one 64x128 tile of e4m3 codes into an unswizzled [64][128 B] buffer; rows >= valid_rows zero-filled (code 0 = +0)
__device__ __forceinline__ void load_kv_tile8(uint32_t sdst, const uint8_t* gsrc, int valid_rows) {
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int idx = threadIdx.x + it * kAttnThreads;
    const int r = idx >> 3, c = idx & 7;
    cp_async_16(sdst + r * 128 + c * 16, gsrc + r * 128 + c * 16, r < valid_rows);
  }
}

// expand a staged code tile into the swizzled bf16 tile load_kv_tile would have produced from bf16(codes); 128 threads
__device__ __forceinline__ void expand_kv_tile8(uint8_t* dst, const uint8_t* codes) {
  const Fp8Scale one = fp8_scale(__float2bfloat16(1.0f));
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int idx = threadIdx.x + it * kAttnThreads;
    const int r = idx >> 3, c = idx & 7;
    uint4 o0, o1;
    fp8x16_dequant(*reinterpret_cast<const uint4*>(codes + r * 128 + c * 16), one, o0, o1);
    *reinterpret_cast<uint4*>(dst + swz(r, 2 * c)) = o0;
    *reinterpret_cast<uint4*>(dst + swz(r, 2 * c + 1)) = o1;
  }
}

struct AttnPrefillParams {
  const bf16* q; long long ldq;        // roped queries [T][ldq], head h at column h*128
  bf16* out; long long ldo;            // [T][ldo]
  const bf16* kcache; const bf16* vcache;  // this layer
  const int32_t* page_table; int max_pages;
  const int32_t* cu_seqlens;           // [B+1] token offsets of each sequence in the packed buffers
  const int32_t* seq_slot;             // [B] row of the page table
  int nh, nkv;
  float scale_log2;                    // (1/sqrt(d)) * log2(e)
};

__global__ void __launch_bounds__(kAttnThreads) attn_prefill_kernel(const AttnPrefillParams p) {
  TraceScope _ts(TK_ATTN_PREFILL);
  pdl_launch_dependents();
  pdl_wait();
  _ts.mark();
  extern __shared__ __align__(1024) uint8_t smem[];
  const int b = blockIdx.z, h = blockIdx.y, qt = blockIdx.x;
  const int tok0 = p.cu_seqlens[b];
  const int len = p.cu_seqlens[b + 1] - tok0;
  const int q0 = qt * 64;
  if (q0 >= len) return;
  const int kvh = h / (p.nh / p.nkv);
  const int slot = p.seq_slot[b];
  const int32_t* pages = p.page_table + (long long)slot * p.max_pages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK = sQ + kTileBytes;      // 2 buffers
  const uint32_t sV = sK + 2 * kTileBytes;  // 2 buffers
  const long long tile_stride = (long long)p.nkv * kPageTokens * kHeadDim;
  const long long head_off = (long long)kvh * kPageTokens * kHeadDim;

  // Q tile (rows beyond the sequence are zero-filled)
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int idx = threadIdx.x + it * kAttnThreads;
    const int r = idx >> 4, c = idx & 15;
    const bool valid = (q0 + r) < len;
    const bf16* src = p.q + (long long)(tok0 + (valid ? q0 + r : 0)) * p.ldq + h * kHeadDim + c * 8;
    cp_async_16(sQ + swz(r, c), src, valid);
  }
  const int ntiles = qt + 1;  // causal: KV tiles 0..qt
  load_kv_tile(sK, p.kcache + (long long)pages[0] * tile_stride + head_off);
  load_kv_tile(sV, p.vcache + (long long)pages[0] * tile_stride + head_off);
  cp_async_commit();

  uint32_t qf[8][4];
  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const int wrow = warp * 16;

  for (int j = 0; j < ntiles; ++j) {
    const int buf = j & 1;
    if (j + 1 < ntiles) {
      const long long pg = pages[j + 1];
      load_kv_tile(sK + (buf ^ 1) * kTileBytes, p.kcache + pg * tile_stride + head_off);
      load_kv_tile(sV + (buf ^ 1) * kTileBytes, p.vcache + pg * tile_stride + head_off);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (j == 0) {
#pragma unroll
      for (int ks = 0; ks < 8; ++ks)
        ldmatrix_x4(qf[ks], sQ + swz(wrow + (lane & 7) + 8 * ((lane >> 3) & 1), 2 * ks + (lane >> 4)));
    }
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    const uint32_t sKb = sK + buf * kTileBytes, sVb = sV + buf * kTileBytes;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bfr[4];
        ldmatrix_x4(bfr, sKb + swz(16 * np + (lane & 7) + 8 * (lane >> 4), 2 * ks + ((lane >> 3) & 1)));
        mma_m16n8k16_bf16(s[2 * np], qf[ks], bfr[0], bfr[1]);
        mma_m16n8k16_bf16(s[2 * np + 1], qf[ks], bfr[2], bfr[3]);
      }
    }
    // scale (log2 domain) + causal mask on the diagonal tile
    const bool diag = (j == qt);
    const int qp0 = q0 + wrow + g, qp1 = qp0 + 8;
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int kp = j * 64 + nt * 8 + 2 * t + e;
        float v0 = s[nt][e] * p.scale_log2, v1 = s[nt][2 + e] * p.scale_log2;
        if (diag && kp > qp0) v0 = -INFINITY;
        if (diag && kp > qp1) v1 = -INFINITY;
        s[nt][e] = v0;
        s[nt][2 + e] = v1;
        mx0 = fmaxf(mx0, v0);
        mx1 = fmaxf(mx1, v1);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);  // finite: key 0 is never masked
    const float c0 = exp2f(m0 - mn0), c1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    l0 *= c0; l1 *= c1;
#pragma unroll
    for (int i = 0; i < 16; ++i) { o[i][0] *= c0; o[i][1] *= c0; o[i][2] *= c1; o[i][3] *= c1; }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = exp2f(s[nt][0] - mn0); s[nt][1] = exp2f(s[nt][1] - mn0);
      s[nt][2] = exp2f(s[nt][2] - mn1); s[nt][3] = exp2f(s[nt][3] - mn1);
      l0 += s[nt][0] + s[nt][1];
      l1 += s[nt][2] + s[nt][3];
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      a[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
      a[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
      a[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int dp = 0; dp < 8; ++dp) {
        uint32_t bfr[4];
        ldmatrix_x4_trans(bfr, sVb + swz(16 * kk + (lane & 7) + 8 * ((lane >> 3) & 1), 2 * dp + (lane >> 4)));
        mma_m16n8k16_bf16(o[2 * dp], a, bfr[0], bfr[1]);
        mma_m16n8k16_bf16(o[2 * dp + 1], a, bfr[2], bfr[3]);
      }
    }
    __syncthreads();
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int r0 = q0 + wrow + g, r1 = r0 + 8;
#pragma unroll
  for (int nt = 0; nt < 16; ++nt) {
    const int col = h * kHeadDim + nt * 8 + 2 * t;
    if (r0 < len)
      *reinterpret_cast<uint32_t*>(p.out + (long long)(tok0 + r0) * p.ldo + col) = pack_bf16x2(o[nt][0] * i0, o[nt][1] * i0);
    if (r1 < len)
      *reinterpret_cast<uint32_t*>(p.out + (long long)(tok0 + r1) * p.ldo + col) = pack_bf16x2(o[nt][2] * i1, o[nt][3] * i1);
  }
}

struct AttnDecodeParams {
  const bf16* q; long long ldq;        // [B][ldq] roped queries of the current token
  bf16* out; long long ldo;            // [B][ldo]
  const bf16* kcache; const bf16* vcache;   // e4m3 codes (one byte per element) in attn_decode_kernel<true>
  const int32_t* page_table; int max_pages;
  const int32_t* seq_slot;             // [B]
  const int32_t* tok_pos;              // [B] position of the current token; context = pos + 1
  int nh, nkv, G, splits;
  float* part_o;                       // [B*nkv][splits][G][128]
  float* part_ml;                      // [B*nkv][splits][G][2]
  float scale_log2;
  // Fused RoPE + KV append: when fuse_rope != 0 the kernel reads the raw QKV projection of the current token
  // (bf16 [B][ld_qkv], or fp32 split-K partials), applies rotate-half RoPE with the same rounding points as
  // rope_kv_kernel, uses the roped q / new k,v directly and appends k,v to the paged cache — one kernel
  // boundary less on the decode critical path.
  int fuse_rope;
  const bf16* qkv; long long ld_qkv;
  const float* qkv_partial; int qkv_splits; long long qkv_split_stride; long long ld_qkv_partial;
  const bf16* qkv_bias;   // [ld_qkv] projection bias added to the summed partials before their bf16 rounding (nullptr = none;
                          // a bf16 `qkv` row already carries it from the GEMM epilogue)
  const bf16* cos_tab; const bf16* sin_tab;
  // Qwen3: per-head RMSNorm of the G q heads (q_norm_w) and the k head (k_norm_w), [128] each, on the bf16-rounded row
  // before RoPE, in common.cuh's qknorm order (so the appended k equals rope_kv_kernel's); both nullptr = none
  const bf16* q_norm_w; const bf16* k_norm_w; float qk_eps;
  bf16* kcache_w; bf16* vcache_w;       // (e4m3 codes in attn_decode_kernel<true>, which appends e4m3(k), e4m3(v))
  // splits > 1: per-(sequence, kv head) arrival counters (zero between launches).  When set, the LAST split CTA to
  // arrive merges the partials itself (in split order: deterministic) and no attn_combine_kernel follows — one kernel
  // boundary less on the tensor-parallel decode path, where few (sequence, kv head) pairs per GPU force the split.
  int* split_counter;
};

// called by every CTA of a split launch after its partial (or its "empty" marker) is in global memory
__device__ __forceinline__ void attn_decode_arrive_and_merge(const AttnDecodeParams& p, int bh, int b, int kvh) {
  __shared__ int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(p.split_counter + bh, 1) == p.splits - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x == 0) p.split_counter[bh] = 0;
  __threadfence();
  const int G = p.G, d = threadIdx.x;
  const long long base = (long long)bh * p.splits * G;
  for (int r = 0; r < G; ++r) {
    float M = -INFINITY;
    for (int s = 0; s < p.splits; ++s) M = fmaxf(M, __ldcg(p.part_ml + (base + (long long)s * G + r) * 2));
    float L = 0.f, acc = 0.f;
    for (int s = 0; s < p.splits; ++s) {
      const long long row = base + (long long)s * G + r;
      const float ms = __ldcg(p.part_ml + row * 2);
      if (ms == -INFINITY) continue;   // empty split: its part_o row was never written
      const float f = exp2f(ms - M);
      L += __ldcg(p.part_ml + row * 2 + 1) * f;
      acc += __ldcg(p.part_o + row * kHeadDim + d) * f;
    }
    p.out[(long long)b * p.ldo + (kvh * G + r) * kHeadDim + d] = __float2bfloat16_rn(acc / L);
  }
}

template <bool KV8>
__global__ void __launch_bounds__(kAttnThreads) attn_decode_kernel(const AttnDecodeParams p) {
  constexpr int STAGES = KV8 ? kDecStages8 : kDecStages;
  TraceScope _ts(TK_ATTN_DECODE);
  pdl_launch_dependents();
  pdl_wait();
  _ts.mark();
  extern __shared__ __align__(1024) uint8_t smem[];
  const int bh = blockIdx.x, split = blockIdx.y;
  const int b = bh / p.nkv, kvh = bh - b * p.nkv;
  const int ctx = p.tok_pos[b] + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int G = p.G;
  const int ntiles = (ctx + 63) >> 6;
  const int per = (ntiles + p.splits - 1) / p.splits;
  const int t0 = split * per, t1 = min(ntiles, t0 + per);
  float* po = p.part_o + ((long long)bh * p.splits + split) * G * kHeadDim;
  float* pml = p.part_ml + ((long long)bh * p.splits + split) * G * 2;
  if (t0 >= t1) {  // empty split (uniform for the CTA)
    if (p.splits > 1 && threadIdx.x < G) { pml[threadIdx.x * 2] = -INFINITY; pml[threadIdx.x * 2 + 1] = 0.f; }
    if (p.splits > 1 && p.split_counter) attn_decode_arrive_and_merge(p, bh, b, kvh);
    return;
  }
  const uint32_t sQ = smem_u32(smem);       // 16 rows x 256 B = 4 KB
  const uint32_t sK = sQ + 4096;                      // bf16: kDecStages x 16 KB; KV8: the one expanded 16 KB tile
  const uint32_t sV = sK + (KV8 ? 1 : kDecStages) * kTileBytes;
  const uint32_t s8 = sQ + 4096 + 2 * kTileBytes;     // KV8: code ring, stage st = K codes at st * 16 KB, V codes 8 KB after
  const int32_t* pages = p.page_table + (long long)p.seq_slot[b] * p.max_pages;
  const long long tile_stride = (long long)p.nkv * kPageTokens * kHeadDim;
  const long long head_off = (long long)kvh * kPageTokens * kHeadDim;

  const int pos = ctx - 1;
  const int jt = pos >> 6;  // KV tile that receives the current token
  float* s_raw = reinterpret_cast<float*>(smem + 4096 + 2 * kDecStages * kTileBytes);   // [(G+2)][128] fp32
  bf16* s_newk = reinterpret_cast<bf16*>(s_raw + 10 * kHeadDim);           // [128]
  bf16* s_newv = s_newk + kHeadDim;                                          // [128]
  const uint8_t* kc8 = reinterpret_cast<const uint8_t*>(p.kcache);
  const uint8_t* vc8 = reinterpret_cast<const uint8_t*>(p.vcache);
  // stage tile jt into ring slot st; rows past the context are zero-filled
  auto load_stage = [&](int st, int jt_, int rows) {
    const long long pg = pages[jt_];
    if constexpr (KV8) {
      load_kv_tile8(s8 + st * 2 * kTile8Bytes, kc8 + pg * tile_stride + head_off, rows);
      load_kv_tile8(s8 + st * 2 * kTile8Bytes + kTile8Bytes, vc8 + pg * tile_stride + head_off, rows);
    } else {
      load_kv_tile(sK + st * kTileBytes, p.kcache + pg * tile_stride + head_off, rows);
      load_kv_tile(sV + st * kTileBytes, p.vcache + pg * tile_stride + head_off, rows);
    }
  };
  // fill the ring: STAGES-1 tiles in flight before any compute (one commit group per ring slot, empty or not)
#pragma unroll
  for (int st = 0; st < STAGES - 1; ++st) {
    if (t0 + st < t1) load_stage(st, t0 + st, ctx - (t0 + st) * 64);   // rows > 0
    cp_async_commit();
  }
  if (p.fuse_rope) {
    const int ngroups = (G + 2) * 16;
    for (int gi = threadIdx.x; gi < ngroups; gi += kAttnThreads) {
      const int hl = gi >> 4, c = (gi & 15) * 8;
      const int col = (hl < G ? (kvh * G + hl) : (hl == G ? p.nh + kvh : p.nh + p.nkv + kvh)) * kHeadDim + c;
      float f[8];
      if (p.qkv_partial) {
        float a[8];
        sum_partials8(p.qkv_partial + (long long)b * p.ld_qkv_partial + col, p.qkv_splits, p.qkv_split_stride, a);
        if (p.qkv_bias) {
#pragma unroll
          for (int i = 0; i < 8; ++i) a[i] += __bfloat162float(p.qkv_bias[col + i]);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] = bf16_round(a[i]);
      } else {
        uint4 u = *reinterpret_cast<const uint4*>(p.qkv + (long long)b * p.ld_qkv + col);
        const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float2 v2 = unpack_bf16x2(uw[i]);
          f[2 * i] = v2.x;
          f[2 * i + 1] = v2.y;
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) s_raw[hl * kHeadDim + c + i] = f[i];
    }
    __syncthreads();
    if (p.q_norm_w) {
      // thread (head hl, part qd) sums the squares of dims 8j + 2qd + {0, 1} and rewrites exactly those dims, so no
      // barrier is needed between the sums and the writes; (G + 1) * 4 <= 36 threads, the quads complete
      const int gi = threadIdx.x;
      const unsigned act = __ballot_sync(0xffffffffu, gi < (G + 1) * 4);
      if (gi < (G + 1) * 4) {
        const int hl = gi >> 2, qd = gi & 3;
        float* row = s_raw + hl * kHeadDim + 2 * qd;
        float sh = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) sh = qknorm_acc(sh, row[8 * j], row[8 * j + 1]);
        sh += __shfl_xor_sync(act, sh, 1);
        sh += __shfl_xor_sync(act, sh, 2);
        const float r = qknorm_rstd(sh, p.qk_eps);
        const bf16* w = (hl < G ? p.q_norm_w : p.k_norm_w) + 2 * qd;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          row[8 * j] = qknorm_apply(row[8 * j], r, __bfloat162float(w[8 * j]));
          row[8 * j + 1] = qknorm_apply(row[8 * j + 1], r, __bfloat162float(w[8 * j + 1]));
        }
      }
      __syncthreads();
    }
    const int items = (G + 1) * 8 + 16;   // roped heads (q heads + k) x 8 threads, then 16 threads copy v
    for (int it = threadIdx.x; it < items; it += kAttnThreads) {
      if (it < (G + 1) * 8) {
        const int hl = it >> 3, c = (it & 7) * 8;
        float cs[8], sn[8], o1[8], o2[8];
        {
          uint4 cu = *reinterpret_cast<const uint4*>(p.cos_tab + (long long)pos * 64 + c);
          uint4 su = *reinterpret_cast<const uint4*>(p.sin_tab + (long long)pos * 64 + c);
          const uint32_t cw[4] = {cu.x, cu.y, cu.z, cu.w}, sw[4] = {su.x, su.y, su.z, su.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float2 a2 = unpack_bf16x2(cw[i]), b2 = unpack_bf16x2(sw[i]);
            cs[2 * i] = a2.x; cs[2 * i + 1] = a2.y;
            sn[2 * i] = b2.x; sn[2 * i + 1] = b2.y;
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float x1 = s_raw[hl * kHeadDim + c + i], x2 = s_raw[hl * kHeadDim + c + 64 + i];
          o1[i] = bf16_round(x1 * cs[i]) + bf16_round(-x2 * sn[i]);
          o2[i] = bf16_round(x2 * cs[i]) + bf16_round(x1 * sn[i]);
          if (KV8 && hl == G) {   // the new k as the cache will give it back
            o1[i] = e4m3_roundtrip(bf16_round(o1[i]));
            o2[i] = e4m3_roundtrip(bf16_round(o2[i]));
          }
        }
        if (hl < G) {
          *reinterpret_cast<uint4*>(smem + swz(hl, c >> 3)) = pack8(o1);
          *reinterpret_cast<uint4*>(smem + swz(hl, (c >> 3) + 8)) = pack8(o2);
        } else {
          *reinterpret_cast<uint4*>(s_newk + c) = pack8(o1);
          *reinterpret_cast<uint4*>(s_newk + c + 64) = pack8(o2);
        }
      } else {
        const int c = (it - (G + 1) * 8) * 8;
        float f[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] = KV8 ? e4m3_roundtrip(s_raw[(G + 1) * kHeadDim + c + i]) : s_raw[(G + 1) * kHeadDim + c + i];
        *reinterpret_cast<uint4*>(s_newv + c) = pack8(f);
      }
    }
    // padding rows of the 16-row Q tile
    for (int idx = threadIdx.x; idx < (16 - G) * 16; idx += kAttnThreads)
      *reinterpret_cast<uint4*>(smem + swz(G + (idx >> 4), idx & 15)) = make_uint4(0, 0, 0, 0);
    __syncthreads();
    if (jt >= t0 && jt < t1 && threadIdx.x < 32) {   // the split that owns the current token appends it to the cache
      const int c = (threadIdx.x & 15) * 8, slot = pos & 63;
      const long long off = (long long)pages[jt] * tile_stride + head_off + slot * kHeadDim + c;
      if constexpr (KV8) {   // s_newk / s_newv hold e4m3 values: converting them back gives their codes exactly
        uint8_t* dst = reinterpret_cast<uint8_t*>(threadIdx.x < 16 ? p.kcache_w : p.vcache_w) + off;
        *reinterpret_cast<uint2*>(dst) = bf16x8_to_e4m3(*reinterpret_cast<const uint4*>((threadIdx.x < 16 ? s_newk : s_newv) + c));
      } else {
        if (threadIdx.x < 16) *reinterpret_cast<uint4*>(p.kcache_w + off) = *reinterpret_cast<const uint4*>(s_newk + c);
        else *reinterpret_cast<uint4*>(p.vcache_w + off) = *reinterpret_cast<const uint4*>(s_newv + c);
      }
    }
  } else {
    // Q: G rows valid, the rest zero
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int idx = threadIdx.x + it * kAttnThreads;
      const int r = idx >> 4, c = idx & 15;
      const bool valid = r < G;
      const bf16* src = p.q + (long long)b * p.ldq + (kvh * G + (valid ? r : 0)) * kHeadDim + c * 8;
      cp_async_16(sQ + swz(r, c), src, valid);
    }
    cp_async_commit();
    cp_async_wait<0>();   // (test path) keep the group accounting of the ring simple
  }

  uint32_t qf[8][4];
  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m0 = -INFINITY, l0 = 0.f;  // only row g (< 8) matters: rows >= G are padding

  for (int j = t0; j < t1; ++j) {
    const int buf = (j - t0) % STAGES;
    cp_async_wait<STAGES - 2>();   // tile j has landed
    __syncthreads();               // ... for every thread, and everyone is done with tile j-1's slot
    {
      const int jn = j + STAGES - 1;   // refill the slot tile j-1 used
      if (jn < t1) load_stage((jn - t0) % STAGES, jn, ctx - jn * 64);
      cp_async_commit();
    }
    if (j == t0) {
#pragma unroll
      for (int ks = 0; ks < 8; ++ks)
        ldmatrix_x4(qf[ks], sQ + swz((lane & 7) + 8 * ((lane >> 3) & 1), 2 * ks + (lane >> 4)));
    }
    const int tb = KV8 ? 0 : buf;   // bf16 tile the MMAs read
    const uint32_t sKb = sK + tb * kTileBytes, sVb = sV + tb * kTileBytes;
    if constexpr (KV8) {
      const uint8_t* codes = smem + 4096 + 2 * kTileBytes + buf * 2 * kTile8Bytes;
      expand_kv_tile8(smem + 4096, codes);
      expand_kv_tile8(smem + 4096 + kTileBytes, codes + kTile8Bytes);
      if (p.fuse_rope && j == jt) __syncthreads();   // the patch below overwrites an expanded row
    }
    if (p.fuse_rope && j == jt) {   // the row of the current token is not in the cache copy that was just staged
      if (threadIdx.x < 32) {
        const int c = threadIdx.x & 15, slot = pos & 63;
        uint8_t* base = smem + 4096 + (threadIdx.x < 16 ? 0 : (KV8 ? 1 : kDecStages) * kTileBytes) + tb * kTileBytes;
        *reinterpret_cast<uint4*>(base + swz(slot, c)) =
            *reinterpret_cast<const uint4*>((threadIdx.x < 16 ? s_newk : s_newv) + c * 8);
      }
      if (!KV8) __syncthreads();
    }
    if (KV8) __syncthreads();       // the expanded (and patched) tile is complete
    float s[2][4];
    s[0][0] = s[0][1] = s[0][2] = s[0][3] = 0.f;
    s[1][0] = s[1][1] = s[1][2] = s[1][3] = 0.f;
    const int trow = warp * 16;  // this warp's 16 tokens of the tile
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      uint32_t bfr[4];
      ldmatrix_x4(bfr, sKb + swz(trow + (lane & 7) + 8 * (lane >> 4), 2 * ks + ((lane >> 3) & 1)));
      mma_m16n8k16_bf16(s[0], qf[ks], bfr[0], bfr[1]);
      mma_m16n8k16_bf16(s[1], qf[ks], bfr[2], bfr[3]);
    }
    float mx = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int kp = j * 64 + trow + nt * 8 + 2 * t + e;
        float v = s[nt][e] * p.scale_log2;
        if (kp >= ctx) v = -INFINITY;
        s[nt][e] = v;
        mx = fmaxf(mx, v);
      }
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float mn = fmaxf(m0, mx);
    const float msafe = (mn == -INFINITY) ? 0.f : mn;  // whole 16-token slice masked and nothing seen yet
    const float c0 = exp2f(m0 - msafe);
    m0 = mn;
    l0 *= c0;
#pragma unroll
    for (int i = 0; i < 16; ++i) { o[i][0] *= c0; o[i][1] *= c0; }
    float pr[2][2];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      pr[nt][0] = exp2f(s[nt][0] - msafe);
      pr[nt][1] = exp2f(s[nt][1] - msafe);
      l0 += pr[nt][0] + pr[nt][1];
    }
    uint32_t a[4];
    a[0] = pack_bf16x2(pr[0][0], pr[0][1]);
    a[1] = 0u;  // rows 8..15 are padding
    a[2] = pack_bf16x2(pr[1][0], pr[1][1]);
    a[3] = 0u;
#pragma unroll
    for (int dp = 0; dp < 8; ++dp) {
      uint32_t bfr[4];
      ldmatrix_x4_trans(bfr, sVb + swz(trow + (lane & 7) + 8 * ((lane >> 3) & 1), 2 * dp + (lane >> 4)));
      mma_m16n8k16_bf16(o[2 * dp], a, bfr[0], bfr[1]);
      mma_m16n8k16_bf16(o[2 * dp + 1], a, bfr[2], bfr[3]);
    }
  }
  cp_async_wait<0>();
  __syncthreads();   // all warps done with the ring before it is reused for the merge
  // ---- merge the 4 warps (each saw a disjoint quarter of every tile) through shared memory
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  float* sm_m = reinterpret_cast<float*>(smem + 4096);  // [4][8]
  float* sm_l = sm_m + 32;                               // [4][8]
  float* sm_o = sm_l + 32;                               // [4][8][128]
  if (t == 0) { sm_m[warp * 8 + g] = m0; sm_l[warp * 8 + g] = l0; }
#pragma unroll
  for (int nt = 0; nt < 16; ++nt) {
    sm_o[(warp * 8 + g) * kHeadDim + nt * 8 + 2 * t] = o[nt][0];
    sm_o[(warp * 8 + g) * kHeadDim + nt * 8 + 2 * t + 1] = o[nt][1];
  }
  __syncthreads();
  const int d = threadIdx.x;  // 128 threads <-> 128 dims
  for (int r = 0; r < G; ++r) {
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < 4; ++w) M = fmaxf(M, sm_m[w * 8 + r]);
    float L = 0.f, acc = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float mw = sm_m[w * 8 + r];
      if (mw == -INFINITY) continue;   // every key this warp saw was masked
      const float f = exp2f(mw - M);
      L += sm_l[w * 8 + r] * f;
      acc += sm_o[(w * 8 + r) * kHeadDim + d] * f;
    }
    if (p.splits == 1) {
      p.out[(long long)b * p.ldo + (kvh * G + r) * kHeadDim + d] = __float2bfloat16_rn(acc / L);
    } else {
      po[r * kHeadDim + d] = acc;
      if (d == 0) { pml[r * 2] = M; pml[r * 2 + 1] = L; }
    }
  }
  if (p.splits > 1 && p.split_counter) attn_decode_arrive_and_merge(p, bh, b, kvh);
}

// one CTA (128 threads) per (batch row, query head)
__global__ void __launch_bounds__(128)
attn_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml, bf16* __restrict__ out,
                    long long ldo, int nkv, int G, int splits) {
  TraceScope _ts(TK_ATTN_COMBINE);
  pdl_launch_dependents();
  pdl_wait();
  _ts.mark();
  const int bhq = blockIdx.x;            // b * nh + head
  const int nh = nkv * G;
  const int b = bhq / nh, head = bhq - b * nh;
  const int kvh = head / G, r = head - kvh * G;
  const long long base = ((long long)(b * nkv + kvh) * splits) * G;
  float M = -INFINITY;
  for (int s = 0; s < splits; ++s) M = fmaxf(M, part_ml[(base + (long long)s * G + r) * 2]);
  float L = 0.f, acc = 0.f;
  const int d = threadIdx.x;
  for (int s = 0; s < splits; ++s) {
    const long long row = base + (long long)s * G + r;
    const float ms = part_ml[row * 2];
    if (ms == -INFINITY) continue;   // empty split: its part_o row was never written
    const float f = exp2f(ms - M);
    L += part_ml[row * 2 + 1] * f;
    acc += part_o[row * kHeadDim + d] * f;
  }
  out[(long long)b * ldo + head * kHeadDim + d] = __float2bfloat16_rn(acc / L);
}

}  // namespace b200
