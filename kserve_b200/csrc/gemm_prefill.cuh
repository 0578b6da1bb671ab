// Persistent, warp-specialised prefill GEMM for sm_90a:  out[M, *] = epi(A[M,K] * B[N,K]^T), 128 x 256 tiles.
//
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx)
//   warpgroups 1-2 : wgmma consumers, one 64-row half of the 128-row tile each (m64n256k16, fp32 accumulators in
//                    registers)
//
// The epilogue works on the accumulator fragment itself: every pair the fused epilogues combine sits in the same
// thread (SwiGLU gate / up columns 32c + x and 32c + 16 + x are fragments j and j + 2, the RoPE pair d / d + 64 is
// fragments j and j + 8).  The bf16 results go to a 128B-swizzled output tile in shared memory that one thread hands
// to TMA stores; the consumers start the next tile's main loop while those stores drain.  Rows past the tile's
// valid extent are never given to TMA: a partial last tile (M known only on the device, MoE experts), an output TMA
// cannot address, and the paged KV-cache rows of EPI_ROPE_KV go out through per-thread stores from the same tile.
#pragma once
#include "gemm_wgmma.cuh"

namespace b200 {

template <int EPI>
struct PrefillCfg {
  static constexpr int kABytes = kGemmBlockM * kGemmBlockK * 2;        // 16 KB
  static constexpr int kStageBytes = kABytes + 256 * kGemmBlockK * 2;  // + 32 KB of weight rows
  static constexpr int kOutCols = (EPI == EPI_SWIGLU) ? 128 : 256;     // bf16 output columns of one tile
  static constexpr int kBoxes = kOutCols / 64;                         // TMA store boxes of [128 rows][64 cols]
  static constexpr int kBoxBytes = kGemmBlockM * 128;
  static constexpr int kOutBytes = kBoxes * kBoxBytes;
  // the 32 KB SwiGLU output tile leaves room for a fourth stage; the 64 KB tiles do not
  static constexpr int kStages = (EPI == EPI_SWIGLU) ? 4 : 3;
  static constexpr int kSmemBytes = kStages * kStageBytes + kOutBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 227 * 1024, "prefill GEMM shared memory exceeds the 227 KB a block may use");
};

// byte offset of output (row, col) in the swizzled tile: box col / 64, 16-byte chunk (col / 8) % 8 swizzled by row % 8
__device__ __forceinline__ uint32_t out_tile_off(int row, int col) {
  return (col >> 6) * (kGemmBlockM * 128) + row * 128 + ((((col >> 3) & 7) ^ (row & 7)) << 4) + (col & 7) * 2;
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}

// residual columns (col, col + 1) of one row; N bounds the valid columns
__device__ __forceinline__ float2 ld_res2(const bf16* row, int col, int N, bool pair) {
  if (pair && col + 1 < N) return unpack_bf16x2(*reinterpret_cast<const uint32_t*>(row + col));
  float2 r;
  r.x = col < N ? __bfloat162float(row[col]) : 0.f;
  r.y = col + 1 < N ? __bfloat162float(row[col + 1]) : 0.f;
  return r;
}

// bias of output columns (col, col + 1); N bounds the valid columns
__device__ __forceinline__ float2 ld_bias2(const bf16* b, int col, int N) {
  float2 r;
  r.x = col < N ? __bfloat162float(b[col]) : 0.f;
  r.y = col + 1 < N ? __bfloat162float(b[col + 1]) : 0.f;
  return r;
}

// tmap_out: `out` as [rows][out columns] with leading dimension ldo, box [128][64], 128B swizzle; used when p.out_tma.
// BIAS (EPI_STORE, EPI_ROPE_KV): add p.bias[column] to the fp32 accumulator before its bf16 rounding; a compile-time
// flag, so the GEMMs without a bias run exactly the code they ran before.
// KV8 (EPI_ROPE_KV): the paged cache holds e4m3 codes; each k / v row goes out as e4m3(bf16 value), 8 codes per store.
// QKNORM (EPI_ROPE_KV, no bias): Qwen3's per-head RMSNorm of q and k (p.rope_q_norm / p.rope_k_norm) between the
// projection's bf16 rounding and RoPE, in common.cuh's qknorm order; a compile-time flag like BIAS.
template <int EPI, bool BIAS = false, bool KV8 = false, bool QKNORM = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_prefill_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                    const __grid_constant__ CUtensorMap tmap_out, const GemmParams p) {
  static_assert(EPI == EPI_STORE || EPI == EPI_STORE_RES || EPI == EPI_SWIGLU || EPI == EPI_ROPE_KV, "row-major epilogues only");
  static_assert(!BIAS || EPI == EPI_STORE || EPI == EPI_ROPE_KV, "bias: QKV epilogues only");
  static_assert(!KV8 || EPI == EPI_ROPE_KV, "FP8 KV cache: the RoPE + KV epilogue only");
  static_assert(!QKNORM || (EPI == EPI_ROPE_KV && !BIAS), "q/k norm: the RoPE + KV epilogue, without a projection bias");
  TraceScope _ts(TK_GEMM + 100 * EPI + 1000 * (p.M >> 7));
  using Cfg = PrefillCfg<EPI>;
  constexpr int STAGES = Cfg::kStages;
  constexpr int BLOCK_N = 256;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* otile = smem + STAGES * Cfg::kStageBytes;   // bf16 output tile, 1024-byte aligned boxes
  uint64_t* bars = reinterpret_cast<uint64_t*>(otile + Cfg::kOutBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (p.out_tma) tma_prefetch_desc(&tmap_out);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrival per MMA warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  int M_rt = p.M;
  if (p.m_rt != nullptr || p.row_off != nullptr) {   // extents produced by the previous kernel
    pdl_wait();
    if (p.m_rt) M_rt = min(p.M, *p.m_rt);
  }
  const int m_tiles_rt = (M_rt <= 0 || p.N <= 0) ? 0 : (M_rt + kGemmBlockM - 1) / kGemmBlockM;
  const int roff = p.row_off ? *p.row_off : 0;   // (read after the wait above: set together with m_rt)

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      pdl_wait();
      int stage = 0;
      uint32_t phase = 0;
      GemmSeg sg;
      for (int idx = 0; gemm_get_seg(p, idx, sg, m_tiles_rt); ++idx) {
        const int a_row = sg.m_t * kGemmBlockM + roff;
        for (int kb = sg.kb0; kb < sg.kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * kGemmBlockK, a_row, p.hint_a);
          tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * kGemmBlockK, sg.n_t * BLOCK_N, p.hint_b);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  // ------------------------------------------------------------------ MMA + epilogue (2 warpgroups)
  setmaxnreg_inc<232>();
  const int half = wg - 1;                 // accumulator rows 64 * half ... + 63 of the tile
  const int t = threadIdx.x - 128 * wg;    // thread of the warpgroup
  const int et = threadIdx.x - 128;        // 0 .. 255
  const int qd = lane & 3;
  const int frag_row = 64 * half + 16 * (warp & 3) + (lane >> 2);   // accumulator rows frag_row, frag_row + 8
  const uint32_t ot = smem_u32(otile);
  const uint64_t out_hint = p.stream_out ? kEvictFirst : kEvictNormal;
  const bool out_vec = ((p.ldo & 7) == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 15) == 0);
  pdl_wait();              // outputs / residual must not be touched before the previous kernel is complete
  int stage = 0;
  uint32_t phase = 0;
  float accum[BLOCK_N / 2];
  GemmSeg sg;
  for (int idx = 0; gemm_get_seg(p, idx, sg, m_tiles_rt); ++idx) {
    const int m_t = sg.m_t, n_t = sg.n_t;
    // ---- main loop: one k-block in flight behind the one being issued
    wgmma_keep(accum);
    int prev = -1;
    for (int kb = sg.kb0; kb < sg.kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
      const uint64_t adesc = make_smem_desc_sw128(sa + half * 64 * 128);
      const uint64_t bdesc = make_smem_desc_sw128(sa + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kGemmBlockK / 16; ++k)
        wgmma_tile<BLOCK_N>(accum, adesc + 2 * k, bdesc + 2 * k, (kb > sg.kb0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);   // the k-block before this one has been consumed
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_keep(accum);
    if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);

    // ---- epilogue: fragment -> bf16 output tile (the previous tile's stores must have read it first)
    const int row0 = m_t * kGemmBlockM;
    const int n0 = n_t * BLOCK_N;
    if (et == 0) bulk_wait_read_all();
    consumer_bar();
    if constexpr (EPI == EPI_STORE || EPI == EPI_STORE_RES) {
      const bf16* rrow[2] = {nullptr, nullptr};
      const bool rpair = ((p.ldo & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.residual) & 3) == 0);
      if constexpr (EPI == EPI_STORE_RES) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = row0 + frag_row + 8 * h;
          rrow[h] = m < M_rt ? p.residual + (long long)(m + roff) * p.ldo + n0 : nullptr;
        }
      }
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = 8 * j + 2 * qd;
        const float2 bb = BIAS ? ld_bias2(p.bias + n0, col, p.N - n0) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float f0 = accum[4 * j + 2 * h], f1 = accum[4 * j + 2 * h + 1];
          if constexpr (BIAS) { f0 += bb.x; f1 += bb.y; }
          if constexpr (EPI == EPI_STORE_RES) {
            if (rrow[h] != nullptr) {
              const float2 r2 = ld_res2(rrow[h], col, p.N - n0, rpair);
              f0 = bf16_round(f0) + r2.x;
              f1 = bf16_round(f1) + r2.y;
            }
          }
          st_shared_u32(ot + out_tile_off(frag_row + 8 * h, col), pack_bf16x2(f0, f1));
        }
      }
    } else if constexpr (EPI == EPI_SWIGLU) {
      // columns [32c, 32c + 16) = gate, [32c + 16, 32c + 32) = up of output columns 16c + x
#pragma unroll
      for (int c = 0; c < BLOCK_N / 32; ++c)
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int jg = 4 * c + jj, ju = jg + 2;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float o[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float g = bf16_round(accum[4 * jg + 2 * h + e]);
              const float up = bf16_round(accum[4 * ju + 2 * h + e]);
              o[e] = bf16_round(silu_f(g)) * up;
            }
            st_shared_u32(ot + out_tile_off(frag_row + 8 * h, 16 * c + 8 * jj + 2 * qd), pack_bf16x2(o[0], o[1]));
          }
        }
    } else {   // EPI_ROPE_KV: the tile is heads 2 n_t, 2 n_t + 1 of [q heads | k heads | v heads] x 128
      // HF bf16 rounding points of apply_rotary_pos_emb (bit-identical to rope_kv_kernel); the projection bias is added
      // to the fp32 accumulator before its one bf16 rounding, i.e. before the rotation as in HF
      int pos[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = row0 + frag_row + 8 * h;
        pos[h] = m < M_rt ? p.rope_tok_pos[m + roff] : 0;
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int head = 2 * n_t + hh;
        const bool hb = BIAS && head < p.rope_nh + 2 * p.rope_nkv;   // (uniform; past the last head there is no bias)
        if (head >= p.rope_nh + p.rope_nkv) {   // v head (or past the last head): copied as is
#pragma unroll
          for (int j = 16 * hh; j < 16 * hh + 16; ++j) {
            const float2 bb = hb ? ld_bias2(p.bias + n0, 8 * j + 2 * qd, p.N - n0) : make_float2(0.f, 0.f);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float f0 = accum[4 * j + 2 * h], f1 = accum[4 * j + 2 * h + 1];
              if (hb) { f0 += bb.x; f1 += bb.y; }
              st_shared_u32(ot + out_tile_off(frag_row + 8 * h, 8 * j + 2 * qd), pack_bf16x2(f0, f1));
            }
          }
        } else {                                  // q or k head: rotate-half RoPE on the pairs (d, d + 64)
          if constexpr (QKNORM) {
            // this thread holds dims 8j + 2qd + {0, 1} (j = 0..15) of rows frag_row and frag_row + 8 of the head: round
            // them to bf16, sum their squares in qknorm order, finish each row's sum across the quad, normalise in place
            const bf16* nw = head < p.rope_nh ? p.rope_q_norm : p.rope_k_norm;
            float ss[2] = {0.f, 0.f};
#pragma unroll
            for (int jl = 0; jl < 16; ++jl) {
              const int j = 16 * hh + jl;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                accum[4 * j + 2 * h] = bf16_round(accum[4 * j + 2 * h]);
                accum[4 * j + 2 * h + 1] = bf16_round(accum[4 * j + 2 * h + 1]);
                ss[h] = qknorm_acc(ss[h], accum[4 * j + 2 * h], accum[4 * j + 2 * h + 1]);
              }
            }
            float rs[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float sh = ss[h];
              sh += __shfl_xor_sync(0xffffffffu, sh, 1);
              sh += __shfl_xor_sync(0xffffffffu, sh, 2);
              rs[h] = qknorm_rstd(sh, p.rope_qk_eps);
            }
#pragma unroll
            for (int jl = 0; jl < 16; ++jl) {
              const int j = 16 * hh + jl;
              const float2 wv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(nw + 8 * jl + 2 * qd));
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                accum[4 * j + 2 * h] = qknorm_apply(accum[4 * j + 2 * h], rs[h], wv.x);
                accum[4 * j + 2 * h + 1] = qknorm_apply(accum[4 * j + 2 * h + 1], rs[h], wv.y);
              }
            }
          }
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j1 = 16 * hh + jj, j2 = j1 + 8;
            const int d = 8 * jj + 2 * qd;
            const float2 ba = hb ? ld_bias2(p.bias + n0, 8 * j1 + 2 * qd, p.N - n0) : make_float2(0.f, 0.f);
            const float2 bc = hb ? ld_bias2(p.bias + n0, 8 * j2 + 2 * qd, p.N - n0) : make_float2(0.f, 0.f);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float2 cs = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.rope_cos + (long long)pos[h] * 64 + d));
              const float2 sn = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.rope_sin + (long long)pos[h] * 64 + d));
              float x0 = accum[4 * j1 + 2 * h], x1 = accum[4 * j1 + 2 * h + 1];
              float y0 = accum[4 * j2 + 2 * h], y1 = accum[4 * j2 + 2 * h + 1];
              if (hb) { x0 += ba.x; x1 += ba.y; y0 += bc.x; y1 += bc.y; }
              const float a0 = bf16_round(x0), a1 = bf16_round(x1);
              const float b0 = bf16_round(y0), b1 = bf16_round(y1);
              const float o1x = bf16_round(a0 * cs.x) + bf16_round(-b0 * sn.x);
              const float o1y = bf16_round(a1 * cs.y) + bf16_round(-b1 * sn.y);
              const float o2x = bf16_round(b0 * cs.x) + bf16_round(a0 * sn.x);
              const float o2y = bf16_round(b1 * cs.y) + bf16_round(a1 * sn.y);
              st_shared_u32(ot + out_tile_off(frag_row + 8 * h, 8 * j1 + 2 * qd), pack_bf16x2(o1x, o1y));
              st_shared_u32(ot + out_tile_off(frag_row + 8 * h, 8 * j2 + 2 * qd), pack_bf16x2(o2x, o2y));
            }
          }
        }
      }
    }
    fence_proxy_async_shared();   // the tile is read by the TMA (async proxy)
    consumer_bar();

    // ---- store: whole tiles by TMA (q heads only for EPI_ROPE_KV), the rest per thread
    const bool tile_tma = p.out_tma && row0 + kGemmBlockM <= M_rt;
    const int oc0 = (EPI == EPI_SWIGLU) ? n0 / 2 : n0;   // first output column of the tile
    if (tile_tma && et == 0) {
#pragma unroll
      for (int b = 0; b < Cfg::kBoxes; ++b) {
        if (EPI == EPI_ROPE_KV && 2 * n_t + b / 2 >= p.rope_nh) continue;
        tma_store_2d(&tmap_out, otile + b * Cfg::kBoxBytes, oc0 + 64 * b, row0 + roff, out_hint);
      }
      bulk_commit_group();
    }
    if (EPI == EPI_ROPE_KV || !tile_tma) {
      // thread -> (tile row r, one half of the tile's output columns)
      constexpr int HC = Cfg::kOutCols / 2;
      const int r = et & (kGemmBlockM - 1), hsel = et >> 7;
      const int m = row0 + r;
      bf16* dst = nullptr;
      uint8_t* dst8 = nullptr;   // KV8: this row's k / v codes
      int nvalid = HC;
      bool vec = out_vec;
      int stream = p.stream_out;
      if (m < M_rt) {
        if constexpr (EPI == EPI_ROPE_KV) {
          const int head = 2 * n_t + hsel;
          if (head < p.rope_nh) {
            if (!tile_tma) dst = reinterpret_cast<bf16*>(p.out) + (long long)(m + roff) * p.ldo + n0 + HC * hsel;
          } else if (head < p.rope_nh + 2 * p.rope_nkv) {
            const int pos = p.rope_tok_pos[m + roff];
            const int page = p.rope_page_table[(long long)p.rope_tok_seq[m + roff] * p.rope_max_pages + (pos >> 6)];
            const long long page_row = (long long)page * p.rope_nkv * 64 + (pos & 63);   // row of kv head 0 in [..][64][128]
            if constexpr (KV8) {
              const long long e0 = head < p.rope_nh + p.rope_nkv ? (page_row + (long long)(head - p.rope_nh) * 64) * 128
                                                                 : (page_row + (long long)(head - p.rope_nh - p.rope_nkv) * 64) * 128;
              dst8 = reinterpret_cast<uint8_t*>(head < p.rope_nh + p.rope_nkv ? p.rope_kcache : p.rope_vcache) + e0;
            } else {
              dst = head < p.rope_nh + p.rope_nkv ? p.rope_kcache + (page_row + (long long)(head - p.rope_nh) * 64) * 128
                                                  : p.rope_vcache + (page_row + (long long)(head - p.rope_nh - p.rope_nkv) * 64) * 128;
            }
            vec = true;
            stream = 0;
          }
        } else {
          const int ncols = (EPI == EPI_SWIGLU) ? p.out_cols : p.N;
          nvalid = min(HC, ncols - (oc0 + HC * hsel));
          if (nvalid > 0) dst = reinterpret_cast<bf16*>(p.out) + (long long)(m + roff) * p.ldo + oc0 + HC * hsel;
        }
      }
      if constexpr (KV8) {
        if (dst8 != nullptr) {
#pragma unroll 4
          for (int c = 0; c < HC; c += 8)
            *reinterpret_cast<uint2*>(dst8 + c) = bf16x8_to_e4m3(ld_shared_v4(ot + out_tile_off(r, HC * hsel + c)));
        }
      }
      if (dst != nullptr) {
#pragma unroll 4
        for (int c = 0; c < HC; c += 8) {
          if (c >= nvalid) break;
          const uint4 v = ld_shared_v4(ot + out_tile_off(r, HC * hsel + c));
          if (vec && c + 8 <= nvalid) {
            st_out_v4(dst + c, v, stream);
          } else {
            const bf16* e = reinterpret_cast<const bf16*>(&v);
            for (int u = 0; u < 8 && c + u < nvalid; ++u) dst[c + u] = e[u];
          }
        }
      }
    }
  }
  if (et == 0) bulk_wait_all();
}

}  // namespace b200
