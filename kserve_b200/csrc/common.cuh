// Common device helpers for the sm_90a kernels: error handling, bf16 helpers and thin
// wrappers over the Hopper PTX used by the hot path (mbarrier, TMA, wgmma).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

namespace b200 {

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------------------------------------
// host-side error plumbing: every C-ABI entry returns an int status; the text is kept per thread.
// ---------------------------------------------------------------------------------------------
void set_last_error(const std::string& msg);

#define B200_CUDA_OK(expr)                                                                       \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      ::b200::set_last_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " at " + \
                             __FILE__ + ":" + std::to_string(__LINE__));                         \
      return -1;                                                                                 \
    }                                                                                            \
  } while (0)

#define B200_REQUIRE(cond, msg)                                                          \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      ::b200::set_last_error(std::string("requirement failed: ") + #cond + ": " + (msg)); \
      return -2;                                                                         \
    }                                                                                    \
  } while (0)

// ---------------------------------------------------------------------------------------------
// small device utilities
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

// Per-head RMSNorm of q and k (Qwen3RMSNorm over one head's 128 dims, between the projection and RoPE).  The prefill
// QKV epilogue, rope_kv_kernel and the decode attention prologue all normalise with these helpers, in this one order of
// the 128 squares, so they produce the same bits from the same bf16 inputs.  The order is the one the wgmma fragment
// gives for free: part qd (0..3) accumulates dims 8j + 2qd and 8j + 2qd + 1 for j = 0..15 in increasing j (the dims quad
// lane qd holds), and the head's sum is (S0 + S1) + (S2 + S3), which two shfl_xor steps (1, then 2) produce in every lane.
__device__ __forceinline__ float qknorm_acc(float s, float a0, float a1) { return fmaf(a1, a1, fmaf(a0, a0, s)); }
__device__ __forceinline__ float qknorm_sum(float s0, float s1, float s2, float s3) { return (s0 + s1) + (s2 + s3); }
// 1 / sqrt(mean of the squares + eps)
__device__ __forceinline__ float qknorm_rstd(float sumsq, float eps) { return rsqrtf(sumsq * (1.0f / 128.0f) + eps); }
// bf16(bf16(a * r) * w): Qwen3RMSNorm casts to the input dtype before the weight multiply
__device__ __forceinline__ float qknorm_apply(float a, float r, float w) { return bf16_round(bf16_round(a * r) * w); }

// FP8 KV cache codes: e4m3(clamp(x, -448, 448)), round to nearest even; NaN stays NaN.  `lo` goes to the lower byte.
__device__ __forceinline__ uint32_t e4m3x2_rn_sat(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
// 8 bf16 (one 16-byte chunk) -> their 8 codes, byte i = element i
__device__ __forceinline__ uint2 bf16x8_to_e4m3(const uint4& v) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t c[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(w[i]);
    c[i] = e4m3x2_rn_sat(f.x, f.y);
  }
  return make_uint2(c[0] | (c[1] << 16), c[2] | (c[3] << 16));
}
// the value an FP8 KV cache gives back for x: float(e4m3(clamp(x))) (exact in bf16 and in half)
__device__ __forceinline__ float e4m3_roundtrip(float x) {
  const uint16_t c = (uint16_t)e4m3x2_rn_sat(x, 0.f);
  uint32_t h2;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(c));
  return __half2float(__ushort_as_half((unsigned short)(h2 & 0xFFFFu)));
}

// 128-bit streaming load that does not allocate in L1 (weights / KV pages are read once per step).
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------------------------------------
// Optional per-CTA timeline (debug): when enabled through b200_debug_trace(), thread 0 of every CTA appends
// {kind, block, globaltimer at entry, at exit}; off by default (one predictable branch per CTA).
// ---------------------------------------------------------------------------------------------
struct TraceRec { unsigned long long t0, t1, tmid; int kind, block; };
__device__ TraceRec* g_trace_buf = nullptr;
__device__ unsigned int g_trace_cap = 0;
__device__ unsigned int g_trace_cnt = 0;
enum TraceKind : int { TK_GEMM = 1, TK_RMSNORM = 2, TK_ROPE = 3, TK_ATTN_DECODE = 4, TK_ATTN_COMBINE = 5, TK_ARGMAX = 6,
                       TK_STEP = 7, TK_EMBED = 8, TK_ATTN_PREFILL = 9, TK_OTHER = 10 };
__device__ __forceinline__ unsigned long long global_timer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
struct TraceScope {
  unsigned long long t0 = 0, tmid = 0;
  int kind;
  __device__ __forceinline__ void mark() { if (threadIdx.x == 0 && t0 != 0) tmid = global_timer(); }
  __device__ __forceinline__ explicit TraceScope(int k) : kind(k) {
    if (threadIdx.x == 0 && g_trace_buf != nullptr) t0 = global_timer();
  }
  __device__ __forceinline__ ~TraceScope() {
    if (threadIdx.x == 0 && t0 != 0) {
      const unsigned int i = atomicAdd(&g_trace_cnt, 1u);
      if (i < g_trace_cap) {
        TraceRec r; r.t0 = t0; r.t1 = global_timer(); r.tmid = tmid; r.kind = kind; r.block = blockIdx.x;
        g_trace_buf[i] = r;
      }
    }
  }
};

// ---------------------------------------------------------------------------------------------
// Recoverable faults of the cross-GPU / cross-CTA waits.  A tensor-parallel peer that died, or was never launched, must
// not take this rank's CUDA context with it: a wait that times out records a code here and the kernel carries on with
// whatever data it has (every later wait then gives up at once), instead of __trap()ing — which would poison the context
// of every rank for good.  The host reads the code at its next synchronisation point (b200_engine_fault), fails the call,
// marks the engine unusable, and the model server reports the model as not ready.  Codes: 1 peer flag, 2 all-reduce
// packet, 3 candidate exchange, 4 stream-K piece.
// ---------------------------------------------------------------------------------------------
__device__ int g_fault_code = 0;
__device__ __forceinline__ bool fault_raised() { return *reinterpret_cast<volatile int*>(&g_fault_code) != 0; }
__device__ __forceinline__ void fault_raise(int code) { atomicCAS(&g_fault_code, 0, code); }
// One step of a bounded spin: false = keep waiting, true = give up (time-out reached, or another wait already failed).
// The bound is wall time (%globaltimer, looked at every 1024 polls): g_wait_timeout_ns, default 5 s — far beyond any
// legitimate wait of a decode step, short enough that a lost peer fails the request instead of hanging the server.
__device__ unsigned long long g_wait_timeout_ns = 5000000000ull;
struct SpinGuard { uint32_t polls = 0; unsigned long long t0 = 0; };
__device__ __forceinline__ bool spin_give_up(SpinGuard& g, int code) {
  if ((++g.polls & 0x3ff) != 0) return false;
  if (fault_raised()) return true;
  const unsigned long long now = global_timer();
  if (g.t0 == 0) { g.t0 = now; return false; }
  if (now - g.t0 > *reinterpret_cast<volatile unsigned long long*>(&g_wait_timeout_ns)) { fault_raise(code); return true; }
  return false;
}

// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch: a kernel lets its successor start (prologue, weight prefetch) while it is
// still running, and blocks only where it first touches data the predecessor produced.  Both are no-ops when
// the kernel was launched without the programmatic-stream-serialization attribute.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug traps (-> a CUDA error the host reports) instead of hanging the GPU.  No function call
// (printf) on the timeout branch: these waits sit between wgmma issues, and a call inside the wgmma pipeline makes ptxas
// serialise every wgmma of the kernel (C7510).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) — 2D tile load, completion on an mbarrier, with an L2 cache hint
// ---------------------------------------------------------------------------------------------
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c_inner,
                                            int c_outer, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c_inner), "r"(c_outer), "l"(hint)
      : "memory");
}
// Asynchronous prefetch of a 2D tile into L2 only (no shared memory): used to pull the next weight slab towards
// the SMs while the kernel is still waiting for its predecessor.
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* map, int c_inner, int c_outer) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(c_inner), "r"(c_outer)
               : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// 2D tile store shared -> global (elements outside the map's extents are not written), tracked by bulk groups.
// Generic-proxy writes of the source tile must be made visible with fence_proxy_async_shared() before the issue.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int c_inner, int c_outer,
                                             uint64_t hint) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3}], [%1], %4;"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(smem_src)), "r"(c_inner), "r"(c_outer), "l"(hint)
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }  // sources reusable
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): all 128 threads of a warpgroup issue it together; the fp32 accumulator of an
// m64nN tile lives in registers, thread t of the warpgroup holding, for i in [0, N/2):
//   row 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),  column 8 * (i / 4) + 2 * (t % 4) + i % 2
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_keep(float (&d)[N]) {   // accumulator registers stay live across wgmma_wait
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Register budget of a warp-specialised kernel: the TMA producer warpgroup gives registers back, the MMA warpgroups take them.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// wgmma shared-memory descriptor for a K-major bf16 tile whose rows are 128 B (64 elements) wide and stored with
// the 128-byte swizzle TMA writes (CU_TENSOR_MAP_SWIZZLE_128B): 8-row groups are SBO = 1024 B apart, LBO is unused
// for swizzled K-major layouts (encoded 1), layout type 1 = 128B swizzle.  Advancing 16 elements (32 B) along K
// inside the swizzle atom is +2 on the descriptor.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// MN-major 128B-swizzled operand (B = V[token][dim], dims contiguous): 8 token rows x 128 B form one swizzle atom,
// atoms along K (tokens) are SBO = 1024 B apart, the next 64-element block along N is LBO further.
__device__ __forceinline__ uint64_t make_smem_desc_sw128_mn(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// D (+)= A[smem desc] * B[smem desc]^T, both K-major (wgmma_ss_nN), and D (+)= A[registers] * B[smem desc] with an
// MN-major B (wgmma_rs_n128_tb).  scale_d == 0 overwrites D.
__device__ __forceinline__ void wgmma_ss_n16(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_ss_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_ss_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_rs_n128_tb(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}

// ---------------------------------------------------------------------------------------------
// legacy warp-level MMA (m16n8k16 bf16) + ldmatrix + cp.async: used by the attention kernels
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_m16n8k16_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void cp_async_16(uint32_t smem_dst, const void* gsrc, bool valid) {
  int sz = valid ? 16 : 0;  // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

}  // namespace b200
