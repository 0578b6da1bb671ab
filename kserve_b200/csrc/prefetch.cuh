// Weight-stream L2 prefetch for the decode step.
//
// A decode step is one long dependent chain of small kernels (7 per layer); each weight-streaming GEMM can only pull
// its weights while it runs, so HBM idles in every gap of the chain (kernel tails, griddepcontrol waits, the norm
// kernels, the epilogue -> next prologue latency): r01 measured 0.69 of the HBM peak with DRAM traffic == algorithmic
// bytes, i.e. pure latency.  The weights, however, depend on nothing.  While GEMM g of the step runs, a tiny kernel on a
// forked branch of the step's CUDA graph issues `cp.async.bulk.prefetch.tensor.2d.L2` for the HEAD of GEMM g+1's weight
// stream: for every CTA of that launch, the first `cap_kb` k-block tiles of exactly the work list (gemm_get_seg) the CTA
// will walk.  The L2 (50 MB on H100) is the staging buffer: HBM keeps streaming through the stalls of the chain and the next
// GEMM finds the start of its stream in L2.  The kernel only issues prefetches and exits (no spinning, no residency).
//
#pragma once
#include "gemm_wgmma.cuh"

namespace b200 {

struct alignas(64) PfGemm {      // one weight-streaming GEMM of the step, in launch order
  CUtensorMap tmap_a;            // the weight operand's tensor map (128 rows x 64 columns boxes)
  GemmSched sched;               // 6 ints
  int grid;                      // CTAs of the GEMM launch
  int pad[9];
};
static_assert(sizeof(PfGemm) % 64 == 0, "the tensor map must stay 64-byte aligned inside the kernel parameter");

constexpr int kPfMaxGemms = 1024;

// grid = G.grid CTAs of one warp: lane l of CTA c prefetches units l, l + 32, ... (< cap_kb) of GEMM CTA c's list
__global__ void __launch_bounds__(32) weight_prefetch_kernel(const __grid_constant__ PfGemm G, int cap_kb) {
  TraceScope _ts(11);
  const int c = blockIdx.x;
  int base = 0;                  // units of this CTA before the current segment
  GemmSeg sg;
  for (int idx = 0; base < cap_kb && gemm_get_seg(G.sched, idx, sg, G.sched.m_tiles, c, G.grid); ++idx) {
    const int n = sg.kb1 - sg.kb0;
    for (int u = (int)threadIdx.x; u < n && base + u < cap_kb; u += 32)
      tma_prefetch_l2_2d(&G.tmap_a, (sg.kb0 + u) * kGemmBlockK, sg.m_t * kGemmBlockM);
    base += n;
  }
}

}  // namespace b200
