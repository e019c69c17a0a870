// A residual-stream GEMM and the LayerNorm that follows it as ONE launch.
//
// The LayerNorm launches of a DiT step each move a few MB of L2-resident data, so they are dominated by launch ramp, one thin wave and drain.  Their
// producers (out-proj, cross-proj, MLP-out, skip and patch-embed linears: blocks.py:128,141,151,156) are swap-AB GEMMs; when one fits a single
// resident wave (on 132 SMs: 9 x 14 tiles of 288 tokens at Be = 8, L = 500) the LayerNorm can run as a tail phase of the same grid behind a
// grid-wide barrier: no second launch, no ramp, the rows are still hot in L2.  The alternative is folding the LayerNorm algebraically into both neighbouring GEMMs (gemm.cuh FoldIn / FoldOut).
#pragma once
#include "elementwise.cuh"
#include "host.cuh"

namespace ezb {

template <int BN, class Epi>
__global__ void __launch_bounds__((GemmCfg<BN, Epi>::THREADS), 1)
gemm_ln_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmShape g, const typename Epi::Params ep,
               const LnParams lp, GridBarrier* bar) {
  extern __shared__ uint8_t smem_dyn[];
  gemm_body<BN, Epi, 1>(tmA, tmB, g, ep, smem_dyn);
  grid_barrier(bar);   // every tile of x is written and visible; the barrier is safe because the grid is at most one CTA per SM (all resident)
  ln_tail(lp);
}

inline int& opt_ln_tail() {
  static int v = [] { const char* e = getenv("EZB_LN_TAIL"); return e ? atoi(e) : 0; }();
  return v;
}

// gemm_swapped (host.cuh, same token width) + LayerNorm tail.  Falls back to two launches when the GEMM does not fit one resident wave.
template <int BN, class Epi>
int gemm_swapped_ln_at(Device& dev, cudaStream_t st, const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, int M_tokens, int N_features,
                       int K, const typename Epi::Params& ep, const LnParams& lp, GridBarrier* bar, bool* fused) {
  *fused = false;
  const int mt = (N_features + GEMM_BM - 1) / GEMM_BM, nt = (M_tokens + BN - 1) / BN, tiles = mt * nt;
  if (tiles > dev.num_sms || (K % 8) || (lda % 8) || (ldw % 8)) return gemm_swapped_at<BN, Epi>(dev, st, A, lda, W, ldw, M_tokens, N_features, K, ep);
  GemmShape g;
  memset(&g, 0, sizeof g);
  g.M = N_features; g.N = M_tokens;
  g.num_m_tiles = mt; g.num_n_tiles = nt;
  g.num_k_blocks = (K + GEMM_BK - 1) / GEMM_BK;
  const CUtensorMap *tA, *tB;
  EZB_TRY(dev.tmaps.get2d(W, (uint64_t)K, (uint64_t)N_features, (uint64_t)ldw, GEMM_BM, &tA));
  EZB_TRY(dev.tmaps.get2d(A, (uint64_t)K, (uint64_t)M_tokens, (uint64_t)lda, gemm_b_box(BN), &tB));
  auto kern = gemm_ln_kernel<BN, Epi>;
  constexpr int smem = GemmCfg<BN, Epi>::BYTES;
  constexpr int THREADS = GemmCfg<BN, Epi>::THREADS;
  static bool attr_set[16] = {};
  if (!attr_set[dev.id & 15]) {
    EZB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set[dev.id & 15] = true;
  }
  GemmProf& gp = gemm_prof();
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (gp.on) {
    if (gp.used + 2 > gp.ev.size()) {
      for (int i = 0; i < 2; ++i) { cudaEvent_t e; EZB_CUDA(cudaEventCreate(&e)); gp.ev.push_back(e); }
    }
    e0 = gp.ev[gp.used]; e1 = gp.ev[gp.used + 1];
    gp.used += 2;
    gp.flops.push_back(2.0 * (double)g.M * (double)g.N * (double)g.num_k_blocks * GEMM_BK);
    EZB_CUDA(cudaEventRecord(e0, st));
  }
  EZB_TRY(launch_k(kern, dim3(tiles), dim3(THREADS), smem, st, 1, *tA, *tB, g, ep, lp, bar));
  if (gp.on) EZB_CUDA(cudaEventRecord(e1, st));
  *fused = true;
  return EZB_OK;
}
template <template <int> class Epi>
int gemm_swapped_ln(Device& dev, cudaStream_t st, const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, int M_tokens, int N_features, int K,
                    const typename Epi<256>::Params& ep, const LnParams& lp, GridBarrier* bar, bool* fused) {
  if (swapped_bn(dev, M_tokens, N_features) == 288)
    return gemm_swapped_ln_at<288, Epi<288>>(dev, st, A, lda, W, ldw, M_tokens, N_features, K, ep, lp, bar, fused);
  return gemm_swapped_ln_at<256, Epi<256>>(dev, st, A, lda, W, ldw, M_tokens, N_features, K, ep, lp, bar, fused);
}

}  // namespace ezb
