// The fused classifier-free guidance + rescale + sampler update of one sample by a cluster of CFG_CLUSTER CTAs (elementwise.cuh describes
// the layout and the reduction above cfg_ddim_kernel).  It lives in a header of its own so that a second translation unit (timeline.cu)
// runs the same code, and so computes the same bits, on rows it pairs differently.
#pragma once
#include "common.cuh"

namespace ezb {

constexpr int CFG_CLUSTER = 8;
__device__ __forceinline__ double ld_dsmem_f64(const double* local, uint32_t rank) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(mapa_u32(smem_u32(local), rank)));
  return v;
}
// The update of one sample by its cluster (after pdl_wait), shared by the DDIM kernels (DPM = false: cfg_ddim_kernel with the scalars of the
// call, cfg_ddim_slots_kernel with those of the sample's slot) and the DPM-Solver++ kernels (DPM = true, elementwise.cuh), which differ only in
// the per-element update after guidance and rescale; timeline_guide_kernel (timeline.cu) runs the DDIM body on paired rows.  out_uncond null: no guidance; noise null: its coefficient (c4 / c6) is 0.
// DDIM: c0..c4 = {sqrt(a), sqrt(1-a), sqrt(a_prev), sqrt(1-a_prev-sigma^2), sigma}.  DPM: c0..c6 = ezb_dpm_slot.coef; history and order2 unused
// by DDIM.
template <bool DPM>
__device__ __forceinline__ void cfg_update_sample(const float* __restrict__ out_text, const float* __restrict__ out_uncond, float* __restrict__ latents,
                                                  const float* __restrict__ noise, const int32_t* __restrict__ lens, int sample, int C, int L, float gs,
                                                  float gr, float c0, float c1, float c2, float c3, float c4, float c5 = 0.f, float c6 = 0.f,
                                                  float* __restrict__ history = nullptr, bool order2 = false) {
  __shared__ double red[4][32];
  __shared__ double part[4];
  const uint32_t rank = cluster_ctarank();
  const size_t base = (size_t)sample * C * L;
  const int len = lens != nullptr ? min(max(lens[sample], 1), L) : L;
  const int n = C * len;
  const bool packed = len == L;   // element i lives at i
  auto at = [&](int i) { return packed ? i : (i / len) * L + i % len; };
  const int per = (((n + CFG_CLUSTER - 1) / CFG_CLUSTER) + 3) & ~3;   // slice of this CTA, multiple of 4 elements
  const int lo = (int)rank * per, hi = (lo + per < n) ? lo + per : n;
  const float* t = out_text + base;
  const float* u = out_uncond ? out_uncond + base : nullptr;
  float ratio = 1.f;
  const bool rescale = u && gr > 0.f;   // uniform over the grid
  if (rescale) {
    double st = 0, st2 = 0, sc = 0, sc2 = 0;
    for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      const int j = at(i);
      const float a = t[j], c = u[j] + gs * (a - u[j]);
      st += a; st2 += (double)a * a; sc += c; sc2 += (double)c * c;
    }
    double v[4] = {st, st2, sc, sc2};
    for (int k = 0; k < 4; ++k) {
      double x = v[k];
      for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
      if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = x;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
      double s = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[threadIdx.x][w];
      part[threadIdx.x] = s;
    }
    cluster_sync_all();   // partials of all CTAs of this sample are visible cluster-wide
    double s[4] = {0, 0, 0, 0};
    for (uint32_t r = 0; r < CFG_CLUSTER; ++r)
#pragma unroll
      for (int k = 0; k < 4; ++k) s[k] += ld_dsmem_f64(&part[k], r);
    const double var_t = (s[1] - s[0] * s[0] / n) / (n - 1), var_c = (s[3] - s[2] * s[2] / n) / (n - 1);
    ratio = (float)(sqrt(var_t) / sqrt(var_c));
    cluster_sync_all();   // nobody exits (releasing its shared memory) while a peer may still read its partials
  }
  float* x = latents + base;
  const float* z = noise ? noise + base : nullptr;
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const int j = at(i);
    float v = t[j];
    if (u) {
      v = u[j] + gs * (v - u[j]);
      if (gr > 0.f) v = gr * (v * ratio) + (1.f - gr) * v;
    }
    const float xi = x[j];
    if constexpr (DPM) {   // m0 = alpha_s x - sigma_s v;  x <- kx x + k0 m0 [+ k1 (r (m0 - m1))] [+ kz z];  history <- m0
      float* m = history + base;
      const float m0 = c0 * xi - c1 * v;
      float prev = c2 * xi + c3 * m0;
      if (order2) prev += c4 * (c5 * (m0 - m[j]));
      if (z) prev += c6 * z[j];
      m[j] = m0;
      x[j] = prev;
    } else {
      const float x0 = c0 * xi - c1 * v, eps = c0 * v + c1 * xi;
      float prev = c2 * x0 + c3 * eps;
      if (z) prev += c4 * z[j];
      x[j] = prev;
    }
  }
}

}  // namespace ezb
