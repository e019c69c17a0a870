// timeline_gather_kernel / timeline_guide_kernel / timeline_blend_kernel: see timeline.cuh for the plan, the tables and the weights.
#include <string.h>

#include "cfg_update.cuh"
#include "timeline.cuh"

namespace ezb {

namespace {

// a(f) of segment [s, e) with transition T (clamped to >= 0), 0 outside [s - T, e + T); in 64-bit so that no table entry overflows
__device__ __forceinline__ float segment_weight(int f, int s, int e, int T) {
  const long long t = max(T, 0), lo = (long long)f - s + t + 1, hi = (long long)e + t - f;
  if (lo <= 0 || hi <= 0) return 0.f;
  const float t1 = (float)(t + 1);
  return fminf(1.f, fminf(__fdiv_rn((float)lo, t1), __fdiv_rn((float)hi, t1)));
}

}  // namespace

__global__ void __launch_bounds__(256) timeline_gather_kernel(const TimelinePlan p, const float* __restrict__ latents, float* __restrict__ windows) {
  const WindowPlan& wp = p.win;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= wp.C * wp.Lw) return;
  const int y = blockIdx.y, c = i / wp.Lw, j = i - c * wp.Lw;
  const int k = y < p.R ? p.rows[4 * y] : y - p.R;   // the window of this row
  float v = 0.f;
  for (int b = 0; b < wp.B; ++b) {
    const ClipWindows cw = clip_windows(wp, b);
    if (k < cw.first || k >= cw.first + cw.count) continue;
    if (j < cw.len) v = latents[((size_t)b * wp.C + c) * wp.Nmax + window_start(wp, cw, k - cw.first) + j];
    break;
  }
  windows[((size_t)y * wp.C + c) * wp.Lw + j] = v;
}

// cfg_ddim_kernel's body with coefficients (1, 0, 0, 1, 0) and no noise, on conditioned row r and the uncond row R + window(r): it writes
// 0 * x0 + 1 * (1 * v + 0 * x) = v, the guided and rescaled v, into `guided` (which must hold finite values).  The uncond pointer is shifted
// so that the body's own row offset (r * C * Lw) lands on row R + window(r).
__global__ void __launch_bounds__(1024) timeline_guide_kernel(const float* __restrict__ model_out, float* __restrict__ guided,
                                                              const int32_t* __restrict__ rows, const int32_t* __restrict__ lens, int R, int W, int C,
                                                              int Lw, float gs, float gr) {
  const int r = blockIdx.x / CFG_CLUSTER;
  const int k = rows[4 * r];
  if (k < 0 || k >= W) return;   // every CTA of the cluster reads the same entry: the cluster leaves whole, before any cluster barrier
  const float* uncond = gs != 0.f ? model_out + (size_t)(R + k - r) * C * Lw : nullptr;
  cfg_update_sample<false>(model_out, uncond, guided, nullptr, lens, r, C, Lw, gs, gr, 1.f, 0.f, 0.f, 1.f, 0.f);
}

// The rows of clip b covering frame f with a(f) > 0, in row order: the first term starts both sums, so one covering row of weight 1 gives
// its v bit for bit, and a one-segment timeline (a = 1 on the whole clip, w * 1.0f == w) gives window_blend_kernel's bits.
__global__ void __launch_bounds__(256) timeline_blend_kernel(const TimelinePlan p, const float* __restrict__ windows, float* __restrict__ out) {
  const WindowPlan& wp = p.win;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= wp.C * wp.Nmax) return;
  const int b = blockIdx.y, c = i / wp.Nmax, f = i - c * wp.Nmax;
  const ClipWindows cw = clip_windows(wp, b);
  if (f >= cw.n) return;
  const int r0 = max(p.spans[2 * b], 0), r1 = min(p.spans[2 * b] + p.spans[2 * b + 1], p.R);
  float acc = 0.f, ws = 0.f;
  bool first = true;
  for (int r = r0; r < r1; ++r) {
    const int4 e = reinterpret_cast<const int4*>(p.rows)[r];   // (window, s, e, T)
    const int k = e.x - cw.first;
    if (k < 0 || k >= cw.count) continue;
    const int j = f - window_start(wp, cw, k);
    if (j < 0 || j >= cw.len) continue;
    const float a = segment_weight(f, e.y, e.z, e.w);
    if (!(a > 0.f)) continue;
    const float w = window_weight(wp, cw, k, j) * a;
    const float v = windows[((size_t)r * wp.C + c) * wp.Lw + j];
    if (first) { acc = w * v; ws = w; first = false; }
    else { acc = fmaf(w, v, acc); ws += w; }
  }
  out[((size_t)b * wp.C + c) * wp.Nmax + f] = __fdiv_rn(acc, ws);
}

cudaError_t timeline_gather_launch(cudaStream_t st, const TimelinePlan& p, const float* latents, float* windows, int uncond) {
  timeline_gather_kernel<<<dim3((unsigned)((p.win.C * p.win.Lw + 255) / 256), p.R + (uncond ? p.win.W : 0)), 256, 0, st>>>(p, latents, windows);
  return cudaGetLastError();
}

cudaError_t timeline_guide_launch(cudaStream_t st, const float* model_out, float* guided, const int32_t* rows, const int32_t* lens, int R, int W,
                                  int C, int Lw, float gs, float gr) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = dim3(R * CFG_CLUSTER);
  cfg.blockDim = dim3(1024);
  cfg.stream = st;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = CFG_CLUSTER; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, timeline_guide_kernel, model_out, guided, rows, lens, R, W, C, Lw, gs, gr);
}

cudaError_t timeline_blend_launch(cudaStream_t st, const TimelinePlan& p, const float* windows, float* out) {
  timeline_blend_kernel<<<dim3((unsigned)((p.win.C * p.win.Nmax + 255) / 256), p.win.B), 256, 0, st>>>(p, windows, out);
  return cudaGetLastError();
}

}  // namespace ezb
