// window_gather_kernel / window_blend_kernel, and their circular counterparts loop_gather_kernel / loop_blend_kernel: see longform.cuh for
// the plans and for why they live in a translation unit of their own.
#include "longform.cuh"

namespace ezb {

__global__ void __launch_bounds__(256) window_gather_kernel(const WindowPlan p, const float* __restrict__ latents, float* __restrict__ windows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.C * p.Lw) return;
  const int r = blockIdx.y, c = i / p.Lw, j = i - c * p.Lw;
  float v = 0.f;
  for (int b = 0; b < p.B; ++b) {
    const ClipWindows cw = clip_windows(p, b);
    if (r < cw.first || r >= cw.first + cw.count) continue;
    if (j < cw.len) v = latents[((size_t)b * p.C + c) * p.Nmax + window_start(p, cw, r - cw.first) + j];
    break;
  }
  windows[(((size_t)blockIdx.z * p.W + r) * p.C + c) * p.Lw + j] = v;
}

// v(f) = sum_k w_k(f - s_k) v_k(f - s_k) / sum_k w_k(f - s_k) over the windows covering frame f, in increasing k, in fp32.  The first term
// starts the sums, so one covering window of weight 1 gives its v bit for bit.
__global__ void __launch_bounds__(256) window_blend_kernel(const WindowPlan p, const float* __restrict__ windows, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.C * p.Nmax) return;
  const int b = blockIdx.y, c = i / p.Nmax, f = i - c * p.Nmax;
  const ClipWindows cw = clip_windows(p, b);
  if (f >= cw.n) return;
  const int H = p.Lw - p.overlap;
  // the evenly spaced windows 0 .. count - 2 covering f, then the last one (which starts at N - len) when it covers f
  const int k_lo = f >= p.Lw ? (f - p.Lw) / H + 1 : 0, k_hi = min(cw.count - 2, f / H);
  float acc = 0.f, ws = 0.f;
  bool first = true;
  auto add = [&](int k, int s) {
    const int row = cw.first + k;
    if (row < 0 || row >= p.W) return;
    const float w = window_weight(p, cw, k, f - s);
    const float v = windows[((size_t)row * p.C + c) * p.Lw + (f - s)];
    if (first) { acc = w * v; ws = w; first = false; }
    else { acc = fmaf(w, v, acc); ws += w; }
  };
  for (int k = k_lo; k <= k_hi; ++k) add(k, k * H);
  const int s_last = cw.n - cw.len;
  if (f >= s_last) add(cw.count - 1, s_last);
  out[((size_t)b * p.C + c) * p.Nmax + f] = __fdiv_rn(acc, ws);
}

// ---- seamless loops
struct LoopWindows { int first, count, n, len, r; };   // len = Lw_b; r: this step's offset, reduced to 0 .. n - 1

__device__ __forceinline__ LoopWindows loop_windows(const LoopPlan& p, int b) {
  const int32_t* e = p.plan + 3 * b;
  const int n = min(max(e[2], 1), p.Nmax);
  int r = p.offsets[b] % n;
  if (r < 0) r += n;
  return LoopWindows{e[0], max(e[1], 1), n, min(n, p.Lw), r};
}
// the unshifted start of window k: floor(k * n / count)
__device__ __forceinline__ int loop_base(const LoopWindows& lw, int k) { return (int)(((long long)k * lw.n) / lw.count); }

__global__ void __launch_bounds__(256) loop_gather_kernel(const LoopPlan p, const float* __restrict__ latents, float* __restrict__ windows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.C * p.Lw) return;
  const int r = blockIdx.y, c = i / p.Lw, j = i - c * p.Lw;
  float v = 0.f;
  for (int b = 0; b < p.B; ++b) {
    const LoopWindows lw = loop_windows(p, b);
    if (r < lw.first || r >= lw.first + lw.count) continue;
    if (j < lw.len) {
      int s = loop_base(lw, r - lw.first) + lw.r;   // < 2n
      if (s >= lw.n) s -= lw.n;
      int f = s + j;                                // < 2n: j < len <= n
      if (f >= lw.n) f -= lw.n;
      v = latents[((size_t)b * p.C + c) * p.Nmax + f];
    }
    break;
  }
  windows[(((size_t)blockIdx.z * p.W + r) * p.C + c) * p.Lw + j] = v;
}

// Frame f sits at g = (f - r) mod n on the unshifted circle.  K = ((g + 1) * count - 1) / n is the last window whose base is <= g; walking
// k = K + 1, ..., count - 1, 0, ..., K (cyclically) visits the windows in strictly decreasing local index j = (g - base_k) mod n, and those
// with j < len cover f.  The first covering term starts both sums, so one covering window of weight 1 gives its v bit for bit.
__global__ void __launch_bounds__(256) loop_blend_kernel(const LoopPlan p, const float* __restrict__ windows, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.C * p.Nmax) return;
  const int b = blockIdx.y, c = i / p.Nmax, f = i - c * p.Nmax;
  const LoopWindows lw = loop_windows(p, b);
  if (f >= lw.n) return;
  int g = f - lw.r;
  if (g < 0) g += lw.n;
  const int K = (int)(((long long)(g + 1) * lw.count - 1) / lw.n);
  const float o1 = (float)(p.overlap + 1);
  float acc = 0.f, ws = 0.f;
  bool first = true;
  for (int m = lw.count - 1; m >= 0; --m) {
    int k = K - m;
    if (k < 0) k += lw.count;
    int j = g - loop_base(lw, k);
    if (j < 0) j += lw.n;
    const int row = lw.first + k;
    if (j >= lw.len || row < 0 || row >= p.W) continue;
    float w = 1.f;
    if (lw.count > 1) w = fminf(w, fminf(__fdiv_rn((float)(j + 1), o1), __fdiv_rn((float)(lw.len - j), o1)));
    const float v = windows[((size_t)row * p.C + c) * p.Lw + j];
    if (first) { acc = w * v; ws = w; first = false; }
    else { acc = fmaf(w, v, acc); ws += w; }
  }
  out[((size_t)b * p.C + c) * p.Nmax + f] = __fdiv_rn(acc, ws);
}

cudaError_t loop_gather_launch(cudaStream_t st, const LoopPlan& p, const float* latents, float* windows, int copies) {
  loop_gather_kernel<<<dim3((unsigned)((p.C * p.Lw + 255) / 256), p.W, copies), 256, 0, st>>>(p, latents, windows);
  return cudaGetLastError();
}

cudaError_t loop_blend_launch(cudaStream_t st, const LoopPlan& p, const float* windows, float* out) {
  loop_blend_kernel<<<dim3((unsigned)((p.C * p.Nmax + 255) / 256), p.B), 256, 0, st>>>(p, windows, out);
  return cudaGetLastError();
}

cudaError_t window_gather_launch(cudaStream_t st, const WindowPlan& p, const float* latents, float* windows, int copies) {
  window_gather_kernel<<<dim3((unsigned)((p.C * p.Lw + 255) / 256), p.W, copies), 256, 0, st>>>(p, latents, windows);
  return cudaGetLastError();
}

cudaError_t window_blend_launch(cudaStream_t st, const WindowPlan& p, const float* windows, float* out) {
  window_blend_kernel<<<dim3((unsigned)((p.C * p.Nmax + 255) / 256), p.B), 256, 0, st>>>(p, windows, out);
  return cudaGetLastError();
}

}  // namespace ezb
