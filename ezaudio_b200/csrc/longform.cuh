// Windowed denoising of clips longer than the denoiser's trained window (MultiDiffusion): the gather of a long latent into overlapping
// window rows and the crossfade blend of the per-window predictions back into one long prediction.  The kernels are compiled in a
// translation unit of their own (longform.cu), as vae_noised.cu is: every kernel of ezb.cu's module keeps its code.
//
// Plan of clip b (N frames, window Lw, overlap O with 1 <= O <= Lw / 2, hop H = Lw - O): N <= Lw is one window [0, N); otherwise
// n = ceil((N - Lw) / H) + 1 windows of Lw frames start at k * H for k < n - 1 and the last at N - Lw.  The weight of window k at its local
// frame j is min(1, left, right), left = (j + 1) / (O + 1) when k > 0 (else 1), right = (Lw - j) / (O + 1) when k < n - 1 (else 1).
// ezaudio_b200.inference.window_plan is the same plan on the host.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ezb {

// plan: DEVICE int32 [B][3] = (first window row, window count, N) per clip, read when the kernels run; the windows of clip b are rows
// first .. first + count - 1 of the W window rows.  Windows are (rows, C, Lw), long latents (B, C, Nmax).
struct WindowPlan { const int32_t* plan; int B, C, Nmax, W, Lw, overlap; };

// clip b's windows as the plan table gives them (n clamped to 1 .. Nmax), window k's start and its weight at local frame j; shared by the
// linear kernels (longform.cu) and the timeline kernels (timeline.cu)
struct ClipWindows { int first, count, n, len; };   // len: frames of each window (Lw, or N when the clip is one short window)

__device__ __forceinline__ ClipWindows clip_windows(const WindowPlan& p, int b) {
  const int32_t* e = p.plan + 3 * b;
  const int n = min(max(e[2], 1), p.Nmax);
  return ClipWindows{e[0], e[1], n, min(n, p.Lw)};
}
__device__ __forceinline__ int window_start(const WindowPlan& p, const ClipWindows& cw, int k) {
  return k == cw.count - 1 ? cw.n - cw.len : k * (p.Lw - p.overlap);
}
// min(1, left, right), each ratio an IEEE division, as window_weights (inference.py) states it
__device__ __forceinline__ float window_weight(const WindowPlan& p, const ClipWindows& cw, int k, int j) {
  const float o1 = (float)(p.overlap + 1);
  float w = 1.f;
  if (k > 0) w = fminf(w, __fdiv_rn((float)(j + 1), o1));
  if (k < cw.count - 1) w = fminf(w, __fdiv_rn((float)(p.Lw - j), o1));
  return w;
}

// latents (B, C, Nmax) -> windows (copies * W, C, Lw): row r (and, when copies == 2, row W + r) holds its window's frames, zeros past them
cudaError_t window_gather_launch(cudaStream_t st, const WindowPlan& p, const float* latents, float* windows, int copies);
// windows (W, C, Lw) -> out (B, C, Nmax): the weighted mean of the windows covering each frame < N; frames >= N are not written
cudaError_t window_blend_launch(cudaStream_t st, const WindowPlan& p, const float* windows, float* out);

// Seamless loops: the same gather and blend on a circle, where frame N - 1 of loop b is followed by frame 0.  Loop b (N frames, table row
// (first, count, N) as above) has windows of Lw_b = min(Lw, N) frames: count == 1 when N <= Lw, else count = ceil(N / (Lw - O)).  At a
// step with offset r (offsets[b], DEVICE int32, read when the kernels run), window k starts at s_k = ((k * N) / count + r) mod N and reads
// frames (s_k + j) mod N, j < Lw_b.  Its weight at local frame j is 1 for a one-window loop, else min(1, (j + 1) / (O + 1),
// (Lw_b - j) / (O + 1)).  ezaudio_b200.inference.loop_plan is the same plan on the host.  These kernels are separate from the linear
// ones: a wrap there would put a branch in shared code and change their machine code.
struct LoopPlan { const int32_t* plan; const int32_t* offsets; int B, C, Nmax, W, Lw, overlap; };

// latents (B, C, Nmax) -> windows (copies * W, C, Lw): row r (and row W + r when copies == 2) holds its window's frames, zeros past Lw_b
cudaError_t loop_gather_launch(cudaStream_t st, const LoopPlan& p, const float* latents, float* windows, int copies);
// windows (W, C, Lw) -> out (B, C, Nmax): frame f < N gets the weighted mean of the windows covering it, summed in decreasing local index
// j (so the order depends only on where f sits in each window, and a common shift of every offset shifts the result exactly); frames
// >= N are not written
cudaError_t loop_blend_launch(cudaStream_t st, const LoopPlan& p, const float* windows, float* out);

}  // namespace ezb
