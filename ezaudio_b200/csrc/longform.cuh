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

// latents (B, C, Nmax) -> windows (copies * W, C, Lw): row r (and, when copies == 2, row W + r) holds its window's frames, zeros past them
cudaError_t window_gather_launch(cudaStream_t st, const WindowPlan& p, const float* latents, float* windows, int copies);
// windows (W, C, Lw) -> out (B, C, Nmax): the weighted mean of the windows covering each frame < N; frames >= N are not written
cudaError_t window_blend_launch(cudaStream_t st, const WindowPlan& p, const float* windows, float* out);

}  // namespace ezb
