// Timelines of prompts over long clips: MultiDiffusion's region-based generation (Bar-Tal et al. 2023) on the time axis.  A clip is
// windowed as in longform.cuh, each window carries one conditioned DiT row per prompt segment active in it, all rows of a window share
// one unconditional row, and the blend weighs every row's prediction by its window's crossfade weight times its segment's weight.  The
// kernels live in a translation unit of their own (timeline.cu), as longform.cu's do: every kernel of ezb.cu's module keeps its code.
//
// Segment [s, e) of a clip of N frames with a transition of T >= 0 frames weighs frame f by
//   a(f) = min(1, (f - s + T + 1) / (T + 1), (e + T - f) / (T + 1)) on [s - T, e + T), 0 elsewhere,
// each ratio an IEEE fp32 division: 1 inside the segment, tapering over T frames on either side, so abutting segments crossfade over 2T
// frames centred on their boundary.  A segment is active in a window when [s - T, e + T) meets it.  ezaudio_b200.inference.segment_weights
// and timeline_plan are the same rules on the host.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "longform.cuh"

namespace ezb {

// win: the window plan of longform.cuh (its DEVICE [B][3] table, W windows).  rows: DEVICE int32 [R][4] = (window, s, e, T) per
// conditioned row, laid out clip by clip, window by window, then in timeline order.  spans: DEVICE int32 [B][2] = (first row, row count)
// per clip.  Every table is read when the kernels run.
struct TimelinePlan { WindowPlan win; const int32_t* rows; const int32_t* spans; int R; };

// latents (B, C, Nmax) -> windows (R [+ W], C, Lw): row r < R holds its window's frames, row R + k (when uncond) window k's; zeros past a
// window's length
cudaError_t timeline_gather_launch(cudaStream_t st, const TimelinePlan& p, const float* latents, float* windows, int uncond);
// model_out (R + W, C, Lw) -> guided (R, C, Lw): row r guided against row R + window(r) over its lens[r] frames, by cfg_update_sample
cudaError_t timeline_guide_launch(cudaStream_t st, const float* model_out, float* guided, const int32_t* rows, const int32_t* lens, int R, int W,
                                  int C, int Lw, float gs, float gr);
// windows (R, C, Lw) -> out (B, C, Nmax): frame f < N of clip b gets sum w a v / sum w a over its rows covering f with a(f) > 0, in row order
cudaError_t timeline_blend_launch(cudaStream_t st, const TimelinePlan& p, const float* windows, float* out);

}  // namespace ezb
