// Oobleck VAE decoder (stable_vae/models/autoencoders.py:149-190; DecoderBlock :82-113; ResidualUnit :38-61;
// SnakeBeta stable_vae/models/blocks.py:317-359; weight_norm stable_vae/models/nn/layers.py:9-14).
// Activations live channels-last ([B, T, C], bf16 tensor-core operands + an fp32 residual stream); every Conv1d /
// ConvTranspose1d is an implicit GEMM on the wgmma kernel (gemm.cuh, conv addressing) with bias, residual add and the
// NEXT layer's SnakeBeta fused into the epilogue.  Weight-norm is folded once at load time.
#pragma once
#include <map>
#include <string>
#include <vector>

#include "elementwise.cuh"
#include "host.cuh"
#include "vae_noised.cuh"

namespace ezb {

// ||v[row, :]|| for weight_norm (norm over all dims except 0)
__global__ void wn_norm_kernel(const float* __restrict__ v, int cols, float* __restrict__ norms) {
  __shared__ float red[32];
  const float* r = v + (size_t)blockIdx.x * cols;
  float s = 0.f;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) s += r[i] * r[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    s = warp_sum(s);
    if (threadIdx.x == 0) norms[blockIdx.x] = sqrtf(s);
  }
}
__device__ __forceinline__ void store_w_split(__nv_bfloat16* tap_base, int c, int C, int kmul, float val) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(val);
  tap_base[c] = hi;
  if (kmul == 3) {
    tap_base[C + c] = hi;
    tap_base[2 * C + c] = __float2bfloat16_rn(val - __bfloat162float(hi));
  }
}
// Conv1d: v [Cout, Cin, K], g [Cout] -> dst [Cout, K taps * cin_pad], per tap [hi(Cin) | hi | lo | 0-pad]
__global__ void pack_conv_w_kernel(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ norms, __nv_bfloat16* __restrict__ dst,
                                   int Cout, int Cin, int K, int cin_pad, int kmul) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)Cout * K * Cin) return;
  const int ci = i % Cin, tap = (i / Cin) % K, co = i / ((size_t)Cin * K);
  const float val = g[co] * v[((size_t)co * Cin + ci) * K + tap] / norms[co];
  store_w_split(dst + ((size_t)co * K + tap) * cin_pad, ci, Cin, kmul, val);
}
// ConvTranspose1d (kernel 2s, stride s, padding p): v [Cin, Cout, 2s], g [Cin] -> dst [s*Cout, 3 taps * cin_pad]
//   out[co, q*s + r] = sum_ci sum_delta x[ci, q + delta] * w[ci, co, r + p - delta*s],  delta = tap - 1
__global__ void pack_convT_w_kernel(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ norms, __nv_bfloat16* __restrict__ dst,
                                    int Cin, int Cout, int s, int pad, int cin_pad, int kmul) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)s * Cout * 3 * Cin) return;
  const int ci = i % Cin, tap = (i / Cin) % 3;
  const int n = i / ((size_t)Cin * 3), r = n / Cout, co = n - r * Cout;
  const int k = r + pad - (tap - 1) * s;
  const float val = (k >= 0 && k < 2 * s) ? g[ci] * v[((size_t)ci * Cout + co) * (2 * s) + k] / norms[ci] : 0.f;
  store_w_split(dst + ((size_t)n * 3 + tap) * cin_pad, ci, Cin, kmul, val);
}
__global__ void snake_prep_kernel(const float* __restrict__ alpha, const float* __restrict__ beta, float* __restrict__ a, float* __restrict__ binv, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < C) { a[i] = expf(alpha[i]); binv[i] = 1.0f / (expf(beta[i]) + 1e-9f); }
}
// Per-sample clip ends (padded batch, lens [B] device int32 in latent frames, read when the kernel runs and clamped to [1, L]): the
// length-aware kernels below treat everything at or past a clip's end as the zero padding a run of that clip alone sees, and write zeros
// there.
__device__ __forceinline__ int clip_frames(const int32_t* lens, int b, int L) { return min(max(lens[b], 1), L); }

// z (B, C, L) fp32 -> channels-last bf16 [B, L, kmul*C]
__global__ void latent_pack_kernel(const float* __restrict__ z, __nv_bfloat16* __restrict__ out, int C, int L, int kmul) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, l = l0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && l < L) ? z[((size_t)b * C + c) * L + l] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int l = l0 + i, c = c0 + threadIdx.x;
    if (l < L && c < C) store_act(out + ((size_t)b * L + l) * kmul * C, c, C, kmul, tile[threadIdx.x][i]);
  }
}
// latent_pack_kernel for a padded batch: frames at or past the clip's end are written as zeros and never read (they may hold NaN)
__global__ void latent_pack_lens_kernel(const float* __restrict__ z, __nv_bfloat16* __restrict__ out, int C, int L, int kmul, const int32_t* __restrict__ lens) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int Lv = clip_frames(lens, b, L);
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, l = l0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && l < Lv) ? z[((size_t)b * C + c) * L + l] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int l = l0 + i, c = c0 + threadIdx.x;
    if (l < L && c < C) store_act(out + ((size_t)b * L + l) * kmul * C, c, C, kmul, tile[threadIdx.x][i]);
  }
}
// last layer: Conv1d(C -> 1, k=7, pad 3, no bias) on the snake-activated channels-last tensor; w folded fp32 [7][C] (C = 128 shipped).
// HBM-bound (245 MB of bf16 activations per 4 clips).  One warp = 32 consecutive output samples: every input row (t0-3 .. t0+34) is read
// once with 8-byte loads (lane = 4 channels, a 256-byte row per warp), multiplied into the up-to-7 outputs it feeds (weights in
// registers), and the 32 per-lane partial sums are reduced with a 31-shuffle transpose-reduction so that lane i ends up with output i.
// Round 2: the rows are fetched in two batches of 19 unconditional loads (row index clamped, contribution zeroed by a select) -- the
// round-1 loop tested `0 <= t < T` around every load, which kept ptxas from hoisting any of them: each warp had ONE 256-byte request in
// flight.  Same accumulation order, bit-identical output.
template <int KMUL>
__global__ void __launch_bounds__(128, 3) wave_out_kernel(const __nv_bfloat16* __restrict__ act, const float* __restrict__ w, float* __restrict__ wav, int C, int T) {
  const int lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int b = blockIdx.y, t0 = chunk * 32;
  if (t0 >= T) return;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  for (int c0 = lane * 4; c0 < C; c0 += 128) {   // C = 128 in the shipped model: one pass
    const __nv_bfloat16* ab = act + (size_t)b * T * KMUL * C + c0;
    float wk[7][4];
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const float4 t = *reinterpret_cast<const float4*>(w + k * C + c0);
      wk[k][0] = t.x; wk[k][1] = t.y; wk[k][2] = t.z; wk[k][3] = t.w;
    }
    constexpr int NB = KMUL == 3 ? 10 : 19;   // rows per batch of loads
#pragma unroll
    for (int r0 = 0; r0 < 38; r0 += NB) {   // input sample t0 - 3 + rr, rr = 0..37, feeds outputs o = rr - k, k = 0..6 (tap k reads x[t + k - 3])
      uint2 u[NB], v[KMUL == 3 ? NB : 1];
#pragma unroll
      for (int i = 0; i < NB; ++i) {
        if (r0 + i >= 38) continue;
        const int t = t0 - 3 + r0 + i;
        const int tc = t < 0 ? 0 : (t >= T ? T - 1 : t);
        const __nv_bfloat16* row = ab + (size_t)tc * KMUL * C;
        u[i] = __ldg(reinterpret_cast<const uint2*>(row));
        if (KMUL == 3) v[i] = __ldg(reinterpret_cast<const uint2*>(row + C));   // split-bf16 operand: hi | lo | hi
      }
#pragma unroll
      for (int i = 0; i < NB; ++i) {
        if (r0 + i >= 38) continue;
        const int rr = r0 + i, t = t0 - 3 + rr;
        const bool ok = t >= 0 && t < T;
        float x[4];
        x[0] = __uint_as_float(u[i].x << 16); x[1] = __uint_as_float(u[i].x & 0xffff0000u);
        x[2] = __uint_as_float(u[i].y << 16); x[3] = __uint_as_float(u[i].y & 0xffff0000u);
        if (KMUL == 3) {
          x[0] += __uint_as_float(v[i].x << 16); x[1] += __uint_as_float(v[i].x & 0xffff0000u);
          x[2] += __uint_as_float(v[i].y << 16); x[3] += __uint_as_float(v[i].y & 0xffff0000u);
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) x[e] = ok ? x[e] : 0.f;
#pragma unroll
        for (int k = 0; k < 7; ++k) {
          const int o = rr - k;
          if (o >= 0 && o < 32) acc[o] = fmaf(wk[k][0], x[0], fmaf(wk[k][1], x[1], fmaf(wk[k][2], x[2], fmaf(wk[k][3], x[3], acc[o]))));
        }
      }
      asm volatile("" ::: "memory");   // keep the next batch's loads behind this batch's arithmetic (register budget)
    }
  }
  // transpose-reduction: after the five steps lane i holds the sum over lanes of acc[i]
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int j = 0; j < off; ++j) {
      const float send = up ? acc[j] : acc[j + off];
      const float keep = up ? acc[j + off] : acc[j];
      acc[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  if (t0 + lane < T) wav[(size_t)b * T + t0 + lane] = acc[0];
}
// Padded batch: wave_out_kernel runs as it is -- the activated rows at or past a clip's end are zeros already (EpiLinearLens), which is
// the zero padding the clip alone sees, so the samples before the end need nothing new -- and this kernel then zeroes the samples of wav
// [B, T] at or past it (hop samples per latent frame; the few just past the end hold the conv's reach into the clip).
__global__ void wave_tail_zero_kernel(float* __restrict__ wav, int T, const int32_t* __restrict__ lens, int hop) {
  const int b = blockIdx.y;
  const int t = clip_frames(lens, b, T / hop) * hop + blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T) wav[(size_t)b * T + t] = 0.f;
}
__global__ void fold_wave_w_kernel(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ norms, float* __restrict__ w, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // v [1, C, 7] -> w [7][C]
  if (i < 7 * C) { const int k = i / C, c = i - k * C; w[i] = g[0] * v[c * 7 + k] / norms[0]; }
}

// encoder stem: Conv1d(1 -> C0, k=7, pad 3) on the raw waveform (autoencoders.py:133) -> channels-last fp32 residual stream
// + bf16 SnakeBeta(next) operand.  w folded fp32 [7][C0].
// LENS: samples at or past the clip's end (hop per latent frame) read as zero, whatever the buffer holds there, and rows at or past it get
// a zero activation (they would be snake(bias)); raw is not written there.
template <bool LENS>
__device__ __forceinline__ void enc_conv_in_body(const float* __restrict__ audio, const float* __restrict__ w, const float* __restrict__ bias,
                                                 const float* __restrict__ sa, const float* __restrict__ sb, float* __restrict__ raw,
                                                 __nv_bfloat16* __restrict__ act, int C, int T, int kmul, const int32_t* lens, int hop) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= (size_t)T * C) return;
  const int t = i / C, c = i - (size_t)t * C;
  const int end = LENS ? clip_frames(lens, b, T / hop) * hop : T;
  if (LENS && t >= end) {
    store_act(act + ((size_t)b * T + t) * kmul * C, c, C, kmul, 0.f);
    return;
  }
  const float* a = audio + (size_t)b * T;
  float v = bias[c];
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    const int tt = t + k - 3;
    if (tt >= 0 && tt < end) v = fmaf(w[k * C + c], a[tt], v);
  }
  raw[((size_t)b * T + t) * C + c] = v;
  const float sn = sinf(v * sa[c]);
  store_act(act + ((size_t)b * T + t) * kmul * C, c, C, kmul, v + sb[c] * sn * sn);
}
__global__ void enc_conv_in_kernel(const float* __restrict__ audio, const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ sa,
                                   const float* __restrict__ sb, float* __restrict__ raw, __nv_bfloat16* __restrict__ act, int C, int T, int kmul) {
  enc_conv_in_body<false>(audio, w, bias, sa, sb, raw, act, C, T, kmul, nullptr, 1);
}
__global__ void enc_conv_in_lens_kernel(const float* __restrict__ audio, const float* __restrict__ w, const float* __restrict__ bias,
                                        const float* __restrict__ sa, const float* __restrict__ sb, float* __restrict__ raw, __nv_bfloat16* __restrict__ act,
                                        int C, int T, int kmul, const int32_t* __restrict__ lens, int hop) {
  enc_conv_in_body<true>(audio, w, bias, sa, sb, raw, act, C, T, kmul, lens, hop);
}
__global__ void fold_conv_in_w_kernel(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ norms, float* __restrict__ w, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // v [C, 1, 7] -> w [7][C]
  if (i < 7 * C) { const int k = i / C, c = i - k * C; w[i] = g[c] * v[c * 7 + k] / norms[c]; }
}
// VAEBottleneck.encode (bottleneck.py:66-70,77-87): enc [B*L, 2*Cz] channels-last (mean | scale) -> z (B, Cz, L)
// LENS: z frames at or past the clip's end are zeros (enc rows there are not read: the encoder's last conv leaves them unwritten)
template <bool LENS>
__device__ __forceinline__ void vae_sample_body(const float* __restrict__ enc, const float* __restrict__ noise, float* __restrict__ z, int Cz, int L,
                                                const int32_t* lens) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= (size_t)Cz * L) return;
  const int c = i / L, l = i - (size_t)c * L;
  if (LENS && l >= clip_frames(lens, b, L)) { z[((size_t)b * Cz + c) * L + l] = 0.f; return; }
  const float* row = enc + ((size_t)b * L + l) * 2 * Cz;
  const float mean = row[c], sc = row[Cz + c];
  const float sp = sc > 20.f ? sc : log1pf(expf(sc));  // F.softplus (threshold 20)
  const float nz = noise ? noise[((size_t)b * Cz + c) * L + l] : 0.f;
  z[((size_t)b * Cz + c) * L + l] = nz * (sp + 1e-4f) + mean;
}
__global__ void vae_sample_kernel(const float* __restrict__ enc, const float* __restrict__ noise, float* __restrict__ z, int Cz, int L) {
  vae_sample_body<false>(enc, noise, z, Cz, L, nullptr);
}
__global__ void vae_sample_lens_kernel(const float* __restrict__ enc, const float* __restrict__ noise, float* __restrict__ z, int Cz, int L,
                                       const int32_t* __restrict__ lens) {
  vae_sample_body<true>(enc, noise, z, Cz, L, lens);
}
struct VaeConv {  // one packed conv / conv-transpose
  __nv_bfloat16* w = nullptr;
  const float* bias = nullptr;
  int cin = 0, cout = 0, taps = 0, center = 0, dil = 1, cin_pad = 0, N = 0, stride = 0;
  size_t w_elems() const { return (size_t)N * taps * cin_pad; }
};
struct VaeSnake { float *a = nullptr, *binv = nullptr; };

// Geometry of the three conv shapes (w and bias left to the caller).  Conv1d(cin -> cout, K taps, dilation, padding dil * (K - 1) / 2):
inline VaeConv vae_conv_geom(int cin, int cout, int K, int dil, int kmul) {
  VaeConv c;
  c.cin = cin; c.cout = cout; c.N = cout; c.taps = K; c.center = (K - 1) / 2; c.dil = dil;
  c.cin_pad = (kmul * cin + 63) / 64 * 64;
  return c;
}
// ConvTranspose1d(cin -> cout, k = 2s, stride s, padding s / 2) (DecoderBlock): three taps over the input, N = s * cout (one column block per phase)
inline VaeConv vae_convT_geom(int cin, int cout, int s, int kmul) {
  VaeConv c = vae_conv_geom(cin, cout, 3, 1, kmul);
  c.N = s * cout; c.stride = s;
  return c;
}
// strided Conv1d(cin -> cout, k = 2s, stride s, pad ceil(s/2)) (EncoderBlock, autoencoders.py:76-77): same packing as a conv
inline VaeConv vae_conv_strided_geom(int cin, int cout, int s, int kmul) {
  VaeConv c = vae_conv_geom(cin, cout, 2 * s, 1, kmul);
  c.stride = s;
  c.center = (s + 1) / 2;  // padding
  return c;
}

// Weight-norm folding and packing from the reference layouts into caller-provided buffers.  `norms` is scratch of one float per dim-0 row.
// Conv1d / strided conv: v [cout, cin, taps], g [cout] -> c.w
inline int vae_pack_conv_w(cudaStream_t st, const VaeConv& c, const float* v, const float* g, float* norms, int kmul) {
  ++launch_counter();
  wn_norm_kernel<<<c.cout, 256, 0, st>>>(v, c.cin * c.taps, norms);
  const size_t n = (size_t)c.cout * c.taps * c.cin;
  ++launch_counter();
  pack_conv_w_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(v, g, norms, c.w, c.cout, c.cin, c.taps, c.cin_pad, kmul);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// ConvTranspose1d: v [cin, cout, 2s], g [cin] -> c.w
inline int vae_pack_convT_w(cudaStream_t st, const VaeConv& c, const float* v, const float* g, float* norms, int kmul) {
  const int s = c.stride;
  ++launch_counter();
  wn_norm_kernel<<<c.cin, 256, 0, st>>>(v, c.cout * 2 * s, norms);
  const size_t n = (size_t)c.N * 3 * c.cin;
  ++launch_counter();
  pack_convT_w_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(v, g, norms, c.w, c.cin, c.cout, s, (s + 1) / 2, c.cin_pad, kmul);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// SnakeBeta(alpha, beta) -> the epilogue's exp(alpha) and 1 / (exp(beta) + 1e-9)
inline int vae_snake_prep(cudaStream_t st, const float* alpha, const float* beta, const VaeSnake& s, int C) {
  ++launch_counter();
  snake_prep_kernel<<<(C + 255) / 256, 256, 0, st>>>(alpha, beta, s.a, s.binv, C);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// the decoder's last conv, v [1, C, 7], g [1] -> w [7][C]
inline int vae_fold_wave_w(cudaStream_t st, const float* v, const float* g, float* norms, float* w, int C) {
  ++launch_counter();
  wn_norm_kernel<<<1, 256, 0, st>>>(v, C * 7, norms);
  ++launch_counter();
  fold_wave_w_kernel<<<(7 * C + 255) / 256, 256, 0, st>>>(v, g, norms, w, C);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// the encoder stem, v [C, 1, 7], g [C] -> w [7][C]
inline int vae_fold_conv_in_w(cudaStream_t st, const float* v, const float* g, float* norms, float* w, int C) {
  ++launch_counter();
  wn_norm_kernel<<<C, 256, 0, st>>>(v, 7, norms);
  ++launch_counter();
  fold_conv_in_w_kernel<<<(7 * C + 255) / 256, 256, 0, st>>>(v, g, norms, w, C);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}

// One implicit-GEMM conv: A [B, T_in, kmul*cin] -> raw_out fp32 [B*T, N] (pre-activation, + resid_in when given) and act_out bf16
// [B, T * phases, kmul*cout] (SnakeBeta(snake) of it, [hi | lo | hi] in bf16x3).  T: input rows, except for a strided conv (output rows,
// the input has T * stride).  resid_in may alias raw_out.
// lens (device [B], or null): clips of lens[b] <= max_len latent frames, frame_rows = T / max_len GEMM rows each, in a batch padded to T
// rows: the EpiLinearLens kernel, which zeroes act_out past each clip's end and leaves raw_out unwritten there.
inline int vae_conv(Device& dev, cudaStream_t st, const VaeConv& c, int kmul, const __nv_bfloat16* A, int B, int T, const float* resid_in,
                    float* raw_out, __nv_bfloat16* act_out, const VaeSnake* snake, const int32_t* lens = nullptr, int max_len = 0) {
  EpiLinearParams e;
  memset(&e, 0, sizeof e);
  e.bias = c.bias;
  e.bias_mod = c.cout;
  e.resid = resid_in; e.ldr = c.N;
  e.out_f32 = raw_out; e.ld32 = c.N;
  e.out_bf16 = act_out;
  const int phases = c.N / c.cout;
  e.ld16 = phases * kmul * c.cout;
  e.split_stride = kmul == 3 ? c.cout : 0;
  e.phase_cols = phases > 1 ? c.cout : 0;
  e.phase_ld16 = kmul * c.cout;
  if (snake) { e.act = ACT_SNAKE; e.act_a = snake->a; e.act_b = snake->binv; }
  ConvAddr ca;
  ca.taps = c.taps; ca.center = c.center; ca.dilation = c.dil; ca.cin_pad = c.cin_pad; ca.T = T; ca.B = B;
  if (c.stride > 1 && c.N == c.cout) { ca.stride = c.stride; ca.pad = c.center; }  // strided conv (T = output length); conv-transpose has N = s*cout
  const int ld = c.taps * c.cin_pad;
  if (lens != nullptr) {
    if (max_len < 1 || T % max_len) return fail(EZB_ERR_SHAPE, "vae_conv: %d rows per clip are not a multiple of the %d padded frames", T, max_len);
    const EpiLinearLensParams el{e, lens, T, max_len, T / max_len};
    return gemm<128, EpiLinearLens<128>>(dev, st, A, kmul * c.cin, c.w, ld, B * T, c.N, kmul * c.cin, el, &ca);
  }
  return gemm<128, EpiLinear<128>>(dev, st, A, kmul * c.cin, c.w, ld, B * T, c.N, kmul * c.cin, e, &ca);
}

// z (B, C, L) fp32 -> act [B, L, kmul*C]
inline int vae_latent_pack(cudaStream_t st, const float* z, __nv_bfloat16* act, int B, int C, int L, int kmul, const int32_t* lens = nullptr) {
  dim3 grid((L + 31) / 32, (C + 31) / 32, B), blk(32, 8);
  ++launch_counter();
  if (lens != nullptr) latent_pack_lens_kernel<<<grid, blk, 0, st>>>(z, act, C, L, kmul, lens);
  else latent_pack_kernel<<<grid, blk, 0, st>>>(z, act, C, L, kmul);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// act [B, T, kmul*C] -> wav [B, T], w folded [7][C]
// lens (device [B] latent frames of `hop` samples, or null): samples at or past a clip's end are zeroed by a second launch
inline int vae_wave_out(cudaStream_t st, const __nv_bfloat16* act, const float* w, float* wav, int B, int C, int T, int kmul,
                        const int32_t* lens = nullptr, int hop = 1) {
  if (C % 4) return fail(EZB_ERR_UNSUPPORTED, "wave_out: %d channels in the last stage (multiple of 4 expected)", C);
  dim3 g2((T + 127) / 128, B);
  ++launch_counter();
  if (kmul == 3) wave_out_kernel<3><<<g2, 128, 0, st>>>(act, w, wav, C, T);
  else wave_out_kernel<1><<<g2, 128, 0, st>>>(act, w, wav, C, T);
  if (lens != nullptr) {
    ++launch_counter();
    wave_tail_zero_kernel<<<dim3((T - hop + 255) / 256 + 1, B), 256, 0, st>>>(wav, T, lens, hop);
  }
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// audio [B, T] -> raw [B, T, C] fp32 and act = SnakeBeta(snake) [B, T, kmul*C], w folded [7][C]
inline int vae_enc_conv_in(cudaStream_t st, const float* audio, const float* w, const float* bias, const VaeSnake& snake, float* raw,
                           __nv_bfloat16* act, int B, int C, int T, int kmul, const int32_t* lens = nullptr, int hop = 1) {
  dim3 grid((unsigned)(((size_t)T * C + 255) / 256), B);
  ++launch_counter();
  if (lens != nullptr) enc_conv_in_lens_kernel<<<grid, 256, 0, st>>>(audio, w, bias, snake.a, snake.binv, raw, act, C, T, kmul, lens, hop);
  else enc_conv_in_kernel<<<grid, 256, 0, st>>>(audio, w, bias, snake.a, snake.binv, raw, act, C, T, kmul);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// enc [B*L, 2*Cz] (mean | scale) -> z (B, Cz, L)
inline int vae_sample(cudaStream_t st, const float* enc, const float* noise, float* z, int B, int Cz, int L, const int32_t* lens = nullptr) {
  dim3 g2((unsigned)(((size_t)Cz * L + 255) / 256), B);
  ++launch_counter();
  if (lens != nullptr) vae_sample_lens_kernel<<<g2, 256, 0, st>>>(enc, noise, z, Cz, L, lens);
  else vae_sample_kernel<<<g2, 256, 0, st>>>(enc, noise, z, Cz, L);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// enc [B*L, 2*Cz] (mean | scale), eps (B, Cz, L), ab [B][2] -> x_t (B, Cz, L): vae_sample_noised_kernel (vae_noised.cu)
inline int vae_sample_noised(cudaStream_t st, const float* enc, const float* noise, const VaeNoised& n, float* x_t, int B, int Cz, int L,
                             const int32_t* lens) {
  ++launch_counter();
  EZB_CUDA(vae_sample_noised_launch(st, enc, noise, n, x_t, B, Cz, L, lens));
  return EZB_OK;
}

struct Vae {
  ezb_vae_desc d;
  Device* dev = nullptr;
  int kmul = 1, nst = 0;
  std::vector<void*> allocs;
  std::map<std::string, std::pair<float*, std::vector<int64_t>>> raw;  // staged fp32 copies until finalize
  std::vector<std::string> expected;
  bool finalized = false;
  VaeConv conv_in;
  std::vector<VaeConv> up;                 // per stage conv-transpose
  std::vector<VaeSnake> up_snake;          // per stage input snake
  std::vector<VaeConv> res7, res1;         // [stage*3 + unit]
  std::vector<VaeSnake> res_s0, res_s2;
  VaeSnake out_snake;
  float* out_w = nullptr;                  // [7][C0]
  std::vector<int> cin_s, cout_s, stride_s;
  __nv_bfloat16 *actA = nullptr, *actB = nullptr;
  float* resid = nullptr;
  size_t elems_per_clip = 0;
  // ---- encoder (OobleckEncoder, autoencoders.py:115-146), present when desc.with_encoder
  float *e_in_w = nullptr, *e_in_b = nullptr;                 // stem conv folded [7][C0], bias
  std::vector<VaeConv> e_res7, e_res1, e_down;              // [stage*3 + unit], per stage strided conv
  std::vector<VaeSnake> e_res_s0, e_res_s2, e_down_snake;
  VaeSnake e_out_snake;
  VaeConv e_out;
  std::vector<int> e_cin, e_cout, e_stride;

  ~Vae() { for (void* p : allocs) cudaFree(p); }
  template <typename T>
  int alloc(T** out, size_t count) {
    void* p = nullptr;
    const size_t bytes = ((count * sizeof(T)) + 255) & ~size_t(255);
    EZB_CUDA(cudaMalloc(&p, bytes));
    EZB_CUDA(cudaMemset(p, 0, bytes));
    allocs.push_back(p);
    *out = reinterpret_cast<T*>(p);
    return EZB_OK;
  }
  void expect_wn(const std::string& k, bool bias) { expected.push_back(k + ".weight_g"); expected.push_back(k + ".weight_v"); if (bias) expected.push_back(k + ".bias"); }
  void expect_snake(const std::string& k) { expected.push_back(k + ".alpha"); expected.push_back(k + ".beta"); }

  int init(const ezb_vae_desc& desc, Device* device) {
    d = desc; dev = device;
    kmul = d.precision == 1 ? 3 : 1;
    nst = d.n_stages;
    if (nst < 1 || nst > 8 || d.out_channels != 1 || d.latent_dim % 32 || d.channels % 8) return fail(EZB_ERR_UNSUPPORTED, "vae config");
    // ConvTranspose1d(k = 2s, stride s, padding ceil(s/2)) makes T*s - 1 frames for odd s; the decoder is built for T*s
    for (int i = 0; i < nst; ++i)
      if (d.strides[i] < 2 || d.strides[i] % 2)
        return fail(EZB_ERR_UNSUPPORTED, "vae decoder stage %d: stride %d (an even stride >= 2 expected)", nst - i, d.strides[i]);
    std::vector<int> mults(1, 1);
    for (int i = 0; i < nst; ++i) mults.push_back(d.c_mults[i]);
    for (int i = nst; i >= 1; --i) { cin_s.push_back(mults[i] * d.channels); cout_s.push_back(mults[i - 1] * d.channels); stride_s.push_back(d.strides[i - 1]); }
    const std::string p = "decoder.layers.";
    expect_wn(p + "0", true);
    for (int j = 0; j < nst; ++j) {
      const std::string q = p + std::to_string(j + 1) + ".layers.";
      expect_snake(q + "0"); expect_wn(q + "1", true);
      for (int u = 0; u < 3; ++u) {
        const std::string ru = q + std::to_string(u + 2) + ".layers.";
        expect_snake(ru + "0"); expect_wn(ru + "1", true); expect_snake(ru + "2"); expect_wn(ru + "3", true);
      }
    }
    expect_snake(p + std::to_string(nst + 1));
    expect_wn(p + std::to_string(nst + 2), false);
    if (d.with_encoder) {
      if (d.in_channels != 1 || d.enc_latent_dim != 2 * d.latent_dim) return fail(EZB_ERR_UNSUPPORTED, "vae encoder config");
      const std::string e = "encoder.layers.";
      expect_wn(e + "0", true);
      for (int i = 0; i < nst; ++i) {
        e_cin.push_back(mults[i] * d.channels); e_cout.push_back(mults[i + 1] * d.channels); e_stride.push_back(d.strides[i]);
        const std::string q = e + std::to_string(i + 1) + ".layers.";
        for (int u = 0; u < 3; ++u) {
          const std::string ru = q + std::to_string(u) + ".layers.";
          expect_snake(ru + "0"); expect_wn(ru + "1", true); expect_snake(ru + "2"); expect_wn(ru + "3", true);
        }
        expect_snake(q + "3"); expect_wn(q + "4", true);
      }
      expect_snake(e + std::to_string(nst + 1));
      expect_wn(e + std::to_string(nst + 2), true);
    }
    // workspace: largest channels-last activation per clip
    size_t T = d.max_latent_len, mx = (size_t)T * cin_s[0];
    for (int j = 0; j < nst; ++j) { T *= stride_s[j]; mx = std::max(mx, T * (size_t)cout_s[j]); }
    mx = std::max(mx, (size_t)d.max_latent_len * d.latent_dim);
    elems_per_clip = mx;
    EZB_TRY(alloc(&actA, mx * d.max_batch * kmul)); EZB_TRY(alloc(&actB, mx * d.max_batch * kmul));
    EZB_TRY(alloc(&resid, mx * d.max_batch));
    return EZB_OK;
  }
  int load_weight(const char* key, const float* data, const int64_t* shape, int ndim, cudaStream_t st) {
    std::string k(key);
    if (std::find(expected.begin(), expected.end(), k) == expected.end()) return fail(EZB_ERR_WEIGHT, "unexpected VAE key '%s'", key);
    size_t n = 1;
    std::vector<int64_t> shp(shape, shape + ndim);
    for (auto v : shp) n *= v;
    float* p = nullptr;
    EZB_TRY(alloc(&p, n));
    EZB_CUDA(cudaMemcpyAsync(p, data, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    raw[k] = std::make_pair(p, shp);
    return EZB_OK;
  }
  int need(const std::string& k, std::vector<int64_t> shape, float** out) {
    auto it = raw.find(k);
    if (it == raw.end()) return fail(EZB_ERR_WEIGHT, "missing VAE key '%s'", k.c_str());
    if (it->second.second != shape) return fail(EZB_ERR_WEIGHT, "shape mismatch for VAE key '%s'", k.c_str());
    *out = it->second.first;
    return EZB_OK;
  }
  // conv geometry c (from vae_*_geom) + the checkpoint entries of key k -> packed weights of this handle
  int pack_conv(const std::string& k, bool bias, VaeConv* c, cudaStream_t st) {
    float *g, *v, *b = nullptr, *norms;
    EZB_TRY(need(k + ".weight_g", {c->cout, 1, 1}, &g));
    EZB_TRY(need(k + ".weight_v", {c->cout, c->cin, c->taps}, &v));
    if (bias) EZB_TRY(need(k + ".bias", {c->cout}, &b));
    EZB_TRY(alloc(&norms, (size_t)c->cout));
    c->bias = b;
    EZB_TRY(alloc(&c->w, c->w_elems()));
    return vae_pack_conv_w(st, *c, v, g, norms, kmul);
  }
  int pack_convT(const std::string& k, VaeConv* c, cudaStream_t st) {
    float *g, *v, *b, *norms;
    EZB_TRY(need(k + ".weight_g", {c->cin, 1, 1}, &g));
    EZB_TRY(need(k + ".weight_v", {c->cin, c->cout, 2 * c->stride}, &v));
    EZB_TRY(need(k + ".bias", {c->cout}, &b));
    EZB_TRY(alloc(&norms, (size_t)c->cin));
    c->bias = b;
    EZB_TRY(alloc(&c->w, c->w_elems()));
    return vae_pack_convT_w(st, *c, v, g, norms, kmul);
  }
  int finalize_encoder(cudaStream_t st) {
    const std::string e = "encoder.layers.";
    const int C0 = e_cin[0];
    {
      float *g, *v, *b, *norms;
      EZB_TRY(need(e + "0.weight_g", {C0, 1, 1}, &g)); EZB_TRY(need(e + "0.weight_v", {C0, 1, 7}, &v)); EZB_TRY(need(e + "0.bias", {C0}, &b));
      EZB_TRY(alloc(&norms, (size_t)C0)); EZB_TRY(alloc(&e_in_w, (size_t)7 * C0));
      EZB_TRY(vae_fold_conv_in_w(st, v, g, norms, e_in_w, C0));
      e_in_b = b;
    }
    e_res7.resize(3 * nst); e_res1.resize(3 * nst); e_res_s0.resize(3 * nst); e_res_s2.resize(3 * nst); e_down.resize(nst); e_down_snake.resize(nst);
    const int dils[3] = {1, 3, 9};
    for (int j = 0; j < nst; ++j) {
      const std::string q = e + std::to_string(j + 1) + ".layers.";
      for (int u = 0; u < 3; ++u) {
        const std::string ru = q + std::to_string(u) + ".layers.";
        EZB_TRY(prep_snake(ru + "0", e_cin[j], &e_res_s0[3 * j + u], st));
        e_res7[3 * j + u] = vae_conv_geom(e_cin[j], e_cin[j], 7, dils[u], kmul);
        EZB_TRY(pack_conv(ru + "1", true, &e_res7[3 * j + u], st));
        EZB_TRY(prep_snake(ru + "2", e_cin[j], &e_res_s2[3 * j + u], st));
        e_res1[3 * j + u] = vae_conv_geom(e_cin[j], e_cin[j], 1, 1, kmul);
        EZB_TRY(pack_conv(ru + "3", true, &e_res1[3 * j + u], st));
      }
      EZB_TRY(prep_snake(q + "3", e_cin[j], &e_down_snake[j], st));
      e_down[j] = vae_conv_strided_geom(e_cin[j], e_cout[j], e_stride[j], kmul);
      EZB_TRY(pack_conv(q + "4", true, &e_down[j], st));
    }
    EZB_TRY(prep_snake(e + std::to_string(nst + 1), e_cout[nst - 1], &e_out_snake, st));
    e_out = vae_conv_geom(e_cout[nst - 1], d.enc_latent_dim, 3, 1, kmul);
    EZB_TRY(pack_conv(e + std::to_string(nst + 2), true, &e_out, st));
    return EZB_OK;
  }
  int prep_snake(const std::string& k, int C, VaeSnake* s, cudaStream_t st) {
    float *al, *be;
    EZB_TRY(need(k + ".alpha", {C}, &al)); EZB_TRY(need(k + ".beta", {C}, &be));
    EZB_TRY(alloc(&s->a, (size_t)C)); EZB_TRY(alloc(&s->binv, (size_t)C));
    return vae_snake_prep(st, al, be, *s, C);
  }
  int finalize(cudaStream_t st) {
    const std::string p = "decoder.layers.";
    conv_in = vae_conv_geom(d.latent_dim, cin_s[0], 7, 1, kmul);
    EZB_TRY(pack_conv(p + "0", true, &conv_in, st));
    up.resize(nst); up_snake.resize(nst); res7.resize(3 * nst); res1.resize(3 * nst); res_s0.resize(3 * nst); res_s2.resize(3 * nst);
    const int dils[3] = {1, 3, 9};
    for (int j = 0; j < nst; ++j) {
      const std::string q = p + std::to_string(j + 1) + ".layers.";
      EZB_TRY(prep_snake(q + "0", cin_s[j], &up_snake[j], st));
      up[j] = vae_convT_geom(cin_s[j], cout_s[j], stride_s[j], kmul);
      EZB_TRY(pack_convT(q + "1", &up[j], st));
      for (int u = 0; u < 3; ++u) {
        const std::string ru = q + std::to_string(u + 2) + ".layers.";
        EZB_TRY(prep_snake(ru + "0", cout_s[j], &res_s0[3 * j + u], st));
        res7[3 * j + u] = vae_conv_geom(cout_s[j], cout_s[j], 7, dils[u], kmul);
        EZB_TRY(pack_conv(ru + "1", true, &res7[3 * j + u], st));
        EZB_TRY(prep_snake(ru + "2", cout_s[j], &res_s2[3 * j + u], st));
        res1[3 * j + u] = vae_conv_geom(cout_s[j], cout_s[j], 1, 1, kmul);
        EZB_TRY(pack_conv(ru + "3", true, &res1[3 * j + u], st));
      }
    }
    const int C0 = cout_s[nst - 1];
    EZB_TRY(prep_snake(p + std::to_string(nst + 1), C0, &out_snake, st));
    {
      float *g, *v, *norms;
      const std::string k = p + std::to_string(nst + 2);
      EZB_TRY(need(k + ".weight_g", {1, 1, 1}, &g)); EZB_TRY(need(k + ".weight_v", {1, C0, 7}, &v));
      EZB_TRY(alloc(&norms, (size_t)1)); EZB_TRY(alloc(&out_w, (size_t)7 * C0));
      EZB_TRY(vae_fold_wave_w(st, v, g, norms, out_w, C0));
    }
    if (d.with_encoder) EZB_TRY(finalize_encoder(st));
    EZB_CUDA(cudaStreamSynchronize(st));
    finalized = true;
    return EZB_OK;
  }

  // lens / lens_max: the per-clip lengths of the encode / decode in flight (null: every clip fills the batch's length)
  const int32_t* lens = nullptr;
  int lens_max = 0;
  int run_conv(cudaStream_t st, const VaeConv& c, const __nv_bfloat16* A, int B, int T, const float* resid_in, float* raw_out, __nv_bfloat16* act_out,
               const VaeSnake* snake) {
    return vae_conv(*dev, st, c, kmul, A, B, T, resid_in, raw_out, act_out, snake, lens, lens_max);
  }

  // audio (B, 1, T) fp32, T = hop * L; noise (B, latent, L) fp32 or null (-> mean); z (B, latent, L) fp32.
  // lens_ (device [B] latent frames, or null): clip b is its first hop * lens_[b] samples; its z frames come out as an encode of the
  // clip alone at that length, the frames past it as zeros, whatever audio and noise hold past the end.
  // noised (or null): z receives the start latent of a variation instead (vae_sample_noised_kernel).
  int encode(const float* audio, const float* noise, float* z, int B, int T, cudaStream_t st, const int32_t* lens_ = nullptr,
             const VaeNoised* noised = nullptr) {
    if (!finalized || !d.with_encoder) return fail(EZB_ERR_STATE, "VAE encoder weights not loaded");
    int hop = 1;
    for (int j = 0; j < nst; ++j) hop *= e_stride[j];
    if (T % hop) return fail(EZB_ERR_SHAPE, "vae_encode: T %d is not a multiple of the hop %d", T, hop);
    const int L = T / hop;
    if (B < 1 || B > d.max_batch || L < 1 || L > d.max_latent_len) return fail(EZB_ERR_SHAPE, "vae_encode: B %d L %d exceed workspace", B, L);
    const int C0 = e_cin[0];
    __nv_bfloat16 *cur = actA, *oth = actB;
    lens = lens_; lens_max = L;
    EZB_TRY(vae_enc_conv_in(st, audio, e_in_w, e_in_b, e_res_s0[0], resid, cur, B, C0, T, kmul, lens, hop));
    int Tc = T;
    for (int j = 0; j < nst; ++j) {
      for (int u = 0; u < 3; ++u) {
        EZB_TRY(run_conv(st, e_res7[3 * j + u], cur, B, Tc, nullptr, nullptr, oth, &e_res_s2[3 * j + u]));
        const bool last = u == 2;
        const VaeSnake* nxt = last ? &e_down_snake[j] : &e_res_s0[3 * j + u + 1];
        EZB_TRY(run_conv(st, e_res1[3 * j + u], oth, B, Tc, resid, last ? nullptr : resid, cur, nxt));
      }
      Tc /= e_stride[j];
      const bool last_stage = j + 1 == nst;
      const VaeSnake* nxt = last_stage ? &e_out_snake : &e_res_s0[3 * (j + 1)];
      EZB_TRY(run_conv(st, e_down[j], cur, B, Tc, nullptr, last_stage ? nullptr : resid, oth, nxt));
      std::swap(cur, oth);
    }
    EZB_TRY(run_conv(st, e_out, cur, B, Tc, nullptr, resid, nullptr, nullptr));  // (mean | scale), channels-last fp32
    if (noised != nullptr) return vae_sample_noised(st, resid, noise, *noised, z, B, d.latent_dim, L, lens);
    return vae_sample(st, resid, noise, z, B, d.latent_dim, L, lens);
  }

  // lens_ (device [B] latent frames, or null): clip b is its first lens_[b] frames; its hop * lens_[b] samples come out as a decode of the
  // clip alone at that length, the samples past them as zeros, whatever z holds past the end (NaN included).
  int decode(const float* z, float* wav, int B, int L, cudaStream_t st, const int32_t* lens_ = nullptr) {
    if (!finalized) return fail(EZB_ERR_STATE, "VAE weights not finalized");
    if (B < 1 || B > d.max_batch || L < 1 || L > d.max_latent_len) return fail(EZB_ERR_SHAPE, "vae_decode: B %d L %d exceed workspace", B, L);
    lens = lens_; lens_max = L;
    EZB_TRY(vae_latent_pack(st, z, actA, B, d.latent_dim, L, kmul, lens));
    __nv_bfloat16 *cur = actA, *oth = actB;
    int T = L;
    EZB_TRY(run_conv(st, conv_in, cur, B, T, nullptr, nullptr, oth, &up_snake[0]));
    std::swap(cur, oth);
    for (int j = 0; j < nst; ++j) {
      // conv-transpose: writes the fp32 residual stream [B, T*s, cout] and the first unit's snake input
      EZB_TRY(run_conv(st, up[j], cur, B, T, nullptr, resid, oth, &res_s0[3 * j]));
      std::swap(cur, oth);
      T *= stride_s[j];
      for (int u = 0; u < 3; ++u) {
        EZB_TRY(run_conv(st, res7[3 * j + u], cur, B, T, nullptr, nullptr, oth, &res_s2[3 * j + u]));
        const bool last = u == 2;
        const VaeSnake* nxt = !last ? &res_s0[3 * j + u + 1] : (j + 1 < nst ? &up_snake[j + 1] : &out_snake);
        EZB_TRY(run_conv(st, res1[3 * j + u], oth, B, T, resid, last ? nullptr : resid, cur, nxt));
      }
    }
    return vae_wave_out(st, cur, out_w, wav, B, cout_s[nst - 1], T, kmul, lens, T / L);
  }
};

}  // namespace ezb
