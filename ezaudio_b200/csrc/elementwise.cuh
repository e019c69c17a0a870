// Bandwidth-bound kernels of the DiT step: LayerNorm(+AdaLN modulate)+cast, per-head qk-LayerNorm + RoPE + head layout,
// patch-embed input packing, final 3-tap conv, time-embedding path, weight repacking, CFG + DDIM / DPM-Solver++ update.
// All fp32 math; bf16 only where a tensor feeds a tensor-core operand.
#pragma once
#include "cfg_update.cuh"
#include "common.cuh"
#include "../../include/ezb200.h"

namespace ezb {

// parity ("split") operand write: A' = [hi | lo | hi] along K (matches W' = [hi | hi | lo]): A'W'^T = hi*hi + lo*hi + hi*lo
__device__ __forceinline__ void store_act(__nv_bfloat16* row, int col, int K, int kmul, float v) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  row[col] = hi;
  if (kmul == 3) {
    row[K + col] = __float2bfloat16_rn(v - __bfloat162float(hi));
    row[2 * K + col] = hi;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm over the (optionally concatenated) row [x | x2 (+x3)], affine, optional AdaLN modulate, cast to bf16.
//   nn.LayerNorm eps 1e-5 (blocks.py:68,83,85,91,100), film_modulate x*(1+scale)+shift (modules.py:15-16),
//   skip path cat[x, skip (+ controlnet skip)] (blocks.py:124-126, udit.py:345-348).
// One warp per row; two passes over an L1/L2-resident row.
struct LnParams {
  const float* x;    // [M, D1]
  const float* x2;   // optional [M, D2] (concatenated after x)
  const float* x3;   // optional, added to x2 element-wise
  int D1, D2;
  const float* w;    // [D1 + D2]
  const float* b;
  const float* shift;  // optional modulation: shift[bidx * mod_bstride + c], scale likewise (c < D1 only, D2 == 0)
  const float* scale;
  int mod_bstride;     // element stride between batch items in shift/scale (0: all share one row)
  int rows_per_batch;
  __nv_bfloat16* out;  // [M, kmul * (D1 + D2)]
  int kmul;
  int M;
  const float* G;      // optional precombined affine for ln_gc_kernel: y = (x - mu) * rstd * G + C with G = w (1 + scale), C = b (1 + scale) + shift
  const float* C;      // (one row for the whole batch: uniform timestep)
};

// x / x2 / x3 are read with ld.global.cg (L2 only): when the LayerNorm runs as the tail phase of the GEMM that produced x (gemm_ln.cuh), rows
// written by other SMs moments ago must not be served from a stale L1 line; for the stand-alone kernels it makes no difference (streaming).
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ void ln_row_generic(const LnParams& p, int row, int lane) {
  const int D = p.D1 + p.D2;
  const float* x = p.x + (size_t)row * p.D1;
  const float* x2 = p.x2 ? p.x2 + (size_t)row * p.D2 : nullptr;
  const float* x3 = p.x3 ? p.x3 + (size_t)row * p.D2 : nullptr;
  float s = 0.f;
  for (int c = lane * 4; c < p.D1; c += 128) {
    const float4 v = ldcg4(x + c);
    s += v.x + v.y + v.z + v.w;
  }
  for (int c = lane * 4; c < p.D2; c += 128) {
    float4 v = ldcg4(x2 + c);
    if (x3) { const float4 u = ldcg4(x3 + c); v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w; }
    s += v.x + v.y + v.z + v.w;
  }
  const float mean = warp_sum(s) / D;
  float q = 0.f;
  for (int c = lane * 4; c < p.D1; c += 128) {
    const float4 v = ldcg4(x + c);
    q += (v.x - mean) * (v.x - mean) + (v.y - mean) * (v.y - mean) + (v.z - mean) * (v.z - mean) + (v.w - mean) * (v.w - mean);
  }
  for (int c = lane * 4; c < p.D2; c += 128) {
    float4 v = ldcg4(x2 + c);
    if (x3) { const float4 u = ldcg4(x3 + c); v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w; }
    q += (v.x - mean) * (v.x - mean) + (v.y - mean) * (v.y - mean) + (v.z - mean) * (v.z - mean) + (v.w - mean) * (v.w - mean);
  }
  float rstd = rsqrtf(warp_sum(q) / D + 1e-5f);
  const bool norm = p.w != nullptr;  // w == NULL: cast only (no normalisation)
  float mu = mean;
  if (!norm) { mu = 0.f; rstd = 1.f; }
  const float *sh = nullptr, *sc = nullptr;
  if (p.shift) {
    const size_t off = (size_t)(row / p.rows_per_batch) * p.mod_bstride;
    sh = p.shift + off;
    sc = p.scale + off;
  }
  __nv_bfloat16* o = p.out + (size_t)row * p.kmul * D;
  for (int c = lane * 4; c < D; c += 128) {
    float4 v;
    if (c < p.D1) {
      v = ldcg4(x + c);
    } else {
      v = ldcg4(x2 + (c - p.D1));
      if (x3) { const float4 u = ldcg4(x3 + (c - p.D1)); v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w; }
    }
    float4 w = make_float4(1.f, 1.f, 1.f, 1.f), b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (norm) { w = *reinterpret_cast<const float4*>(p.w + c); b = *reinterpret_cast<const float4*>(p.b + c); }
    float y[4] = {(v.x - mu) * rstd * w.x + b.x, (v.y - mu) * rstd * w.y + b.y, (v.z - mu) * rstd * w.z + b.z, (v.w - mu) * rstd * w.w + b.w};
    if (sh) {
      const float4 a = *reinterpret_cast<const float4*>(sc + c), d = *reinterpret_cast<const float4*>(sh + c);
      y[0] = y[0] * (1.f + a.x) + d.x; y[1] = y[1] * (1.f + a.y) + d.y; y[2] = y[2] * (1.f + a.z) + d.z; y[3] = y[3] * (1.f + a.w) + d.w;
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) store_act(o, c + e, D, p.kmul, y[e]);
  }
}
__global__ void __launch_bounds__(256) ln_mod_cast_kernel(const LnParams p) {
  pdl_launch();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= p.M) return;
  ln_row_generic(p, warp, lane);
}

// Register-resident variant for the hot shapes (single source, D = 128 * NCH): the row is read once, both moments come
// from registers (two-pass formula, same numerics as above), 8-byte bf16 stores.
template <int NCH>
__device__ __forceinline__ void ln_row_reg(const LnParams& p, int row, int lane) {
  constexpr int D = NCH * 128;
  const float* x = p.x + (size_t)row * D;
  float4 v[NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) v[i] = ldcg4(x + 4 * (lane + 32 * i));
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) * (1.0f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + 1e-5f);
  const float4 *w4 = reinterpret_cast<const float4*>(p.w), *b4 = reinterpret_cast<const float4*>(p.b);
  const float4 *sh4 = nullptr, *sc4 = nullptr;
  if (p.shift) {
    const size_t off = (size_t)(row / p.rows_per_batch) * p.mod_bstride;
    sh4 = reinterpret_cast<const float4*>(p.shift + off);
    sc4 = reinterpret_cast<const float4*>(p.scale + off);
  }
  __nv_bfloat16* o = p.out + (size_t)row * D;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c4 = lane + 32 * i;
    const float4 w = __ldg(w4 + c4), b = __ldg(b4 + c4);
    float y0 = (v[i].x - mean) * rstd * w.x + b.x, y1 = (v[i].y - mean) * rstd * w.y + b.y;
    float y2 = (v[i].z - mean) * rstd * w.z + b.z, y3 = (v[i].w - mean) * rstd * w.w + b.w;
    if (sh4) {
      const float4 a = __ldg(sc4 + c4), d = __ldg(sh4 + c4);
      y0 = y0 * (1.f + a.x) + d.x; y1 = y1 * (1.f + a.y) + d.y; y2 = y2 * (1.f + a.z) + d.z; y3 = y3 * (1.f + a.w) + d.w;
    }
    *reinterpret_cast<uint2*>(o + 4 * c4) = make_uint2(pack_bf16(y0, y1), pack_bf16(y2, y3));
  }
}
// One warp per row, 4 rows per 128-thread block.  MINB = minimum CTAs per SM: 1 -> 79 registers, 6 CTAs per SM = 888 of the 1000 CTAs of an
// M = 4000 launch resident (a second, nearly empty wave); 8 -> <= 64 registers, one wave.  Run-time choice (option "ln_variant").
template <int NCH, int MINB>
__global__ void __launch_bounds__(128, MINB) ln_mod_cast_reg_kernel(const LnParams p) {
  pdl_launch();
  pdl_wait();
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= p.M) return;
  ln_row_reg<NCH>(p, row, lane);
}
// Variant with the affine precombined per timestep (G, C: fold_gc_kernel) and held in REGISTERS across rows.  In the kernel above every warp
// re-reads weight, bias, scale and shift (4 x 4.6 KB) for its one row: 27 warps per SM pull ~500 KB of parameters through L1 for 124 KB of
// activations.  Here a warp loads G and C once (2 x 36 registers per lane) and walks its rows in a strided loop.
template <int NCH>
__global__ void __launch_bounds__(128, 4) ln_gc_kernel(const LnParams p) {
  pdl_launch();
  pdl_wait();
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31, gw = blockIdx.x * 4 + (threadIdx.x >> 5), nw = gridDim.x * 4;
  if (gw >= p.M) return;
  float4 g[NCH], c[NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    g[i] = __ldg(reinterpret_cast<const float4*>(p.G) + lane + 32 * i);
    c[i] = __ldg(reinterpret_cast<const float4*>(p.C) + lane + 32 * i);
  }
  for (int row = gw; row < p.M; row += nw) {
    const float* x = p.x + (size_t)row * D;
    float4 v[NCH];
#pragma unroll
    for (int i = 0; i < NCH; ++i) v[i] = ldcg4(x + 4 * (lane + 32 * i));
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) * (1.0f / D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const float a = v[i].x - mean, b = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (cc * cc + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + 1e-5f);
    __nv_bfloat16* o = p.out + (size_t)row * D;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const float y0 = fmaf((v[i].x - mean) * rstd, g[i].x, c[i].x), y1 = fmaf((v[i].y - mean) * rstd, g[i].y, c[i].y);
      const float y2 = fmaf((v[i].z - mean) * rstd, g[i].z, c[i].z), y3 = fmaf((v[i].w - mean) * rstd, g[i].w, c[i].w);
      *reinterpret_cast<uint2*>(o + 4 * (lane + 32 * i)) = make_uint2(pack_bf16(y0, y1), pack_bf16(y2, y3));
    }
  }
}
// skip_norm of the out-blocks (blocks.py:124-126): LayerNorm over the concatenated row [x | x2 (+ x3)] with D1 = D2 = 128 NCH, held in registers (one
// pass; the generic kernel above walks the row three times).  No modulation.  One warp per row, 4 rows per 128-thread block.
template <int NCH>
__global__ void __launch_bounds__(128) ln_cat_reg_kernel(const LnParams p) {
  pdl_launch();
  pdl_wait();
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= p.M) return;
  constexpr int D1 = NCH * 128, D = 2 * D1;
  const float* x = p.x + (size_t)row * D1;
  const float* x2 = p.x2 + (size_t)row * D1;
  float4 v[2 * NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    v[i] = ldcg4(x + 4 * (lane + 32 * i));
    v[NCH + i] = ldcg4(x2 + 4 * (lane + 32 * i));
  }
  if (p.x3 != nullptr) {
    const float* x3 = p.x3 + (size_t)row * D1;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const float4 u = ldcg4(x3 + 4 * (lane + 32 * i));
      v[NCH + i].x += u.x; v[NCH + i].y += u.y; v[NCH + i].z += u.z; v[NCH + i].w += u.w;
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 2 * NCH; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) * (1.0f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 2 * NCH; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + 1e-5f);
  const float4 *w4 = reinterpret_cast<const float4*>(p.w), *b4 = reinterpret_cast<const float4*>(p.b);
  __nv_bfloat16* o = p.out + (size_t)row * D;
#pragma unroll
  for (int i = 0; i < 2 * NCH; ++i) {
    const int c4 = (i < NCH ? 0 : D1 / 4) + lane + 32 * (i < NCH ? i : i - NCH);
    const float4 w = __ldg(w4 + c4), b = __ldg(b4 + c4);
    const float y0 = (v[i].x - mean) * rstd * w.x + b.x, y1 = (v[i].y - mean) * rstd * w.y + b.y;
    const float y2 = (v[i].z - mean) * rstd * w.z + b.z, y3 = (v[i].w - mean) * rstd * w.w + b.w;
    *reinterpret_cast<uint2*>(o + 4 * c4) = make_uint2(pack_bf16(y0, y1), pack_bf16(y2, y3));
  }
}
// LayerNorm as the tail phase of another kernel (gemm_ln.cuh): every warp of the (persistent, fully resident) grid takes rows in a strided loop
__device__ __forceinline__ bool ln_reg_eligible(const LnParams& p) { return p.kmul == 1 && p.x2 == nullptr && p.w != nullptr && (p.D1 == 1152 || p.D1 == 1024); }
__device__ __forceinline__ void ln_tail(const LnParams& p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const bool reg = ln_reg_eligible(p);
  for (int row = blockIdx.x * nw + warp; row < p.M; row += gridDim.x * nw) {
    if (reg) {
      if (p.D1 == 1152) ln_row_reg<9>(p, row, lane);
      else ln_row_reg<8>(p, row, lane);
    } else {
      ln_row_generic(p, row, lane);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// FP8 mode: e4m3 operands with one fp32 scale per row, s = amax / 448 and q = e4m3(v * (448 / amax)) saturated (amax = 0: q = 0, s = 0).
__device__ __forceinline__ float e4m3_inv_scale(float amax) { return amax > 0.f ? 448.f / amax : 0.f; }
__device__ __forceinline__ uint32_t pack_e4m3x2(float lo, float hi) {   // round to nearest even, saturated to +-448; lo -> the low byte
  unsigned short r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) { return pack_e4m3x2(a, b) | (pack_e4m3x2(c, d) << 16); }
struct LnFp8Out {
  uint8_t* q;   // [M, D1] e4m3
  float* s;     // [M] row scales
};
// LayerNorm (+ AdaLN modulate) of x [M, D1] to e4m3 rows: the operand of the FP8 QKV and GEGLU projections.  The row stays in registers
// (D1 <= 128 NCH; EXACT: D1 == 128 NCH), so its amax costs one warp reduction.  Affine from the precombined per-timestep tables (p.G, p.C,
// as ln_gc_kernel) when set, else weight, bias and the per-batch shift / scale (as ln_row_generic).  One warp per row, rows in a strided loop.
template <int NCH, bool EXACT>
__global__ void __launch_bounds__(128) ln_fp8_kernel(const LnParams p, const LnFp8Out o) {
  pdl_launch();
  pdl_wait();
  const int D = EXACT ? NCH * 128 : p.D1;
  const int lane = threadIdx.x & 31, gw = blockIdx.x * 4 + (threadIdx.x >> 5), nw = gridDim.x * 4;
  for (int row = gw; row < p.M; row += nw) {
    const float* x = p.x + (size_t)row * D;
    float4 v[NCH];
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c4 = lane + 32 * i;
      v[i] = (EXACT || 4 * c4 < D) ? ldcg4(x + 4 * c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) / D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      if (!EXACT && 4 * (lane + 32 * i) >= D) continue;
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) / D + 1e-5f);
    const float *sh = nullptr, *sc = nullptr;
    if (p.G == nullptr && p.shift != nullptr) {
      const size_t off = (size_t)(row / p.rows_per_batch) * p.mod_bstride;
      sh = p.shift + off;
      sc = p.scale + off;
    }
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c4 = lane + 32 * i;
      if (!EXACT && 4 * c4 >= D) continue;
      float y[4] = {(v[i].x - mean) * rstd, (v[i].y - mean) * rstd, (v[i].z - mean) * rstd, (v[i].w - mean) * rstd};
      if (p.G != nullptr) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(p.G) + c4), c = __ldg(reinterpret_cast<const float4*>(p.C) + c4);
        y[0] = fmaf(y[0], g.x, c.x); y[1] = fmaf(y[1], g.y, c.y); y[2] = fmaf(y[2], g.z, c.z); y[3] = fmaf(y[3], g.w, c.w);
      } else {
        const float4 w = __ldg(reinterpret_cast<const float4*>(p.w) + c4), b = __ldg(reinterpret_cast<const float4*>(p.b) + c4);
        y[0] = y[0] * w.x + b.x; y[1] = y[1] * w.y + b.y; y[2] = y[2] * w.z + b.z; y[3] = y[3] * w.w + b.w;
        if (sh) {
          const float4 a = *reinterpret_cast<const float4*>(sc + 4 * c4), d = *reinterpret_cast<const float4*>(sh + 4 * c4);
          y[0] = y[0] * (1.f + a.x) + d.x; y[1] = y[1] * (1.f + a.y) + d.y; y[2] = y[2] * (1.f + a.z) + d.z; y[3] = y[3] * (1.f + a.w) + d.w;
        }
      }
      v[i] = make_float4(y[0], y[1], y[2], y[3]);
      amax = fmaxf(amax, fmaxf(fmaxf(fabsf(y[0]), fabsf(y[1])), fmaxf(fabsf(y[2]), fabsf(y[3]))));
    }
    amax = warp_max(amax);
    const float inv = e4m3_inv_scale(amax);
    uint32_t* out = reinterpret_cast<uint32_t*>(o.q + (size_t)row * D);
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c4 = lane + 32 * i;
      if (!EXACT && 4 * c4 >= D) continue;
      out[c4] = pack_e4m3x4(v[i].x * inv, v[i].y * inv, v[i].z * inv, v[i].w * inv);
    }
    if (lane == 0) o.s[row] = amax / 448.f;
  }
}
// FP8 mode, at finalize: rows of a packed bf16 weight [N, K] -> e4m3 [N, K] with per-row scales (the same rule as ln_fp8_kernel).  One warp per row.
__global__ void __launch_bounds__(256) quant_rows_e4m3_kernel(const __nv_bfloat16* __restrict__ W, int N, int K, uint8_t* __restrict__ Q, float* __restrict__ S) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= N) return;
  const __nv_bfloat16* w = W + (size_t)row * K;
  float amax = 0.f;
  for (int k = lane; k < K; k += 32) amax = fmaxf(amax, fabsf(__bfloat162float(w[k])));
  amax = warp_max(amax);
  const float inv = e4m3_inv_scale(amax);
  for (int k = lane; k < K; k += 32) Q[(size_t)row * K + k] = (uint8_t)pack_e4m3x2(__bfloat162float(w[k]) * inv, 0.f);
  if (lane == 0) S[row] = amax / 448.f;
}

// ---------------------------------------------------------------------------------------------------------------
// Per-head LayerNorm(dh, affine) on q / k (attention.py:63-65,141-142), NeoX rotate-half RoPE with fp32 tables on
// positions 0..L-1 (rotary.py:6-18,72-84; pairs (i, i+dh/2), freq 1e4^(-2i/dh)), and head-major layout for attention:
//   section 0 (q), 1 (k): dst[b, h, l, 0..dh)  (row pitch dst_ld, zero padding beyond dh pre-cleared)
//   section 2 (v)       : fp32 path -> same layout; tensor-core path -> transposed vt[b, h, d, l] (pitch Lpad)
// One warp per (token, head); lane owns dims lane, lane+32, lane+64 (dh <= 96).
template <typename TIn>
struct QkPrepParams {
  const TIn* in;  // [M, ld_in]: GEMM output, sections at column offsets col_off[s]
  int ld_in;
  int col_off[3];
  int n_sections;        // self: 3 (q,k,v); cross q: 1; cross kv: sections k,v -> use sec_kind
  int sec_kind[3];       // 0 q, 1 k, 2 v
  const float* nw[2];    // LN weight for q, k
  const float* nb[2];
  int use_rope;
  const float* inv_freq;  // [dh/2] (attn.rotary.inv_freq buffer of the checkpoint)
  int B, L, H, dh;
  float* f32_out[3];            // optional fp32 [B,H,L,dh] per section (SIMT attention)
  __nv_bfloat16* bf_out[3];     // optional bf16: q,k -> [B,H,L,ld_qk]; v -> vt [B,H,dv_pad,Lpad]
  int ld_qk, Lpad, dv_pad;
};

__device__ __forceinline__ float ld_as_float(const float* p) { return *p; }
__device__ __forceinline__ float ld_as_float(const __nv_bfloat16* p) { return __bfloat162float(*p); }

template <typename TIn>
__global__ void __launch_bounds__(256) qk_prep_kernel(const QkPrepParams<TIn> p) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int total = p.B * p.L * p.H * p.n_sections;
  if (wid >= total) return;
  const int h = wid % p.H;
  const int sec = (wid / p.H) % p.n_sections;
  const int tok = wid / (p.H * p.n_sections);
  const int b = tok / p.L, l = tok - b * p.L;
  const int kind = p.sec_kind[sec];
  const TIn* src = p.in + (size_t)tok * p.ld_in + p.col_off[sec] + h * p.dh;
  float v[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) v[i] = (lane + 32 * i < p.dh) ? ld_as_float(src + lane + 32 * i) : 0.f;
  if (kind < 2) {
    const float mean = warp_sum(v[0] + v[1] + v[2]) / p.dh;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) if (lane + 32 * i < p.dh) q += (v[i] - mean) * (v[i] - mean);
    const float rstd = rsqrtf(warp_sum(q) / p.dh + 1e-5f);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int d = lane + 32 * i;
      if (d < p.dh) v[i] = (v[i] - mean) * rstd * p.nw[kind][d] + p.nb[kind][d];
    }
    if (p.use_rope) {
      // stage through shuffles is awkward for arbitrary dh: use a small smem exchange per warp instead
      __shared__ float xch[8][96];
      float* xw = xch[threadIdx.x >> 5];
#pragma unroll
      for (int i = 0; i < 3; ++i) if (lane + 32 * i < p.dh) xw[lane + 32 * i] = v[i];
      __syncwarp();
      const int half = p.dh >> 1;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const int d = lane + 32 * i;
        if (d < p.dh) {
          const int fi = d < half ? d : d - half;
          float sn, cs;
          sincosf((float)l * p.inv_freq[fi], &sn, &cs);
          const float other = d < half ? -xw[d + half] : xw[d - half];
          v[i] = v[i] * cs + other * sn;
        }
      }
    }
  }
  const size_t bh = (size_t)b * p.H + h;
  if (p.f32_out[sec]) {
    float* o = p.f32_out[sec] + (bh * p.L + l) * p.dh;
#pragma unroll
    for (int i = 0; i < 3; ++i) if (lane + 32 * i < p.dh) o[lane + 32 * i] = v[i];
  }
  if (p.bf_out[sec]) {
    if (kind < 2) {
      __nv_bfloat16* o = p.bf_out[sec] + (bh * p.L + l) * p.ld_qk;
#pragma unroll
      for (int i = 0; i < 3; ++i) if (lane + 32 * i < p.dh) o[lane + 32 * i] = __float2bfloat16_rn(v[i]);
    } else {
      __nv_bfloat16* o = p.bf_out[sec] + bh * p.dv_pad * p.Lpad + l;
#pragma unroll
      for (int i = 0; i < 3; ++i) if (lane + 32 * i < p.dh) o[(size_t)(lane + 32 * i) * p.Lpad] = __float2bfloat16_rn(v[i]);
      for (int dpad = p.dh + lane; dpad < p.dv_pad; dpad += 32) o[(size_t)dpad * p.Lpad] = __float2bfloat16_rn(0.f);  // zero pad rows
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// MaskDiT input assembly (conditioners.py:150-153,174-176) + transpose for the k=1 patch-embed conv (modules.py:100-111):
//   A[b*L + l, :] = [ x[b,:,l] | gt[b,:,l] or mask_embed (where gt is NULL or gt_mask[b,l]) | mask channel | 0-pad ]
//   mask channel = gt ? gt_mask[b,l] : 1          (mae_mask[:,0:1,:]: ones when gt is None)
__global__ void patch_pack_kernel(const float* __restrict__ x, const float* __restrict__ gt, const uint8_t* __restrict__ gt_mask,
                                  const float* __restrict__ mask_embed, __nv_bfloat16* __restrict__ out, int B, int C, int L, int Kp, int kmul) {
  pdl_launch();
  pdl_wait();
  __shared__ float tile[32][33];
  const int b = blockIdx.z, l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;  // c0 over 2C channels
  const int tx = threadIdx.x, ty = threadIdx.y;                            // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, l = l0 + tx;
    float v = 0.f;
    if (l < L) {
      if (c < C) v = x[((size_t)b * C + c) * L + l];
      else {
        const int cg = c - C;
        const bool masked = (gt == nullptr) || (gt_mask != nullptr && gt_mask[(size_t)b * L + l]);
        v = masked ? mask_embed[cg] : gt[((size_t)b * C + cg) * L + l];
      }
    }
    tile[i][tx] = v;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int l = l0 + i, c = c0 + tx;
    if (l < L) store_act(out + ((size_t)b * L + l) * kmul * Kp, c, Kp, kmul, tile[tx][i]);
  }
  if (blockIdx.y == 0 && ty == 0) {  // mask channel + zero pad
    const int l = l0 + tx;
    if (l < L) {
      const float m = gt ? (gt_mask && gt_mask[(size_t)b * L + l] ? 1.f : 0.f) : 1.f;
      __nv_bfloat16* o = out + ((size_t)b * L + l) * kmul * Kp;
      store_act(o, 2 * C, Kp, kmul, m);
      for (int c = 2 * C + 1; c < Kp; ++c) store_act(o, c, Kp, kmul, 0.f);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// FinalBlock tail (blocks.py:207-211): y [B*L, C] token-major -> unpatchify (transpose) -> Conv1d(C, C, k=3, pad=1).
// w packed [3][Cin][Cout].  CTA = 32 positions x all C = 128 output channels, 512 threads = 4 input-channel groups x 128; within a group
// thread = 4 output channels x 8 positions, so one input channel costs 10 broadcast LDS + 3 coalesced float4 weight loads for 96 FMAs; the four
// groups' partial sums meet in shared memory.  (Four warps per SM walking all 128 input channels cannot hide the L2 latency of the weight
// loads; this one: 16 warps.)
// lens ([B] device, or null): clip b ends at lens[b] frames of the padded L.  Frames at or past it are the zero halo a solo run of that
// length sees, and are not written.
constexpr int FC_GROUPS = 4;
__global__ void __launch_bounds__(128 * FC_GROUPS) final_conv_kernel(const float* __restrict__ y, const float* __restrict__ wp, const float* __restrict__ bias,
                                                                     float* __restrict__ out, int B, int C, int L, const int32_t* __restrict__ lens) {
  pdl_launch();
  pdl_wait();
  constexpr int TL = 32, TP = TL + 2 + 2;  // 34 positions (+2 so that the 10-wide window of the last thread group stays in bounds)
  extern __shared__ float sy[];             // [C][TP] channel-major, then [FC_GROUPS - 1][128][32] partial sums
  float* red = sy + (size_t)C * TP;
  const int b = blockIdx.y, l0 = blockIdx.x * TL;
  const int len = lens != nullptr ? min(max(lens[b], 1), L) : L;
  if (l0 >= len) return;   // CTA-uniform: a tile of padding only
  for (int i = threadIdx.x; i < (TL + 2) * C; i += blockDim.x) {
    const int r = i / C, c = i - r * C, l = l0 + r - 1;
    sy[c * TP + r] = (l >= 0 && l < len) ? y[((size_t)b * L + l) * C + c] : 0.f;
  }
  __syncthreads();
  const int gq = threadIdx.x >> 7, t128 = threadIdx.x & 127;
  const int tq = t128 >> 5;                  // positions tq*8 .. tq*8+7 of the tile
  const int cq = (C + FC_GROUPS - 1) / FC_GROUPS, ci0 = gq * cq, ci1 = ci0 + cq < C ? ci0 + cq : C;
  for (int cb = 0; cb < C; cb += 128) {   // C = 128 shipped: one pass.  The trip count is uniform (barriers inside); lanes beyond C idle.
    const int co = cb + (t128 & 31) * 4;
    const bool live = co < C;
    float acc[8][4];
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gq == 0 && live) bv = *reinterpret_cast<const float4*>(bias + co);
#pragma unroll
    for (int t = 0; t < 8; ++t) { acc[t][0] = bv.x; acc[t][1] = bv.y; acc[t][2] = bv.z; acc[t][3] = bv.w; }
#pragma unroll 4
    for (int ci = ci0; ci < (live ? ci1 : ci0); ++ci) {
      float4 w[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) w[k] = __ldg(reinterpret_cast<const float4*>(wp + ((size_t)k * C + ci) * C + co));
      float x[10];
#pragma unroll
      for (int t = 0; t < 10; ++t) x[t] = sy[ci * TP + tq * 8 + t];
#pragma unroll
      for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          acc[t][0] = fmaf(w[k].x, x[t + k], acc[t][0]);
          acc[t][1] = fmaf(w[k].y, x[t + k], acc[t][1]);
          acc[t][2] = fmaf(w[k].z, x[t + k], acc[t][2]);
          acc[t][3] = fmaf(w[k].w, x[t + k], acc[t][3]);
        }
    }
    if (gq > 0) {
      float* rr = red + ((size_t)(gq - 1) * 128 + t128) * 32;
#pragma unroll
      for (int t = 0; t < 8; ++t) *reinterpret_cast<float4*>(rr + t * 4) = make_float4(acc[t][0], acc[t][1], acc[t][2], acc[t][3]);
    }
    __syncthreads();
    if (gq == 0 && live) {
#pragma unroll
      for (int q = 0; q < FC_GROUPS - 1; ++q) {
        const float* rr = red + ((size_t)q * 128 + t128) * 32;
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const float4 v = *reinterpret_cast<const float4*>(rr + t * 4);
          acc[t][0] += v.x; acc[t][1] += v.y; acc[t][2] += v.z; acc[t][3] += v.w;
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int l = l0 + tq * 8 + t;
          if (l < len) out[((size_t)b * C + co + e) * L + l] = acc[t][e];
        }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Small-M linear for the time path (fp32 weights, R <= a few hundred rows): out[r, n] = act(in[r,:] . W[n,:] + bias[n]) + add[r, n]
// One warp per output feature; the weight row lives in registers and is reused across all rows.
__global__ void __launch_bounds__(256) small_linear_kernel(const float* __restrict__ in, int ld_in, const float* __restrict__ W, const float* __restrict__ bias,
                                                           const float* __restrict__ add, int ld_add, float* __restrict__ out, int ld_out, int R, int N, int K,
                                                           int act /*0 none, 1 silu*/, float out_scale) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (n >= N) return;
  constexpr int MAXK = 40;  // K <= 1280 per pass
  for (int k0 = 0; k0 < K; k0 += 32 * MAXK) {
    float w[MAXK];
#pragma unroll
    for (int i = 0; i < MAXK; ++i) { const int k = k0 + lane + 32 * i; w[i] = k < K ? W[(size_t)n * K + k] : 0.f; }
    for (int r = 0; r < R; ++r) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < MAXK; ++i) { const int k = k0 + lane + 32 * i; if (k < K) s = fmaf(w[i], in[(size_t)r * ld_in + k], s); }
      s = warp_sum(s);
      if (lane == 0) {
        float* o = out + (size_t)r * ld_out + n;
        float v = (k0 == 0 ? 0.f : *o) + s;
        if (k0 + 32 * MAXK >= K) {
          v = v * out_scale + (bias ? bias[n] : 0.f);
          if (act == 1) v = silu(v);
          if (add) v += add[(size_t)r * ld_add + n];
        }
        *o = v;
      }
    }
  }
}

// RoPE table (rotary.py:48-70): cs[l][i] = (cos, sin)(l * inv_freq[i]), fp32, i < dh/2 (token-major: a thread reads its
// token's dh/2 pairs as 9 full 32-byte sectors; the frequency-major alternative is strided)
__global__ void rope_table_kernel(const float* __restrict__ inv_freq, float2* __restrict__ cs, int L, int half) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L * half) return;
  const int l = i / half, f = i - l * half;
  float s, c;
  sincosf((float)l * inv_freq[f], &s, &c);
  cs[i] = make_float2(c, s);
}
// timestep_embedding (modules.py:19-39): [cos(t f_i) | sin(t f_i)], f_i = exp(-ln(1e4) i / 128), dim 256
__global__ void timestep_embed_kernel(const float* __restrict__ t, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 128) return;
  const int r = i / 128, j = i - r * 128;
  const float f = expf(-9.210340371976184f * (float)j / 128.0f);
  float s, c;
  sincosf(t[r] * f, &s, &c);
  out[r * 256 + j] = c;
  out[r * 256 + 128 + j] = s;
}
__global__ void silu_inplace_kernel(float* x, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = silu(x[i]);
}
// mod[r, blk, :] += table[blk, :]  (scale_shift_table[None] + time_ada, blocks.py:43-45)
__global__ void add_rowvec_kernel(float* __restrict__ dst, int ld_dst, const float* __restrict__ vec, int R, int N) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)R * N) return;
  const int r = i / N, c = i - (size_t)r * N;
  dst[(size_t)r * ld_dst + c] += vec[c];
}

// ---------------------------------------------------------------------------------------------------------------
// Weight repacking fp32 [N, K] (reference layout) -> bf16 [N', kmul*Kpad] rows; optional GEGLU tile interleave
// (dst row = tile*BN + {0,HALF} + j) and row offset (QKV / KV concatenation).  Split mode writes W' = [hi | hi | lo].
// heads3 mode (h3_dh > 0): rows are heads of one of the q / k / v sections; global head g = h3_head_off + n / dh goes to row
// (g / 3) * h3_bn + (g % 3) * dh + n % dh of the packed QKV weight (three heads per N-tile, see EpiHeads<DH, 3>).
__global__ void pack_weight_kernel(const float* __restrict__ src, int N, int K, __nv_bfloat16* __restrict__ dst, int Kpad, int kmul, int row_off,
                                   int geglu_inner, int geglu_half, int h3_dh, int h3_head_off, int h3_bn) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)N * Kpad) return;
  const int n = i / Kpad, k = i - (size_t)n * Kpad;
  int dn = n + row_off;
  if (geglu_inner > 0) {
    const int g = n >= geglu_inner, m = g ? n - geglu_inner : n;
    dn = (m / geglu_half) * (2 * geglu_half) + g * geglu_half + (m % geglu_half);
  }
  if (h3_dh > 0) {
    const int g = h3_head_off + n / h3_dh;
    dn = (g / 3) * h3_bn + (g % 3) * h3_dh + n % h3_dh;
  }
  const float v = k < K ? src[(size_t)n * K + k] : 0.f;
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  __nv_bfloat16* o = dst + (size_t)dn * kmul * Kpad;
  o[k] = hi;
  if (kmul == 3) {
    o[Kpad + k] = hi;
    o[2 * Kpad + k] = __float2bfloat16_rn(v - __bfloat162float(hi));
  }
}
__global__ void pack_geglu_bias_kernel(const float* __restrict__ src, float* __restrict__ dst, int inner, int half) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= 2 * inner) return;
  const int g = n >= inner, m = g ? n - inner : n;
  dst[(m / half) * (2 * half) + g * half + (m % half)] = src[n];
}
// generic strided permute copy fp32: dst[a, b, c] = src[...]: used for conv weight transposes at load time
__global__ void permute3_kernel(const float* __restrict__ src, float* __restrict__ dst, int d0, int d1, int d2, int s0, int s1, int s2) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)d0 * d1 * d2) return;
  const int c = i % d2, b = (i / d2) % d1, a = i / ((size_t)d1 * d2);
  dst[i] = src[(size_t)a * s0 + (size_t)b * s1 + (size_t)c * s2];
}

// ---------------------------------------------------------------------------------------------------------------
// Classifier-free guidance + rescale (src/inference.py:12-23,88-93) fused with the DDIM v-prediction update
// (diffusers DDIMScheduler.step, SURVEY Appendix B).  coef = {sqrt(a), sqrt(1-a), sqrt(a_prev), sqrt(1-a_prev-sigma^2), sigma}.
// One CLUSTER of CFG_CLUSTER CTAs per sample (one CTA per sample would leave all but a handful of SMs idle):
// every CTA reduces the four sums of its slice (double accumulation, fixed order -> deterministic), the partials are exchanged
// through distributed shared memory, every CTA forms the same ratio and updates its slice.
// Tensors are [B, C, L].  lens ([B] device, or null = L): sample b covers the first lens[b] frames of each channel.  Its n = C * lens[b]
// elements are walked in the order of a solo call on a [1, C, lens[b]] tensor (element i at (i / lens[b]) * L + i % lens[b]), so sums and
// updates are bit-identical to that call; the padded frames are not touched.
// CFG_CLUSTER and cfg_update_sample, the update of one sample by its cluster: cfg_update.cuh.
__global__ void __launch_bounds__(1024) cfg_ddim_kernel(const float* __restrict__ out_text, const float* __restrict__ out_uncond, float* __restrict__ latents,
                                                        const float* __restrict__ noise, const int32_t* __restrict__ lens, int C, int L, float gs, float gr,
                                                        float c0, float c1, float c2, float c3, float c4) {
  pdl_launch();
  pdl_wait();
  cfg_update_sample<false>(out_text, out_uncond, latents, noise, lens, blockIdx.x / CFG_CLUSTER, C, L, gs, gr, c0, c1, c2, c3, c4);
}
// The same update with the constants of each sample read from its slot (ezb_ddim_slot, device memory), so that one captured launch serves
// samples at different points of different schedules.  out_uncond = the B uncond rows, used by slots with EZB_SLOT_CFG; a slot without
// EZB_SLOT_ACTIVE leaves its latents untouched; noise is read only by slots with sigma != 0.
__global__ void __launch_bounds__(1024) cfg_ddim_slots_kernel(const float* __restrict__ out_text, const float* __restrict__ out_uncond,
                                                              float* __restrict__ latents, const float* __restrict__ noise,
                                                              const int32_t* __restrict__ lens, const ezb_ddim_slot* __restrict__ slots, int C, int L) {
  pdl_launch();
  pdl_wait();
  const int sample = blockIdx.x / CFG_CLUSTER;
  const ezb_ddim_slot s = slots[sample];
  if (!(s.flags & EZB_SLOT_ACTIVE)) return;   // every CTA of the cluster reads the same slot: the cluster leaves whole, before any cluster barrier
  cfg_update_sample<false>(out_text, (s.flags & EZB_SLOT_CFG) ? out_uncond : nullptr, latents, s.coef[4] != 0.f ? noise : nullptr, lens, sample, C, L,
                           s.guidance_scale, s.guidance_rescale, s.coef[0], s.coef[1], s.coef[2], s.coef[3], s.coef[4]);
}

// Classifier-free guidance + rescale fused with the DPM-Solver++ multistep update (diffusers DPMSolverMultistepScheduler, dpmsolver++ and
// sde-dpmsolver++, midpoint; ezaudio_b200/scheduler.py): cfg_update_sample<true>, the same clusters, slices, element order and rescale
// reduction as the DDIM update.  Per element, with v the guided model output and c = ezb_dpm_slot.coef = {alpha_s, sigma_s, kx, k0, k1, r, kz}:
//   m0 = alpha_s x - sigma_s v ;  x <- kx x + k0 m0 [+ k1 (r (m0 - m1))]_order2 [+ kz z]_noise ;  history <- m0
// m1 (the previous step's m0) is read from history only at order 2; noise null: kz == 0.
__global__ void __launch_bounds__(1024) cfg_dpm_kernel(const float* __restrict__ out_text, const float* __restrict__ out_uncond, float* __restrict__ latents,
                                                       float* __restrict__ history, const float* __restrict__ noise, const int32_t* __restrict__ lens,
                                                       int C, int L, const ezb_dpm_slot s) {
  pdl_launch();
  pdl_wait();
  cfg_update_sample<true>(out_text, out_uncond, latents, noise, lens, blockIdx.x / CFG_CLUSTER, C, L, s.guidance_scale, s.guidance_rescale, s.coef[0],
                          s.coef[1], s.coef[2], s.coef[3], s.coef[4], s.coef[5], s.coef[6], history, (s.flags & EZB_SLOT_ORDER2) != 0);
}
// Per-sample constants from ezb_dpm_slot (device memory), as cfg_ddim_slots_kernel: a slot without EZB_SLOT_ACTIVE (a free slot, or one that
// runs DDIM) leaves its latents and history untouched; noise is read only by slots with kz != 0.
__global__ void __launch_bounds__(1024) cfg_dpm_slots_kernel(const float* __restrict__ out_text, const float* __restrict__ out_uncond,
                                                             float* __restrict__ latents, float* __restrict__ history, const float* __restrict__ noise,
                                                             const int32_t* __restrict__ lens, const ezb_dpm_slot* __restrict__ slots, int C, int L) {
  pdl_launch();
  pdl_wait();
  const int sample = blockIdx.x / CFG_CLUSTER;
  const ezb_dpm_slot s = slots[sample];
  if (!(s.flags & EZB_SLOT_ACTIVE)) return;   // the cluster leaves whole, before any cluster barrier
  cfg_update_sample<true>(out_text, (s.flags & EZB_SLOT_CFG) ? out_uncond : nullptr, latents, s.coef[6] != 0.f ? noise : nullptr, lens, sample, C, L,
                          s.guidance_scale, s.guidance_rescale, s.coef[0], s.coef[1], s.coef[2], s.coef[3], s.coef[4], s.coef[5], s.coef[6], history,
                          (s.flags & EZB_SLOT_ORDER2) != 0);
}

// Per-sample modulation rows from DEVICE timestep indices (Dit::select_mod): sample b gets row t_index[b] (clamped to [0, n_t)) of the AdaLN
// table mod [n_t, ldm4 float4] and of the FinalBlock table modf [n_t, ldf4 float4] (null: none) in mod_b / modf_b.  The indices are read when
// the kernel runs, so a replayed graph follows later copies into them.
__global__ void __launch_bounds__(256) gather_mod_kernel(const int32_t* __restrict__ t_index, int n_t, const float4* __restrict__ mod, int ldm4,
                                                         const float4* __restrict__ modf, int ldf4, float4* __restrict__ mod_b, float4* __restrict__ modf_b) {
  pdl_launch();
  pdl_wait();
  const int b = blockIdx.y;
  const int t = min(max(t_index[b], 0), n_t - 1);
  const int n = ldm4 + (modf ? ldf4 : 0);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (i < ldm4) mod_b[(size_t)b * ldm4 + i] = mod[(size_t)t * ldm4 + i];
    else modf_b[(size_t)b * ldf4 + (i - ldm4)] = modf[(size_t)t * ldf4 + (i - ldm4)];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Tables of the folded LayerNorm (gemm.cuh, FoldIn / FoldOut), built once per schedule by ezb_dit_set_timesteps:
//   G[t][k] = w[k] (1 + scale_t[k]),  C[t][k] = b[k] (1 + scale_t[k]) + shift_t[k]            (fold_gc_kernel; no modulation: G = w, C = b)
//   U[t][n] = sum_k G[t][k] W[n][k],  V[t][n] = sum_k C[t][k] W[n][k] (+ bias[n])             (fold_uv_kernel; W = the PACKED bf16 weight the
//   GEMM itself multiplies with, so U and V are in the GEMM's own column order and consistent with its operand rounding)
__global__ void fold_gc_kernel(const float* __restrict__ w, const float* __restrict__ b, const float* __restrict__ shift, const float* __restrict__ scale,
                               int ld_mod, float* __restrict__ G, float* __restrict__ Cc, int R, int D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * D) return;
  const int r = i / D, k = i - r * D;
  const float sc = scale ? scale[(size_t)r * ld_mod + k] : 0.f, sh = shift ? shift[(size_t)r * ld_mod + k] : 0.f;
  G[i] = w[k] * (1.f + sc);
  Cc[i] = b[k] * (1.f + sc) + sh;
}
__global__ void __launch_bounds__(256) fold_uv_kernel(const __nv_bfloat16* __restrict__ W, int ldw, const float* __restrict__ G, const float* __restrict__ Cc,
                                                      const float* __restrict__ add_v, float* __restrict__ U, float* __restrict__ V, int N, int K, int R) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (n >= N) return;
  constexpr int MAXK = 72;  // K <= 2304 (the normalised width: D, or 2 D on the skip path)
  float w[MAXK];
#pragma unroll
  for (int i = 0; i < MAXK; ++i) { const int k = lane + 32 * i; w[i] = k < K ? __bfloat162float(W[(size_t)n * ldw + k]) : 0.f; }
  const float add = add_v ? add_v[n] : 0.f;
  for (int r = 0; r < R; ++r) {
    float su = 0.f, sv = 0.f;
#pragma unroll
    for (int i = 0; i < MAXK; ++i) {
      const int k = lane + 32 * i;
      if (k < K) { su = fmaf(w[i], G[(size_t)r * K + k], su); sv = fmaf(w[i], Cc[(size_t)r * K + k], sv); }
    }
    su = warp_sum(su); sv = warp_sum(sv);
    if (lane == 0) { U[(size_t)r * N + n] = su; V[(size_t)r * N + n] = sv + add; }
  }
}

// timestep values of ezb_dit_set_timesteps, passed BY VALUE in chunks (no host staging buffer, so the call needs no synchronisation)
struct TimestepChunk { float v[240]; };
__global__ void fill_timesteps_kernel(float* __restrict__ dst, const TimestepChunk c, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = c.v[i];
}

}  // namespace ezb

namespace ezb {
// Direct 1-D convolution for the (tiny) ControlNet stem (controlnet.py:29-36,65-84): one thread per output element.
// in [B,Cin,Tin] (channel cin_real..Cin-1 read as zero: the eval-time all-zero mask channel), out [B,Cout,Tout] or
// transposed [B,Tout,Cout].
__global__ void conv1d_direct_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ out, int B,
                                     int Cin, int cin_real, int Tin, int Cout, int Tout, int K, int stride, int pad, int act, int transposed) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * Cout * Tout) return;
  int b, co, t;
  if (transposed) { co = i % Cout; t = (i / Cout) % Tout; b = i / ((size_t)Cout * Tout); }
  else { t = i % Tout; co = (i / Tout) % Cout; b = i / ((size_t)Cout * Tout); }
  float acc = bias[co];
  for (int ci = 0; ci < cin_real; ++ci)
    for (int k = 0; k < K; ++k) {
      const int ti = t * stride + k - pad;
      if (ti >= 0 && ti < Tin) acc = fmaf(w[((size_t)co * Cin + ci) * K + k], in[((size_t)b * cin_real + ci) * Tin + ti], acc);
    }
  if (act == 1) acc = silu(acc);
  out[i] = acc;
}
}  // namespace ezb

namespace ezb {
// ---------------------------------------------------------------------------------------------------------------------------------
// EnergyExtractor (src/models/conditions/energy.py:19-56): per frame f (hop `hop`, window `win`, reflect padding (win-hop)/2 both sides)
//   e_f = mean_{j<win} a[reflect(f*hop + j - pad)]^2 ; g_f = 10*log10(max(e_f, 10^(min_db/10)))
//   norm: g_f = (g_f - min_db) / (max_f g_f - min_db + 1e-8) ; quantize_levels q>0: round(g*(q-1))/(q-1).
// One CTA per clip: the frame energies stay in shared memory between the reduction over frames and the normalisation.
// Memory-bound (each sample is read win/hop = 8 times, all but the first from L1/L2); runs once per generate call.
__global__ void __launch_bounds__(1024) energy_kernel(const float* __restrict__ audio, float* __restrict__ out, int T, int n_frames, int hop,
                                                      int win, float min_db, float floor_e, int norm, int qlevels) {
  extern __shared__ float e_db[];  // n_frames
  __shared__ float red[32];
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* a = audio + (size_t)b * T;
  const int pad = (win - hop) / 2;
  float wmax = -INFINITY;
  for (int f = warp; f < n_frames; f += nw) {
    float acc = 0.f;
    const int base = f * hop - pad;
    for (int j = lane; j < win; j += 32) {
      int i = base + j;
      if (i < 0) i = -i;                      // F.pad(mode='reflect'): no edge repeat
      if (i >= T) i = 2 * (T - 1) - i;
      const float v = __ldg(a + i);
      acc = fmaf(v, v, acc);
    }
    acc = warp_sum(acc);
    const float g = 10.f * log10f(fmaxf(acc / (float)win, floor_e));
    if (lane == 0) e_db[f] = g;
    wmax = fmaxf(wmax, g);
  }
  if (lane == 0) red[warp] = wmax;
  __syncthreads();
  float mx = red[0];
  for (int i = 1; i < nw; ++i) mx = fmaxf(mx, red[i]);
  for (int f = threadIdx.x; f < n_frames; f += blockDim.x) {
    float g = e_db[f];
    if (norm) g = (g - min_db) / (mx - min_db + 1e-8f);
    if (qlevels > 1) g = rintf(g * (float)(qlevels - 1)) / (float)(qlevels - 1);
    out[(size_t)b * n_frames + f] = g;
  }
}
}  // namespace ezb

namespace ezb {
// ---------------------------------------------------------------------------------------------------------------------------------
// Waveform pre / post-processing around the path (SURVEY 8(f) row 4), device-side so that clips never bounce through the host:
//   wave_prepare : gt / (max|gt| + 1e-9), optional noise gate |x| <= thr -> 0, pad / crop to T_out   (api/ezaudio.py:147,
//                  api/controlnet.py:119-133).  One CTA per clip: block max-abs reduction, then a scaled copy.
//   wave_splice  : output_audio[start : start + n] = pred[:n]                                         (api/ezaudio.py:198-203)
//   wave_to_pcm16: float -> 16-bit PCM with saturation (soundfile.write's default WAV subtype)         (t2a_demo.py:13,20)
// All three are HBM-bound copies: 4-8 bytes per sample.
__global__ void __launch_bounds__(1024) wave_prepare_kernel(const float* __restrict__ in, float* __restrict__ out, int T_in, int T_out, float eps,
                                                            float gate, int normalize) {
  __shared__ float red[32];
  __shared__ float inv_s;
  const int b = blockIdx.x;
  const float* a = in + (size_t)b * T_in;
  float inv = 1.f;
  if (normalize) {
    float m = 0.f;
    for (int i = threadIdx.x; i < T_in; i += blockDim.x) m = fmaxf(m, fabsf(a[i]));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      float mx = red[0];
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
      inv_s = mx + eps;
    }
    __syncthreads();
    inv = inv_s;
  }
  float* o = out + (size_t)b * T_out;
  for (int i = threadIdx.x; i < T_out; i += blockDim.x) {
    float v = 0.f;
    if (i < T_in) {
      v = normalize ? a[i] / inv : a[i];   // a true division like numpy's (not a reciprocal multiply): bit-identical to the reference's float32 result
      if (gate > 0.f && fabsf(v) <= gate) v = 0.f;
    }
    o[i] = v;
  }
}
__global__ void wave_splice_kernel(float* __restrict__ dst, const float* __restrict__ src, long long start, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[start + i] = src[i];
}
__global__ void wave_to_pcm16_kernel(const float* __restrict__ in, int16_t* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = fminf(fmaxf(in[i] * 32768.0f, -32768.0f), 32767.0f);
  out[i] = (int16_t)__float2int_rn(v);
}
}  // namespace ezb
