// fp32 CUDA-core attention: softmax(q k^T * scale [+ bias] [+ key mask]) v   (attention.py:107-110, mask attention.py:30-37;
// with scale 1 and a relative-position bias: T5Attention).
// Used by the bf16x3 parity mode (fp32-grade numerics) and as the on-device comparator of the tensor-core kernel.
// q,k,v fp32 [B,H,L,dh]; out bf16 [B, Lq, H*dh] token-major (A operand of the output projection).
// lens ([B] device, or null): sample b holds lens[b] valid tokens (padded batch of clips of different lengths).  Keys at or past it are
// skipped like the keys past Lk of a solo run (same bits for the valid rows, nothing from the padded tokens reaches them); query rows at
// or past it are written as zeros.  VARLEN = false (lens null) compiles the uniform-length kernel without any of this.
#pragma once
#include "elementwise.cuh"

namespace ezb {

constexpr int SA_TK = 64;   // keys per smem tile
constexpr int SA_QW = 8;    // queries per warp
constexpr int SA_WARPS = 4;

// Shared-memory traffic is what bounds this kernel (one T5 layer: 160 heads x 100 x 100 x 64): round 2a read K values once per d and reused them for the
// warp's 8 queries but still issued 10 scalar LDS per 16 FMAs in the score loop and one SHFL per (key, query) in P V (512 per tile per warp).  Now
// (dh % 4 == 0): K rows at a 16-byte-aligned pitch whose quarter-warp LDS.128 phases are conflict-free, q / k / p read as float4 (10 LDS.128 per 64
// FMAs), and the probabilities go through a per-warp shared tile and come back as broadcast LDS.128 (no shuffles).  Every accumulator still sums in the
// same order (d ascending, keys ascending), so the output bits are unchanged.
template <bool VARLEN>
__global__ void __launch_bounds__(SA_WARPS * 32) attn_simt_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                                                  const uint8_t* __restrict__ key_mask, __nv_bfloat16* __restrict__ out, int H, int Lq,
                                                                  int Lk, int dh, float scale, int kmul, const int32_t* __restrict__ lens,
                                                                  const float* __restrict__ bias = nullptr /* [H, Lq, Lk] added to the scores (T5) */) {
  extern __shared__ __align__(16) float sm[];
  const int ldk = ((dh >> 2) & 1) ? dh : dh + 4;   // pitch / 4 odd: the 8 lanes of an LDS.128 phase hit 8 different 16-byte bank groups
  float* sK = sm;                       // [SA_TK][ldk]
  float* sV = sK + SA_TK * ldk;         // [SA_TK][dh]
  float* sQ = sV + SA_TK * dh;          // [SA_WARPS*SA_QW][dh]
  float* sP = sQ + SA_WARPS * SA_QW * dh;   // [SA_WARPS][SA_QW][SA_TK]
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * (SA_WARPS * SA_QW);
  const int D = H * dh;
  int lk = Lk, lq = Lq;   // valid keys / query rows of this sample
  if (VARLEN) {
    const int n = max(lens[b], 1);
    lk = min(n, lk); lq = min(n, lq);
  }
  if (VARLEN && q0 >= lq) {   // a tile of padded query rows (CTA-uniform): zeros
    for (int i = threadIdx.x; i < SA_WARPS * SA_QW * dh; i += blockDim.x) {
      const int qrow = q0 + i / dh;
      if (qrow < Lq) store_act(out + ((size_t)b * Lq + qrow) * kmul * D, h * dh + i % dh, D, kmul, 0.f);
    }
    return;
  }
  const float* qb = q + (size_t)bh * Lq * dh;
  const float* kb = k + (size_t)bh * Lk * dh;
  const float* vb = v + (size_t)bh * Lk * dh;
  for (int i = threadIdx.x; i < SA_WARPS * SA_QW * dh; i += blockDim.x) {
    const int r = i / dh, d = i - r * dh;
    sQ[i] = (q0 + r < lq) ? qb[(size_t)(q0 + r) * dh + d] * scale : 0.f;
  }
  float m[SA_QW], l[SA_QW], acc[SA_QW][3];
#pragma unroll
  for (int i = 0; i < SA_QW; ++i) { m[i] = -INFINITY; l[i] = 0.f; acc[i][0] = acc[i][1] = acc[i][2] = 0.f; }
  float* sPw = sP + warp * (SA_QW * SA_TK);
  for (int k0 = 0; k0 < lk; k0 += SA_TK) {
    __syncthreads();
    for (int i = threadIdx.x; i < SA_TK * dh; i += blockDim.x) {
      const int r = i / dh, d = i - r * dh;
      const bool ok = k0 + r < lk;
      sK[r * ldk + d] = ok ? kb[(size_t)(k0 + r) * dh + d] : 0.f;
      sV[r * dh + d] = ok ? vb[(size_t)(k0 + r) * dh + d] : 0.f;
    }
    __syncthreads();
    const bool in0 = k0 + lane < lk, in1 = k0 + lane + 32 < lk;
    bool ok0 = in0, ok1 = in1;
    if (key_mask) {
      ok0 = ok0 && key_mask[(size_t)b * Lk + k0 + lane];
      ok1 = ok1 && key_mask[(size_t)b * Lk + k0 + lane + 32];
    }
    // A masked key scores -inf, so a query whose keys are all masked has l = 0 and is written as zeros (as the tensor-core kernels and SDPA
    // do).  T5 (bias != null) masks additively with finfo(float32).min instead, as transformers does: the masked scores all stay -FLT_MAX
    // after the subtract a - mn, so a fully masked row becomes the mean of V over the lk keys.  The zero-filled tile padding past lk stays
    // -inf in both modes.
    const float masked = bias != nullptr ? -3.40282347e38f : -INFINITY;
    // scores of this warp's SA_QW queries against the lane's two keys
    float s0[SA_QW], s1[SA_QW];
#pragma unroll
    for (int qi = 0; qi < SA_QW; ++qi) { s0[qi] = 0.f; s1[qi] = 0.f; }
    const float* qw = sQ + (warp * SA_QW) * dh;
    const float* kr0 = sK + lane * ldk;
    const float* kr1 = sK + (lane + 32) * ldk;
#pragma unroll 2
    for (int d = 0; d < dh; d += 4) {
      const float4 ka = *reinterpret_cast<const float4*>(kr0 + d), kc = *reinterpret_cast<const float4*>(kr1 + d);
#pragma unroll
      for (int qi = 0; qi < SA_QW; ++qi) {
        const float4 qv = *reinterpret_cast<const float4*>(qw + qi * dh + d);
        s0[qi] = fmaf(qv.w, ka.w, fmaf(qv.z, ka.z, fmaf(qv.y, ka.y, fmaf(qv.x, ka.x, s0[qi]))));
        s1[qi] = fmaf(qv.w, kc.w, fmaf(qv.z, kc.z, fmaf(qv.y, kc.y, fmaf(qv.x, kc.x, s1[qi]))));
      }
    }
#pragma unroll
    for (int qi = 0; qi < SA_QW; ++qi) {
      float a0 = s0[qi], a1 = s1[qi];
      if (bias != nullptr) {
        const int qrow = q0 + warp * SA_QW + qi;
        if (qrow < Lq) {
          const float* br = bias + ((size_t)h * Lq + qrow) * Lk + k0;
          if (k0 + lane < Lk) a0 += br[lane];
          if (k0 + lane + 32 < Lk) a1 += br[lane + 32];
        }
      }
      a0 = ok0 ? a0 : (in0 ? masked : -INFINITY);
      a1 = ok1 ? a1 : (in1 ? masked : -INFINITY);
      const float mn = fmaxf(m[qi], warp_max(fmaxf(a0, a1)));
      const float corr = (mn == -INFINITY) ? 1.f : expf(m[qi] - mn);
      const float p0 = (mn == -INFINITY) ? 0.f : expf(a0 - mn);
      const float p1 = (mn == -INFINITY) ? 0.f : expf(a1 - mn);
      l[qi] = l[qi] * corr + warp_sum(p0 + p1);
      m[qi] = mn;
      acc[qi][0] *= corr; acc[qi][1] *= corr; acc[qi][2] *= corr;
      sPw[qi * SA_TK + lane] = p0;
      sPw[qi * SA_TK + lane + 32] = p1;
    }
    __syncwarp();
    // P V: a V row is read once and reused by all queries; four keys' probabilities per broadcast LDS.128
    const bool d1 = lane + 32 < dh, d2 = lane + 64 < dh;
#pragma unroll 2
    for (int j = 0; j < SA_TK; j += 4) {
      float v0[4], v1[4], v2[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float* vr = sV + (j + t) * dh;
        v0[t] = vr[lane]; v1[t] = d1 ? vr[lane + 32] : 0.f; v2[t] = d2 ? vr[lane + 64] : 0.f;
      }
#pragma unroll
      for (int qi = 0; qi < SA_QW; ++qi) {
        const float4 pj = *reinterpret_cast<const float4*>(sPw + qi * SA_TK + j);
        const float pp[4] = {pj.x, pj.y, pj.z, pj.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          acc[qi][0] = fmaf(pp[t], v0[t], acc[qi][0]);
          acc[qi][1] = fmaf(pp[t], v1[t], acc[qi][1]);
          acc[qi][2] = fmaf(pp[t], v2[t], acc[qi][2]);
        }
      }
    }
    __syncwarp();   // the probabilities of this tile are consumed before the next tile overwrites them
  }
#pragma unroll
  for (int qi = 0; qi < SA_QW; ++qi) {
    const int qrow = q0 + warp * SA_QW + qi;
    if (qrow >= Lq) continue;
    const float inv = l[qi] > 0.f ? 1.f / l[qi] : 0.f;   // l = 0: every key masked (acc is 0 too)
    const bool valid = !VARLEN || qrow < lq;
    __nv_bfloat16* o = out + ((size_t)b * Lq + qrow) * kmul * D;
#pragma unroll
    for (int i = 0; i < 3; ++i)
      if (lane + 32 * i < dh) store_act(o, h * dh + lane + 32 * i, D, kmul, valid ? acc[qi][i] * inv : 0.f);
  }
}

// dh must be a multiple of 4 (float4 rows)
inline size_t attn_simt_smem(int dh) { return sizeof(float) * (SA_TK * (dh + 4) + SA_TK * dh + SA_WARPS * SA_QW * dh + SA_WARPS * SA_QW * SA_TK); }

}  // namespace ezb
