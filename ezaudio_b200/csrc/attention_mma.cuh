// Tensor-core flash attention for sm_90a: O = softmax(Q K^T / sqrt(dh) [+ key mask]) V.
// Replaces F.scaled_dot_product_attention in src/models/utils/attention.py:107-110 (self: mask None; cross: bool key mask built
// by attention.py:30-37).
//
// A warp owns 16 query rows of one (b, h) and walks all key blocks with the online softmax (running max / sum in fp32, exp2 domain).
// S = Q K^T and O += P V are mma.sync m16n8k16 (bf16 in, fp32 accumulate); the S accumulator fragments are re-packed in registers as
// the bf16 A fragments of P, so P never leaves the registers.  K and V^T blocks are staged in shared memory with cp.async (zero fill
// beyond the true length and beyond dh).  Variants (the A/B options of attention_variant()):
//   generation 6 (default)  4 warps = 64 query rows per CTA, 64-key blocks, double-buffered
//   generation 4            8 warps = 128 query rows per CTA (each K / V^T block feeds twice as many rows)
//     + RES                 one CTA per (b, h): all key blocks of the head (Lk <= 512) are loaded once and stay resident while the CTA
//                           walks every query tile of that head (K / V^T read from L2 once per head instead of once per query tile)
//   generation 7            4 warps, 128-key blocks (half as many block barriers and rescales per key)
//   generation 8 (default for dh 64 / 72)  TMA-fed, warp-specialised wgmma kernel of attention_wgmma.cuh; other head dims run generation 6
// Layouts as produced by the QKV GEMM epilogue: Q, K [B*H, L, DHP] bf16; V^T [B*H, DVP, Lkpad] bf16.  Output [B, Lq, H*dh] bf16
// token-major.
// Padded batches (self-attention of clips of different lengths, p.lens): sample b holds len = lens[b] valid tokens.  Keys at or past len are
// zero-filled like the keys past Lk of a solo run, so valid rows see exactly what a run at Lq = Lk = len sees (bit-identical) and nothing
// in the padded tokens (not even NaN) reaches them; query rows at or past len are written as zeros.  Those kernels are the VARLEN = true
// instantiations; without lens the VARLEN = false ones run, compiled without any of this.
#pragma once
#include "attention_wgmma.cuh"
#include "host.cuh"

namespace ezb {

constexpr int AM_RES_KEYS = 512;   // longest key sequence the resident variant holds

__device__ __forceinline__ void cp_async16(void* dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

struct AttnMmaParams {
  const __nv_bfloat16 *q, *k, *vt;
  const uint8_t* key_mask;  // [B, Lk] or null
  const int32_t* lens;      // [B] valid tokens per sample (device; clamped to [1, min(Lq, Lk)]) or null: all Lq / Lk valid
  __nv_bfloat16* out;       // [B, Lq, H*dh]
  int H, Lq, Lk, Lkpad, dh, dhp, dvp;
  float scale_log2;         // (1/sqrt(dh)) * log2(e)
  int poly;                 // exponentials on the FMA pipe (one in four, ex2_poly): 0 none, 1 every warp, 2 odd warps only
  int halves;               // 1: the P V MMAs of a key block are issued after each half of its P; 0: after each 16-key slice
  int dbg;                  // profiling only (results are garbage): 1 no exp2, 8 no P V MMAs, 16 no S MMAs
};

// 2^x on the FMA pipe (Cody-Waite split + degree-3 minimax polynomial on [-0.5, 0.5], max relative error 7.8e-5 -- far below the bf16
// rounding of P): used for one element in four so that the MUFU is not the only unit working through the scores.
__device__ __forceinline__ float ex2_poly(float x) {
  x = fmaxf(x, -125.f);
  const float t = x + 12582912.f;          // 1.5 * 2^23: the integer part lands in the low mantissa bits
  const float f = x - (t - 12582912.f);    // [-0.5, 0.5]
  float q = fmaf(0.05508868f, f, 0.24260405f);
  q = fmaf(q, f, 0.69327623f);
  q = fmaf(q, f, 0.99992895f);
  return __int_as_float(__float_as_int(q) + (__float_as_int(t) << 23));
}

// DK: dh rounded up to 16 (the MMA K of Q K^T and the N of P V); WARPS x 16 query rows per tile; KB keys per block
template <int DK, int KB>
struct AttnMmaSmem {
  static constexpr int KP = DK + 8;   // smem pitches (bf16): 16 B of padding puts the fragment reads of a warp on distinct banks
  static constexpr int VP = KB + 8;
  static constexpr int K_ELEMS = KB * KP, V_ELEMS = DK * VP;
  static constexpr size_t bytes(int nbuf) { return (size_t)nbuf * (K_ELEMS + V_ELEMS) * sizeof(__nv_bfloat16); }
};
template <int DK, int WARPS, int KB, bool RES, bool VARLEN>
__global__ void __launch_bounds__(WARPS * 32) attn_mma_kernel(const AttnMmaParams p) {
  using SM = AttnMmaSmem<DK, KB>;
  constexpr int KP = SM::KP, VP = SM::VP;
  constexpr int NT = DK / 8;        // 8-column tiles of O
  constexpr int QROWS = 16 * WARPS;
  extern __shared__ __align__(16) uint8_t am_smem[];
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(am_smem);                                   // [nbuf][KB * KP]
  __nv_bfloat16* sV = sK + (RES ? AM_RES_KEYS / KB : 2) * SM::K_ELEMS;                               // [nbuf][DK * VP]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y, b = bh / p.H, h = bh - b * p.H;
  const __nv_bfloat16* kb = p.k + (size_t)bh * p.Lk * p.dhp;
  const __nv_bfloat16* vb = p.vt + (size_t)bh * p.dvp * p.Lkpad;
  const uint8_t* mask = p.key_mask != nullptr ? p.key_mask + (size_t)b * p.Lk : nullptr;
  // valid keys / query rows of this sample.  The 128-key-block variants have no register to spare across the key loop (ptxas spills): they
  // re-read the length where it is needed instead of holding it.
  auto valid = [&](int n) { return VARLEN ? min(max(p.lens[b], 1), n) : n; };
  const int lk0 = valid(p.Lk), lq0 = valid(p.Lq);
  auto klen = [&] { return KB == 128 ? valid(p.Lk) : lk0; };
  auto qlen = [&] { return KB == 128 ? valid(p.Lq) : lq0; };
  const int nblk = (lk0 + KB - 1) / KB;
  const int nqt = (p.Lq + QROWS - 1) / QROWS;
  const bool use_poly = p.poly == 1 || (p.poly == 2 && (warp & 1));   // warp-uniform
  const bool no_exp = p.dbg & 1, no_pv = p.dbg & 8, no_s = p.dbg & 16;

  auto load_block = [&](int buf, int k0) {
    const int lk = klen();
    __nv_bfloat16* dK = sK + buf * SM::K_ELEMS;
    __nv_bfloat16* dV = sV + buf * SM::V_ELEMS;
    for (int c = threadIdx.x; c < KB * (DK / 8); c += WARPS * 32) {   // K rows: 8-column chunks
      const int r = c / (DK / 8), col = (c - r * (DK / 8)) * 8, key = k0 + r;
      const bool ok = key < lk && col < p.dh;
      cp_async16(dK + r * KP + col, ok ? kb + (size_t)key * p.dhp + col : kb, ok ? 16 : 0);
    }
    for (int c = threadIdx.x; c < DK * (KB / 8); c += WARPS * 32) {   // V^T rows: 8-key chunks
      const int d = c / (KB / 8), key = k0 + (c - d * (KB / 8)) * 8;
      const int n = d < p.dh ? (lk - key < 8 ? lk - key : 8) : 0;
      cp_async16(dV + d * VP + key - k0, n > 0 ? vb + (size_t)d * p.Lkpad + key : vb, n > 0 ? 2 * n : 0);
    }
    cp_async_commit();
  };
  if (RES) {   // every key block of the head, once
    for (int blk = 0; blk < nblk; ++blk) load_block(blk, blk * KB);
    cp_async_wait<0>();
    __syncthreads();
  }

  for (int qt = RES ? 0 : blockIdx.x; qt < (RES ? nqt : blockIdx.x + 1); ++qt) {
    const int q0 = qt * QROWS + warp * 16;
    if (VARLEN && qt * QROWS >= qlen()) {   // a tile of padded query rows (CTA-uniform): zeros, no key block is loaded
      __nv_bfloat16* ob = p.out + (size_t)b * p.Lq * (p.H * p.dh) + (size_t)h * p.dh;
      for (int i = threadIdx.x; i < QROWS * (p.dh / 2); i += WARPS * 32) {
        const int r = qt * QROWS + i / (p.dh / 2), col = 2 * (i % (p.dh / 2));
        if (r < p.Lq) *reinterpret_cast<uint32_t*>(ob + (size_t)r * (p.H * p.dh) + col) = 0u;
      }
      continue;
    }
    if (!RES) load_block(0, 0);
    // Q fragments of this warp's 16 rows, zero beyond the sample's valid rows and beyond dh
    uint32_t qa[DK / 16][4];
    {
      const int lq = qlen();
      const __nv_bfloat16* qb = p.q + (size_t)bh * p.Lq * p.dhp;
#pragma unroll
      for (int ks = 0; ks < DK / 16; ++ks) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = q0 + g + 8 * (i & 1), col = ks * 16 + 2 * t + 8 * (i >> 1);
          qa[ks][i] = (row < lq && col < p.dh) ? *reinterpret_cast<const uint32_t*>(qb + (size_t)row * p.dhp + col) : 0u;
        }
      }
    }
    float o[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows g and g + 8

    for (int blk = 0; blk < nblk; ++blk) {
      const int k0 = blk * KB, buf = RES ? blk : (blk & 1);
      if (!RES) {
        if (blk + 1 < nblk) { load_block(buf ^ 1, k0 + KB); cp_async_wait<1>(); }
        else cp_async_wait<0>();
        __syncthreads();
      }
      const __nv_bfloat16* K = sK + buf * SM::K_ELEMS;
      const __nv_bfloat16* V = sV + buf * SM::V_ELEMS;
      float s[KB / 8][4];
#pragma unroll
      for (int j = 0; j < KB / 8; ++j) {
        s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
        if (no_s) continue;
#pragma unroll
        for (int ks = 0; ks < DK / 16; ++ks) {
          const __nv_bfloat16* kr = K + (8 * j + g) * KP + ks * 16 + 2 * t;
          mma_bf16_16816(s[j], qa[ks], *reinterpret_cast<const uint32_t*>(kr), *reinterpret_cast<const uint32_t*>(kr + 8));
        }
      }
      // scale, key mask, block row max
      float bm0 = -INFINITY, bm1 = -INFINITY;
      const int lk = klen();
#pragma unroll
      for (int j = 0; j < KB / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = k0 + 8 * j + 2 * t + e;
          const bool ok = key < lk && (mask == nullptr || mask[key] != 0);
          s[j][e] = ok ? s[j][e] * p.scale_log2 : -INFINITY;
          s[j][2 + e] = ok ? s[j][2 + e] * p.scale_log2 : -INFINITY;
          bm0 = fmaxf(bm0, s[j][e]);
          bm1 = fmaxf(bm1, s[j][2 + e]);
        }
      }
#pragma unroll
      for (int o2 = 1; o2 <= 2; o2 <<= 1) {
        bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, o2));
        bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, o2));
      }
      const float nm0 = fmaxf(m0, bm0), nm1 = fmaxf(m1, bm1);
      const float off0 = nm0 == -INFINITY ? 0.f : nm0, off1 = nm1 == -INFINITY ? 0.f : nm1;   // a row with no valid key yet
      const float c0 = exp2f(m0 - off0), c1 = exp2f(m1 - off1);
      m0 = nm0; m1 = nm1;
      l0 *= c0; l1 *= c1;
#pragma unroll
      for (int j = 0; j < NT; ++j) { o[j][0] *= c0; o[j][1] *= c0; o[j][2] *= c1; o[j][3] *= c1; }
      // P = exp2(s - m) -> bf16 A fragments (two adjacent 8-key tiles = one 16-key MMA step); the P V MMAs follow each 16-key slice or,
      // with p.halves, each half of the block
      constexpr int HALF = KB / 32;
      uint32_t pa[KB / 16][4];
      auto pv = [&](int kk) {
        if (no_pv) return;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const __nv_bfloat16* vr = V + (8 * j + g) * VP + kk * 16 + 2 * t;
          mma_bf16_16816(o[j], pa[kk], *reinterpret_cast<const uint32_t*>(vr), *reinterpret_cast<const uint32_t*>(vr + 8));
        }
      };
#pragma unroll
      for (int kk = 0; kk < KB / 16; ++kk) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int j = 2 * kk + hh;
          float p0, p1, p2, p3;
          if (no_exp) {
            p0 = s[j][0]; p1 = s[j][1]; p2 = s[j][2]; p3 = s[j][3];
          } else {
            p0 = exp2f(s[j][0] - off0); p1 = exp2f(s[j][1] - off0); p2 = exp2f(s[j][2] - off1);
            p3 = use_poly ? ex2_poly(s[j][3] - off1) : exp2f(s[j][3] - off1);
          }
          const uint32_t lo = pack_bf16(p0, p1), hi = pack_bf16(p2, p3);
          // the row sums use the bf16-rounded probabilities the P V product sees
          const __nv_bfloat162 lo2 = *reinterpret_cast<const __nv_bfloat162*>(&lo), hi2 = *reinterpret_cast<const __nv_bfloat162*>(&hi);
          l0 += __low2float(lo2) + __high2float(lo2);
          l1 += __low2float(hi2) + __high2float(hi2);
          pa[kk][2 * hh] = lo;
          pa[kk][2 * hh + 1] = hi;
        }
        if (!p.halves) {
          pv(kk);
        } else if ((kk + 1) % HALF == 0) {
#pragma unroll
          for (int k2 = kk + 1 - HALF; k2 <= kk; ++k2) pv(k2);
        }
      }
      if (!RES) __syncthreads();   // the buffer is refilled by the next block's prefetch
    }
#pragma unroll
    for (int o2 = 1; o2 <= 2; o2 <<= 1) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, o2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, o2);
    }
    const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
    const int ld = p.H * p.dh;
    const int r0 = q0 + g, r1 = q0 + g + 8, lq = qlen();
    __nv_bfloat16* ob = p.out + (size_t)b * p.Lq * ld + (size_t)h * p.dh;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const int col = 8 * j + 2 * t;
      if (col < p.dh) {
        if (r0 < p.Lq) *reinterpret_cast<uint32_t*>(ob + (size_t)r0 * ld + col) = (!VARLEN || r0 < lq) ? pack_bf16(o[j][0] * i0, o[j][1] * i0) : 0u;
        if (r1 < p.Lq) *reinterpret_cast<uint32_t*>(ob + (size_t)r1 * ld + col) = (!VARLEN || r1 < lq) ? pack_bf16(o[j][2] * i1, o[j][3] * i1) : 0u;
      }
    }
  }
}

// Kernel variant selection (A/B switches, see the file comment).  opt_attn6: bit 0 = generation 6 (else 4); bit 1 = the odd warps of a
// generation-6 CTA take one exp2 in four on the FMA pipe while the even warps stay on the MUFU (the two warp halves share the SM's MUFU);
// bit 2 = generation 6 issues the P V MMAs after each half of a key block instead of after each 16-key slice.  opt_attn_pp: bit 1's
// split for generation 4.
constexpr int ATTN6_DEFAULT = 5;
inline int& opt_attn6() {
  static int v = [] { const char* e = getenv("EZB_ATTN6"); return e ? atoi(e) : ATTN6_DEFAULT; }();
  return v;
}
inline int& opt_attn7() {
  static int v = [] { const char* e = getenv("EZB_ATTN7"); return e ? atoi(e) : 0; }();
  return v;
}
inline int& opt_attn_res() {   // generation 4 with K / V^T resident per (b, h); falls back above AM_RES_KEYS keys
  static int v = [] { const char* e = getenv("EZB_ATTN_RES"); return e ? atoi(e) : 0; }();
  return v;
}
inline int& opt_attn_poly() {   // one exp2 in four on the FMA pipe (ex2_poly), every warp
  static int v = 0;
  return v;
}
inline int& opt_attn_dbg() {     // profiling only, see AttnMmaParams::dbg
  static int v = 0;
  return v;
}
inline int& opt_attn_pp() {
  static int v = [] { const char* e = getenv("EZB_ATTN_PP"); return e ? atoi(e) : 0; }();
  return v;
}
// generation 8 (attention_wgmma.cuh); it runs only while attn6 and attn7 are at their defaults, so that a non-default value of either still
// selects its generation
inline int& opt_attn8() {
  static int v = [] { const char* e = getenv("EZB_ATTN8"); return e ? atoi(e) : 1; }();
  return v;
}
inline int attention_variant() {
  if (opt_attn7()) return 7;
  if (opt_attn8() && opt_attn6() == ATTN6_DEFAULT) return 8;
  return (opt_attn6() & 1) ? 6 : 4;
}

template <int DK, int WARPS, int KB, bool RES>
int attn_mma_launch(cudaStream_t st, const AttnMmaParams& p, int B, int H) {
  auto kern = p.lens ? attn_mma_kernel<DK, WARPS, KB, RES, true> : attn_mma_kernel<DK, WARPS, KB, RES, false>;
  const size_t smem = AttnMmaSmem<DK, KB>::bytes(RES ? AM_RES_KEYS / KB : 2);
  static int attr_set[2] = {-1, -1};   // function attributes are per device and kernel
  int dev = 0;
  EZB_CUDA(cudaGetDevice(&dev));
  if (smem > 48 * 1024 && attr_set[p.lens != nullptr] != dev) {
    EZB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set[p.lens != nullptr] = dev;
  }
  const dim3 grid(RES ? 1 : (p.Lq + 16 * WARPS - 1) / (16 * WARPS), B * H);
  ++launch_counter();
  ++attn_launch_counts()[KB == 128 ? 7 : WARPS == 8 ? 4 : 6];
  kern<<<grid, WARPS * 32, smem, st>>>(p);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
template <int DK>
int attn_mma_dispatch(cudaStream_t st, const AttnMmaParams& p, int B, int H, int variant) {
  if (variant == 7) return attn_mma_launch<DK, 4, 128, false>(st, p, B, H);
  if (variant == 4) {
    if (opt_attn_res() && p.Lk <= AM_RES_KEYS) return attn_mma_launch<DK, 8, 64, true>(st, p, B, H);
    return attn_mma_launch<DK, 8, 64, false>(st, p, B, H);
  }
  return attn_mma_launch<DK, 4, 64, false>(st, p, B, H);
}

// variant: 4, 6, 7 or 8 (see the file comment); 0 = the one the options select (generation 8 falls back to 6 for a head dimension other
// than 64 or 72)
// lens: [B] valid tokens per sample (device) or null, see the file comment
inline int attention_mma(Device& dev, cudaStream_t st, const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* vt, const uint8_t* key_mask,
                         __nv_bfloat16* out, int B, int H, int Lq, int Lk, int Lkpad, int dh, int dhp, int dvp, float scale, int variant = 0,
                         const int32_t* lens = nullptr) {
  if (dh % 8 || dh > 80) return fail(EZB_ERR_UNSUPPORTED, "attention: head dimension %d (multiples of 8 up to 80)", dh);
  if (dhp < dh || dhp % 8 || dvp < dh || Lkpad < Lk || Lkpad % 8) return fail(EZB_ERR_SHAPE, "attention: pitches dhp %d dvp %d Lkpad %d", dhp, dvp, Lkpad);
  if (B < 1 || H < 1 || Lq < 1 || Lk < 1) return fail(EZB_ERR_SHAPE, "attention: empty problem");
  AttnMmaParams p;
  p.q = q; p.k = k; p.vt = vt; p.key_mask = key_mask; p.lens = lens; p.out = out;
  p.H = H; p.Lq = Lq; p.Lk = Lk; p.Lkpad = Lkpad; p.dh = dh; p.dhp = dhp; p.dvp = dvp;
  p.scale_log2 = scale * 1.4426950408889634f;
  const bool forced = variant != 0;
  if (variant == 0) variant = attention_variant();
  if (variant == 8) {
    if (dh == 64 || dh == 72 || forced) return attention_wgmma(dev, st, q, k, vt, key_mask, out, B, H, Lq, Lk, Lkpad, dh, dhp, dvp, scale, lens);
    variant = 6;
  }
  const bool split = (variant == 6 && (opt_attn6() & 2)) || (variant == 4 && opt_attn_pp());
  p.poly = opt_attn_poly() ? 1 : split ? 2 : 0;
  p.halves = variant == 6 && (opt_attn6() & 4);
  p.dbg = opt_attn_dbg();
  return dh <= 64 ? attn_mma_dispatch<64>(st, p, B, H, variant) : attn_mma_dispatch<80>(st, p, B, H, variant);
}

}  // namespace ezb
