// Persistent warp-specialised wgmma GEMM for sm_90a:  C[M,N] = A[M,K] * W[N,K]^T  (bf16 in, fp32 accumulate)
//
//   last warp           TMA producer : cp.async.bulk.tensor tiles of A (128 x 64) and W (BN x 64) into a STAGES-deep smem ring
//   warpgroups 0..      consumers    : the first one or two warpgroups issue wgmma.mma_async m64nBNk16 (accumulator in registers,
//                                      64 rows per warpgroup; a single MMA warpgroup takes both 64-row halves), release each ring
//                                      slot once its MMAs have completed, then park the finished 128 x BN fp32 tile in shared memory
//                                      (over the ring, which is idle then); every consumer warp runs the fused epilogue on 32 rows
//                                      (thread == row) of it.  The producer refills the ring for the next tile once the epilogue is done.
//   An epilogue that works on the wgmma fragment itself (FRAG: the plain GEGLU, EpiGegluFrag, and the plain Q/K/V heads, EpiHeadsFrag) keeps
//   the accumulator out of the ring instead: the producer streams the next tile's k-blocks while the MMA warpgroups run the epilogue from
//   their registers.
//
// A can also be addressed as an implicit-GEMM operand of a 1-D convolution over channels-last activations
// [B, T, C]: k-block kb -> tap = kb / cin_blocks, rows shifted by (tap - center) * dilation with TMA zero fill at
// the clip edges (used by the Oobleck decoder: stable_vae/models/autoencoders.py:38-113).
//
// Reference ops this kernel replaces: every nn.Linear on the DiT step (src/models/utils/attention.py:127-129,148;
// src/models/utils/modules.py:266,366; src/models/blocks.py:101; src/models/udit.py:94-97) and the VAE's
// Conv1d / ConvTranspose1d (stable_vae/models/autoencoders.py:46-52,97-99,167,183).
#pragma once
#include "common.cuh"

namespace ezb {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
#ifdef EZB_GEMM_DEBUG
#define EZB_DBG(...) __VA_ARGS__
#else
#define EZB_DBG(...)
#endif
constexpr int GEMM_SMEM_BUDGET = 227 * 1024 - 2048;  // dynamic smem per CTA minus alignment slack and barriers
// Rows of one TMA box of the BN-row operand tile: boxes and wgmma N stop at 256, so a wider tile (the 288-token swap-AB tile) is loaded
// as two boxes and multiplied as two halves.
constexpr int gemm_b_box(int bn) { return bn > 256 ? bn / 2 : bn; }

struct GemmShape {
  int M, N;
  int num_k_blocks;    // K / 64 (rounded up; TMA zero-fills the tail)
  int num_m_tiles, num_n_tiles;
  // implicit-conv addressing of A (taps == 0 -> plain 2-D A[M,K])
  int taps, center, dilation, cin_blocks, T, tiles_per_batch;
  int stride, pad;     // stride > 1: strided conv (VAE encoder): A is a 4-D map [B, T/stride, stride, C], tap k reads row q*stride + k - pad
  unsigned long long* dbg;  // optional cycle counters of CTA 0 (builds with -DEZB_GEMM_DEBUG): [0] warpgroup 0 mainloop incl. its full-slot waits,
                            // [1] consumer wait for the accumulator tile (FRAG: for the output tile's previous store), [2] producer wait for
                            // empty slots, [3] unused, [4] warp 0 epilogue, [5] total
  // L2 prefetch of the weights the NEXT GEMM of the step will stream (host.cuh WeightSeq): every layer's weights are read once per step,
  // i.e. from HBM, and a kernel's first k-blocks pay that latency on top of its ramp.
  const char* pf;
  unsigned int pf_bytes;    // multiple of 16
};

// CTA c of `nctas` asks the L2 for its share (16 KB pieces, round-robin) of [pf, pf + bytes): a hint, no completion to wait for
__device__ __forceinline__ void prefetch_weights_l2(const char* pf, unsigned int bytes, unsigned int cta, unsigned int nctas) {
  constexpr unsigned int CH = 16384;
  for (unsigned int off = cta * CH; off < bytes; off += nctas * CH) {
    const unsigned int n = bytes - off < CH ? bytes - off : CH;
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(__cvta_generic_to_global(pf + off)), "r"(n) : "memory");
  }
}

enum { ACT_NONE = 0, ACT_SILU = 1, ACT_SNAKE = 2 };

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm folded into the GEMMs on either side of it (fast mode; blocks.py:137,149,155 and modules.py:15-16):
//     h = ((x - mu) * rstd) * g + c,   g = w (1 + scale), c = b (1 + scale) + shift        (LayerNorm affine + AdaLN modulate)
//     h W^T = rstd * ( (x g) W^T  -  mu * u ) + v,      u[n] = sum_k g[k] W[n,k],  v[n] = sum_k c[k] W[n,k]
// The GEMM that WRITES the residual stream x (FoldOut) also writes A = bf16(x * g) -- the operand of the GEMM that follows the
// LayerNorm -- and per-row partial sums (sum x, sum x^2), one slot per 32-feature lane group: slot-major [slots][ld_st], fixed
// summation order, so the result is deterministic.  The GEMM that FOLLOWS the LayerNorm (FoldIn) turns the partials into (mu, rstd)
// per row and applies the per-row affine to its accumulator.  No LayerNorm pass, no extra launch; u, v come from per-timestep tables.
struct FoldIn {
  const float2* st0;   // partials of the row (or of the first half of a concatenated row); null: no fold
  const float2* st1;   // second source (skip path: LayerNorm over [x | skip]) or null
  int slots0, slots1, ld_st;
  float inv_dim;       // 1 / (normalised width)
  const float* u;      // [N] in this GEMM's (packed) output-column order
  const float* v;
};
struct FoldOut {
  float2* st;          // null: nothing to emit
  int ld_st;
  __nv_bfloat16* a0; int ld0; const float* g0;   // a0[token, f] = bf16(x * g0[f])  (g0 null: plain cast)
  __nv_bfloat16* a1; int ld1; const float* g1;   // optional second consumer of the same x (null: none)
};
__device__ __forceinline__ void fold_row_stats(const FoldIn& f, int row, float& rstd, float& nmr) {
  float s1 = 0.f, s2 = 0.f;
#pragma unroll 4
  for (int s = 0; s < f.slots0; ++s) { const float2 p = f.st0[(size_t)s * f.ld_st + row]; s1 += p.x; s2 += p.y; }
#pragma unroll 4
  for (int s = 0; s < f.slots1; ++s) { const float2 p = f.st1[(size_t)s * f.ld_st + row]; s1 += p.x; s2 += p.y; }
  const float mean = s1 * f.inv_dim;
  const float var = fmaxf(s2 * f.inv_dim - mean * mean, 0.f);
  rstd = rsqrtf(var + 1e-5f);
  nmr = -mean * rstd;
}
// x[j] (j = 0..31) per lane -> lane L ends with sum over the 32 lanes of x[L]: 31 shuffles instead of 32 x 5
__device__ __forceinline__ float warp_transpose_sum(float (&x)[32], int lane) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const bool up = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < o; ++i) {
      const float send = up ? x[i] : x[i + o];
      const float keep = up ? x[i + o] : x[i];
      x[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
  return x[0];
}

// out_f32 receives the pre-activation value, out_bf16 the post-activation one (either may be null).
struct EpiLinearParams {
  const float* bias;       // [N] or [bias_mod]
  int bias_mod;            // 0: bias[col]; >0: bias[col % bias_mod] (conv-transpose phases share one bias)
  const float* resid;      // optional residual input, row stride ldr
  int ldr;
  const float* gate;       // optional: v = resid + (1 - gate[b, col]) * v, b = row / rows_per_batch
  int gate_bstride;
  int rows_per_batch;
  float* out_f32;
  int ld32;
  __nv_bfloat16* out_bf16;
  int ld16;
  int split_stride;        // >0: parity mode, write [hi | lo | hi] at col, col+s, col+2s
  int act;
  const float* act_a;      // snake: exp(alpha)[c], c = col % bias_mod (or col)
  const float* act_b;      // snake: 1 / (exp(beta)[c] + 1e-9)
  float out_scale;         // v = (acc + bias) * out_scale (before residual); 0 is treated as 1
  int phase_cols;          // >0 (conv-transpose): bf16 column = (col / phase_cols) * phase_ld16 + col % phase_cols
  int phase_ld16;
  FoldIn fin;              // swap-AB epilogue only: LayerNorm folded in / out (see above)
  FoldOut fout;
};

// ---------------------------------------------------------------------------------------------------------------
// The finished accumulator tile in shared memory, as an epilogue warp sees it: its 32 rows (row = lane), fp32, `pitch` floats apart.
// pitch = BN + 4 keeps the 16-byte row reads of 8 consecutive lanes on distinct banks.
struct AccRows {
  const float* base;
  int pitch;
};
template <int N>
__device__ __forceinline__ void acc_ld(const AccRows& a, int col, int lane, uint32_t* r) {
  const float4* p = reinterpret_cast<const float4*>(a.base + lane * a.pitch + col);
#pragma unroll
  for (int i = 0; i < N / 4; ++i) {
    const float4 v = p[i];
    r[4 * i] = __float_as_uint(v.x); r[4 * i + 1] = __float_as_uint(v.y); r[4 * i + 2] = __float_as_uint(v.z); r[4 * i + 3] = __float_as_uint(v.w);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Epilogue staging: a warp reads its 32 accumulator rows (thread == row), transposes 64-column chunks through
// a private 8 KB smem tile (XOR-swizzled 8-byte granules: conflict-free both ways) and then works with lane == column
// pair, so every global access is a fully coalesced 128/256-byte row segment.
constexpr int EPI_STAGE_FLOATS = 32 * 64;

template <int PITCH = 64>
__device__ __forceinline__ void stage_put(float* st, int r, int g, float a, float b) {
  *reinterpret_cast<float2*>(st + r * PITCH + 2 * (g ^ (r & (PITCH / 2 - 1)))) = make_float2(a, b);
}
template <int PITCH = 64>
__device__ __forceinline__ float2 stage_get(const float* st, int rr, int lane) {
  return *reinterpret_cast<const float2*>(st + rr * PITCH + 2 * (lane ^ (rr & (PITCH / 2 - 1))));
}
__device__ __forceinline__ void store_bf16x2(__nv_bfloat16* p, int split_stride, float a, float b) {
  const uint32_t hi = pack_bf16(a, b);
  *reinterpret_cast<uint32_t*>(p) = hi;
  if (split_stride > 0) {
    const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&hi);
    *reinterpret_cast<uint32_t*>(p + split_stride) = pack_bf16(a - __low2float(h), b - __high2float(h));
    *reinterpret_cast<uint32_t*>(p + 2 * split_stride) = hi;
  }
}

struct RowCtx {
  const float* st; int lane, nv, row0, brow;
  float b0, b1; float2 g0, g1; float sa0, sa1, sb0, sb1;
  float* o32; int ld32; __nv_bfloat16* o16; int ld16;
};
template <bool RESID, bool GATE, bool F32, bool BF16, int ACT>
__device__ __forceinline__ void rows_t(const RowCtx& c, const float2* x) {
  float* o32 = c.o32;
  __nv_bfloat16* o16 = c.o16;
#pragma unroll
  for (int rr = 0; rr < 32; ++rr) {
    if (rr >= c.nv) break;
    const float2 acc = stage_get(c.st, rr, c.lane);
    float v0 = acc.x + c.b0, v1 = acc.y + c.b1;
    if (RESID) {
      if (GATE) {
        const bool second = c.row0 + rr >= c.brow;
        v0 = fmaf(second ? c.g1.x : c.g0.x, v0, x[rr].x);
        v1 = fmaf(second ? c.g1.y : c.g0.y, v1, x[rr].y);
      } else {
        v0 += x[rr].x;
        v1 += x[rr].y;
      }
    }
    if (F32) { *reinterpret_cast<float2*>(o32) = make_float2(v0, v1); o32 += c.ld32; }
    if (BF16) {
      if (ACT == ACT_SILU) { v0 = silu(v0); v1 = silu(v1); }
      if (ACT == ACT_SNAKE) {  // bf16 throughput path: MUFU sine (the result is rounded to bf16); bf16x3 uses the exact sinf (rows_generic)
        const float s0 = __sinf(v0 * c.sa0), s1 = __sinf(v1 * c.sa1);
        v0 = fmaf(c.sb0 * s0, s0, v0);
        v1 = fmaf(c.sb1 * s1, s1, v1);
      }
      *reinterpret_cast<uint32_t*>(o16) = pack_bf16(v0, v1);
      o16 += c.ld16;
    }
  }
}
__device__ __forceinline__ void rows_generic(const EpiLinearParams& ep, const RowCtx& c, const float2* x, int col, int c16) {
  const float osc = ep.out_scale != 0.f ? ep.out_scale : 1.f;
#pragma unroll
  for (int rr = 0; rr < 32; ++rr) {
    if (rr >= c.nv) break;
    const int row = c.row0 + rr;
    const float2 acc = stage_get(c.st, rr, c.lane);
    float v0 = (acc.x + c.b0) * osc, v1 = (acc.y + c.b1) * osc;
    if (ep.resid != nullptr) {
      if (ep.gate != nullptr) {
        float2 g = row >= c.brow ? c.g1 : c.g0;
        if (ep.rows_per_batch < 32) {  // short clips (L < 32, api/ezaudio.py:160-172 crops to any length): a warp's rows span > 2 batch items
          g = *reinterpret_cast<const float2*>(ep.gate + (size_t)(row / ep.rows_per_batch) * ep.gate_bstride + col);
          g.x = 1.0f - g.x; g.y = 1.0f - g.y;
        }
        v0 = x[rr].x + g.x * v0;
        v1 = x[rr].y + g.y * v1;
      } else {
        v0 += x[rr].x;
        v1 += x[rr].y;
      }
    }
    if (ep.out_f32 != nullptr) *reinterpret_cast<float2*>(ep.out_f32 + (size_t)row * ep.ld32 + col) = make_float2(v0, v1);
    if (ep.out_bf16 != nullptr) {
      if (ep.act == ACT_SILU) {
        v0 = silu(v0);
        v1 = silu(v1);
      } else if (ep.act == ACT_SNAKE) {
        const float s0 = sinf(v0 * c.sa0), s1 = sinf(v1 * c.sa1);
        v0 = v0 + c.sb0 * s0 * s0;
        v1 = v1 + c.sb1 * s1 * s1;
      }
      store_bf16x2(ep.out_bf16 + (size_t)row * ep.ld16 + c16, ep.split_stride, v0, v1);
    }
  }
}

template <int BN>
struct EpiLinear {
  using Params = EpiLinearParams;
  static constexpr int EPI_WARPS = BN >= 128 ? 8 : 4;       // two warps per 32-row group split the tile's columns
  static constexpr bool WIDE_REGS = false;                  // true: run with GemmCfg::PRODUCER_WG
  static constexpr int STAGE_FLOATS = EPI_STAGE_FLOATS;
  // row0: global row of this warp's first accumulator row; nvalid: rows of the 32 that exist (<= 0: none);
  // [c_begin, c_end): this warp's column range inside the tile; wait(): blocks until the accumulator is complete.
  template <class Wait>
  static __device__ __forceinline__ void run(const Params& ep, float* st, const AccRows& ar, int row0, int nvalid, int n0, int N, int lane, int c_begin,
                                             int c_end, Wait wait) {
    const int nv = nvalid < 32 ? nvalid : 32;
    bool waited = false;
#pragma unroll 1
    for (int c = c_begin; c < c_end; c += 64) {
      const int col = n0 + c + 2 * lane;
      const bool col_ok = (c + 2 * lane < c_end) && col < N;
      // operands that do not depend on the accumulator are fetched first (and, for the first chunk, before the wait)
      float2 x[32];
      if (ep.resid != nullptr) {
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          x[i] = make_float2(0.f, 0.f);
          if (col_ok && i < nv) x[i] = *reinterpret_cast<const float2*>(ep.resid + (size_t)(row0 + i) * ep.ldr + col);
        }
      }
      float b0 = 0.f, b1 = 0.f, sa0 = 0.f, sa1 = 0.f, sb0 = 0.f, sb1 = 0.f;
      float2 g0 = make_float2(0.f, 0.f), g1 = g0;
      int brow = 0x7fffffff;  // first row that belongs to the second batch item touched by this warp
      if (col_ok) {
        const int ch = ep.bias_mod > 0 ? col % ep.bias_mod : col;
        if (ep.bias != nullptr) { b0 = ep.bias[ch]; b1 = ep.bias[ch + 1]; }
        if (ep.act == ACT_SNAKE) { sa0 = ep.act_a[ch]; sa1 = ep.act_a[ch + 1]; sb0 = ep.act_b[ch]; sb1 = ep.act_b[ch + 1]; }
        if (ep.gate != nullptr && nv > 0) {
          const int b0i = row0 / ep.rows_per_batch;
          brow = (b0i + 1) * ep.rows_per_batch;
          g0 = *reinterpret_cast<const float2*>(ep.gate + (size_t)b0i * ep.gate_bstride + col);
          if (brow < row0 + nv) g1 = *reinterpret_cast<const float2*>(ep.gate + (size_t)(b0i + 1) * ep.gate_bstride + col);
          g0.x = 1.0f - g0.x; g0.y = 1.0f - g0.y; g1.x = 1.0f - g1.x; g1.y = 1.0f - g1.y;
        }
      }
      if (!waited) { wait(); waited = true; }
      __syncwarp();
#pragma unroll
      for (int hc = 0; hc < 2; ++hc) {  // two 32-column halves: 32 accumulator registers live next to the 64 prefetched residual values (one 64-wide
        uint32_t r[32];                 // load spilled 780 bytes per thread under the 168-register cap of this 320-thread CTA)
        acc_ld<32>(ar, c + 32 * hc, lane, r);
#pragma unroll
        for (int g = 0; g < 16; ++g) stage_put(st, lane, 16 * hc + g, __uint_as_float(r[2 * g]), __uint_as_float(r[2 * g + 1]));
      }
      __syncwarp();
      if (col_ok) {
        const int c16 = ep.phase_cols > 0 ? (col / ep.phase_cols) * ep.phase_ld16 + col % ep.phase_cols : col;
        const int code = (ep.resid != nullptr ? 1 : 0) | (ep.gate != nullptr ? 2 : 0) | (ep.out_f32 != nullptr ? 4 : 0) | (ep.out_bf16 != nullptr ? 8 : 0) |
                         (ep.act << 4) | ((ep.split_stride > 0 || ep.out_scale != 0.f || (ep.gate != nullptr && ep.rows_per_batch < 32)) ? 256 : 0);
        const RowCtx rc{st, lane, nv, row0, brow, b0, b1, g0, g1, sa0, sa1, sb0, sb1,
                        ep.out_f32 != nullptr ? ep.out_f32 + (size_t)row0 * ep.ld32 + col : nullptr, ep.ld32,
                        ep.out_bf16 != nullptr ? ep.out_bf16 + (size_t)row0 * ep.ld16 + c16 : nullptr, ep.ld16};
        switch (code) {
          case 4: rows_t<false, false, true, false, ACT_NONE>(rc, x); break;             // bias -> f32
          case 7: rows_t<true, true, true, false, ACT_NONE>(rc, x); break;               // gated residual (in place)
          case 5: rows_t<true, false, true, false, ACT_NONE>(rc, x); break;              // residual
          case 8: rows_t<false, false, false, true, ACT_NONE>(rc, x); break;             // bf16
          case 8 | (ACT_SILU << 4): rows_t<false, false, false, true, ACT_SILU>(rc, x); break;
          case 8 | (ACT_SNAKE << 4): rows_t<false, false, false, true, ACT_SNAKE>(rc, x); break;       // conv7
          case 12 | (ACT_SNAKE << 4): rows_t<false, false, true, true, ACT_SNAKE>(rc, x); break;       // conv-transpose
          case 13 | (ACT_SNAKE << 4): rows_t<true, false, true, true, ACT_SNAKE>(rc, x); break;        // conv1 + residual
          case 9 | (ACT_SNAKE << 4): rows_t<true, false, false, true, ACT_SNAKE>(rc, x); break;        // last conv1 of a block
          default: rows_generic(ep, rc, x, col, c16); break;
        }
      }
    }
    if (!waited) wait();
  }
};

// EpiLinear for the convs of a padded batch of clips of different lengths (conv addressing only: rows are (clip, t), rows_per_clip per
// clip, and a tile never straddles clips).  Clip b ends at row end = clamp(lens[b], 1, max_len) * frame_rows of this layer.  Rows below it
// go through EpiLinear with the row count a run of that clip alone at its own length has (nvalid = end - t0), so they are the same bits;
// rows at or past it are stored as zeros to out_bf16 ([hi | lo | hi] included) -- the operand the next conv reads is then the zero halo
// the TMA fill gives the solo run -- and out_f32 is not written there.  lens is read when the kernel runs.
struct EpiLinearLensParams {
  EpiLinearParams lin;
  const int32_t* lens;     // [B] device, latent frames per clip
  int rows_per_clip;       // GEMM rows per clip (ConvAddr::T)
  int max_len;             // padded length in latent frames
  int frame_rows;          // GEMM rows of this layer per latent frame
};
template <int BN>
struct EpiLinearLens {
  using Params = EpiLinearLensParams;
  static constexpr int EPI_WARPS = EpiLinear<BN>::EPI_WARPS;
  static constexpr bool WIDE_REGS = false;
  static constexpr int STAGE_FLOATS = EPI_STAGE_FLOATS;
  template <class Wait>
  static __device__ __forceinline__ void run(const Params& ep, float* st, const AccRows& ar, int row0, int nvalid, int n0, int N, int lane, int c_begin,
                                             int c_end, Wait wait) {
    if (nvalid <= 0) { wait(); return; }   // this warp's rows lie past the padded length (row0 may belong to the next clip)
    const int b = row0 / ep.rows_per_clip, t0 = row0 - b * ep.rows_per_clip;
    const int end = min(max(ep.lens[b], 1), ep.max_len) * ep.frame_rows;
    const int live = min(nvalid, end - t0);
    EpiLinear<BN>::run(ep.lin, st, ar, row0, live, n0, N, lane, c_begin, c_end, wait);
    const EpiLinearParams& e = ep.lin;
    const int nv = nvalid < 32 ? nvalid : 32;
    if (e.out_bf16 == nullptr || live >= nv) return;
    for (int c = c_begin; c < c_end; c += 64) {
      const int col = n0 + c + 2 * lane;
      if (c + 2 * lane >= c_end || col >= N) continue;
      const int c16 = e.phase_cols > 0 ? (col / e.phase_cols) * e.phase_ld16 + col % e.phase_cols : col;
      for (int rr = live > 0 ? live : 0; rr < nv; ++rr) store_bf16x2(e.out_bf16 + (size_t)(row0 + rr) * e.ld16 + c16, e.split_stride, 0.f, 0.f);
    }
  }
};

// bias -> f32 with a per-sample scale read when the kernel runs: out[row, col] = (acc + bias[col]) * scale[row / rows_per_batch], the float
// operations rows_generic applies with a uniform out_scale, so a sample whose scale equals it comes out with the same bits.  A scale of 0 gives
// zeros (the uniform out_scale treats 0 as 1).  The ControlNet zero-linears of a batch of requests with different conditioning scales.
struct EpiLinearScaledParams {
  EpiLinearParams lin;     // bias, out_f32, ld32 (nothing else is read)
  const float* scale;      // [B] device
  int rows_per_batch;
};
template <int BN>
struct EpiLinearScaled {
  using Params = EpiLinearScaledParams;
  static constexpr int EPI_WARPS = EpiLinear<BN>::EPI_WARPS;
  static constexpr bool WIDE_REGS = false;
  static constexpr int STAGE_FLOATS = EPI_STAGE_FLOATS;
  template <class Wait>
  static __device__ __forceinline__ void run(const Params& ep, float* st, const AccRows& ar, int row0, int nvalid, int n0, int N, int lane, int c_begin,
                                             int c_end, Wait wait) {
    const EpiLinearParams& e = ep.lin;
    const int nv = nvalid < 32 ? nvalid : 32;
    wait();
#pragma unroll 1
    for (int c = c_begin; c < c_end; c += 64) {
      const int col = n0 + c + 2 * lane;
      const bool col_ok = (c + 2 * lane < c_end) && col < N;
      __syncwarp();
#pragma unroll
      for (int hc = 0; hc < 2; ++hc) {
        uint32_t r[32];
        acc_ld<32>(ar, c + 32 * hc, lane, r);
#pragma unroll
        for (int g = 0; g < 16; ++g) stage_put(st, lane, 16 * hc + g, __uint_as_float(r[2 * g]), __uint_as_float(r[2 * g + 1]));
      }
      __syncwarp();
      if (!col_ok) continue;
      const float b0 = e.bias != nullptr ? e.bias[col] : 0.f, b1 = e.bias != nullptr ? e.bias[col + 1] : 0.f;
#pragma unroll 4
      for (int rr = 0; rr < nv; ++rr) {
        const int row = row0 + rr;
        const float s = ep.scale[row / ep.rows_per_batch];
        const float2 acc = stage_get(st, rr, lane);
        *reinterpret_cast<float2*>(e.out_f32 + (size_t)row * e.ld32 + col) = make_float2((acc.x + b0) * s, (acc.y + b1) * s);
      }
    }
  }
};

// GEGLU (src/models/utils/modules.py:274-277): W rows are packed so that an N-tile of BN columns holds BN/2 hidden
// features followed by the BN/2 matching gate features; out[row, n0/2 + j] = (h_j + bh_j) * gelu_erf(g_j + bg_j).
struct EpiGegluParams {
  const float* bias;  // packed like the weight rows
  __nv_bfloat16* out_bf16;
  int ld16;
  int split_stride;
  FoldIn fin;         // LayerNorm folded into this GEMM (fin.v already contains the bias)
};
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// h * gelu(g) with erf from Abramowitz-Stegun 7.1.26 (|err| <= 1.5e-7 + 2 ulp of the MUFU rcp / ex2): 2 MUFU + ~14 FP32 ops.
// Used by the bf16 throughput path only (its output is rounded to bf16, 4e-3 relative); bf16x3 calls the exact erff.
__device__ __forceinline__ float geglu_fast(float h, float g) {
  const float z = g * 0.70710678118654752440f, az = fabsf(z);
  const float t = rcp_approx(fmaf(0.3275911f, az, 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = ex2_approx(az * az * -1.4426950408889634f);
  const float erf_abs = fmaf(-p * t, e, 1.0f);
  const float erf_s = copysignf(erf_abs, z);
  return h * (0.5f * g) * (1.0f + erf_s);
}

template <int BN, bool FOLD = false>
struct EpiGeglu {
  using Params = EpiGegluParams;
  static constexpr int HALF = BN / 2;
  static constexpr int EPI_WARPS = BN == 256 ? 8 : 4;   // 8 warps: each takes 64 of the tile's 128 output features
  static constexpr bool WIDE_REGS = false;
  static constexpr int STAGE_FLOATS = 32 * 32;          // 64 packed bf16 per row
  template <class Wait>
  static __device__ __forceinline__ void run(const Params& ep, float* st, const AccRows& ar, int row0, int nvalid, int n0, int N, int lane, int c_begin,
                                             int c_end, Wait wait) {
    constexpr bool fold = FOLD;
    float rstd = 1.f, nmr = 0.f;
    if (fold && lane < nvalid) fold_row_stats(ep.fin, row0 + lane, rstd, nmr);   // before the accumulator wait
    wait();
    // c_begin/c_end are expressed in accumulator columns of the whole tile: map them to output-feature ranges
    const int f_begin = c_begin / 2, f_end = c_end / 2;
#pragma unroll 1
    for (int c = f_begin; c < f_end; c += 64) {  // 64 output features per pass, gated in the thread == row layout
      if (n0 + c >= N) break;
      if (ep.split_stride > 0) {  // bf16x3 parity mode: exact erf, per-thread row stores of [hi | lo | hi]
        uint32_t h[32], g[32];
#pragma unroll 1
        for (int q4 = 0; q4 < 2; ++q4) {
          __syncwarp();
          acc_ld<32>(ar, c + q4 * 32, lane, h);
          acc_ld<32>(ar, HALF + c + q4 * 32, lane, g);
          if (lane < nvalid) {
            __nv_bfloat16* o = ep.out_bf16 + (size_t)(row0 + lane) * ep.ld16 + (n0 / 2 + c + q4 * 32);
#pragma unroll
            for (int j = 0; j < 32; j += 2) {
              const float o0 = (__uint_as_float(h[j]) + ep.bias[n0 + c + q4 * 32 + j]) * gelu_erf(__uint_as_float(g[j]) + ep.bias[n0 + HALF + c + q4 * 32 + j]);
              const float o1 = (__uint_as_float(h[j + 1]) + ep.bias[n0 + c + q4 * 32 + j + 1]) * gelu_erf(__uint_as_float(g[j + 1]) + ep.bias[n0 + HALF + c + q4 * 32 + j + 1]);
              store_bf16x2(o + j, ep.split_stride, o0, o1);
            }
          }
        }
        continue;
      }
      uint32_t pk[32];  // 64 bf16 results of this thread's row
#pragma unroll
      for (int q4 = 0; q4 < 2; ++q4) {
        uint32_t h[32], g[32];
        __syncwarp();
        acc_ld<32>(ar, c + q4 * 32, lane, h);
        acc_ld<32>(ar, HALF + c + q4 * 32, lane, g);
        if (fold) {   // warp-uniform: h = rstd * acc - rstd * mu * u + (v + bias)
          const float* bh = ep.fin.v + n0 + c + q4 * 32;
          const float* bg = ep.fin.v + n0 + HALF + c + q4 * 32;
          const float* uh = ep.fin.u + n0 + c + q4 * 32;
          const float* ug = ep.fin.u + n0 + HALF + c + q4 * 32;
#pragma unroll
          for (int j = 0; j < 32; j += 2) {
            const float o0 = geglu_fast(fmaf(__uint_as_float(h[j]), rstd, fmaf(nmr, __ldg(uh + j), __ldg(bh + j))),
                                        fmaf(__uint_as_float(g[j]), rstd, fmaf(nmr, __ldg(ug + j), __ldg(bg + j))));
            const float o1 = geglu_fast(fmaf(__uint_as_float(h[j + 1]), rstd, fmaf(nmr, __ldg(uh + j + 1), __ldg(bh + j + 1))),
                                        fmaf(__uint_as_float(g[j + 1]), rstd, fmaf(nmr, __ldg(ug + j + 1), __ldg(bg + j + 1))));
            pk[q4 * 16 + j / 2] = pack_bf16(o0, o1);
          }
        } else {
        const float* bh = ep.bias + n0 + c + q4 * 32;
        const float* bg = ep.bias + n0 + HALF + c + q4 * 32;
#pragma unroll
        for (int j = 0; j < 32; j += 2) {
          const float o0 = geglu_fast(__uint_as_float(h[j]) + __ldg(bh + j), __uint_as_float(g[j]) + __ldg(bg + j));
          const float o1 = geglu_fast(__uint_as_float(h[j + 1]) + __ldg(bh + j + 1), __uint_as_float(g[j + 1]) + __ldg(bg + j + 1));
          pk[q4 * 16 + j / 2] = pack_bf16(o0, o1);
        }
        }
      }
      __syncwarp();
#pragma unroll
      for (int gq = 0; gq < 16; ++gq) stage_put<32>(st, lane, gq, __uint_as_float(pk[2 * gq]), __uint_as_float(pk[2 * gq + 1]));
      __syncwarp();
      // 16 lanes cover one 128-byte row segment (64 bf16): the two half-warps take alternate rows
      const int hl = lane & 15, hw = lane >> 4;
      __nv_bfloat16* obase = ep.out_bf16 + (size_t)row0 * ep.ld16 + (n0 / 2 + c + 4 * hl);
#pragma unroll 4
      for (int rp = 0; rp < 16; ++rp) {
        const int rr = 2 * rp + hw;
        if (rr < nvalid) *reinterpret_cast<float2*>(obase + (size_t)rr * ep.ld16) = stage_get<32>(st, rr, hl);
      }
    }
  }
};

// The GEGLU epilogue of the plain bf16 path (no LayerNorm fold, no bf16x3 split) on the wgmma fragment, for gemm_body's overlapped schedule
// (FRAG): the accumulator stays in the MMA warpgroup's registers, so the ring never holds it and the producer streams the next tile's k-blocks
// while this runs.  In the m64n256 fragment hidden column j and gate column j + 128 of a row sit in the same thread (registers 4i.. and
// 4(i + 16)..), so the gate is applied in place with EpiGeglu's float operations in EpiGeglu's order: the output is bit-identical.  Each
// warpgroup writes its 64 x 128 bf16 result into its own 16 KB smem tile (two 64 x 64 boxes in the TMA 128-byte swizzle, conflict-free for
// the fragment's 4-byte writes) and stores it with two TMA box stores through `out`, a map of out_bf16 [M, N / 2] (pitch ld16) with
// {64 features, 64 rows} boxes, built by gemm2: its bounds clip rows >= M and the empty padding tile of an odd M-tile count.
// Params: bias, out_bf16, ld16 as for EpiGeglu; split_stride must be 0 and fin unset.
// Barrier of MMA warpgroup wg's 128 threads (ids 2 and 3; id 1 is the parked schedule's consumer barrier).  Constant ids, so that ptxas reserves
// only the barriers the kernel uses.
__device__ __forceinline__ void warpgroup_bar_sync(int wg) {
  if (wg == 0) named_bar_sync(2, 128);
  else named_bar_sync(3, 128);
}
struct EpiGegluFrag {
  using Params = EpiGegluParams;
  static constexpr bool FRAG = true;
  static constexpr int EPI_WARPS = 8;                   // two MMA warpgroups, one 64-row half each
  static constexpr bool WIDE_REGS = false;
  static constexpr int STAGE_FLOATS = 32 * 32;          // 8 warps x 4 KB = two 16 KB output tiles
  static constexpr int HALF = 128;
  // d: this thread's m64n256 fragment of the warpgroup's rows m0 + 64 wg ..; tile: the warpgroup's 16 KB output tile (1024-byte aligned)
  static __device__ __forceinline__ void frag(const Params& ep, const CUtensorMap* out, float (&d)[128], uint8_t* tile, int m0, int n0, const GemmShape&,
                                              int wg, int lg, int lane) {
    const int q = lane & 3;
    const int r0 = 16 * lg + (lane >> 2);   // row of registers 4i, 4i + 1; registers 4i + 2, 4i + 3 hold row r0 + 8 (same swizzle phase)
    const float2* bh = reinterpret_cast<const float2*>(ep.bias + n0) + q;
    const float2* bg = reinterpret_cast<const float2*>(ep.bias + n0 + HALF) + q;
#pragma unroll
    for (int i = 0; i < 16; ++i) {   // output columns 8i + 2q, 8i + 2q + 1: box i / 8, 16-byte chunk i % 8 of the box row
      const float2 b_h = __ldg(bh + 4 * i), b_g = __ldg(bg + 4 * i);
      const uint32_t lo = pack_bf16(geglu_fast(d[4 * i] + b_h.x, d[64 + 4 * i] + b_g.x), geglu_fast(d[4 * i + 1] + b_h.y, d[64 + 4 * i + 1] + b_g.y));
      const uint32_t hi = pack_bf16(geglu_fast(d[4 * i + 2] + b_h.x, d[64 + 4 * i + 2] + b_g.x), geglu_fast(d[4 * i + 3] + b_h.y, d[64 + 4 * i + 3] + b_g.y));
      uint8_t* p = tile + (i >> 3) * 8192 + r0 * 128 + (((i & 7) ^ (r0 & 7)) << 4) + 4 * q;
      *reinterpret_cast<uint32_t*>(p) = lo;
      *reinterpret_cast<uint32_t*>(p + 8 * 128) = hi;
    }
    fence_proxy_async_smem();        // the generic writes above, before the TMA engine reads the tile
    warpgroup_bar_sync(wg);
    if ((threadIdx.x & 127) == 0) {
      tma_store_2d(out, tile, n0 / 2, m0 + 64 * wg);
      tma_store_2d(out, tile + 8192, n0 / 2 + 64, m0 + 64 * wg);
      bulk_commit_group();
    }
  }
};
// Epilogues that run on the register fragment declare FRAG = true; the others (no FRAG member) use the parked-tile schedule.  A FRAG epilogue
// may hand its warpgroup's tile to bulk async stores issued by the warpgroup's thread 0: gemm_body has that thread wait until they have
// read it before the next frag() call (then a warpgroup barrier), and until they are complete before the CTA exits.
template <class E>
constexpr auto epi_frag_impl(int) -> decltype(E::FRAG) { return E::FRAG; }
template <class E>
constexpr bool epi_frag_impl(long) { return false; }
template <class E>
constexpr bool epi_frag() { return epi_frag_impl<E>(0); }

// ---------------------------------------------------------------------------------------------------------------
// Transposed ("swap-AB") linear epilogue.  For N_out = 1152-wide layers the natural 128/144-column tiles spend more operand
// bytes per flop and a 256-column tile does not divide 1152.  Computing C^T = W A^T instead puts the 1152 output features on the
// accumulator ROWS (9 tiles of 128) and 256 or 288 tokens on the columns (host.cuh swapped_bn picks the width).  A thread now owns one output
// feature; for a given token the 32 lanes of a warp hold 32 consecutive features, so residual loads and stores are 128-byte coalesced without
// any staging.  Each of the two warps of a 32-feature group owns BN / 2 tokens, walked in chunks of up to 32: at BN = 288 that is 4.5 chunks,
// and the half chunk stops at the warp's range so that no warp writes another warp's tokens.
__device__ __forceinline__ int swap_chunk_tokens(int c, int c_end, int t0, int N) {   // tokens of the chunk at tile column c (first token t0)
  int n = c_end - c;
  if (N - t0 < n) n = N - t0;
  return n < 32 ? n : 32;
}
template <int BN>
struct EpiLinearT {
  using Params = EpiLinearParams;   // bias/gate indexed by feature, resid/out_f32 [token, feature]; bf16/act/split unsupported
  static constexpr int EPI_WARPS = 8;
  static constexpr bool WIDE_REGS = false;
  static constexpr int STAGE_FLOATS = 0;
  // residual values of one chunk of nt <= 32 tokens (feature f of tokens t0 .. t0+nt-1)
  static __device__ __forceinline__ void load_resid(const Params& ep, float (&x)[32], int t0, int nt, int f, bool f_ok) {
#pragma unroll
    for (int j = 0; j < 32; ++j) x[j] = (f_ok && j < nt) ? ep.resid[(size_t)(t0 + j) * ep.ldr + f] : 0.f;
  }
  template <class Wait>
  static __device__ __forceinline__ void run(const Params& ep, float* st, const AccRows& ar, int row0, int nvalid, int n0, int N, int lane, int c_begin,
                                             int c_end, Wait wait) {
    const int f = row0 + lane;                 // output feature of this thread
    const bool f_ok = lane < nvalid;
    const float bias = (ep.bias != nullptr && f_ok) ? ep.bias[f] : 0.f;
    bool waited = false;
    // The epilogue does not overlap the next tile's mainloop, so it is exposed: the residual of chunk c + 1 is fetched while chunk c is
    // processed (and the first chunk's before the accumulator wait), instead of one L2 round trip per chunk on the critical path.
    float x[32];
    if (ep.resid != nullptr && n0 + c_begin < N) load_resid(ep, x, n0 + c_begin, swap_chunk_tokens(c_begin, c_end, n0 + c_begin, N), f, f_ok);
#pragma unroll 1
    for (int c = c_begin; c < c_end; c += 32) {
      const int t0 = n0 + c;                   // first token of this chunk
      if (t0 >= N) break;                      // warp-uniform
      const int nt = swap_chunk_tokens(c, c_end, t0, N);
      float xn[32];
      const bool more = ep.resid != nullptr && c + 32 < c_end && t0 + 32 < N;
      if (more) load_resid(ep, xn, t0 + 32, swap_chunk_tokens(c + 32, c_end, t0 + 32, N), f, f_ok);
      float g0 = 1.f, g1 = 1.f;
      int btok = 0x7fffffff;                   // first token that belongs to the second batch item of this chunk
      if (ep.gate != nullptr && f_ok) {
        const int b0i = t0 / ep.rows_per_batch;
        btok = (b0i + 1) * ep.rows_per_batch;
        g0 = 1.0f - ep.gate[(size_t)b0i * ep.gate_bstride + f];
        if (btok < t0 + nt) g1 = 1.0f - ep.gate[(size_t)(b0i + 1) * ep.gate_bstride + f];
      }
      if (!waited) { wait(); waited = true; }
      uint32_t r[32];
      __syncwarp();
      acc_ld<32>(ar, c, lane, r);
      if (f_ok) {
        float* o = ep.out_f32 + (size_t)t0 * ep.ld32 + f;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          if (j >= nt) break;
          float v = __uint_as_float(r[j]) + bias;
          if (ep.resid != nullptr) v = fmaf((t0 + j >= btok) ? g1 : g0, v, x[j]);
          o[(size_t)j * ep.ld32] = v;
        }
      }
      if (more) {
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = xn[j];
      }
    }
    if (!waited) wait();
  }
};

// Fold-capable variant (LayerNorm folded in / out, see FoldIn / FoldOut).  Kept apart from EpiLinearT on purpose: the extra outputs and the
// warp transposes lengthen this epilogue, which matters when the LayerNorm is not folded.
template <int BN>
struct EpiLinearTF {
  using Params = EpiLinearParams;   // bias/gate indexed by feature, resid/out_f32 [token, feature]; bf16/act/split unsupported
  static constexpr int EPI_WARPS = 8;
  static constexpr bool WIDE_REGS = false;
  static constexpr int STAGE_FLOATS = 0;
  template <class Wait>
  static __device__ __forceinline__ void run(const Params& ep, float* st, const AccRows& ar, int row0, int nvalid, int n0, int N, int lane, int c_begin,
                                             int c_end, Wait wait) {
    const int f = row0 + lane;                 // output feature of this thread
    const bool f_ok = lane < nvalid;
    const float bias = (ep.bias != nullptr && f_ok) ? ep.bias[f] : 0.f;
    const bool fold_in = ep.fin.u != nullptr, fold_out = ep.fout.st != nullptr && nvalid > 0;
    float uf = 0.f, vf = 0.f, ga = 1.f, gb = 1.f;
    if (fold_in && f_ok) { uf = ep.fin.u[f]; vf = ep.fin.v[f]; }
    if (fold_out && f_ok) {
      if (ep.fout.g0 != nullptr) ga = ep.fout.g0[f];
      if (ep.fout.a1 != nullptr && ep.fout.g1 != nullptr) gb = ep.fout.g1[f];
    }
    bool waited = false;
#pragma unroll 1
    for (int c = c_begin; c < c_end; c += 32) {
      const int t0 = n0 + c;                   // first token of this chunk
      if (t0 >= N) break;                      // warp-uniform
      const int nt = swap_chunk_tokens(c, c_end, t0, N);
      float x[32];
      if (ep.resid != nullptr) {
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = (f_ok && j < nt) ? ep.resid[(size_t)(t0 + j) * ep.ldr + f] : 0.f;
      }
      float g0 = 1.f, g1 = 1.f;
      int btok = 0x7fffffff;                   // first token that belongs to the second batch item of this chunk
      if (ep.gate != nullptr && f_ok) {
        const int b0i = t0 / ep.rows_per_batch;
        btok = (b0i + 1) * ep.rows_per_batch;
        g0 = 1.0f - ep.gate[(size_t)b0i * ep.gate_bstride + f];
        if (btok < t0 + nt) g1 = 1.0f - ep.gate[(size_t)(b0i + 1) * ep.gate_bstride + f];
      }
      float rs_l = 1.f, nm_l = 0.f;            // LayerNorm statistics of token t0 + lane (fold-in)
      if (fold_in && lane < nt) fold_row_stats(ep.fin, t0 + lane, rs_l, nm_l);
      if (!waited) { wait(); waited = true; }
      uint32_t r[32];
      __syncwarp();
      acc_ld<32>(ar, c, lane, r);
      float val[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        float acc = __uint_as_float(r[j]);
        if (fold_in) {                           // warp-uniform branch; the shuffles run on all lanes
          const float rs = __shfl_sync(0xffffffffu, rs_l, j), nm = __shfl_sync(0xffffffffu, nm_l, j);
          acc = fmaf(acc, rs, fmaf(nm, uf, vf));
        }
        float v = acc + bias;
        float gj = (t0 + j >= btok) ? g1 : g0;
        if (ep.resid != nullptr) v = fmaf(gj, v, x[j]);
        val[j] = (f_ok && j < nt) ? v : 0.f;
      }
      if (f_ok) {
        float* o = ep.out_f32 + (size_t)t0 * ep.ld32 + f;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          if (j >= nt) break;
          o[(size_t)j * ep.ld32] = val[j];
        }
        if (fold_out) {                          // operand(s) of the GEMM(s) behind the LayerNorm(s) that read this x
          __nv_bfloat16* a = ep.fout.a0 + (size_t)t0 * ep.fout.ld0 + f;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            if (j >= nt) break;
            a[(size_t)j * ep.fout.ld0] = __float2bfloat16_rn(val[j] * ga);
          }
          if (ep.fout.a1 != nullptr) {
            __nv_bfloat16* a2 = ep.fout.a1 + (size_t)t0 * ep.fout.ld1 + f;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              if (j >= nt) break;
              a2[(size_t)j * ep.fout.ld1] = __float2bfloat16_rn(val[j] * gb);
            }
          }
        }
      }
      if (fold_out) {                            // per-token partial sums over this warp's 32 features -> slot row0 / 32
        float sq[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) sq[j] = val[j] * val[j];
        const float s1 = warp_transpose_sum(val, lane), s2 = warp_transpose_sum(sq, lane);
        if (lane < nt) ep.fout.st[(size_t)(row0 >> 5) * ep.fout.ld_st + t0 + lane] = make_float2(s1, s2);
      }
    }
    if (!waited) wait();
  }
};

// FP8 mode (gemm_fp8_kernel): e4m3 operands with per-row scales; the MMA warpgroups multiply the fp32 accumulator by sa[row] * sw[col] as they
// park it in shared memory, so the epilogues see the dequantised tile and run unchanged.
struct Fp8Scales {
  const float* sa;   // [M] per token row (A operand)
  const float* sw;   // [N] per output feature (W operand, in its packed row order)
};

// Shared-memory plan of one CTA: the STAGES-deep operand ring (which also holds the finished fp32 accumulator tile between the
// mainloop and the epilogue of a tile), the epilogues' per-warp transpose tiles, the barriers.  A ring slot holds one 64-wide k-block.
template <int BN, class Epi>
struct GemmCfg {
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int EPI_WARPS = Epi::EPI_WARPS;
  // Every consumer warpgroup issues wgmma over the full BN columns.  One warpgroup: both 64-row halves of the tile.  Two: one half each.
  static constexpr int MMA_WG = EPI_WARPS / 4;
  static_assert(MMA_WG == 1 || MMA_WG == 2, "one or two consumer warpgroups");
  static constexpr int NSUB = MMA_WG == 2 ? 1 : 2;                // 64-row halves per warpgroup
  // Consumer warpgroups + the producer warp.  A CTA of 9..12 warps puts three warps on one SM sub-partition, which caps every thread at 168
  // registers: too few for the 144 accumulators of a 288-wide tile (ptxas spills and serialises the wgmma), and for the 224-wide heads tile,
  // whose 112 accumulators and two dh-wide epilogue rows per thread spill 1.4 KB (the epilogue asks with WIDE_REGS).  These run a whole
  // producer warpgroup (one active warp) that hands registers to the consumers with setmaxnreg: 384 x 168 = 128 x 40 + 256 x 232.
  static constexpr bool PRODUCER_WG = BN > 256 || Epi::WIDE_REGS;
  static constexpr int THREADS = 32 * EPI_WARPS + (PRODUCER_WG ? 128 : 32);
  static constexpr int REGS_LAUNCH = (65536 / THREADS) & ~7;                        // what __launch_bounds__(THREADS, 1) lets ptxas allocate
  static constexpr int REGS_PRODUCER = 40;
  static constexpr int REGS_CONSUMER = ((THREADS * REGS_LAUNCH - 128 * REGS_PRODUCER) / (32 * EPI_WARPS)) & ~7;
  // setmaxnreg.inc waits for free registers: the split must not ask for more than the launch allocated
  static_assert(!PRODUCER_WG || (EPI_WARPS == 8 && 128 * REGS_PRODUCER + 32 * EPI_WARPS * REGS_CONSUMER <= THREADS * REGS_LAUNCH &&
                                 REGS_CONSUMER >= 224), "register split");
  static constexpr int NH = BN > 256 ? 2 : 1;   // wgmma N stops at 256: a wider tile is issued as two halves, HN columns each
  static constexpr int HN = BN / NH;
  // FRAG (epi_frag): the epilogue runs on the accumulator registers, the ring never holds the tile
  static constexpr bool FRAG = epi_frag<Epi>();
  static constexpr int ACC_PITCH = BN + 4;
  static constexpr int ACC_BYTES = FRAG ? 0 : GEMM_BM * ACC_PITCH * 4;
  static constexpr int STAGE_BYTES = EPI_WARPS * Epi::STAGE_FLOATS * 4;   // one transpose tile per epilogue warp
  static constexpr int FIT = (GEMM_SMEM_BUDGET - STAGE_BYTES) / (A_BYTES + B_BYTES);
  static constexpr int STAGES = FIT > 8 ? 8 : FIT;
  static constexpr int RING = STAGES * (A_BYTES + B_BYTES) > ACC_BYTES ? STAGES * (A_BYTES + B_BYTES) : ACC_BYTES;
  static_assert(!FRAG || (RING % 1024 == 0 && MMA_WG == 2 && NH == 1), "FRAG: 1024-byte aligned output tiles, one 64-row half per warpgroup");
  static constexpr int BYTES = 1024 /*align slack*/ + RING + STAGE_BYTES + (2 * STAGES + 1) * 8;
  static_assert(STAGES >= 2, "smem budget");
  static_assert(BYTES <= 227 * 1024, "smem budget");
};

// One consumer warpgroup's k-loop over a tile: all BN accumulator columns of NSUB 64-row halves from 64-row block row64 (slot s is released
// once wgmma.wait_group shows its MMAs complete, while slot s + 1's are in flight).  Returns with every MMA of this warpgroup complete.
// FP8: the ring slots hold 128-element e4m3 k-blocks (the same 128-byte rows), issued as four k32 MMAs at the bf16 descriptor steps.
template <int BN, class Epi, int MC, bool FP8 = false>
__device__ __forceinline__ void gemm_mainloop(float (&d)[GemmCfg<BN, Epi>::NSUB][GemmCfg<BN, Epi>::NH][GemmCfg<BN, Epi>::HN / 2],
                                              int row64, const uint8_t* sA, const uint8_t* sB, uint64_t* full, uint64_t* empty, int num_k_blocks,
                                              uint32_t& stage, uint32_t& phase) {
  using SM = GemmCfg<BN, Epi>;
  constexpr int NSUB = SM::NSUB, NH = SM::NH, HN = SM::HN;
  // One thread per warpgroup arrives on the slot's barrier in every CTA of the cluster, without a release fence: the slot's only readers
  // are this warpgroup's wgmma (async proxy), complete at the wgmma.wait_group before the release; its only writer is a producer's TMA
  // (async proxy), issued after that producer's try_wait has observed the arrival; and no generic-proxy data is published through `empty`.
  // A .release.cluster arrive would put two fences (MEMBAR.ALL.CTA + MEMBAR.ALL.GPU) in front of every arrive of every k-block, and the
  // warpgroup's next .sync.aligned wgmma would wait for them.
  auto release = [&](uint32_t s) {
    if ((threadIdx.x & 127) == 0) {
      if (MC == 1) mbar_arrive(&empty[s]);
      else for (int r = 0; r < MC; ++r) mbar_arrive_cluster_nofence(mapa_u32(smem_u32(&empty[s]), r));
    }
  };
  static_assert(HN <= 256 && HN % 8 == 0, "BN");   // HN % 8: the second half starts on a 1024-byte swizzle atom
  uint32_t prev = 0;
  for (int kb = 0; kb < num_k_blocks; ++kb) {
    mbar_wait(&full[stage], phase);
    wgmma_fence();
    const uint32_t a0 = smem_u32(sA + stage * SM::A_BYTES + row64 * 8192);
    const uint32_t b0 = smem_u32(sB + stage * SM::B_BYTES);
#pragma unroll
    for (int k = 0; k < GEMM_BK / 16; ++k) {
#pragma unroll
      for (int s = 0; s < NSUB; ++s)
#pragma unroll
        for (int h = 0; h < NH; ++h)
          if constexpr (FP8) WgmmaE4m3<HN>::mma(d[s][h], wgmma_desc_sw128(a0 + s * 8192) + 2 * k, wgmma_desc_sw128(b0 + h * HN * 128) + 2 * k, (kb | k) != 0);
          else Wgmma<HN>::mma(d[s][h], wgmma_desc_sw128(a0 + s * 8192) + 2 * k, wgmma_desc_sw128(b0 + h * HN * 128) + 2 * k, (kb | k) != 0);
    }
    wgmma_commit();
    if (kb > 0) { wgmma_wait<1>(); release(prev); }
    prev = stage;
    if (++stage == SM::STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  release(prev);
#pragma unroll
  for (int s = 0; s < NSUB; ++s)
#pragma unroll
    for (int h = 0; h < NH; ++h) wgmma_fence_regs(d[s][h]);
}

// Parked-tile schedule: the k-loop, then, after every warpgroup's MMAs have completed, the fragments written into the accumulator tile in
// shared memory (over the ring).  FP8: the accumulator is dequantised with the scales of global rows m0 + .. (< M) and columns n0 + .. on its
// way to shared memory.
template <int BN, class Epi, int MC, bool FP8 = false>
__device__ __forceinline__ void gemm_mma_part(int row64, const uint8_t* sA, const uint8_t* sB, float* sAcc, uint64_t* full, uint64_t* empty,
                                              int num_k_blocks, uint32_t& stage, uint32_t& phase, int lg, int lane, const Fp8Scales& fs = Fp8Scales{},
                                              int m0 = 0, int M = 0, int n0 = 0) {
  using SM = GemmCfg<BN, Epi>;
  constexpr int NSUB = SM::NSUB, NH = SM::NH, HN = SM::HN;
  float d[NSUB][NH][HN / 2];
  gemm_mainloop<BN, Epi, MC, FP8>(d, row64, sA, sB, full, empty, num_k_blocks, stage, phase);
  named_bar_sync(1, 32 * SM::EPI_WARPS);   // every MMA of the tile has completed: the ring may now hold the accumulator
  // m64nN fragment: register 4i + {0,1} -> row 16 * (warp % 4) + lane / 4, columns 8i + 2 (lane % 4) + {0,1}; 4i + {2,3} -> row + 8
  if constexpr (FP8) {
#pragma unroll
    for (int s = 0; s < NSUB; ++s) {
      const int r = m0 + (row64 + s) * 64 + 16 * lg + (lane >> 2);
      const float sa0 = r < M ? fs.sa[r] : 0.f, sa1 = r + 8 < M ? fs.sa[r + 8] : 0.f;
#pragma unroll
      for (int h = 0; h < NH; ++h) {
        const float2* sw = reinterpret_cast<const float2*>(fs.sw + n0 + h * HN + 2 * (lane & 3));
#pragma unroll
        for (int i = 0; i < HN / 8; ++i) {
          const float2 w = __ldg(sw + 4 * i);
          d[s][h][4 * i] *= sa0 * w.x; d[s][h][4 * i + 1] *= sa0 * w.y;
          d[s][h][4 * i + 2] *= sa1 * w.x; d[s][h][4 * i + 3] *= sa1 * w.y;
        }
      }
    }
  }
#pragma unroll
  for (int s = 0; s < NSUB; ++s) {
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      float* r0 = sAcc + (size_t)((row64 + s) * 64 + 16 * lg + (lane >> 2)) * SM::ACC_PITCH + h * HN + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < HN / 8; ++i) {
        *reinterpret_cast<float2*>(r0 + 8 * i) = make_float2(d[s][h][4 * i], d[s][h][4 * i + 1]);
        *reinterpret_cast<float2*>(r0 + 8 * SM::ACC_PITCH + 8 * i) = make_float2(d[s][h][4 * i + 2], d[s][h][4 * i + 3]);
      }
    }
  }
}

// MC > 1: launched as clusters of MC CTAs with consecutive blockIdx.x = consecutive M tiles of the SAME N tile (host guarantees
// num_m_tiles % MC == 0 and gridDim.x % MC == 0, so the CTAs of a cluster walk the same number of tiles in step).
// The N-side operand tile (BN rows x 64 columns) is then fetched ONCE per cluster: tmB is a map with SUBROWS-row boxes, CTA rank r issues
// the sub-boxes j = r, r + MC, ... with .multicast::cluster, every CTA still expects the full A + B bytes on its own `full` barrier, a
// stage is free again only when the MMA warpgroups of all MC CTAs have released it (`empty` counts their arrivals), and the ring is
// refilled for the next tile only when every CTA of the cluster has finished reading its accumulator out of it (`acc_free`; parked-tile
// schedule only: a FRAG epilogue never puts the accumulator in the ring).
// FIRST_PHASE: another GEMM phase follows in the same kernel (mlp_fused_kernel): the barriers are invalidated at the end so that the next
// phase may lay out its own in the same shared memory.
template <int BN>
struct McSub { static constexpr int ROWS = BN % 32 == 0 ? 32 : 16; };
// Per-thread register budget of the executing warpgroup (all its threads execute it); inc waits until the pool has the registers.
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int BN, class Epi, int MC = 1, bool FIRST_PHASE = false, bool FP8 = false>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmShape& g, const typename Epi::Params& ep, uint8_t* smem_raw,
                                          const Fp8Scales& fs = Fp8Scales{}, const CUtensorMap* tmC = nullptr) {
  using SM = GemmCfg<BN, Epi>;
  constexpr int KB_ELEMS = FP8 ? 2 * GEMM_BK : GEMM_BK;   // elements per 128-byte k-block row
  // BN > 256: two TMA boxes and two wgmma halves per warpgroup, single CTA, one 64-row half per MMA warpgroup (the 288-token swap-AB tile)
  static_assert(BN % 16 == 0 && BN >= 64 && (BN <= 256 || (BN <= 512 && BN % 32 == 0 && MC == 1 && SM::MMA_WG == 2)), "BN");
  static_assert(MC >= 1 && MC <= 8 && BN % McSub<BN>::ROWS == 0, "MC");
  constexpr int STAGES = SM::STAGES, EPI_WARPS = SM::EPI_WARPS, NSUB = SM::NSUB;
  constexpr uint16_t MC_MASK = static_cast<uint16_t>((1u << MC) - 1u);
  // 1024-byte alignment (128-byte swizzle atoms) by pointer arithmetic on the __shared__ array (a round trip through uintptr_t loses the
  // address space and turns every staging access into a generic LD.E / ST.E)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * SM::A_BYTES;
  float* sAcc = reinterpret_cast<float*>(smem);
  float* sStage = reinterpret_cast<float*>(smem + SM::RING);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + SM::RING + SM::STAGE_BYTES);
  uint64_t* empty = full + STAGES;
  uint64_t* acc_free = empty + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = g.num_m_tiles * g.num_n_tiles;
  constexpr int PRODUCER = EPI_WARPS;

  if (warp == PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], SM::MMA_WG * MC);
    }
    mbar_init(acc_free, EPI_WARPS * MC);
    fence_mbar_init();
  }
  __syncthreads();
  if (MC > 1) cluster_sync_all();  // peers multicast into our stages and arrive on our barriers: they must exist first
  pdl_launch();
  if (warp == PRODUCER && g.pf_bytes != 0) {   // constant data: no need to wait for the previous kernel
    if (elect_one()) prefetch_weights_l2(g.pf, g.pf_bytes, blockIdx.x, gridDim.x);
    __syncwarp();
  }
  pdl_wait();  // everything above overlapped the previous kernel's tail; global memory is touched only below
  EZB_DBG(const bool dbg = g.dbg != nullptr && blockIdx.x == 0; const long long t_start = clock64(); long long w0 = 0, w1 = 0, w4 = 0;)

  if (warp >= PRODUCER) {
    // ------------------------------------------------ TMA producer (warp-uniform loop, copies issued under elect.sync); the other warps of a
    // producer warpgroup (GemmCfg::PRODUCER_WG) only give their registers away
    if constexpr (SM::PRODUCER_WG) setmaxnreg_dec<SM::REGS_PRODUCER>();
    uint32_t stage = 0, phase = 0, af_phase = 0;
    bool first = true;
    for (int tile = warp == PRODUCER ? (int)blockIdx.x : num_tiles; tile < num_tiles; tile += gridDim.x) {
      const int mt = tile % g.num_m_tiles, nt = tile / g.num_m_tiles;
      const int n0 = nt * BN;
      // parked-tile schedule: the ring held the previous tile's accumulator.  FRAG: the producer runs ahead into the next tile, limited by
      // `empty` alone (which counts the releases of every MMA warpgroup of the cluster before a slot is multicast into again).
      if (!SM::FRAG && !first) { mbar_wait(acc_free, af_phase); af_phase ^= 1; }
      first = false;
      for (int kb = 0; kb < g.num_k_blocks; ++kb) {
        EZB_DBG(const long long tq = clock64();)
        mbar_wait(&empty[stage], phase ^ 1);
        EZB_DBG(w0 += clock64() - tq;)
        if (elect_one()) {
          mbar_expect_tx(&full[stage], SM::A_BYTES + SM::B_BYTES);
          uint8_t* dA = sA + stage * SM::A_BYTES;
          uint8_t* dB = sB + stage * SM::B_BYTES;
          if (g.taps == 0) {
            tma_load_2d(dA, &tmA, &full[stage], kb * KB_ELEMS, mt * GEMM_BM);
          } else {
            const int tap = kb / g.cin_blocks, cb = kb - tap * g.cin_blocks;
            const int bidx = mt / g.tiles_per_batch, t0 = (mt - bidx * g.tiles_per_batch) * GEMM_BM;
            if (g.stride > 1) {
              const int off = tap - g.pad;                                   // input row = q * stride + off
              const int r = ((off % g.stride) + g.stride) % g.stride, dq = (off - r) / g.stride;
              tma_load_4d(dA, &tmA, &full[stage], cb * GEMM_BK, r, t0 + dq, bidx);
            } else {
              tma_load_3d(dA, &tmA, &full[stage], cb * GEMM_BK, t0 + (tap - g.center) * g.dilation, bidx);
            }
          }
          if (MC == 1) {
            constexpr int BOX = gemm_b_box(BN);
#pragma unroll
            for (int j = 0; j < BN / BOX; ++j) tma_load_2d(dB + j * BOX * 128, &tmB, &full[stage], kb * KB_ELEMS, n0 + j * BOX);
          } else {
            constexpr int SR = McSub<BN>::ROWS;
            for (int j = (int)cluster_ctarank(); j < BN / SR; j += MC)
              tma_load_2d_mc(dB + j * SR * 128, &tmB, &full[stage], kb * KB_ELEMS, n0 + j * SR, MC_MASK);
          }
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ------------------------------------------------ consumers: wgmma mainloop (MMA warpgroups), accumulator -> smem, epilogue (all)
    if constexpr (SM::PRODUCER_WG) setmaxnreg_inc<SM::REGS_CONSUMER>();
    const int wg = warp >> 2, lg = warp & 3;
    uint32_t stage = 0, phase = 0;
    if constexpr (SM::FRAG) {
      // Overlapped schedule: mainloop, then the epilogue on this warpgroup's registers, then straight into the next tile, whose first k-blocks
      // the producer has already loaded.  Counters: [0] mainloop, [1] wait for the output tile's previous store, [4] epilogue.
      static_assert(!FP8 && !FIRST_PHASE, "FRAG: bf16 kernels of one phase (gemm_frag_kernel)");
      uint8_t* tile_buf = reinterpret_cast<uint8_t*>(sStage) + wg * (SM::STAGE_BYTES / 2);
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mt = tile % g.num_m_tiles, nt = tile / g.num_m_tiles;
        EZB_DBG(const long long tm = clock64();)
        // defined before the mainloop (whose first MMA ignores it) so that the previous tile's accumulator is not kept live through the
        // epilogue as the operand of that first MMA: with it, the heads epilogue's dh-wide rows spilled
        float d[NSUB][SM::NH][SM::HN / 2] = {};
        gemm_mainloop<BN, Epi, MC>(d, wg * NSUB, sA, sB, full, empty, g.num_k_blocks, stage, phase);
        EZB_DBG(const long long ta = clock64(); w0 += ta - tm;)
        if ((threadIdx.x & 127) == 0) bulk_wait_group_read<0>();   // the previous tile's store has left this warpgroup's output tile
        warpgroup_bar_sync(wg);
        EZB_DBG(const long long te = clock64(); w1 += te - ta;)
        Epi::frag(ep, tmC, d[0][0], tile_buf, mt * GEMM_BM, nt * BN, g, wg, lg, lane);
        EZB_DBG(w4 += clock64() - te;)
      }
      if ((threadIdx.x & 127) == 0) bulk_wait_group<0>();
    } else
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mt = tile % g.num_m_tiles, nt = tile / g.num_m_tiles;
      EZB_DBG(const long long tm = clock64();)
      gemm_mma_part<BN, Epi, MC, FP8>(wg * NSUB, sA, sB, sAcc, full, empty, g.num_k_blocks, stage, phase, lg, lane, fs, mt * GEMM_BM, g.M, nt * BN);
      EZB_DBG(const long long ta = clock64(); w0 += ta - tm;)
      named_bar_sync(1, 32 * EPI_WARPS);     // accumulator tile complete in shared memory
      EZB_DBG(const long long te = clock64(); w1 += te - ta;)
      int row0, nvalid;
      if (g.taps == 0) {
        row0 = mt * GEMM_BM + lg * 32;
        nvalid = g.M - row0;
      } else {  // rows are (batch, t): tiles never straddle clips
        const int bidx = mt / g.tiles_per_batch, t0 = (mt - bidx * g.tiles_per_batch) * GEMM_BM + lg * 32;
        row0 = bidx * g.T + t0;
        nvalid = g.T - t0;
      }
      constexpr int CW = BN / (EPI_WARPS / 4);  // columns per warp
      const AccRows ar{sAcc + lg * 32 * SM::ACC_PITCH, SM::ACC_PITCH};
      Epi::run(ep, sStage + warp * Epi::STAGE_FLOATS, ar, row0, nvalid, nt * BN, g.N, lane, wg * CW, (wg + 1) * CW, []() {});
      EZB_DBG(w4 += clock64() - te;)
      fence_proxy_async_smem();   // this warp's generic accesses to the ring are ordered before the producer's next TMA writes into it
      __syncwarp();
      if (lane == 0) {   // cluster-scope release (once per tile): the epilogue's generic reads of the ring precede the peers' multicast into it
        if (MC == 1) mbar_arrive(acc_free);
        else for (int r = 0; r < MC; ++r) mbar_arrive_cluster(mapa_u32(smem_u32(acc_free), r));
      }
    }
    if constexpr (SM::PRODUCER_WG) setmaxnreg_dec<SM::REGS_LAUNCH>();
  }
  EZB_DBG(if (dbg && lane == 0) {
    if (warp == PRODUCER) atomicAdd(&g.dbg[2], (unsigned long long)w0);
    if (warp == 0) {
      atomicAdd(&g.dbg[0], (unsigned long long)w0); atomicAdd(&g.dbg[1], (unsigned long long)w1); atomicAdd(&g.dbg[4], (unsigned long long)w4);
      atomicAdd(&g.dbg[5], (unsigned long long)(clock64() - t_start));
    }
  })
  __syncthreads();
  // The producer warpgroup takes its registers back (the launch split, for whatever follows: gemm_ln_kernel's tail) only once every consumer
  // warp has given its extra ones back: setmaxnreg allocates per warp from the CTA's pool, so a producer-warpgroup warp that asked earlier
  // (its idle warps reach this point at once) could take registers a consumer warp's setmaxnreg.inc is still waiting for, and both would wait
  // for ever.
  if constexpr (SM::PRODUCER_WG) if (warp >= PRODUCER) setmaxnreg_inc<SM::REGS_LAUNCH>();
  if (MC > 1) cluster_sync_all();  // nobody leaves while a peer may still multicast into this CTA or arrive on its barriers
  if (FIRST_PHASE) {
    if (warp == PRODUCER && lane == 0) {
      for (int i = 0; i < STAGES; ++i) { mbar_inval(&full[i]); mbar_inval(&empty[i]); }
      mbar_inval(acc_free);
    }
    __syncthreads();
  }
}
template <int BN, class Epi, int MC = 1>
__global__ void __launch_bounds__((GemmCfg<BN, Epi>::THREADS), 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmShape g,
                  const typename Epi::Params ep) {
  extern __shared__ uint8_t smem_dyn[];
  gemm_body<BN, Epi, MC>(tmA, tmB, g, ep, smem_dyn);
}
// gemm_wgmma_kernel<BN, Epi, 2> for an epilogue on the register fragment (epi_frag): tmC is the map its output stores go through.
template <int BN, class Epi>
__global__ void __launch_bounds__((GemmCfg<BN, Epi>::THREADS), 1)
gemm_frag_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
                 const GemmShape g, const typename Epi::Params ep) {
  extern __shared__ uint8_t smem_dyn[];
  gemm_body<BN, Epi, 2>(tmA, tmB, g, ep, smem_dyn, Fp8Scales{}, &tmC);
}
// FP8 twin of gemm_wgmma_kernel<BN, Epi, 2> (2-CTA clusters, W tile multicast): A [M, K] and W [N, K] e4m3 through UINT8 tensor maps with
// 128-element k-blocks (num_k_blocks = K / 128), dequantised by the per-row scales fs (see Fp8Scales).
template <int BN, class Epi>
__global__ void __launch_bounds__((GemmCfg<BN, Epi>::THREADS), 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmShape g, const typename Epi::Params ep,
                const Fp8Scales fs) {
  extern __shared__ uint8_t smem_dyn[];
  gemm_body<BN, Epi, 2, false, true>(tmA, tmB, g, ep, smem_dyn, fs);
}

}  // namespace ezb

namespace ezb {
// ---------------------------------------------------------------------------------------------------------------
// Fused "heads" epilogue for the Q/K/V projections (attention.py:127-129,137-144; rotary.py:6-18,72-84): an N-tile holds two
// whole heads, a thread owns one token row, so the per-head LayerNorm(dh) and the rotate-half RoPE are in-thread.
//   kind 0/1 (q/k): LN affine -> RoPE (optional) -> bf16 rows [b*H + h, l, 0..dh) (pitch ld_qk), written 144/128 B-coalesced
//                   through the staging tile;
//   kind 2   (v)  : bf16 V^T [b*H + h, d, l] (pitch Lpad): for a fixed d a warp stores 32 consecutive tokens (64 B).
struct EpiHeadsParams {
  int D, H, L;                 // model width, heads, tokens per batch item
  int kind[3];                 // section (n / D) -> 0 q, 1 k, 2 v
  float nw[2][72];             // LayerNorm(dh) weight / bias for q, k -- BY VALUE: they live in the constant bank, so the
  float nb[2][72];             // normalisation FFMAs take them as operands instead of issuing 2 x dh loads per token
  const float2* rope;          // [L][dh/2] (cos, sin) table or null
  int rope_ld;
  int rope_mufu;               // 1: evaluate cos/sin with the MUFU (__sincosf) from inv_freq instead of reading the table
  float inv_freq[36];          // rotary.py:41-42 (checkpoint buffer), by value -> constant bank
  int rope_kinds;              // bit k set: apply RoPE to kind k
  __nv_bfloat16* out[3];       // per kind: q rows, k rows, v^T
  int ld_qk, dvp, Lpad;
  int dbg;                     // profiling instantiation only (option heads_dbg; results garbage): 1 no RoPE, 2 no per-head LayerNorm, 4 no V^T stores, 8 no q / k stores
  FoldIn fin;                  // LayerNorm (+ AdaLN modulate) of the block input folded into this projection
};

// The per-row steps of the heads epilogue, shared by the parked-tile (EpiHeads) and register-fragment (EpiHeadsFrag) schedules so that both
// run the same float operations in the same order.  Head hh of the N-tile at n0 -> section (q / k / v of the reference column order) and head
// index; false: the tile's pair slot hh lies past N.
constexpr int heads_bn(int dh, int hpt) { return hpt == 3 ? (dh == 72 ? 224 : 3 * dh) : 2 * dh; }
template <int DH, int HPT>
__device__ __forceinline__ bool head_of_tile(const EpiHeadsParams& ep, int n0, int hh, int N, int& sec, int& head) {
  if (HPT == 3) {
    const int g = (n0 / heads_bn(DH, HPT)) * 3 + hh;   // global head index in [q heads | k heads | v heads]
    sec = g / ep.H;
    head = g - sec * ep.H;
    return true;
  }
  const int n = n0 + hh * DH;
  if (n >= N) return false;
  sec = n / ep.D;
  head = (n - sec * ep.D) / DH;
  return true;
}
// LayerNorm(dh) with the affine of `kind` (0 q, 1 k), then rotate-half RoPE at position l, in place on one token row of one head.
template <int DH, bool DBG>
__device__ __forceinline__ void head_ln_rope(const EpiHeadsParams& ep, float (&v)[DH], int kind, int l) {
  float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < DH; ++i) { s1[i & 3] += v[i]; s2[i & 3] = fmaf(v[i], v[i], s2[i & 3]); }
  const float mean = ((s1[0] + s1[1]) + (s1[2] + s1[3])) * (1.0f / DH);
  const float var = fmaxf(((s2[0] + s2[1]) + (s2[2] + s2[3])) * (1.0f / DH) - mean * mean, 0.f);
  const float rstd = rsqrtf(var + 1e-5f);
  const float nmr = -mean * rstd;
  if (DBG && (ep.dbg & 2)) {
  } else if (kind == 0) {
#pragma unroll
    for (int i = 0; i < DH; ++i) v[i] = fmaf(fmaf(v[i], rstd, nmr), ep.nw[0][i], ep.nb[0][i]);
  } else {
#pragma unroll
    for (int i = 0; i < DH; ++i) v[i] = fmaf(fmaf(v[i], rstd, nmr), ep.nw[1][i], ep.nb[1][i]);
  }
  if (ep.rope != nullptr && ((ep.rope_kinds >> kind) & 1) && !(DBG && (ep.dbg & 1))) {
    const float2* cs = ep.rope + (size_t)l * (DH / 2);
    const float lf = (float)l;
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) {
      float2 c;
      if (ep.rope_mufu) __sincosf(lf * ep.inv_freq[i], &c.y, &c.x);
      else c = __ldg(cs + i);
      const float a = v[i], bq = v[i + DH / 2];
      v[i] = a * c.x - bq * c.y;
      v[i + DH / 2] = bq * c.x + a * c.y;
    }
  }
}
// q / k row bh * L + l as dh bf16 with 16-byte stores (out[kind] 16-byte aligned, ld_qk a multiple of 8)
template <int DH>
__device__ __forceinline__ void head_store_row(const EpiHeadsParams& ep, const float (&v)[DH], int kind, size_t bh, int l) {
  uint4* dst = reinterpret_cast<uint4*>(ep.out[kind] + (bh * ep.L + l) * (size_t)ep.ld_qk);
#pragma unroll
  for (int g = 0; g < DH / 8; ++g)
    dst[g] = make_uint4(pack_bf16(v[8 * g], v[8 * g + 1]), pack_bf16(v[8 * g + 2], v[8 * g + 3]), pack_bf16(v[8 * g + 4], v[8 * g + 5]),
                        pack_bf16(v[8 * g + 6], v[8 * g + 7]));
}
// V^T column l of head bh: dh values, then zeros up to dvp
template <int DH>
__device__ __forceinline__ void head_store_vt(const EpiHeadsParams& ep, const float (&v)[DH], size_t bh, int l) {
  __nv_bfloat16* dst = ep.out[2] + bh * ep.dvp * ep.Lpad + l;
#pragma unroll
  for (int i = 0; i < DH; ++i) { *dst = __float2bfloat16_rn(v[i]); dst += ep.Lpad; }
  for (int i = DH; i < ep.dvp; ++i) { *dst = __float2bfloat16_rn(0.f); dst += ep.Lpad; }
}

// HPT = 2: tile = two adjacent heads of the reference column order (N-tile 2*dh).  HPT = 3: the packed QKV layout -- the
// 3H heads of [q | k | v] are regrouped three per tile (N-tile 224 for dh = 72: 3 x 72 + 8 zero columns; 192 for dh = 64), which
// makes the tile wide enough for the tensor pipe (narrow tiles are operand-bandwidth bound).
// Eight epilogue warps, two per 32-row group: warpgroup wg takes heads wg, wg + 2 of the tile on the group's rows, i.e. one head each at HPT = 2;
// at HPT = 3 warpgroup 0 takes heads 0 and 2 and warpgroup 1 head 1 (12 head x row-group units on 8 warps take two rounds however they are
// dealt).  The packed tile runs with the producer warpgroup's registers (GemmCfg::PRODUCER_WG): 112 accumulators per thread in the mainloop,
// two dh-wide rows per thread in the epilogue.
template <int DH, int HPT = 2, bool FOLD = false, bool DBG = false>
struct EpiHeads {
  using Params = EpiHeadsParams;
  static constexpr int BN = heads_bn(DH, HPT);
  static constexpr int EPI_WARPS = 8;
  static constexpr bool WIDE_REGS = HPT == 3;
  static constexpr int STAGE_FLOATS = EPI_STAGE_FLOATS;
  template <class Wait>
  static __device__ __forceinline__ void run(const Params& ep, float* st, const AccRows& ar, int row0, int nvalid, int n0, int N, int lane, int c_begin,
                                             int c_end, Wait wait) {
    const int row = row0 + lane;
    const bool row_ok = lane < nvalid;
    constexpr bool fold = FOLD;
    float f_rstd = 1.f, f_nmr = 0.f;
    if (fold && row_ok) fold_row_stats(ep.fin, row, f_rstd, f_nmr);   // issued before the accumulator wait
    wait();
    const int b = row_ok ? row / ep.L : 0, l = row_ok ? row - b * ep.L : 0;
#pragma unroll 1
    for (int hh = threadIdx.x >> 7; hh < HPT; hh += 2) {   // gemm_body's consumer warp 4 wg + (32-row group): heads wg, wg + 2
      int sec, head;
      if (!head_of_tile<DH, HPT>(ep, n0, hh, N, sec, head)) break;
      const int kind = ep.kind[sec];
      uint32_t r[DH];
      __syncwarp();
      acc_ld<64>(ar, hh * DH, lane, r);
      if constexpr (DH == 72) acc_ld<8>(ar, hh * DH + 64, lane, r + 64);
      float v[DH];
#pragma unroll
      for (int i = 0; i < DH; ++i) v[i] = __uint_as_float(r[i]);
      if (fold) {  // warp-uniform: per-row affine of the folded LayerNorm; u, v are the same for every row (uniform 16-byte loads)
        const float4* u4 = reinterpret_cast<const float4*>(ep.fin.u + n0 + hh * DH);
        const float4* v4 = reinterpret_cast<const float4*>(ep.fin.v + n0 + hh * DH);
#pragma unroll
        for (int i = 0; i < DH / 4; ++i) {
          const float4 uu = __ldg(u4 + i), vv = __ldg(v4 + i);
          v[4 * i] = fmaf(v[4 * i], f_rstd, fmaf(f_nmr, uu.x, vv.x));
          v[4 * i + 1] = fmaf(v[4 * i + 1], f_rstd, fmaf(f_nmr, uu.y, vv.y));
          v[4 * i + 2] = fmaf(v[4 * i + 2], f_rstd, fmaf(f_nmr, uu.z, vv.z));
          v[4 * i + 3] = fmaf(v[4 * i + 3], f_rstd, fmaf(f_nmr, uu.w, vv.w));
        }
      }
      const size_t bh = (size_t)b * ep.H + head;
      if (kind < 2) {
        head_ln_rope<DH, DBG>(ep, v, kind, l);
        // bf16 pairs -> staging granules (4 bf16 each) -> coalesced row stores
#pragma unroll
        for (int g = 0; g < DH / 4; ++g)
          stage_put(st, lane, g, __uint_as_float(pack_bf16(v[4 * g], v[4 * g + 1])), __uint_as_float(pack_bf16(v[4 * g + 2], v[4 * g + 3])));
        __syncwarp();
        if (lane < DH / 4 && !(DBG && (ep.dbg & 8))) {
          const int rb0 = row0 / ep.L, rl0 = row0 - rb0 * ep.L;
          __nv_bfloat16* base = ep.out[kind] + 4 * lane;
          const size_t head_rows = (size_t)ep.L * ep.ld_qk;
          const int nv = nvalid < 32 ? nvalid : 32;
#pragma unroll 4
          for (int rr = 0; rr < nv; ++rr) {
            int rl = rl0 + rr, rb = rb0;
            while (rl >= ep.L) { rl -= ep.L; ++rb; }   // normally at most one wrap (L >= 32); short contexts may wrap more
            *reinterpret_cast<float2*>(base + ((size_t)rb * ep.H + head) * head_rows + (size_t)rl * ep.ld_qk) = stage_get(st, rr, lane);
          }
        }
      } else if (row_ok && !(DBG && (ep.dbg & 4))) {
        head_store_vt<DH>(ep, v, bh, l);
      }
    }
  }
};

// The heads epilogue of the plain bf16 path (no LayerNorm fold, no profiling) on the wgmma fragment, for gemm_body's overlapped schedule (FRAG):
// the accumulator stays in the MMA warpgroups' registers, so the producer streams the next tile's k-blocks while this runs, and the ring gets
// the shared memory the parked tile and the staging tiles took (4 stages of the 224-wide tile instead of 3).  Each MMA warpgroup moves one head
// slice at a time (its 64 rows x dh fp32) from the fragment into its own shared-memory buffer; its first two warps take head hh, its last two
// head hh + 1, one token row per thread, and run EpiHeads' per-row code on them; each thread stores its own q / k row with 16-byte stores
// (head_store_row) where EpiHeads transposes it through the staging tile, so the outputs are the same bits.
template <int DH, int HPT>
struct EpiHeadsFrag {
  using Params = EpiHeadsParams;
  static constexpr bool FRAG = true;
  static constexpr int BN = heads_bn(DH, HPT);
  static constexpr int EPI_WARPS = 8;
  static constexpr bool WIDE_REGS = true;              // the producer warpgroup's registers: dh-wide rows next to the fragment, spill-free
  static constexpr int PITCH = DH + 4;                 // the thread == row 16-byte reads of 8 consecutive rows hit distinct banks
  static constexpr int STAGE_FLOATS = 64 * PITCH / 4;  // a warpgroup's four warps share one 64-row head slice
  static_assert(DH % 8 == 0, "head slices start on a fragment register quad");
  // d: this thread's m64nBN fragment of the warpgroup's rows m0 + 64 wg ..; tile: the warpgroup's head-slice buffer.  Rows >= g.M are not stored.
  static __device__ __forceinline__ void frag(const Params& ep, const CUtensorMap*, float (&d)[BN / 2], uint8_t* tile, int m0, int n0, const GemmShape& g,
                                              int wg, int lg, int lane) {
    float* buf = reinterpret_cast<float*>(tile);
    const int t = threadIdx.x & 127, half = t >> 6;   // half: warps 0-1 or 2-3 of the warpgroup
    const int row = m0 + 64 * wg + (t & 63);
    const bool row_ok = row < g.M;
    const int b = row_ok ? row / ep.L : 0, l = row_ok ? row - b * ep.L : 0;
    float* w0 = buf + (16 * lg + (lane >> 2)) * PITCH + 2 * (lane & 3);   // fragment row r0 (registers 4i, 4i + 1); r0 + 8: 4i + 2, 4i + 3
    const float4* rd = reinterpret_cast<const float4*>(buf + (t & 63) * PITCH);
#pragma unroll
    for (int p = 0; p < HPT; p += 2) {
      float v[DH];
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int hh = p + s;
        if (hh >= HPT) break;
        if (hh > 0) warpgroup_bar_sync(wg);   // the buffer's previous head has been read (gemm_body's barrier covers the previous tile)
#pragma unroll
        for (int i = 0; i < DH / 8; ++i) {
          const int j = 4 * (hh * DH / 8 + i);
          *reinterpret_cast<float2*>(w0 + 8 * i) = make_float2(d[j], d[j + 1]);
          *reinterpret_cast<float2*>(w0 + 8 * PITCH + 8 * i) = make_float2(d[j + 2], d[j + 3]);
        }
        warpgroup_bar_sync(wg);
        if (half == s) {
#pragma unroll
          for (int i = 0; i < DH / 4; ++i) {
            const float4 x = rd[i];
            v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
          }
        }
      }
      const int hh = p + half;
      int sec, head;
      if (hh >= HPT || !head_of_tile<DH, HPT>(ep, n0, hh, g.N, sec, head)) continue;
      const int kind = ep.kind[sec];
      const size_t bh = (size_t)b * ep.H + head;
      if (kind < 2) {
        head_ln_rope<DH, false>(ep, v, kind, l);
        if (row_ok) head_store_row<DH>(ep, v, kind, bh, l);
      } else if (row_ok) {
        head_store_vt<DH>(ep, v, bh, l);
      }
    }
  }
};

}  // namespace ezb

namespace ezb {
// ---------------------------------------------------------------------------------------------------------------
// The MLP of a DiT block (modules.py:263-277,366) as ONE persistent launch: phase 1 = the GEGLU projection (2-CTA cluster tiles, EpiGeglu), a
// grid-wide barrier, phase 2 = the output projection with its gated-residual epilogue (swap-AB tiles, EpiLinearT, incl. the LayerNorm fold
// outputs for the next block).  The grid is one CTA per SM (all co-resident), launched as clusters of two for phase 1.  Phase 2 reads the
// bf16 intermediate that phase 1 wrote with ordinary stores through TMA, hence the generic->async proxy fence after the barrier.
struct GridBarrier { unsigned int count; unsigned int gen; };
__device__ __forceinline__ void grid_barrier(GridBarrier* b) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();   // this CTA's global writes (all threads, ordered by the barrier above) before the arrive
    unsigned int gen;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(gen) : "l"(&b->gen) : "memory");
    if (atomicAdd(&b->count, 1u) == gridDim.x - 1) {
      b->count = 0;
      __threadfence();
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(&b->gen), "r"(gen + 1) : "memory");
    } else {
      unsigned int cur;
      do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cur) : "l"(&b->gen) : "memory");
      } while (cur == gen);
    }
  }
  __syncthreads();
  asm volatile("fence.proxy.async;" ::: "memory");
}
template <int BN1, class Epi1, class Epi2>
__global__ void __launch_bounds__((GemmCfg<BN1, Epi1>::THREADS), 1)
mlp_fused_kernel(const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmB1, const GemmShape g1, const typename Epi1::Params ep1,
                 const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2, const GemmShape g2, const typename Epi2::Params ep2,
                 GridBarrier* bar) {
  static_assert(GemmCfg<BN1, Epi1>::THREADS == GemmCfg<256, Epi2>::THREADS, "both phases use the same warp roles");
  extern __shared__ uint8_t smem_dyn[];
  gemm_body<BN1, Epi1, 2, true>(tmA1, tmB1, g1, ep1, smem_dyn);
  grid_barrier(bar);
  gemm_body<256, Epi2, 1>(tmA2, tmB2, g2, ep2, smem_dyn);
}

}  // namespace ezb
