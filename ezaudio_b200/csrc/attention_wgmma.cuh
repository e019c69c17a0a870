// Generation 8 of the tensor-core attention (sm_90a): O = softmax(Q K^T / sqrt(dh) [+ key mask]) V on warpgroup MMAs, fed by TMA.
//
// A CTA owns 128 query rows of one (b, h): two consumer warpgroups of 64 rows each, plus one producer warp that loads the Q tile once and the
// K / V^T key blocks (128 keys) into a two-stage ring (full / empty mbarriers, as in gemm_body).  Per key block a consumer warpgroup
//   issues S = Q K^T (SS wgmma, N = 128 keys) and O += P V of the PREVIOUS block (RS wgmma: P is the previous S accumulator re-packed to bf16 in
//   registers, N = the padded head width), then runs the online softmax of S while that P V product is on the tensor cores.
// The two consumer warpgroups take turns issuing their MMAs (named barriers 1 and 2), so one warpgroup's exponentials run under the other's
// wgmma.  At dh = 72 one score costs 320 padded MMA FLOPs and one exp2, and the SM's tensor rate over its MUFU rate is ~256 FLOPs per
// exponential: without this overlap the exponentials alone would hold the kernel near half of the tensor peak.
//
// Layouts are the ones the QKV epilogue writes (no producer change): Q, K bf16 [B*H, L, dhp]; V^T bf16 [B*H, dvp, Lkpad]; output bf16
// [B, Lq, H*dh].  The tensor maps are 3-D {cols, rows, B*H} with the extent of the head (dh columns of Q / K; dh rows and Lk keys of V^T), so
// TMA zero-fills everything past a head's end and never reads the next head's data or the padding past Lk.  A dh = 72 row is one 64-column box
// with the 128-byte swizzle plus one 16-column box with the 32-byte swizzle (columns 72..79 zero-filled): 5 k16 steps.
//
// Numerics as generation 6 (attention_mma.cuh): exp2-domain online softmax with scale_log2, P rounded to bf16, row sums over the rounded P,
// offset 0 for a row without a valid key yet, 1/l = 0 for an empty row.  Tiles and the key-block order depend only on (Lq, Lk, dh), so a
// (b, h) gives the same bits whatever else is in the batch.
// Padded batches (p.lens): keys at or past lens[b] score -inf, key blocks wholly past it are not loaded, and in the one block that straddles it
// the V^T columns past the end are zeroed in shared memory before the P V product (0 * NaN would be NaN): valid rows are bit-identical to a
// run at L = lens[b].  Query rows at or past lens[b] are written as zeros; a tile wholly past it writes zeros and loads nothing.
#pragma once
#include "host.cuh"

namespace ezb {

// launches per attention generation (4, 6, 7, 8) since the library was loaded, process-wide: ezb_attn_launch_count
inline unsigned long long* attn_launch_counts() {
  static unsigned long long n[9] = {};
  return n;
}

constexpr int AW_QROWS = 128;                // query rows per CTA: two consumer warpgroups of 64
constexpr int AW_KB = 128;                   // keys per block
constexpr int AW_STAGES = 2;                 // K / V^T ring depth
constexpr int AW_PRODUCER = 8;               // warp index of the TMA producer (first warp of the third warpgroup)
constexpr int AW_THREADS = 3 * 128;
// registers per thread after the split (setmaxnreg): the producer warpgroup gives its registers to the consumers, whose S, P and O fragments
// (64 + 32 + DK / 2 per thread) do not fit the 168 of an even split
constexpr int AW_REGS_PRODUCER = 24, AW_REGS_CONSUMER = 240;

struct AttnWgParams {
  const uint8_t* key_mask;  // [B, Lk] or null
  const int32_t* lens;      // [B] (device) or null, see the file comment
  __nv_bfloat16* out;       // [B, Lq, H*dh]
  int H, Lq, Lk, dh;
  float scale_log2;         // (1/sqrt(dh)) * log2(e)
};

// DK: head width padded to the MMA (64 for dh 64, 80 for dh 72).  Offsets from a 1024-byte aligned base; every TMA box starts on a multiple
// of 1024 B, so the swizzle pattern TMA writes is the one the wgmma descriptors assume.
template <int DK>
struct AttnWgSmem {
  static constexpr bool TAIL = DK == 80;                       // the 16-column, 32-byte swizzled box of columns 64..79
  static constexpr int Q_MAIN = AW_QROWS * 128, Q_BYTES = Q_MAIN + (TAIL ? AW_QROWS * 32 : 0);
  static constexpr int K_MAIN = AW_KB * 128, K_BYTES = K_MAIN + (TAIL ? AW_KB * 32 : 0);
  static constexpr int V_BOX = DK * 128;                       // DK rows of 64 keys
  static constexpr int STAGE = K_BYTES + (AW_KB / 64) * V_BOX;
  static constexpr int BAR = Q_BYTES + AW_STAGES * STAGE;
  static constexpr size_t BYTES = BAR + (1 + 2 * AW_STAGES) * 8 + 1024;
  static_assert(Q_BYTES % 1024 == 0 && K_BYTES % 1024 == 0 && V_BOX % 1024 == 0, "box alignment");
};

__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
template <int R>
__device__ __forceinline__ void fence_regs_u32(uint32_t (&d)[R][4]) {
#pragma unroll
  for (int i = 0; i < R; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(d[i][j])::"memory");
}

template <int DK, bool VARLEN, bool MASKED>
__global__ void __launch_bounds__(AW_THREADS, 1)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmQt, const __grid_constant__ CUtensorMap tmK,
                  const __grid_constant__ CUtensorMap tmKt, const __grid_constant__ CUtensorMap tmV, const AttnWgParams p) {
  using SM = AttnWgSmem<DK>;
  extern __shared__ uint8_t aw_smem_raw[];
  uint8_t* smem = aw_smem_raw + ((1024u - (smem_u32(aw_smem_raw) & 1023u)) & 1023u);
  uint64_t* full_q = reinterpret_cast<uint64_t*>(smem + SM::BAR);
  uint64_t* full = full_q + 1;
  uint64_t* empty = full + AW_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, bh = blockIdx.y, b = bh / p.H, h = bh - b * p.H;

  if (threadIdx.x == 0) {
    mbar_init(full_q, 1);
    for (int i = 0; i < AW_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);   // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  if (warp == AW_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    if (SM::TAIL) { tma_prefetch_desc(&tmQt); tma_prefetch_desc(&tmKt); }
  }
  __syncthreads();
  pdl_launch();
  pdl_wait();   // global memory (q / k / v^T, lens, mask, out) is touched only below

  const int lk = VARLEN ? min(max(p.lens[b], 1), p.Lk) : p.Lk;
  const int lq = VARLEN ? min(max(p.lens[b], 1), p.Lq) : p.Lq;
  const int ld = p.H * p.dh;
  __nv_bfloat16* ob = p.out + (size_t)b * p.Lq * ld + (size_t)h * p.dh;
  if (VARLEN && qt * AW_QROWS >= lq) {   // a tile of padded query rows (CTA-uniform): zeros, nothing is loaded
    for (int i = threadIdx.x; i < AW_QROWS * (p.dh / 2); i += AW_THREADS) {
      const int r = qt * AW_QROWS + i / (p.dh / 2), col = 2 * (i % (p.dh / 2));
      if (r < p.Lq) *reinterpret_cast<uint32_t*>(ob + (size_t)r * ld + col) = 0u;
    }
    return;
  }
  const int nblk = (lk + AW_KB - 1) / AW_KB;

  if (warp >= AW_PRODUCER) {
    // ------------------------------------------------ TMA producer (one thread; the other warps only give their registers away)
    setmaxnreg_dec<AW_REGS_PRODUCER>();
    if (warp == AW_PRODUCER && lane == 0) {
      mbar_expect_tx(full_q, SM::Q_BYTES);
      tma_load_3d(smem, &tmQ, full_q, 0, qt * AW_QROWS, bh);
      if (SM::TAIL) tma_load_3d(smem + SM::Q_MAIN, &tmQt, full_q, 64, qt * AW_QROWS, bh);
      uint32_t stage = 0, phase = 0;
      for (int blk = 0; blk < nblk; ++blk) {
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_expect_tx(&full[stage], SM::STAGE);
        uint8_t* st = smem + SM::Q_BYTES + stage * SM::STAGE;
        const int k0 = blk * AW_KB;
        tma_load_3d(st, &tmK, &full[stage], 0, k0, bh);
        if (SM::TAIL) tma_load_3d(st + SM::K_MAIN, &tmKt, &full[stage], 64, k0, bh);
#pragma unroll
        for (int v = 0; v < AW_KB / 64; ++v) tma_load_3d(st + SM::K_BYTES + v * SM::V_BOX, &tmV, &full[stage], k0 + 64 * v, 0, bh);
        if (++stage == AW_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ------------------------------------------------ consumers: warpgroup wg owns query rows 64 wg .. 64 wg + 63 of the tile
  setmaxnreg_inc<AW_REGS_CONSUMER>();
  const int wg = warp >> 2, wl = warp & 3, g = lane >> 2, t = lane & 3;
  const uint8_t* mask = MASKED ? p.key_mask + (size_t)b * p.Lk : nullptr;
  const uint32_t q_main = smem_u32(smem + wg * 64 * 128), q_tail = smem_u32(smem + SM::Q_MAIN + wg * 64 * 32);
  const int my_bar = 1 + wg, other_bar = 2 - wg;   // warpgroup 0 issues first
  float o[DK / 2];
#pragma unroll
  for (int i = 0; i < DK / 2; ++i) o[i] = 0.f;
  float s[AW_KB / 2];
  uint32_t pa[AW_KB / 16][4];
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows g and g + 8 of this warp's 16

  auto stage_base = [&](uint32_t st) { return smem + SM::Q_BYTES + st * SM::STAGE; };
  auto pv = [&](uint32_t st) {
    const uint32_t v0 = smem_u32(stage_base(st) + SM::K_BYTES);
#pragma unroll
    for (int kk = 0; kk < AW_KB / 16; ++kk) WgmmaRS<DK>::mma(o, pa[kk], wgmma_desc_sw128(v0 + (kk >> 2) * SM::V_BOX) + 2 * (kk & 3), 1);
  };
  auto release = [&](uint32_t st) {
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[st]);
  };

  // S = Q K^T of the block in stage st (one commit group)
  auto issue_s = [&](uint32_t st) {
    const uint32_t kb = smem_u32(stage_base(st));
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) Wgmma<AW_KB>::mma(s, wgmma_desc_sw128(q_main) + 2 * ks, wgmma_desc_sw128(kb) + 2 * ks, ks != 0);
    if (SM::TAIL) Wgmma<AW_KB>::mma(s, wgmma_desc_sw32(q_tail), wgmma_desc_sw32(kb + SM::K_MAIN), 1);
    wgmma_commit();
  };
  // online softmax of the block at key k0 (stage st): S -> unnormalised fp32 P in place, new row maxima, O / l rescale factors.  Masking is
  // branch-free (every register the next wgmma reads is written on a uniform path, so ptxas need not serialise the wgmma).
  auto softmax = [&](int k0, uint32_t st, float& c0, float& c1) {
#pragma unroll
    for (int j = 0; j < AW_KB / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = k0 + 8 * j + 2 * t + e;
        bool ok = key < lk;
        if (MASKED) ok = ok && mask[key] != 0;
        s[4 * j + e] = ok ? s[4 * j + e] : -INFINITY;
        s[4 * j + 2 + e] = ok ? s[4 * j + 2 + e] : -INFINITY;
      }
    }
    float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < AW_KB / 8; ++j) {
      bm0 = fmaxf(bm0, fmaxf(s[4 * j], s[4 * j + 1]));
      bm1 = fmaxf(bm1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
    }
#pragma unroll
    for (int o2 = 1; o2 <= 2; o2 <<= 1) {
      bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, o2));
      bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, o2));
    }
    const float nm0 = fmaxf(m0, bm0 * p.scale_log2), nm1 = fmaxf(m1, bm1 * p.scale_log2);
    const float off0 = nm0 == -INFINITY ? 0.f : nm0, off1 = nm1 == -INFINITY ? 0.f : nm1;   // a row with no valid key yet
    c0 = exp2f(m0 - off0);
    c1 = exp2f(m1 - off1);
    m0 = nm0; m1 = nm1;
#pragma unroll
    for (int j = 0; j < AW_KB / 8; ++j) {
      s[4 * j] = exp2f(fmaf(s[4 * j], p.scale_log2, -off0));
      s[4 * j + 1] = exp2f(fmaf(s[4 * j + 1], p.scale_log2, -off0));
      s[4 * j + 2] = exp2f(fmaf(s[4 * j + 2], p.scale_log2, -off1));
      s[4 * j + 3] = exp2f(fmaf(s[4 * j + 3], p.scale_log2, -off1));
    }
    if (VARLEN && k0 + AW_KB > lk) {
      // the block that straddles the sample's end: V^T columns past it may hold anything (NaN included) and P is 0 there, so zero them
      // before this block's P V product reads them (both warpgroups write the same zeros; each orders its own writes before its wgmma)
      uint8_t* vb = stage_base(st) + SM::K_BYTES;
      const int c_lo = lk - k0, n = AW_KB - c_lo;
      for (int i = threadIdx.x & 127; i < DK * n; i += 128) {
        const int d = i / n, c = c_lo + (i - d * n);
        const int byte = (c & 63) * 2;
        *reinterpret_cast<__nv_bfloat16*>(vb + (c >> 6) * SM::V_BOX + d * 128 + ((((byte >> 4) ^ (d & 7)) << 4) | (byte & 15))) = __float2bfloat16(0.f);
      }
      fence_proxy_async_smem();
      named_bar_sync(3 + wg, 128);
    }
  };
  // O and l rescaled, P packed to the bf16 A fragments of the next P V product
  auto absorb = [&](float c0, float c1) {
    l0 *= c0; l1 *= c1;
#pragma unroll
    for (int j = 0; j < DK / 8; ++j) { o[4 * j] *= c0; o[4 * j + 1] *= c0; o[4 * j + 2] *= c1; o[4 * j + 3] *= c1; }
#pragma unroll
    for (int kk = 0; kk < AW_KB / 16; ++kk) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int j = 2 * kk + hh;
        const uint32_t lo = pack_bf16(s[4 * j], s[4 * j + 1]), hi = pack_bf16(s[4 * j + 2], s[4 * j + 3]);
        // the row sums use the bf16-rounded probabilities the P V product sees
        const __nv_bfloat162 lo2 = *reinterpret_cast<const __nv_bfloat162*>(&lo), hi2 = *reinterpret_cast<const __nv_bfloat162*>(&hi);
        l0 += __low2float(lo2) + __high2float(lo2);
        l1 += __low2float(hi2) + __high2float(hi2);
        pa[kk][2 * hh] = lo;
        pa[kk][2 * hh + 1] = hi;
      }
    }
  };

  if (wg == 1) named_bar_arrive(1, 256);
  mbar_wait(full_q, 0);
  float c0, c1;
  // block 0: nothing to overlap its softmax with
  mbar_wait(&full[0], 0);
  named_bar_sync(my_bar, 256);
  wgmma_fence();
  issue_s(0);
  named_bar_arrive(other_bar, 256);
  wgmma_wait<0>();
  wgmma_fence_regs(s);
  softmax(0, 0, c0, c1);
  absorb(c0, c1);
  uint32_t prev = 0, stage = 1 % AW_STAGES, phase = AW_STAGES == 1;
  for (int blk = 1; blk < nblk; ++blk) {
    const int k0 = blk * AW_KB;
    mbar_wait(&full[stage], phase);
    named_bar_sync(my_bar, 256);
    wgmma_fence();
    issue_s(stage);
    pv(prev);   // the previous block's P V runs under this block's softmax
    wgmma_commit();
    named_bar_arrive(other_bar, 256);
    wgmma_wait<1>();
    wgmma_fence_regs(s);
    softmax(k0, stage, c0, c1);
    // the previous block's P V is done: its stage goes back to the producer, and O and P may be rewritten
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    fence_regs_u32(pa);
    release(prev);
    absorb(c0, c1);
    prev = stage;
    if (++stage == AW_STAGES) { stage = 0; phase ^= 1; }
  }
  // the last block's P V (warpgroup 1 has no successor turn to hand over)
  named_bar_sync(my_bar, 256);
  wgmma_fence();
  pv(prev);
  wgmma_commit();
  if (wg == 0) named_bar_arrive(other_bar, 256);
  wgmma_wait<0>();
  wgmma_fence_regs(o);
  release(prev);

#pragma unroll
  for (int o2 = 1; o2 <= 2; o2 <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, o2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, o2);
  }
  const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
  const int r0 = qt * AW_QROWS + wg * 64 + wl * 16 + g, r1 = r0 + 8;
#pragma unroll
  for (int j = 0; j < DK / 8; ++j) {
    const int col = 8 * j + 2 * t;
    if (col < p.dh) {
      if (r0 < p.Lq) *reinterpret_cast<uint32_t*>(ob + (size_t)r0 * ld + col) = (!VARLEN || r0 < lq) ? pack_bf16(o[4 * j] * i0, o[4 * j + 1] * i0) : 0u;
      if (r1 < p.Lq) *reinterpret_cast<uint32_t*>(ob + (size_t)r1 * ld + col) = (!VARLEN || r1 < lq) ? pack_bf16(o[4 * j + 2] * i1, o[4 * j + 3] * i1) : 0u;
    }
  }
}

template <int DK>
int attn_wgmma_launch(Device& dev, cudaStream_t st, const CUtensorMap* const (&tm)[5], const AttnWgParams& p, int B, int H) {
  const int which = (p.lens != nullptr) * 2 + (p.key_mask != nullptr);
  auto kern = which == 3 ? attn_wgmma_kernel<DK, true, true> : which == 2 ? attn_wgmma_kernel<DK, true, false>
            : which == 1 ? attn_wgmma_kernel<DK, false, true> : attn_wgmma_kernel<DK, false, false>;
  const size_t smem = AttnWgSmem<DK>::BYTES;
  static int attr_set[4][16];   // function attributes are per device and kernel; 0: not yet, else device id + 1
  int& set = attr_set[which][dev.id & 15];
  if (set != dev.id + 1) {
    EZB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    set = dev.id + 1;
  }
  ++attn_launch_counts()[8];
  return launch_k(kern, dim3((p.Lq + AW_QROWS - 1) / AW_QROWS, B * H), dim3(AW_THREADS), smem, st, 1, *tm[0], *tm[1], *tm[2], *tm[3], *tm[4], p);
}

// dh 64 or 72; q, k [B*H, L, dhp] and vt [B*H, dvp, Lkpad] as attention_mma() takes them; lens: [B] valid tokens per sample (device) or null
inline int attention_wgmma(Device& dev, cudaStream_t st, const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* vt, const uint8_t* key_mask,
                           __nv_bfloat16* out, int B, int H, int Lq, int Lk, int Lkpad, int dh, int dhp, int dvp, float scale, const int32_t* lens) {
  if (dh != 64 && dh != 72) return fail(EZB_ERR_UNSUPPORTED, "attention generation 8: head dimension %d (64 or 72)", dh);
  const int DK = dh == 64 ? 64 : 80;
  const uint64_t BH = (uint64_t)B * H;
  const CUtensorMap* tm[5];
  EZB_TRY(dev.tmaps.get3d_box(q, dh, Lq, BH, dhp, (uint64_t)Lq * dhp, 64, AW_QROWS, &tm[0]));
  EZB_TRY(dev.tmaps.get3d_box(k, dh, Lk, BH, dhp, (uint64_t)Lk * dhp, 64, AW_KB, &tm[2]));
  EZB_TRY(dev.tmaps.get3d_box(vt, Lk, dh, BH, Lkpad, (uint64_t)dvp * Lkpad, 64, DK, &tm[4]));
  if (DK == 80) {
    EZB_TRY(dev.tmaps.get3d_box(q, dh, Lq, BH, dhp, (uint64_t)Lq * dhp, 16, AW_QROWS, &tm[1]));
    EZB_TRY(dev.tmaps.get3d_box(k, dh, Lk, BH, dhp, (uint64_t)Lk * dhp, 16, AW_KB, &tm[3]));
  } else {
    tm[1] = tm[0]; tm[3] = tm[2];   // unused
  }
  AttnWgParams p;
  p.key_mask = key_mask; p.lens = lens; p.out = out;
  p.H = H; p.Lq = Lq; p.Lk = Lk; p.dh = dh;
  p.scale_log2 = scale * 1.4426950408889634f;
  return DK == 64 ? attn_wgmma_launch<64>(dev, st, tm, p, B, H) : attn_wgmma_launch<80>(dev, st, tm, p, B, H);
}

}  // namespace ezb
