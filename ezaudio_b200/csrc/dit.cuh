// DiT / ControlNet instance: packed weights, workspace, step-invariant caches and the per-step launch sequence.
// Reference: src/models/udit.py:281-362 (UDiT.forward), src/models/blocks.py:120-160 (DiTBlock._forward),
// src/models/conditioners.py:156-183 (MaskDiT.forward), src/models/controlnet.py:252-315 (DiTControlNet.forward).
#pragma once
#include <functional>
#include <set>
#include <vector>

#include "attention_simt.cuh"
#include "attention_mma.cuh"
#include "host.cuh"
#include "gemm_ln.cuh"

namespace ezb {

typedef __nv_bfloat16 bf16;

struct BlockW {
  bf16 *qkv = nullptr, *proj = nullptr, *cq = nullptr, *ckv = nullptr, *cproj = nullptr, *mlp1 = nullptr, *mlp2 = nullptr, *skip = nullptr;
  float *b_proj = nullptr, *b_cproj = nullptr, *b_mlp1 = nullptr, *b_mlp2 = nullptr, *b_skip = nullptr;
  float *n1w = nullptr, *n1b = nullptr, *n2w = nullptr, *n2b = nullptr, *n3w = nullptr, *n3b = nullptr, *ncw = nullptr, *ncb = nullptr, *snw = nullptr,
        *snb = nullptr;
  float *nqw = nullptr, *nqb = nullptr, *nkw = nullptr, *nkb = nullptr, *cnqw = nullptr, *cnqb = nullptr, *cnkw = nullptr, *cnkb = nullptr;
  float *table = nullptr, *lora_a = nullptr, *lora_b = nullptr, *inv_freq = nullptr;
  bf16* zero_w = nullptr;
  float* zero_b = nullptr;
  float h_nq[2][96] = {}, h_nk[2][96] = {}, h_cnq[2][96] = {}, h_cnk[2][96] = {};  // host copies [weight|bias][dh] of the per-head LayerNorms
  // folded-LayerNorm tables (gemm.cuh FoldIn / FoldOut): per timestep [T][.] for the modulated sites 1 (norm1 -> QKV) and 3 (norm3 -> GEGLU),
  // static for site 2 (norm2 -> cross-Q) and the skip path (skip_norm -> skip_linear)
  float *g1 = nullptr, *u1 = nullptr, *v1 = nullptr, *g3 = nullptr, *u3 = nullptr, *v3 = nullptr, *u2 = nullptr, *v2 = nullptr, *us = nullptr, *vs = nullptr;
  float2 *st_skip = nullptr, *st_a = nullptr, *st_b = nullptr, *st_out = nullptr;   // per-row partial sums written by the residual-stream GEMMs
  float *lnG1 = nullptr, *lnC1 = nullptr, *lnG3 = nullptr, *lnC3 = nullptr;   // [T][D]: norm1 / norm3 affine x AdaLN modulation precombined per timestep (ln_gc_kernel)
  // per-clip cross-attention K / V^T caches
  float *kc32 = nullptr, *vc32 = nullptr;
  bf16 *kc16 = nullptr, *vtc16 = nullptr;
  // FP8 mode: e4m3 copies of the packed QKV and GEGLU weights with per-row scales (quantised at finalize)
  uint8_t *qkv8 = nullptr, *mlp18 = nullptr;
  float *s_qkv = nullptr, *s_mlp1 = nullptr;
};

struct WeightSpec {
  std::vector<int64_t> shape;
  std::function<int(const float*, cudaStream_t)> load;
  bool loaded = false;
};

constexpr int KP_PATCH_ALIGN = 8;

// ---------------------------------------------------------------- launches of the step's bandwidth kernels (elementwise.cuh)
// Shared by Dit and the kernel-level test hook (ezb_test_step), so that a test runs exactly the launch the model makes.
// LayerNorm kernel: LN_AUTO = what option "ln_variant" selects for these parameters; the others force one kernel, which the caller has
// checked can take them.
enum LnVariant { LN_AUTO = 0, LN_GENERIC = 1, LN_REG1 = 2, LN_REG8 = 3, LN_GC = 4, LN_CAT = 5 };
inline int ln_select(const LnParams& p) {
  if (p.kmul == 1 && p.x2 == nullptr && p.w != nullptr && (p.D1 == 1152 || p.D1 == 1024)) {
    if (opt_ln_variant() == 2 && p.G != nullptr && (p.shift == nullptr || p.mod_bstride == 0)) return LN_GC;
    return opt_ln_variant() == 1 ? LN_REG8 : LN_REG1;
  }
  if (p.kmul == 1 && opt_ln_variant() == 2 && p.x2 != nullptr && p.w != nullptr && p.shift == nullptr && p.D1 == p.D2 && (p.D1 == 1152 || p.D1 == 1024))
    return LN_CAT;
  return LN_GENERIC;
}
// launches per LayerNorm kernel (indexed by LnVariant) since the library was loaded, process-wide: ezb_ln_launch_count
inline unsigned long long* ln_launch_counts() {
  static unsigned long long n[LN_CAT + 1] = {};
  return n;
}
inline int ln_launch(const Device& dev, cudaStream_t st, const LnParams& p, int variant = LN_AUTO) {
  const int M = p.M;
  const bool d9 = p.D1 == 1152;
  if (variant == LN_AUTO) variant = ln_select(p);
  ++ln_launch_counts()[variant];
  switch (variant) {
    case LN_GC: {   // warps walk rows in a strided loop: at most 4 CTAs per SM
      const int grid = dev.num_sms * 4 < (M + 3) / 4 ? dev.num_sms * 4 : (M + 3) / 4;
      if (d9) return launch_k(ln_gc_kernel<9>, dim3(grid), dim3(128), 0, st, 1, p);
      return launch_k(ln_gc_kernel<8>, dim3(grid), dim3(128), 0, st, 1, p);
    }
    case LN_REG8:
      if (d9) return launch_k(ln_mod_cast_reg_kernel<9, 8>, dim3((M + 3) / 4), dim3(128), 0, st, 1, p);
      return launch_k(ln_mod_cast_reg_kernel<8, 8>, dim3((M + 3) / 4), dim3(128), 0, st, 1, p);
    case LN_REG1:
      if (d9) return launch_k(ln_mod_cast_reg_kernel<9, 1>, dim3((M + 3) / 4), dim3(128), 0, st, 1, p);
      return launch_k(ln_mod_cast_reg_kernel<8, 1>, dim3((M + 3) / 4), dim3(128), 0, st, 1, p);
    case LN_CAT:
      if (d9) return launch_k(ln_cat_reg_kernel<9>, dim3((M + 3) / 4), dim3(128), 0, st, 1, p);
      return launch_k(ln_cat_reg_kernel<8>, dim3((M + 3) / 4), dim3(128), 0, st, 1, p);
    default:
      return launch_k(ln_mod_cast_kernel, dim3((M + 7) / 8), dim3(256), 0, st, 1, p);
  }
}
template <typename TIn>
inline int qk_prep_launch(cudaStream_t st, const QkPrepParams<TIn>& p) {   // one warp per (token, section, head)
  const int total = p.B * p.L * p.H * p.n_sections;
  ++launch_counter();
  qk_prep_kernel<TIn><<<(total + 7) / 8, 256, 0, st>>>(p);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
inline int patch_pack_launch(cudaStream_t st, const float* x, const float* gt, const uint8_t* gt_mask, const float* mask_embed, bf16* out, int B, int C, int L,
                             int Kp, int kmul) {
  if ((2 * C) % 32) return fail(EZB_ERR_UNSUPPORTED, "latent_chans must be a multiple of 16");
  dim3 grid((L + 31) / 32, (2 * C) / 32, B), blockd(32, 8);
  return launch_k(patch_pack_kernel, grid, blockd, 0, st, 1, x, gt, gt_mask, mask_embed, out, B, C, L, Kp, kmul);
}
inline int final_conv_launch(const Device& dev, cudaStream_t st, const float* y, const float* wp, const float* bias, float* out, int B, int C, int L,
                             const int32_t* lens) {
  if (C % 4) return fail(EZB_ERR_UNSUPPORTED, "final conv: %d channels (multiple of 4 expected)", C);
  const size_t smem = ((size_t)36 * C + (size_t)(FC_GROUPS - 1) * 128 * 32) * sizeof(float);
  static bool fc_attr[16] = {};   // function attributes are per device
  if (!fc_attr[dev.id & 15]) { EZB_CUDA(cudaFuncSetAttribute(final_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024)); fc_attr[dev.id & 15] = true; }
  if (smem > 160 * 1024) return fail(EZB_ERR_UNSUPPORTED, "final conv: %d channels exceed the shared-memory tile", C);
  return launch_k(final_conv_kernel, dim3((L + 31) / 32, B), dim3(128 * FC_GROUPS), smem, st, 1, y, wp, bias, out, B, C, L, lens);
}
inline int small_linear_launch(cudaStream_t st, const float* in, int ld_in, const float* W, const float* bias, const float* add, int ld_add, float* out, int ld_out,
                               int R, int N, int K, int act, float scale) {   // one warp per output feature
  ++launch_counter();
  small_linear_kernel<<<(N + 7) / 8, 256, 0, st>>>(in, ld_in, W, bias, add, ld_add, out, ld_out, R, N, K, act, scale);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
inline int timestep_embed_launch(cudaStream_t st, const float* t, float* out, int n) {
  ++launch_counter();
  timestep_embed_kernel<<<(n * 128 + 255) / 256, 256, 0, st>>>(t, out, n);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// Tables of the folded LayerNorm (elementwise.cuh fold_gc_kernel / fold_uv_kernel), as Dit::build_fold_tables and Dit::finalize build them.
// fold_uv_kernel keeps a lane's share of a W row in 72 registers: K <= 72 * 32.
constexpr int FOLD_MAX_K = 72 * 32;
inline int fold_gc_launch(cudaStream_t st, const float* w, const float* b, const float* shift, const float* scale, int ld_mod, float* G, float* Cc, int R,
                          int D) {
  ++launch_counter();
  fold_gc_kernel<<<(R * D + 255) / 256, 256, 0, st>>>(w, b, shift, scale, ld_mod, G, Cc, R, D);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
inline int fold_uv_launch(cudaStream_t st, const bf16* W, int ldw, const float* G, const float* Cc, const float* add_v, float* U, float* V, int N, int K,
                          int R) {
  if (K > FOLD_MAX_K) return fail(EZB_ERR_UNSUPPORTED, "fold_uv: K %d", K);
  ++launch_counter();
  fold_uv_kernel<<<(N + 7) / 8, 256, 0, st>>>(W, ldw, G, Cc, add_v, U, V, N, K, R);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}

// Does Dit::lin run this linear as swap-AB tiles (host.cuh gemm_swapped) rather than on the 128-wide N-tiles of EpiLinear?  Only fp32-output
// layers without a uniform scale, in bf16 operands, on at least 512 tokens (m_select, 0: M) or with a folded LayerNorm; clips of fewer than 32
// rows stay on EpiLinear, whose generic path looks up each row's gate.  Shared with the test hook ezb_test_linear.
inline bool lin_takes_swap_ab(const EpiLinearParams& e, int M, int m_select, bool pair, bool swap_ab, int kmul) {
  const bool folded = e.fin.u != nullptr || e.fout.st != nullptr;
  const bool short_clips = e.gate != nullptr && e.rows_per_batch < 32;
  return pair && swap_ab && kmul == 1 && e.out_bf16 == nullptr && e.out_f32 != nullptr && e.out_scale == 0.f && e.bias_mod == 0 && !short_clips &&
         ((m_select ? m_select : M) >= 512 || folded);
}

struct FoldCtx {
  bool on = false;
  int t = 0;                  // timestep index (uniform over the batch)
  const float2* st_x = nullptr;
};

struct Dit {
  ezb_dit_desc d;
  Device* dev = nullptr;
  int D, H, dh, inner, r, C, nblk, half, kmul, Kp;
  int DHP, DVP;  // tensor-core attention paddings: q/k row pitch, v^T rows
  bool use_tc_attention = true;
  std::vector<void*> allocs;
  std::map<std::string, WeightSpec> specs;
  bool finalized = false;
  std::vector<BlockW> blk;
  // trunk weights
  bf16 *w_patch = nullptr, *w_ce0 = nullptr, *w_ce2 = nullptr, *w_final = nullptr;
  float *b_patch = nullptr, *b_ce0 = nullptr, *b_ce2 = nullptr, *b_final = nullptr;
  float *te_w0 = nullptr, *te_b0 = nullptr, *te_w2 = nullptr, *te_b2 = nullptr, *ta_w = nullptr, *ta_b = nullptr, *taf_w = nullptr, *taf_b = nullptr;
  float *fn_w = nullptr, *fn_b = nullptr, *fc_w = nullptr, *fc_b = nullptr, *mask_embed = nullptr;
  // controlnet stem (fp32, tiny)
  float *cs_in_w = nullptr, *cs_in_b = nullptr, *cs_me = nullptr, *cs_c0_w = nullptr, *cs_c0_b = nullptr, *cs_c1_w = nullptr, *cs_c1_b = nullptr,
        *cs_out_w = nullptr, *cs_out_b = nullptr;
  // workspace
  float *x0 = nullptr, *xa = nullptr, *xb = nullptr, *ybuf = nullptr, *ctx_emb = nullptr, *cond_emb = nullptr, *cs_t0 = nullptr, *cs_t1 = nullptr, *cs_t2 = nullptr;
  std::vector<float*> skips;
  bf16 *act = nullptr, *a_patch = nullptr, *attn_out = nullptr, *mid = nullptr;
  void* qkv = nullptr;  // bf16 (fast) or fp32 (parity) [M, 3D]
  float *q32 = nullptr, *k32 = nullptr, *v32 = nullptr;
  bf16 *q16 = nullptr, *k16 = nullptr, *vt16 = nullptr;
  uint8_t* ctx_mask = nullptr;
  float *t_vals = nullptr, *t_emb = nullptr, *t_h = nullptr, *t_tok = nullptr, *t_ada = nullptr, *t_lora = nullptr, *mod = nullptr, *mod_final = nullptr,
        *mod_b = nullptr, *modf_b = nullptr;
  int n_timesteps = 0, ctx_Be = 0, ctx_Lc = 0, ctx_Lpad = 0;
  // ControlNet condition cache (ezb_controlnet_set_condition): the stem's output [cond_Be, cond_L, D], apart from the cond_emb scratch that
  // ezb_controlnet_forward writes on every call
  float* cond_cache = nullptr;
  int cond_Be = 0, cond_L = 0;
  float2* rope_cs = nullptr;
  float h_inv_freq[48] = {};
  bool fused_heads = false;
  bool pair = true;       // 2-CTA cluster GEMMs sharing the weight tile (host.cuh gemm2)
  bool swap_ab = true;    // swap-AB tiles for the fp32-output N = D layers
  // LayerNorm folded into the neighbouring GEMMs (fast mode, uniform timestep): see gemm.cuh
  bool fold_cfg = false;  // handle built with the fold tables / buffers
  int fold_T = 0;         // timesteps the per-timestep tables hold
  int fold_n = 0;         // timesteps currently tabulated (0: tables not valid for the current schedule)
  int st_slots = 0, n_qkv = 0;
  size_t st_ld = 0;
  float *gc_G = nullptr, *gc_C = nullptr, *gF = nullptr, *uF = nullptr, *vF = nullptr;
  float2* st_x0 = nullptr;
  float *lnGF = nullptr, *lnCF = nullptr;   // FinalBlock norm, per timestep
  int gc_T = 0, gc_n = 0;                   // capacity / timesteps currently tabulated
  GridBarrier* grid_bar = nullptr;   // mlp_fused_kernel's self-resetting grid barrier
  std::vector<bf16*> cat;   // MaskDiT: per in-block [Mx, 2D] = [x of the paired out-block * snw[:D] | this block's output * snw[D:]]; ControlNet: [Mx, D] plain cast
  int geglu_bn = 128;     // N-tile of the GEGLU GEMM: packing group = geglu_bn / 2
  int qkv3_bn = 0;        // >0: self-attention QKV weight packed three heads per N-tile of this width (EpiHeads<DH,3>)
  const int32_t* lens = nullptr;   // forward(): valid frames per sample of the padded batch (device [Be]) or null; read by self-attention and the final conv
  // FP8 mode (precision 2): norm1 -> QKV and norm3 -> GEGLU run on e4m3 operands (ln8 writes act8 / act8_s), everything else as in bf16 mode
  bool fp8 = false;
  uint8_t* act8 = nullptr;
  float* act8_s = nullptr;

  ~Dit() {
    for (void* p : allocs) cudaFree(p);
  }
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

  // ---------------------------------------------------------------- weight registry
  void reg(const std::string& key, std::vector<int64_t> shape, std::function<int(const float*, cudaStream_t)> fn) {
    WeightSpec s;
    s.shape = std::move(shape);
    s.load = std::move(fn);
    specs[key] = std::move(s);
  }
  int reg_f32(const std::string& key, std::vector<int64_t> shape, float** dst) {
    size_t n = 1;
    for (auto v : shape) n *= v;
    EZB_TRY(alloc(dst, n));
    float* p = *dst;
    reg(key, shape, [p, n](const float* src, cudaStream_t st) -> int {
      EZB_CUDA(cudaMemcpyAsync(p, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
      return EZB_OK;
    });
    return EZB_OK;
  }
  // fp32 [N, K] -> rows [row_off, row_off+N) of bf16 dst [Ntot, kmul*Kpad]
  void reg_linear(const std::string& key, int N, int K, bf16* dst, int Kpad, int row_off, int geglu_inner = 0, std::vector<int64_t> shape = {},
                  int h3_head_off = -1) {
    const int km = kmul, gh = geglu_bn / 2;
    const int h3dh = h3_head_off >= 0 ? dh : 0, h3off = h3_head_off >= 0 ? h3_head_off : 0, h3bn = qkv3_bn;
    if (shape.empty()) shape = {N, K};
    reg(key, shape, [=](const float* src, cudaStream_t st) -> int {
      const size_t n = (size_t)N * Kpad;
      ++launch_counter();
      pack_weight_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, N, K, dst, Kpad, km, row_off, geglu_inner, gh, h3dh, h3off, h3bn);
      EZB_CUDA(cudaGetLastError());
      return EZB_OK;
    });
  }
  int alloc_w(bf16** dst, int N, int Kpad) { return alloc(dst, (size_t)N * kmul * Kpad); }

  int init(const ezb_dit_desc& desc, Device* device) {
    d = desc;
    dev = device;
    D = d.embed_dim; H = d.num_heads; inner = d.inner_dim; r = d.ada_rank; C = d.latent_chans;
    if (D <= 0 || H <= 0 || D % H) return fail(EZB_ERR_UNSUPPORTED, "embed_dim %d / num_heads %d", D, H);
    dh = D / H;
    half = d.depth / 2;
    nblk = d.is_controlnet ? half : d.depth + 1;
    kmul = d.precision == 1 ? 3 : 1;
    if (d.precision < 0 || d.precision > 2) return fail(EZB_ERR_UNSUPPORTED, "precision %d", d.precision);
    fp8 = d.precision == 2;
    pair = opt_pair_gemm() != 0;
    swap_ab = opt_swap_ab() != 0;
    geglu_bn = (pair && inner % 128 == 0) ? 256 : 128;
    qkv3_bn = (pair && d.precision != 1 && (D / H == 72 || D / H == 64) && H % 2 == 0 && opt_qkv3()) ? (D / H == 72 ? 224 : 192) : 0;
    if (dh > 96 || dh % 8 || D % 16 || inner % 64 || d.context_dim % 8 || d.depth % 2)
      return fail(EZB_ERR_UNSUPPORTED, "unsupported dims: D %d dh %d inner %d ctx %d depth %d", D, dh, inner, d.context_dim, d.depth);
    if (fp8 && (qkv3_bn == 0 || D > 1152))
      return fail(EZB_ERR_UNSUPPORTED, "fp8: needs the packed QKV (head dim 64 or 72, an even head count, options pair_gemm and qkv3 on) "
                  "and embed_dim <= 1152 (D %d dh %d H %d)", D, dh, H);
    if (d.max_batch < 1 || d.max_batch > 256 || d.max_len < 1 || d.max_ctx_len < 1 || d.max_timesteps < 1) return fail(EZB_ERR_ARG, "workspace bounds");
    Kp = (2 * C + 1 + KP_PATCH_ALIGN - 1) / KP_PATCH_ALIGN * KP_PATCH_ALIGN;
    // q / k row pitch: dh = 72 rows are 80 elements (160 bytes: 64 columns behind a SWIZZLE_128B box + a 16-column SWIZZLE_32B tail box, TMA only
    // needs 16-byte strides); the round-1 pitch of 128 moved 1.56x the algorithmic bytes (ncu dram__bytes_read 43.2 MB vs 27.6 MB)
    DHP = dh == 72 ? (opt_dhp80() ? 80 : 128) : (dh + 63) / 64 * 64;
    DVP = (dh + 15) / 16 * 16;
    use_tc_attention = (d.precision != 1);
    blk.resize(nblk);
    const std::string pre = d.is_controlnet ? "" : "model.";
    // ---- trunk
    EZB_TRY(reg_f32("mask_embed", {C}, &mask_embed));  // controlnet handles take the MaskDiT's mask_embed too (x257 is built from it)
    EZB_TRY(alloc_w(&w_patch, D, Kp));
    reg_linear(pre + "patch_embed.proj.weight", D, 2 * C + 1, w_patch, Kp, 0, 0, {D, 2 * C + 1, 1});
    EZB_TRY(reg_f32(pre + "patch_embed.proj.bias", {D}, &b_patch));
    EZB_TRY(reg_f32(pre + "time_embed.mlp.0.weight", {D, 256}, &te_w0));
    EZB_TRY(reg_f32(pre + "time_embed.mlp.0.bias", {D}, &te_b0));
    EZB_TRY(reg_f32(pre + "time_embed.mlp.2.weight", {D, D}, &te_w2));
    EZB_TRY(reg_f32(pre + "time_embed.mlp.2.bias", {D}, &te_b2));
    EZB_TRY(reg_f32(pre + "time_ada.weight", {6 * D, D}, &ta_w));
    EZB_TRY(reg_f32(pre + "time_ada.bias", {6 * D}, &ta_b));
    if (!d.is_controlnet) {
      EZB_TRY(reg_f32(pre + "time_ada_final.weight", {2 * D, D}, &taf_w));
      EZB_TRY(reg_f32(pre + "time_ada_final.bias", {2 * D}, &taf_b));
    }
    EZB_TRY(alloc_w(&w_ce0, D, d.context_dim));
    reg_linear(pre + "context_embed.0.weight", D, d.context_dim, w_ce0, d.context_dim, 0);
    EZB_TRY(reg_f32(pre + "context_embed.0.bias", {D}, &b_ce0));
    EZB_TRY(alloc_w(&w_ce2, D, D));
    reg_linear(pre + "context_embed.2.weight", D, D, w_ce2, D, 0);
    EZB_TRY(reg_f32(pre + "context_embed.2.bias", {D}, &b_ce2));
    // ---- blocks
    for (int i = 0; i < nblk; ++i) {
      BlockW& w = blk[i];
      std::string p;
      const bool is_out = !d.is_controlnet && i > half;
      if (d.is_controlnet || i < half) p = pre + "in_blocks." + std::to_string(i);
      else if (i == half) p = pre + "mid_block";
      else p = pre + "out_blocks." + std::to_string(i - half - 1);
      EZB_TRY(reg_f32(p + ".norm1.weight", {D}, &w.n1w)); EZB_TRY(reg_f32(p + ".norm1.bias", {D}, &w.n1b));
      EZB_TRY(reg_f32(p + ".norm2.weight", {D}, &w.n2w)); EZB_TRY(reg_f32(p + ".norm2.bias", {D}, &w.n2b));
      EZB_TRY(reg_f32(p + ".norm3.weight", {D}, &w.n3w)); EZB_TRY(reg_f32(p + ".norm3.bias", {D}, &w.n3b));
      EZB_TRY(reg_f32(p + ".norm_context.weight", {D}, &w.ncw)); EZB_TRY(reg_f32(p + ".norm_context.bias", {D}, &w.ncb));
      if (qkv3_bn > 0) {
        EZB_TRY(alloc_w(&w.qkv, H * qkv3_bn, D));  // zero-initialised: the 8 pad rows of every 224-row tile stay 0
        reg_linear(p + ".attn.to_q.weight", D, D, w.qkv, D, 0, 0, {}, 0);
        reg_linear(p + ".attn.to_k.weight", D, D, w.qkv, D, 0, 0, {}, H);
        reg_linear(p + ".attn.to_v.weight", D, D, w.qkv, D, 0, 0, {}, 2 * H);
      } else {
        EZB_TRY(alloc_w(&w.qkv, 3 * D, D));
        reg_linear(p + ".attn.to_q.weight", D, D, w.qkv, D, 0);
        reg_linear(p + ".attn.to_k.weight", D, D, w.qkv, D, D);
        reg_linear(p + ".attn.to_v.weight", D, D, w.qkv, D, 2 * D);
      }
      EZB_TRY(reg_f32(p + ".attn.norm_q.weight", {dh}, &w.nqw)); EZB_TRY(reg_f32(p + ".attn.norm_q.bias", {dh}, &w.nqb));
      EZB_TRY(reg_f32(p + ".attn.norm_k.weight", {dh}, &w.nkw)); EZB_TRY(reg_f32(p + ".attn.norm_k.bias", {dh}, &w.nkb));
      EZB_TRY(alloc_w(&w.proj, D, D));
      reg_linear(p + ".attn.proj.weight", D, D, w.proj, D, 0);
      EZB_TRY(reg_f32(p + ".attn.proj.bias", {D}, &w.b_proj));
      EZB_TRY(reg_f32(p + ".attn.rotary.inv_freq", {dh / 2}, &w.inv_freq));
      EZB_TRY(alloc_w(&w.cq, D, D));
      reg_linear(p + ".cross_attn.to_q.weight", D, D, w.cq, D, 0);
      EZB_TRY(alloc_w(&w.ckv, 2 * D, D));
      reg_linear(p + ".cross_attn.to_k.weight", D, D, w.ckv, D, 0);
      reg_linear(p + ".cross_attn.to_v.weight", D, D, w.ckv, D, D);
      EZB_TRY(reg_f32(p + ".cross_attn.norm_q.weight", {dh}, &w.cnqw)); EZB_TRY(reg_f32(p + ".cross_attn.norm_q.bias", {dh}, &w.cnqb));
      EZB_TRY(reg_f32(p + ".cross_attn.norm_k.weight", {dh}, &w.cnkw)); EZB_TRY(reg_f32(p + ".cross_attn.norm_k.bias", {dh}, &w.cnkb));
      EZB_TRY(alloc_w(&w.cproj, D, D));
      reg_linear(p + ".cross_attn.proj.weight", D, D, w.cproj, D, 0);
      EZB_TRY(reg_f32(p + ".cross_attn.proj.bias", {D}, &w.b_cproj));
      EZB_TRY(alloc_w(&w.mlp1, 2 * inner, D));
      reg_linear(p + ".mlp.net.0.proj.weight", 2 * inner, D, w.mlp1, D, 0, inner);
      EZB_TRY(alloc(&w.b_mlp1, (size_t)2 * inner));
      {
        float* dst = w.b_mlp1;
        const int in_ = inner, gh = geglu_bn / 2;
        reg(p + ".mlp.net.0.proj.bias", {2 * inner}, [dst, in_, gh](const float* src, cudaStream_t st) -> int {
          ++launch_counter();
          pack_geglu_bias_kernel<<<(2 * in_ + 255) / 256, 256, 0, st>>>(src, dst, in_, gh);
          EZB_CUDA(cudaGetLastError());
          return EZB_OK;
        });
      }
      if (fp8) {
        EZB_TRY(alloc(&w.qkv8, (size_t)H * qkv3_bn * D)); EZB_TRY(alloc(&w.s_qkv, (size_t)H * qkv3_bn));
        EZB_TRY(alloc(&w.mlp18, (size_t)2 * inner * D)); EZB_TRY(alloc(&w.s_mlp1, (size_t)2 * inner));
      }
      EZB_TRY(alloc_w(&w.mlp2, D, inner));
      reg_linear(p + ".mlp.net.2.weight", D, inner, w.mlp2, inner, 0);
      EZB_TRY(reg_f32(p + ".mlp.net.2.bias", {D}, &w.b_mlp2));
      EZB_TRY(reg_f32(p + ".adaln.scale_shift_table", {6, D}, &w.table));
      EZB_TRY(reg_f32(p + ".adaln.lora_a.weight", {6 * r, D}, &w.lora_a));
      EZB_TRY(reg_f32(p + ".adaln.lora_b.weight", {6 * D, 6 * r}, &w.lora_b));
      if (is_out) {
        EZB_TRY(reg_f32(p + ".skip_norm.weight", {2 * D}, &w.snw)); EZB_TRY(reg_f32(p + ".skip_norm.bias", {2 * D}, &w.snb));
        EZB_TRY(alloc_w(&w.skip, D, 2 * D));
        reg_linear(p + ".skip_linear.weight", D, 2 * D, w.skip, 2 * D, 0);
        EZB_TRY(reg_f32(p + ".skip_linear.bias", {D}, &w.b_skip));
      }
      if (d.is_controlnet) {
        EZB_TRY(alloc_w(&w.zero_w, D, D));
        reg_linear("controlnet_zero_blocks." + std::to_string(i) + ".weight", D, D, w.zero_w, D, 0);
        EZB_TRY(reg_f32("controlnet_zero_blocks." + std::to_string(i) + ".bias", {D}, &w.zero_b));
      }
    }
    if (!d.is_controlnet) {
      EZB_TRY(reg_f32("model.final_block.norm.weight", {D}, &fn_w)); EZB_TRY(reg_f32("model.final_block.norm.bias", {D}, &fn_b));
      EZB_TRY(alloc_w(&w_final, C, D));
      reg_linear("model.final_block.linear.weight", C, D, w_final, D, 0);
      EZB_TRY(reg_f32("model.final_block.linear.bias", {C}, &b_final));
      EZB_TRY(alloc(&fc_w, (size_t)3 * C * C));
      {
        float* dst = fc_w;
        const int c = C;
        reg("model.final_block.final_layer.weight", {C, C, 3}, [dst, c](const float* src, cudaStream_t st) -> int {
          // [co][ci][k] -> [k][ci][co]
          ++launch_counter();
          permute3_kernel<<<(3 * c * c + 255) / 256, 256, 0, st>>>(src, dst, 3, c, c, 1, 3, 3 * c);
          EZB_CUDA(cudaGetLastError());
          return EZB_OK;
        });
      }
      EZB_TRY(reg_f32("model.final_block.final_layer.bias", {C}, &fc_b));
    } else {
      const int c0 = d.cond_c0, c1 = d.cond_c1;
      EZB_TRY(reg_f32("controlnet_pre.conv_in.weight", {c0, 1, 1}, &cs_in_w)); EZB_TRY(reg_f32("controlnet_pre.conv_in.bias", {c0}, &cs_in_b));
      EZB_TRY(reg_f32("controlnet_pre.mask_embed", {c0}, &cs_me));
      EZB_TRY(reg_f32("controlnet_pre.blocks.0.0.weight", {c0 + 1, c0 + 1, 3}, &cs_c0_w)); EZB_TRY(reg_f32("controlnet_pre.blocks.0.0.bias", {c0 + 1}, &cs_c0_b));
      EZB_TRY(reg_f32("controlnet_pre.blocks.0.2.weight", {c1, c0 + 1, 3}, &cs_c1_w)); EZB_TRY(reg_f32("controlnet_pre.blocks.0.2.bias", {c1}, &cs_c1_b));
      EZB_TRY(reg_f32("controlnet_pre.conv_out.weight", {D, c1, 1}, &cs_out_w)); EZB_TRY(reg_f32("controlnet_pre.conv_out.bias", {D}, &cs_out_b));
    }
    // ---- workspace
    const size_t Mx = (size_t)d.max_batch * d.max_len, Mc = (size_t)d.max_batch * d.max_ctx_len;
    const size_t Mmax = Mx > Mc ? Mx : Mc;
    EZB_TRY(alloc(&x0, Mx * D)); EZB_TRY(alloc(&xa, Mx * D)); EZB_TRY(alloc(&xb, Mx * D));
    skips.resize(half);
    for (int i = 0; i < half; ++i) EZB_TRY(alloc(&skips[i], Mx * D));
    const size_t act_cols = (size_t)kmul * (2 * D > d.context_dim ? 2 * D : d.context_dim);
    EZB_TRY(alloc(&act, Mmax * act_cols));
    EZB_TRY(alloc(&a_patch, Mx * kmul * Kp));
    EZB_TRY(alloc(&attn_out, Mmax * kmul * D));
    EZB_TRY(alloc(&mid, Mx * kmul * inner));
    {
      float* q4 = nullptr;
      EZB_TRY(alloc(&q4, Mmax * 3 * D));
      qkv = q4;
    }
    if (!use_tc_attention) {
      EZB_TRY(alloc(&q32, Mx * D)); EZB_TRY(alloc(&k32, Mx * D)); EZB_TRY(alloc(&v32, Mx * D));
    } else {
      const size_t Lp = ((size_t)d.max_len + 7) / 8 * 8;
      EZB_TRY(alloc(&q16, Mx * H * DHP)); EZB_TRY(alloc(&k16, Mx * H * DHP));
      EZB_TRY(alloc(&vt16, (size_t)d.max_batch * H * DVP * Lp));
    }
    EZB_TRY(alloc(&rope_cs, (size_t)d.max_len * (dh / 2)));
    fused_heads = use_tc_attention && (dh == 64 || dh == 72) && (H % 2 == 0);
    EZB_TRY(alloc(&ctx_emb, Mc * D));
    EZB_TRY(alloc(&ctx_mask, Mc));
    const size_t Lcp = ((size_t)d.max_ctx_len + 7) / 8 * 8;
    for (int i = 0; i < nblk; ++i) {
      if (!use_tc_attention) {
        EZB_TRY(alloc(&blk[i].kc32, Mc * D)); EZB_TRY(alloc(&blk[i].vc32, Mc * D));
      } else {
        EZB_TRY(alloc(&blk[i].kc16, Mc * H * DHP));
        EZB_TRY(alloc(&blk[i].vtc16, (size_t)d.max_batch * H * DVP * Lcp));
      }
    }
    EZB_TRY(alloc(&grid_bar, (size_t)1));
    if (fp8) { EZB_TRY(alloc(&act8, Mx * D)); EZB_TRY(alloc(&act8_s, Mx)); }
    if (d.precision != 1 && (D == 1152 || D == 1024)) {   // precombined LayerNorm affine tables (ln_gc_kernel)
      gc_T = d.max_timesteps < 128 ? d.max_timesteps : 128;
      for (int i = 0; i < nblk; ++i) {
        EZB_TRY(alloc(&blk[i].lnG1, (size_t)gc_T * D)); EZB_TRY(alloc(&blk[i].lnC1, (size_t)gc_T * D));
        EZB_TRY(alloc(&blk[i].lnG3, (size_t)gc_T * D)); EZB_TRY(alloc(&blk[i].lnC3, (size_t)gc_T * D));
      }
      if (!d.is_controlnet) { EZB_TRY(alloc(&lnGF, (size_t)gc_T * D)); EZB_TRY(alloc(&lnCF, (size_t)gc_T * D)); }
    }
    // ---- folded LayerNorm: tables + operand / statistics buffers
    fold_cfg = opt_fold() != 0 && d.precision == 0 && pair && swap_ab && fused_heads && D <= 2304 / 2;
    if (fold_cfg) {
      fold_T = d.max_timesteps < 128 ? d.max_timesteps : 128;
      st_slots = (D + 31) / 32;
      st_ld = Mx;
      n_qkv = qkv3_bn > 0 ? H * qkv3_bn : 3 * D;
      const size_t FT = fold_T;
      EZB_TRY(alloc(&gc_G, FT * 2 * D)); EZB_TRY(alloc(&gc_C, FT * 2 * D));
      EZB_TRY(alloc(&st_x0, (size_t)st_slots * st_ld));
      cat.resize(half);
      for (int i = 0; i < half; ++i) EZB_TRY(alloc(&cat[i], Mx * (d.is_controlnet ? D : 2 * D)));
      for (int i = 0; i < nblk; ++i) {
        BlockW& w = blk[i];
        EZB_TRY(alloc(&w.g1, FT * D)); EZB_TRY(alloc(&w.u1, FT * n_qkv)); EZB_TRY(alloc(&w.v1, FT * n_qkv));
        EZB_TRY(alloc(&w.g3, FT * D)); EZB_TRY(alloc(&w.u3, FT * 2 * inner)); EZB_TRY(alloc(&w.v3, FT * 2 * inner));
        EZB_TRY(alloc(&w.u2, (size_t)D)); EZB_TRY(alloc(&w.v2, (size_t)D));
        if (!d.is_controlnet && i > half) { EZB_TRY(alloc(&w.us, (size_t)D)); EZB_TRY(alloc(&w.vs, (size_t)D)); }
        EZB_TRY(alloc(&w.st_skip, (size_t)st_slots * st_ld)); EZB_TRY(alloc(&w.st_a, (size_t)st_slots * st_ld));
        EZB_TRY(alloc(&w.st_b, (size_t)st_slots * st_ld)); EZB_TRY(alloc(&w.st_out, (size_t)st_slots * st_ld));
      }
      if (!d.is_controlnet) { EZB_TRY(alloc(&gF, FT * D)); EZB_TRY(alloc(&uF, FT * C)); EZB_TRY(alloc(&vF, FT * C)); }
    }
    const size_t T = d.max_timesteps;
    EZB_TRY(alloc(&t_vals, T)); EZB_TRY(alloc(&t_emb, T * 256)); EZB_TRY(alloc(&t_h, T * D)); EZB_TRY(alloc(&t_tok, T * D));
    EZB_TRY(alloc(&t_ada, T * 6 * D)); EZB_TRY(alloc(&t_lora, T * 6 * r));
    EZB_TRY(alloc(&mod, T * nblk * 6 * D));
    EZB_TRY(alloc(&mod_b, (size_t)d.max_batch * nblk * 6 * D));
    if (!d.is_controlnet) {
      EZB_TRY(alloc(&mod_final, T * 2 * D));
      EZB_TRY(alloc(&modf_b, (size_t)d.max_batch * 2 * D));
      EZB_TRY(alloc(&ybuf, Mx * C));
    } else {
      EZB_TRY(alloc(&cond_emb, Mx * D));
      EZB_TRY(alloc(&cond_cache, Mx * D));
      EZB_TRY(alloc(&cs_t0, (size_t)d.max_batch * (d.cond_c0 + 1) * 2 * d.max_len));
      EZB_TRY(alloc(&cs_t1, (size_t)d.max_batch * (d.cond_c0 + 1) * 2 * d.max_len));
      EZB_TRY(alloc(&cs_t2, (size_t)d.max_batch * d.cond_c1 * d.max_len));
    }
    return EZB_OK;
  }

  int load_weight(const char* key, const float* data, const int64_t* shape, int ndim, cudaStream_t st) {
    auto it = specs.find(key);
    if (it == specs.end()) return fail(EZB_ERR_WEIGHT, "unexpected state-dict key '%s'", key);
    WeightSpec& s = it->second;
    bool ok = (int)s.shape.size() == ndim;
    for (int i = 0; ok && i < ndim; ++i) ok = s.shape[i] == shape[i];
    if (!ok) return fail(EZB_ERR_WEIGHT, "shape mismatch for '%s'", key);
    EZB_TRY(s.load(data, st));
    s.loaded = true;
    return EZB_OK;
  }
  int finalize() {
    for (auto& kv : specs)
      if (!kv.second.loaded) return fail(EZB_ERR_WEIGHT, "missing state-dict key '%s'", kv.first.c_str());
    EZB_CUDA(cudaDeviceSynchronize());
    EZB_CUDA(cudaMemcpy(h_inv_freq, blk[0].inv_freq, (dh / 2) * sizeof(float), cudaMemcpyDeviceToHost));
    for (auto& w : blk) {  // the fused heads epilogue takes these by value (constant bank)
      EZB_CUDA(cudaMemcpy(w.h_nq[0], w.nqw, dh * sizeof(float), cudaMemcpyDeviceToHost)); EZB_CUDA(cudaMemcpy(w.h_nq[1], w.nqb, dh * sizeof(float), cudaMemcpyDeviceToHost));
      EZB_CUDA(cudaMemcpy(w.h_nk[0], w.nkw, dh * sizeof(float), cudaMemcpyDeviceToHost)); EZB_CUDA(cudaMemcpy(w.h_nk[1], w.nkb, dh * sizeof(float), cudaMemcpyDeviceToHost));
      EZB_CUDA(cudaMemcpy(w.h_cnq[0], w.cnqw, dh * sizeof(float), cudaMemcpyDeviceToHost)); EZB_CUDA(cudaMemcpy(w.h_cnq[1], w.cnqb, dh * sizeof(float), cudaMemcpyDeviceToHost));
      EZB_CUDA(cudaMemcpy(w.h_cnk[0], w.cnkw, dh * sizeof(float), cudaMemcpyDeviceToHost)); EZB_CUDA(cudaMemcpy(w.h_cnk[1], w.cnkb, dh * sizeof(float), cudaMemcpyDeviceToHost));
    }
    {
      const int n = d.max_len * (dh / 2);
      ++launch_counter();
      rope_table_kernel<<<(n + 255) / 256, 256>>>(blk[0].inv_freq, rope_cs, d.max_len, dh / 2);
      EZB_CUDA(cudaGetLastError());
      EZB_CUDA(cudaDeviceSynchronize());
    }
    if (fp8) {  // after the packing permutations: a row scale follows its row
      for (auto& w : blk) {
        EZB_TRY(quant_rows(w.qkv, H * qkv3_bn, D, w.qkv8, w.s_qkv));
        EZB_TRY(quant_rows(w.mlp1, 2 * inner, D, w.mlp18, w.s_mlp1));
      }
      EZB_CUDA(cudaDeviceSynchronize());
    }
    if (fold_cfg) {  // static sites: norm2 -> cross-Q and skip_norm -> skip_linear (no modulation: G = weight, C = bias)
      for (int i = 0; i < nblk; ++i) {
        BlockW& w = blk[i];
        EZB_TRY(fold_uv(0, w.cq, D, w.n2w, w.n2b, nullptr, w.u2, w.v2, D, D, 1));
        if (w.us) EZB_TRY(fold_uv(0, w.skip, 2 * D, w.snw, w.snb, nullptr, w.us, w.vs, D, 2 * D, 1));
      }
      EZB_CUDA(cudaDeviceSynchronize());
    }
    finalized = true;
    return EZB_OK;
  }
  int quant_rows(const bf16* W, int N, int K, uint8_t* Q, float* S) {
    ++launch_counter();
    quant_rows_e4m3_kernel<<<(N + 7) / 8, 256>>>(W, N, K, Q, S);
    EZB_CUDA(cudaGetLastError());
    return EZB_OK;
  }
  int fold_uv(cudaStream_t st, const bf16* W, int ldw, const float* G, const float* Cc, const float* add_v, float* U, float* V, int N, int K, int R) {
    return fold_uv_launch(st, W, ldw, G, Cc, add_v, U, V, N, K, R);
  }
  // per-timestep tables of the modulated sites (called at the end of set_timesteps)
  int build_gc_tables(int n, cudaStream_t st) {
    gc_n = 0;
    if (gc_T == 0 || n > gc_T) return EZB_OK;
    const int ldm = nblk * 6 * D;
    auto gc = [&](const float* w_, const float* b_, const float* shift, const float* scale, int ld, float* G, float* Cc) -> int {
      return fold_gc_launch(st, w_, b_, shift, scale, ld, G, Cc, n, D);
    };
    for (int i = 0; i < nblk; ++i) {
      BlockW& w = blk[i];
      const float* m = mod + (size_t)i * 6 * D;
      EZB_TRY(gc(w.n1w, w.n1b, m + 0 * D, m + 1 * D, ldm, w.lnG1, w.lnC1));
      EZB_TRY(gc(w.n3w, w.n3b, m + 3 * D, m + 4 * D, ldm, w.lnG3, w.lnC3));
    }
    if (!d.is_controlnet) EZB_TRY(gc(fn_w, fn_b, mod_final, mod_final + D, 2 * D, lnGF, lnCF));
    gc_n = n;
    return EZB_OK;
  }
  int build_fold_tables(int n, cudaStream_t st) {
    EZB_TRY(build_gc_tables(n, st));
    fold_n = 0;
    if (!fold_cfg || n > fold_T) return EZB_OK;
    const int ldm = nblk * 6 * D;
    auto gc = [&](const float* w_, const float* b_, const float* shift, const float* scale, int ld, float* G) -> int {
      return fold_gc_launch(st, w_, b_, shift, scale, ld, G, gc_C, n, D);
    };
    for (int i = 0; i < nblk; ++i) {
      BlockW& w = blk[i];
      const float* m = mod + (size_t)i * 6 * D;   // [t] stride ldm: shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp
      EZB_TRY(gc(w.n1w, w.n1b, m + 0 * D, m + 1 * D, ldm, w.g1));
      EZB_TRY(fold_uv(st, w.qkv, D, w.g1, gc_C, nullptr, w.u1, w.v1, n_qkv, D, n));
      EZB_TRY(gc(w.n3w, w.n3b, m + 3 * D, m + 4 * D, ldm, w.g3));
      EZB_TRY(fold_uv(st, w.mlp1, D, w.g3, gc_C, w.b_mlp1, w.u3, w.v3, 2 * inner, D, n));   // v3 carries the (packed) GEGLU bias
    }
    if (!d.is_controlnet) {  // FinalBlock: shift, scale = time_ada_final.chunk(2) (blocks.py:204)
      EZB_TRY(gc(fn_w, fn_b, mod_final, mod_final + D, 2 * D, gF));
      EZB_TRY(fold_uv(st, w_final, D, gF, gc_C, nullptr, uF, vF, C, D, n));
    }
    fold_n = n;
    return EZB_OK;
  }

  // ---------------------------------------------------------------- launch helpers
  LnParams ln_params(const float* x, int D1, const float* x2, const float* x3, int D2, const float* w, const float* b, const float* shift, const float* scale,
                     int mod_bstride, int rows_per_batch, bf16* out, int M) {
    LnParams p;
    p.x = x; p.x2 = x2; p.x3 = x3; p.D1 = D1; p.D2 = D2; p.w = w; p.b = b; p.shift = shift; p.scale = scale; p.mod_bstride = mod_bstride;
    p.rows_per_batch = rows_per_batch; p.out = out; p.kmul = kmul; p.M = M;
    p.G = nullptr; p.C = nullptr;
    // precombined affine (ln_gc_kernel): static norms directly, modulated ones from the per-timestep tables when the batch shares one timestep
    if (x2 == nullptr && w != nullptr && gc_T > 0) {
      if (shift == nullptr) { p.G = w; p.C = b; }
      else if (mod_bstride == 0 && gc_n > 0) {
        const size_t ldm = (size_t)nblk * 6 * D;
        if (shift >= mod && shift < mod + (size_t)n_timesteps * ldm) {
          const size_t off = (size_t)(shift - mod), t = off / ldm, r = off % ldm, bi = r / (6 * D), site = (r % (6 * D)) / D;   // site 0: norm1, 3: norm3
          if ((int)t < gc_n && (site == 0 || site == 3)) {
            p.G = (site == 0 ? blk[bi].lnG1 : blk[bi].lnG3) + t * D;
            p.C = (site == 0 ? blk[bi].lnC1 : blk[bi].lnC3) + t * D;
          }
        } else if (mod_final && shift >= mod_final && shift < mod_final + (size_t)n_timesteps * 2 * D) {
          const size_t t = (size_t)(shift - mod_final) / (2 * D);
          if ((int)t < gc_n) { p.G = lnGF + t * D; p.C = lnCF + t * D; }
        }
      }
    }
    return p;
  }
  int ln(cudaStream_t st, const LnParams& p) {
    if (opt_skip() & 1) return EZB_OK;
    return ln_launch(*dev, st, p);   // p.kmul == kmul (ln_params)
  }
  // FP8 mode: LayerNorm (+ modulate) of p.x to e4m3 act8 with row scales act8_s (p.out is not written)
  int ln8(cudaStream_t st, const LnParams& p) {
    if (opt_skip() & 1) return EZB_OK;
    if (p.x2 != nullptr || p.w == nullptr || p.D1 > 1152) return fail(EZB_ERR_UNSUPPORTED, "fp8 LayerNorm: single source of at most 1152 features");
    const int M = p.M, grid = dev->num_sms * 4 < (M + 3) / 4 ? dev->num_sms * 4 : (M + 3) / 4;
    const LnFp8Out o{act8, act8_s};
    if (p.D1 == 1152) return launch_k(ln_fp8_kernel<9, true>, dim3(grid), dim3(128), 0, st, 1, p, o);
    if (p.D1 == 1024) return launch_k(ln_fp8_kernel<8, true>, dim3(grid), dim3(128), 0, st, 1, p, o);
    return launch_k(ln_fp8_kernel<9, false>, dim3(grid), dim3(128), 0, st, 1, p, o);
  }
  int ln(cudaStream_t st, const float* x, int D1, const float* x2, const float* x3, int D2, const float* w, const float* b, const float* shift,
         const float* scale, int mod_bstride, int rows_per_batch, bf16* out, int M) {
    return ln(st, ln_params(x, D1, x2, x3, D2, w, b, shift, scale, mod_bstride, rows_per_batch, out, M));
  }
  EpiLinearParams epi() {
    EpiLinearParams e;
    memset(&e, 0, sizeof e);
    return e;
  }
  // `tail`: the LayerNorm that reads this GEMM's fp32 output; when the GEMM is a one-wave swap-AB launch it runs as the tail phase of the same
  // kernel (gemm_ln.cuh) and *tail_done is set, otherwise the caller launches it separately.
  // `m_select` (0: M): the token count the kernel is chosen for (context_rows: the whole batch, so that a part of it comes out bit-identical).
  int lin(cudaStream_t st, const bf16* A, int K, const bf16* W, int M, int N, const EpiLinearParams& e, const LnParams* tail = nullptr, bool* tail_done = nullptr,
          int m_select = 0) {
    if ((opt_skip() & 8) && e.out_f32 != nullptr && e.out_bf16 == nullptr) return EZB_OK;
    // fp32-output layers (residual / gated-residual / plain): swap-AB tiles of 128 features x 256 or 288 tokens (host.cuh swapped_bn)
    const bool folded = e.fin.u != nullptr || e.fout.st != nullptr;   // fold epilogues exist in the swap-AB kernel only
    if (lin_takes_swap_ab(e, M, m_select, pair, swap_ab, kmul)) {
      if (folded) return gemm_swapped<EpiLinearTF>(*dev, st, A, K, W, K, M, N, K, e);
      if (tail != nullptr && tail_done != nullptr && opt_ln_tail() && !(opt_skip() & 9))
        return gemm_swapped_ln<EpiLinearT>(*dev, st, A, K, W, K, M, N, K, e, *tail, grid_bar, tail_done);
      return opt_swap_mc() ? gemm_swapped_mc<EpiLinearT, 3>(*dev, st, A, K, W, K, M, N, K, e)
                           : gemm_swapped<EpiLinearT>(*dev, st, A, K, W, K, M, N, K, e);
    }
    if (folded) return fail(EZB_ERR_STATE, "folded LayerNorm epilogue requested on a GEMM that is not a swap-AB launch");
    if (pair) return gemm2<128, EpiLinear<128>>(*dev, st, A, kmul * K, W, kmul * K, M, N, kmul * K, e);
    return gemm<128, EpiLinear<128>>(*dev, st, A, kmul * K, W, kmul * K, M, N, kmul * K, e);
  }
  FoldIn fold_in(const float2* st0, const float2* st1, int width, const float* u, const float* v) {
    FoldIn f;
    memset(&f, 0, sizeof f);
    f.st0 = st0; f.st1 = st1; f.slots0 = st_slots; f.slots1 = st1 ? st_slots : 0; f.ld_st = (int)st_ld; f.inv_dim = 1.0f / (float)width; f.u = u; f.v = v;
    return f;
  }
  FoldOut fold_out(float2* stp, bf16* a0, int ld0, const float* g0, bf16* a1 = nullptr, int ld1 = 0, const float* g1 = nullptr) {
    FoldOut f;
    memset(&f, 0, sizeof f);
    f.st = stp; f.ld_st = (int)st_ld; f.a0 = a0; f.ld0 = ld0; f.g0 = g0; f.a1 = a1; f.ld1 = ld1; f.g1 = g1;
    return f;
  }
  int small_lin(cudaStream_t st, const float* in, int ld_in, const float* W, const float* bias, const float* add, int ld_add, float* out, int ld_out, int R,
                int N, int K, int act, float scale) {
    return small_linear_launch(st, in, ld_in, W, bias, add, ld_add, out, ld_out, R, N, K, act, scale);
  }
  // head layout for attention from a GEMM output holding `nsec` sections
  int qk_prep(cudaStream_t st, int ld_in, int nsec, const int* col_off, const int* kinds, const float* nqw_, const float* nqb_, const float* nkw_,
              const float* nkb_, const float* inv_freq, int B, int L, float* const* f32o, bf16* const* bfo, int Lpad) {
    auto fill = [&](auto& p) {
      p.ld_in = ld_in; p.n_sections = nsec;
      for (int i = 0; i < 3; ++i) { p.col_off[i] = i < nsec ? col_off[i] : 0; p.sec_kind[i] = i < nsec ? kinds[i] : 0; p.f32_out[i] = i < nsec ? f32o[i] : nullptr; p.bf_out[i] = i < nsec ? bfo[i] : nullptr; }
      p.nw[0] = nqw_; p.nb[0] = nqb_; p.nw[1] = nkw_; p.nb[1] = nkb_; p.use_rope = inv_freq != nullptr; p.inv_freq = inv_freq;
      p.B = B; p.L = L; p.H = H; p.dh = dh; p.ld_qk = DHP; p.Lpad = Lpad; p.dv_pad = DVP;
    };
    if (kmul == 3) {
      QkPrepParams<float> p; p.in = reinterpret_cast<const float*>(qkv); fill(p);
      return qk_prep_launch(st, p);
    }
    QkPrepParams<bf16> p; p.in = reinterpret_cast<const bf16*>(qkv); fill(p);
    return qk_prep_launch(st, p);
  }
  // Q/K/V projection with the fused per-head LN + RoPE + attention-layout epilogue (fast mode)
  EpiHeadsParams heads_params(int N, const int* kinds, const float (*nq)[96], const float (*nk)[96], bool rope, int L, bf16* qo, bf16* ko, bf16* vto,
                              int Lpad, const FoldIn* fin) {
    EpiHeadsParams e;
    memset(&e, 0, sizeof e);
    if (fin) e.fin = *fin;
    for (int i = 0; i < dh && i < 72; ++i) {
      if (nq) { e.nw[0][i] = nq[0][i]; e.nb[0][i] = nq[1][i]; }
      if (nk) { e.nw[1][i] = nk[0][i]; e.nb[1][i] = nk[1][i]; }
    }
    e.D = D; e.H = H; e.L = L;
    for (int i = 0; i < 3; ++i) e.kind[i] = i < N / D ? kinds[i] : 0;
    e.rope = rope ? rope_cs : nullptr; e.rope_kinds = 3; e.rope_ld = d.max_len;
    e.rope_mufu = opt_rope_mufu();
    for (int i = 0; i < dh / 2 && i < 36; ++i) e.inv_freq[i] = h_inv_freq[i];
    e.out[0] = qo; e.out[1] = ko; e.out[2] = vto;
    e.ld_qk = DHP; e.dvp = DVP; e.Lpad = Lpad;
    return e;
  }
  int lin_heads(cudaStream_t st, const bf16* A, const bf16* W, int M, int N, const int* kinds, const float (*nq)[96], const float (*nk)[96], bool rope,
                int L, bf16* qo, bf16* ko, bf16* vto, int Lpad, const FoldIn* fin = nullptr) {
    if (opt_skip() & 4) return EZB_OK;
    EpiHeadsParams e = heads_params(N, kinds, nq, nk, rope, L, qo, ko, vto, Lpad, fin);
    const bool fo = fin != nullptr;
    int variant;
    if (qkv3_bn > 0 && N == 3 * D) {  // packed self-attention QKV: three heads per tile
      if (dh == 72 && opt_heads_dbg() && !fo) e.dbg = opt_heads_dbg();   // profiling instantiation
      variant = HEADS_PACKED3;
    } else if (!pair || (opt_cq_single() && !fo && N == D && dh == 72)) {   // cross-Q as 256 single-CTA tiles of 128 x 144 (1.73 waves of half-size tiles)
      variant = HEADS_SINGLE;
    } else {
      variant = HEADS_PAIR;
    }
    return heads_gemm(*dev, st, A, W, M, N, dh, variant, e);
  }
  // GEMM whose output feeds qk_prep: bf16 [M,N] in fast mode, fp32 in parity mode
  int lin_to_qkv(cudaStream_t st, const bf16* A, int K, const bf16* W, int M, int N) {
    EpiLinearParams e = epi();
    if (kmul == 3) { e.out_f32 = reinterpret_cast<float*>(qkv); e.ld32 = N; }
    else { e.out_bf16 = reinterpret_cast<bf16*>(qkv); e.ld16 = N; }
    return lin(st, A, K, W, M, N, e);
  }
  // lens_: valid tokens per sample (self-attention of a padded batch) or null
  int attention(cudaStream_t st, const float* q32_, const float* k32_, const float* v32_, const bf16* q16_, const bf16* k16_, const bf16* vt16_,
                const uint8_t* mask, int B, int Lq, int Lk, int Lkpad, const int32_t* lens_ = nullptr) {
    const float scale = 1.0f / sqrtf((float)dh);
    if (opt_skip() & 2) return EZB_OK;
    if (!use_tc_attention) {
      if (dh % 4) return fail(EZB_ERR_UNSUPPORTED, "fp32 attention: head dimension %d is not a multiple of 4", dh);
      const size_t smem = attn_simt_smem(dh);
      static bool set[16] = {};  // function attributes are per device
      if (!set[dev->id & 15]) {
        EZB_CUDA(cudaFuncSetAttribute(attn_simt_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        EZB_CUDA(cudaFuncSetAttribute(attn_simt_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        set[dev->id & 15] = true;
      }
      dim3 grid((Lq + SA_WARPS * SA_QW - 1) / (SA_WARPS * SA_QW), B * H);
      ++launch_counter();
      auto kern = lens_ ? attn_simt_kernel<true> : attn_simt_kernel<false>;
      kern<<<grid, SA_WARPS * 32, smem, st>>>(q32_, k32_, v32_, mask, attn_out, H, Lq, Lk, dh, scale, kmul, lens_, nullptr);
      EZB_CUDA(cudaGetLastError());
      return EZB_OK;
    }
    return attention_mma(*dev, st, q16_, k16_, vt16_, mask, attn_out, B, H, Lq, Lk, Lkpad, dh, DHP, DVP, scale, 0, lens_);
  }

  // ---------------------------------------------------------------- step-invariant precompute
  int set_context(const float* ctx, const uint8_t* mask, int Be, int Lc, cudaStream_t st) {
    if (!finalized) return fail(EZB_ERR_STATE, "weights not finalized");
    if (Be < 1 || Be > d.max_batch || Lc < 1 || Lc > d.max_ctx_len) return fail(EZB_ERR_SHAPE, "set_context: Be %d Lc %d exceed workspace", Be, Lc);
    dev->tmaps.trim();
    ctx_Be = Be; ctx_Lc = Lc; ctx_Lpad = (Lc + 7) / 8 * 8;
    return context_rows(ctx, mask, 0, Be, st);
  }
  // rows [row0, row0 + n) of the layout the last set_context established (ezb_dit_set_context_rows)
  int set_context_rows(const float* ctx, const uint8_t* mask, int row0, int n, int Lc, cudaStream_t st) {
    if (!finalized) return fail(EZB_ERR_STATE, "weights not finalized");
    if (ctx_Be < 1) return fail(EZB_ERR_STATE, "set_context_rows: no ezb_dit_set_context call established the context layout");
    if (Lc != ctx_Lc) return fail(EZB_ERR_STATE, "set_context_rows: Lc %d differs from the context layout (Lc %d)", Lc, ctx_Lc);
    if (row0 < 0 || n < 1 || row0 + n > ctx_Be) return fail(EZB_ERR_SHAPE, "set_context_rows: rows [%d, %d) outside the batch of %d", row0, row0 + n, ctx_Be);
    dev->tmaps.trim();
    return context_rows(ctx, mask, row0, n, st);
  }
  // The context path of clips [row0, row0 + n) (ctx, mask: their rows only).  Every kernel works per token or per clip, and the one launch whose
  // kernel depends on the token count (context_embed's fp32-output linear, Dit::lin) is chosen for the whole batch, so a row comes out as a call
  // on the whole batch computes it.
  int context_rows(const float* ctx, const uint8_t* mask, int row0, int n, cudaStream_t st) {
    const int Lc = ctx_Lc, Mc = n * Lc, cd = d.context_dim;
    const size_t r0 = (size_t)row0 * Lc, kq = (size_t)row0 * H * Lc * DHP, kv = (size_t)row0 * H * DVP * ctx_Lpad, k32 = (size_t)row0 * H * Lc * dh;
    EZB_CUDA(cudaMemcpyAsync(ctx_mask + r0, mask, (size_t)Mc, cudaMemcpyDeviceToDevice, st));
    EZB_TRY(ln(st, ctx, cd, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr, 0, 1, act, Mc));  // cast only
    EpiLinearParams e = epi();
    e.bias = b_ce0; e.out_bf16 = attn_out; e.ld16 = kmul * D; e.split_stride = kmul == 3 ? D : 0; e.act = ACT_SILU;
    EZB_TRY(lin(st, act, cd, w_ce0, Mc, D, e));
    e = epi();
    e.bias = b_ce2; e.out_f32 = ctx_emb + r0 * D; e.ld32 = D;
    EZB_TRY(lin(st, attn_out, D, w_ce2, Mc, D, e, nullptr, nullptr, ctx_Be * Lc));
    for (int i = 0; i < nblk; ++i) {
      BlockW& w = blk[i];
      bf16* kc16 = w.kc16 ? w.kc16 + kq : nullptr;
      bf16* vtc16 = w.vtc16 ? w.vtc16 + kv : nullptr;
      EZB_TRY(ln(st, ctx_emb + r0 * D, D, nullptr, nullptr, 0, w.ncw, w.ncb, nullptr, nullptr, 0, 1, act, Mc));
      const int off[2] = {0, D}, kinds[2] = {1, 2};
      if (fused_heads) {
        EZB_TRY(lin_heads(st, act, w.ckv, Mc, 2 * D, kinds, nullptr, w.h_cnk, false, Lc, nullptr, kc16, vtc16, ctx_Lpad));
        continue;
      }
      EZB_TRY(lin_to_qkv(st, act, D, w.ckv, Mc, 2 * D));
      float* f32o[2] = {w.kc32 ? w.kc32 + k32 : nullptr, w.vc32 ? w.vc32 + k32 : nullptr};
      bf16* bfo[2] = {kc16, vtc16};
      if (use_tc_attention) EZB_CUDA(cudaMemsetAsync(vtc16, 0, (size_t)n * H * DVP * ctx_Lpad * sizeof(bf16), st));
      EZB_TRY(qk_prep(st, 2 * D, 2, off, kinds, nullptr, nullptr, w.cnkw, w.cnkb, nullptr, n, Lc, f32o, bfo, ctx_Lpad));
    }
    return EZB_OK;
  }

  int set_timesteps(const int64_t* ts, int n, cudaStream_t st) {
    if (!finalized) return fail(EZB_ERR_STATE, "weights not finalized");
    if (n < 1 || n > d.max_timesteps) return fail(EZB_ERR_SHAPE, "set_timesteps: n %d exceeds max_timesteps %d", n, d.max_timesteps);
    for (int i0 = 0; i0 < n; i0 += 240) {  // values travel by value in the kernel parameters: no host staging buffer, no synchronisation
      TimestepChunk c;
      const int m = n - i0 < 240 ? n - i0 : 240;
      for (int i = 0; i < 240; ++i) c.v[i] = i < m ? (float)ts[i0 + i] : 0.f;
      ++launch_counter();
      fill_timesteps_kernel<<<1, 256, 0, st>>>(t_vals + i0, c, m);
    }
    EZB_TRY(timestep_embed_launch(st, t_vals, t_emb, n));
    EZB_TRY(small_lin(st, t_emb, 256, te_w0, te_b0, nullptr, 0, t_h, D, n, D, 256, 1, 1.f));
    EZB_TRY(small_lin(st, t_h, D, te_w2, te_b2, nullptr, 0, t_tok, D, n, D, D, 1, 1.f));  // time_act SiLU folded (udit.py:313)
    EZB_TRY(small_lin(st, t_tok, D, ta_w, ta_b, nullptr, 0, t_ada, 6 * D, n, 6 * D, D, 0, 1.f));
    if (!d.is_controlnet) EZB_TRY(small_lin(st, t_tok, D, taf_w, taf_b, nullptr, 0, mod_final, 2 * D, n, 2 * D, D, 0, 1.f));
    const int ldm = nblk * 6 * D;
    for (int i = 0; i < nblk; ++i) {
      BlockW& w = blk[i];
      EZB_TRY(small_lin(st, t_tok, D, w.lora_a, nullptr, nullptr, 0, t_lora, 6 * r, n, 6 * r, D, 0, 1.f));
      EZB_TRY(small_lin(st, t_lora, 6 * r, w.lora_b, nullptr, t_ada, 6 * D, mod + (size_t)i * 6 * D, ldm, n, 6 * D, 6 * r, 0, d.ada_scaling));
      ++launch_counter();
      add_rowvec_kernel<<<(unsigned)(((size_t)n * 6 * D + 255) / 256), 256, 0, st>>>(mod + (size_t)i * 6 * D, ldm, w.table, n, 6 * D);
    }
    EZB_CUDA(cudaGetLastError());
    n_timesteps = n;
    return build_fold_tables(n, st);
  }

  // modulation rows for this call: uniform timestep -> point into the table (batch stride 0); else gather per sample.  Device indices (tdev)
  // are always gathered, by a kernel, into the same per-sample rows the host-index gather fills.
  int select_mod(cudaStream_t st, const int32_t* tidx, int tall, const int32_t* tdev, int Be, const float** mod_rows, const float** modf_rows, int* bstride,
                 int* bstride_f) {
    const int ldm = nblk * 6 * D;
    if (tdev) {
      if (n_timesteps < 1) return fail(EZB_ERR_STATE, "device t_index without a timestep table; call ezb_dit_set_timesteps first");
      const int n4 = (ldm + (mod_final ? 2 * D : 0)) / 4, gx = (n4 + 255) / 256 < 64 ? (n4 + 255) / 256 : 64;
      EZB_TRY(launch_k(gather_mod_kernel, dim3(gx, Be), dim3(256), 0, st, 1, tdev, n_timesteps, reinterpret_cast<const float4*>(mod), ldm / 4,
                       reinterpret_cast<const float4*>(mod_final), 2 * D / 4, reinterpret_cast<float4*>(mod_b), reinterpret_cast<float4*>(modf_b)));
      *mod_rows = mod_b; *bstride = ldm; *modf_rows = mod_final ? modf_b : nullptr; *bstride_f = 2 * D;
      return EZB_OK;
    }
    bool uniform = true;
    int t0 = tidx ? tidx[0] : tall;
    for (int i = 0; tidx && i < Be; ++i) {
      if (tidx[i] < 0 || tidx[i] >= n_timesteps) return fail(EZB_ERR_ARG, "t_index %d out of range (n=%d)", tidx[i], n_timesteps);
      uniform = uniform && tidx[i] == t0;
    }
    if (t0 < 0 || t0 >= n_timesteps) return fail(EZB_ERR_ARG, "t_index %d out of range (n=%d); call ezb_dit_set_timesteps first", t0, n_timesteps);
    if (uniform) {
      *mod_rows = mod + (size_t)t0 * ldm; *bstride = 0;
      *modf_rows = mod_final ? mod_final + (size_t)t0 * 2 * D : nullptr; *bstride_f = 0;
    } else {
      for (int i = 0; i < Be; ++i) {
        EZB_CUDA(cudaMemcpyAsync(mod_b + (size_t)i * ldm, mod + (size_t)tidx[i] * ldm, (size_t)ldm * sizeof(float), cudaMemcpyDeviceToDevice, st));
        if (mod_final) EZB_CUDA(cudaMemcpyAsync(modf_b + (size_t)i * 2 * D, mod_final + (size_t)tidx[i] * 2 * D, (size_t)2 * D * sizeof(float), cudaMemcpyDeviceToDevice, st));
      }
      *mod_rows = mod_b; *bstride = ldm; *modf_rows = modf_b; *bstride_f = 2 * D;
    }
    return EZB_OK;
  }

  // ---------------------------------------------------------------- one DiT block (blocks.py:120-160)
  // x_in: residual stream entering; x_out: buffer the block's first residual write goes to (later ops update it in place).
  // Fold mode (fc.on): no LayerNorm pass is launched.  On entry `act` (or, for an out-block, the left half of cat[si]) already holds
  // bf16(x_in * g) and fc.st_x the row statistics of x_in, both written by the GEMM that produced x_in; every residual-stream GEMM of
  // the block does the same for the LayerNorm that follows it (gemm.cuh FoldIn / FoldOut).
  // what reads the OUTPUT of block i: operand buffer(s) + multiplier(s) for the MLP-out epilogue
  FoldOut block_output_fold(int i, int t) {
    BlockW& w = blk[i];
    if (d.is_controlnet) {  // next in-block's norm1 (if any) + the zero-linear of this block (plain cast)
      if (i + 1 < half) return fold_out(w.st_out, act, D, blk[i + 1].g1 + (size_t)t * D, cat[i], D, nullptr);
      return fold_out(w.st_out, cat[i], D, nullptr);
    }
    if (i < half) {   // in-block: norm1 of block i+1, and the skip half of the out-block that pops skip i
      const int ob = half + 1 + (half - 1 - i);
      return fold_out(w.st_out, act, D, blk[i + 1].g1 + (size_t)t * D, cat[i] + D, 2 * D, blk[ob].snw + D);
    }
    if (i < nblk - 1) {  // mid / out-block followed by an out-block: the x half of its concatenated skip_norm input
      const int si = half - 1 - (i + 1 - half - 1);
      return fold_out(w.st_out, cat[si], 2 * D, blk[i + 1].snw);
    }
    return fold_out(w.st_out, act, D, gF + (size_t)t * D);   // last block: FinalBlock norm
  }
  // LayerNorm tails (gemm_ln.cuh): `entry_ln_done` = the LayerNorm this block starts with (norm1, or skip_norm for an out-block) was already
  // executed by the kernel that produced x_in; `next_ln` / `next_done` = the LayerNorm that reads this block's output, for its MLP-out GEMM.
  int block(cudaStream_t st, int i, const float* x_in, float* x_out, const float* skip, const float* cskip, const float* modr, int mbs, int Be, int L,
            FoldCtx fc = FoldCtx(), bool entry_ln_done = false, const LnParams* next_ln = nullptr, bool* next_done = nullptr) {
    BlockW& w = blk[i];
    const int M = Be * L;
    const float* m = modr + (size_t)i * 6 * D;  // shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp (blocks.py:132-133)
    const float2* st1 = fc.st_x;                // statistics of the tensor norm1 sees
    bool fold1 = fc.on;                         // norm1 folded?
    bool ln2_done = false, ln3_done = false;
    if (skip) {  // out-blocks: x = skip_linear(LN_2D(cat[x, skip (+ controlnet skip)]))  (blocks.py:124-128, udit.py:345-348)
      const int si = half - 1 - (i - half - 1);
      EpiLinearParams e = epi();
      e.bias = w.b_skip; e.out_f32 = x_out; e.ld32 = D;
      if (fc.on && cskip == nullptr) {   // both halves of cat[si] and their statistics are in place
        e.fin = fold_in(fc.st_x, blk[si].st_out, 2 * D, w.us, w.vs);
        e.fout = fold_out(w.st_skip, act, D, w.g1 + (size_t)fc.t * D);
        st1 = w.st_skip;
        EZB_TRY(lin(st, cat[si], 2 * D, w.skip, M, D, e));
      } else {  // ControlNet skips are added to the skip half before the norm: LayerNorm kernels for skip_norm and norm1 of this block
        // (`act` is this GEMM's own operand here, so its epilogue cannot also write the norm1 operand into it)
        if (!entry_ln_done) EZB_TRY(ln(st, x_in, D, skip, cskip, D, w.snw, w.snb, nullptr, nullptr, 0, L, act, M));
        const LnParams p1 = ln_params(x_out, D, nullptr, nullptr, 0, w.n1w, w.n1b, m + 0 * D, m + 1 * D, mbs, L, act, M);
        entry_ln_done = false;   // from here on: "norm1 done?"
        EZB_TRY(lin(st, act, 2 * D, w.skip, M, D, e, fp8 ? nullptr : &p1, &entry_ln_done));   // the tail runs behind a grid barrier: nobody reads `act` any more
        fold1 = false;
      }
      x_in = x_out;
    }
    // --- self-attention (blocks.py:137-141)
    if (fp8) EZB_TRY(ln8(st, ln_params(x_in, D, nullptr, nullptr, 0, w.n1w, w.n1b, m + 0 * D, m + 1 * D, mbs, L, act, M)));
    else if (!fold1 && !entry_ln_done) EZB_TRY(ln(st, x_in, D, nullptr, nullptr, 0, w.n1w, w.n1b, m + 0 * D, m + 1 * D, mbs, L, act, M));
    if (fused_heads) {
      const int kinds[3] = {0, 1, 2};
      const int Lp = (L + 7) / 8 * 8;
      FoldIn f1 = fold_in(st1, nullptr, D, w.u1 + (size_t)fc.t * n_qkv, w.v1 + (size_t)fc.t * n_qkv);
      if (fp8) {
        if (!(opt_skip() & 4))
          EZB_TRY(heads_gemm_fp8(*dev, st, act8, act8_s, w.qkv8, w.s_qkv, M, dh, heads_params(3 * D, kinds, w.h_nq, w.h_nk, true, L, q16, k16, vt16, Lp, nullptr)));
      } else {
        EZB_TRY(lin_heads(st, act, w.qkv, M, 3 * D, kinds, w.h_nq, w.h_nk, true, L, q16, k16, vt16, Lp, fold1 ? &f1 : nullptr));
      }
      EZB_TRY(attention(st, q32, k32, v32, q16, k16, vt16, nullptr, Be, L, L, Lp, lens));
    } else {
      EZB_TRY(lin_to_qkv(st, act, D, w.qkv, M, 3 * D));
      const int off[3] = {0, D, 2 * D}, kinds[3] = {0, 1, 2};
      float* f32o[3] = {q32, k32, v32};
      bf16* bfo[3] = {q16, k16, vt16};
      const int Lp = (L + 7) / 8 * 8;
      EZB_TRY(qk_prep(st, 3 * D, 3, off, kinds, w.nqw, w.nqb, w.nkw, w.nkb, w.inv_freq, Be, L, f32o, bfo, Lp));
      EZB_TRY(attention(st, q32, k32, v32, q16, k16, vt16, nullptr, Be, L, L, Lp, lens));
    }
    {
      EpiLinearParams e = epi();
      e.bias = w.b_proj; e.resid = x_in; e.ldr = D; e.gate = m + 2 * D; e.gate_bstride = mbs; e.rows_per_batch = L; e.out_f32 = x_out; e.ld32 = D;
      if (fc.on) e.fout = fold_out(w.st_a, act, D, w.n2w);   // norm2 has no modulation: g = its weight
      const LnParams p2 = ln_params(x_out, D, nullptr, nullptr, 0, w.n2w, w.n2b, nullptr, nullptr, 0, L, act, M);
      EZB_TRY(lin(st, attn_out, D, w.proj, M, D, e, fc.on ? nullptr : &p2, &ln2_done));
    }
    // --- cross-attention (blocks.py:147-151): no modulation, no gate
    if (!fc.on && !ln2_done) EZB_TRY(ln(st, x_out, D, nullptr, nullptr, 0, w.n2w, w.n2b, nullptr, nullptr, 0, L, act, M));
    if (fused_heads) {
      const int kinds[1] = {0};
      FoldIn f2 = fold_in(w.st_a, nullptr, D, w.u2, w.v2);
      EZB_TRY(lin_heads(st, act, w.cq, M, D, kinds, w.h_cnq, nullptr, false, L, q16, nullptr, nullptr, 0, fc.on ? &f2 : nullptr));
      EZB_TRY(attention(st, q32, w.kc32, w.vc32, q16, w.kc16, w.vtc16, ctx_mask, Be, L, ctx_Lc, ctx_Lpad));
    } else {
      EZB_TRY(lin_to_qkv(st, act, D, w.cq, M, D));
      const int off[1] = {0}, kinds[1] = {0};
      float* f32o[1] = {q32};
      bf16* bfo[1] = {q16};
      EZB_TRY(qk_prep(st, D, 1, off, kinds, w.cnqw, w.cnqb, nullptr, nullptr, nullptr, Be, L, f32o, bfo, 0));
      EZB_TRY(attention(st, q32, w.kc32, w.vc32, q16, w.kc16, w.vtc16, ctx_mask, Be, L, ctx_Lc, ctx_Lpad));
    }
    {
      EpiLinearParams e = epi();
      e.bias = w.b_cproj; e.resid = x_out; e.ldr = D; e.out_f32 = x_out; e.ld32 = D;
      if (fc.on) e.fout = fold_out(w.st_b, act, D, w.g3 + (size_t)fc.t * D);
      const LnParams p3 = ln_params(x_out, D, nullptr, nullptr, 0, w.n3w, w.n3b, m + 3 * D, m + 4 * D, mbs, L, act, M);
      EZB_TRY(lin(st, attn_out, D, w.cproj, M, D, e, fc.on || fp8 ? nullptr : &p3, &ln3_done));
    }
    // --- GEGLU MLP (blocks.py:155-156; modules.py:263-277,366)
    if (fp8) EZB_TRY(ln8(st, ln_params(x_out, D, nullptr, nullptr, 0, w.n3w, w.n3b, m + 3 * D, m + 4 * D, mbs, L, act, M)));
    else if (!fc.on && !ln3_done) EZB_TRY(ln(st, x_out, D, nullptr, nullptr, 0, w.n3w, w.n3b, m + 3 * D, m + 4 * D, mbs, L, act, M));
    {
      EpiGegluParams g;
      memset(&g, 0, sizeof g);
      g.bias = w.b_mlp1; g.out_bf16 = mid; g.ld16 = kmul * inner; g.split_stride = kmul == 3 ? inner : 0;
      if (fc.on) g.fin = fold_in(w.st_b, nullptr, D, w.u3 + (size_t)fc.t * 2 * inner, w.v3 + (size_t)fc.t * 2 * inner);
      EpiLinearParams e = epi();
      e.bias = w.b_mlp2; e.resid = x_out; e.ldr = D; e.gate = m + 5 * D; e.gate_bstride = mbs; e.rows_per_batch = L; e.out_f32 = x_out; e.ld32 = D;
      if (fc.on) e.fout = block_output_fold(i, fc.t);
      if (!fp8 && opt_mlp_fused() && geglu_bn == 256 && kmul == 1 && swap_ab && !(opt_skip() & 24) && L >= 32) {
        // the whole MLP as one persistent launch (north_star: "MLP GEMM + act + GEMM as one persistent kernel")
        if (fc.on) EZB_TRY((mlp_fused<EpiGeglu<256, true>, EpiLinearTF<256>>(*dev, st, act, w.mlp1, M, 2 * inner, D, g, mid, w.mlp2, D, inner, e, grid_bar)));
        else EZB_TRY((mlp_fused<EpiGeglu<256>, EpiLinearT<256>>(*dev, st, act, w.mlp1, M, 2 * inner, D, g, mid, w.mlp2, D, inner, e, grid_bar)));
        return EZB_OK;
      }
      if (opt_skip() & 16) {}
      else if (fp8 && geglu_bn == 256) EZB_TRY((gemm2_fp8<256, EpiGeglu<256>>(*dev, st, act8, act8_s, w.mlp18, w.s_mlp1, M, 2 * inner, D, g)));
      else if (fp8) EZB_TRY((gemm2_fp8<128, EpiGeglu<128>>(*dev, st, act8, act8_s, w.mlp18, w.s_mlp1, M, 2 * inner, D, g)));   // inner % 128 != 0
      else if (geglu_bn == 256 && fc.on) EZB_TRY((gemm2<256, EpiGeglu<256, true>>(*dev, st, act, kmul * D, w.mlp1, kmul * D, M, 2 * inner, kmul * D, g)));
      else if (geglu_bn == 256) EZB_TRY(gemm2_geglu(*dev, st, act, kmul * D, w.mlp1, kmul * D, M, 2 * inner, kmul * D, g));
      else if (fc.on) EZB_TRY((gemm<128, EpiGeglu<128, true>>(*dev, st, act, kmul * D, w.mlp1, kmul * D, M, 2 * inner, kmul * D, g)));
      else EZB_TRY((gemm<128, EpiGeglu<128>>(*dev, st, act, kmul * D, w.mlp1, kmul * D, M, 2 * inner, kmul * D, g)));
      if (opt_mlp2_pair() && pair && kmul == 1 && !fc.on)   // MLP-out on 2-CTA cluster tiles (128 tokens x 128 features, thread = token row) instead of swap-AB
        EZB_TRY((gemm2<128, EpiLinear<128>>(*dev, st, mid, inner, w.mlp2, inner, M, D, inner, e)));
      else
      EZB_TRY(lin(st, mid, inner, w.mlp2, M, D, e, fc.on ? nullptr : next_ln, next_done));
    }
    return EZB_OK;
  }

  int embed(cudaStream_t st, const float* x, const float* gt, const uint8_t* gt_mask, const float* resid, int Be, int L, const FoldCtx& fc = FoldCtx(),
            const LnParams* next_ln = nullptr, bool* next_done = nullptr) {
    EZB_TRY(patch_pack_launch(st, x, gt, gt_mask, mask_embed, a_patch, Be, C, L, Kp, kmul));
    EpiLinearParams e = epi();
    e.bias = b_patch; e.out_f32 = x0; e.ld32 = D; e.resid = resid; e.ldr = D;
    if (fc.on) e.fout = fold_out(st_x0, act, D, blk[0].g1 + (size_t)fc.t * D);
    return lin(st, a_patch, Kp, w_patch, Be * L, D, e, fc.on ? nullptr : next_ln, next_done);
  }
  // fold mode for this call: tables valid for the schedule and one timestep for the whole batch
  FoldCtx fold_ctx(int mbs, const float* modr, int L) {
    FoldCtx fc;
    if (fold_cfg && fold_n > 0 && mbs == 0 && L >= 32) {
      const int t = (int)((modr - mod) / ((size_t)nblk * 6 * D));
      if (t >= 0 && t < fold_n) { fc.on = true; fc.t = t; }
    }
    return fc;
  }

  int check_call(int Be, int L) {
    if (!finalized) return fail(EZB_ERR_STATE, "weights not finalized");
    if (Be < 1 || Be > d.max_batch || L < 1 || L > d.max_len) return fail(EZB_ERR_SHAPE, "Be %d / L %d exceed workspace (%d, %d)", Be, L, d.max_batch, d.max_len);
    if (Be != ctx_Be) return fail(EZB_ERR_STATE, "batch %d differs from the context set by ezb_dit_set_context (%d)", Be, ctx_Be);
    return EZB_OK;
  }

  // lens_ (device [Be] or null): sample b is a clip of lens_[b] <= L frames padded to L.  Only self-attention and the final conv mix
  // frames; both stop at the clip end, so its frames come out as a solo forward at that length computes them.  Every other kernel works
  // per token.
  // tdev (device [Be] or null): per-sample timestep indices read on the device, in place of tidx / tall.
  int forward(const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall, const float* const* cskips, float* out, int Be, int L,
              const int32_t* lens_, cudaStream_t st, const int32_t* tdev = nullptr) {
    if (d.is_controlnet) return fail(EZB_ERR_STATE, "ezb_dit_forward called on a controlnet handle");
    EZB_TRY(check_call(Be, L));
    lens = lens_;
    dev->tmaps.trim();
    WeightSeqScope ws(dev, this, cskips ? 1 : 0, ((long long)Be << 32) | (unsigned)L);   // L2 prefetch of the next GEMM's weights (host.cuh)
    const float *modr, *modf;
    int mbs, mbsf;
    EZB_TRY(select_mod(st, tidx, tall, tdev, Be, &modr, &modf, &mbs, &mbsf));
    FoldCtx fc = fold_ctx(mbs, modr, L);
    const int M = Be * L;
    // the LayerNorm that opens block i, as parameters for the tail phase of the GEMM that produces its input x (gemm_ln.cuh)
    auto entry_ln = [&](int i, const float* xin) -> LnParams {
      if (i > half) {   // out-block: skip_norm over [x | skip (+ controlnet skip)]
        const int si = half - 1 - (i - half - 1);
        return ln_params(xin, D, skips[si], cskips ? cskips[si] : nullptr, D, blk[i].snw, blk[i].snb, nullptr, nullptr, 0, L, act, M);
      }
      const float* mi = modr + (size_t)i * 6 * D;
      return ln_params(xin, D, nullptr, nullptr, 0, blk[i].n1w, blk[i].n1b, mi + 0 * D, mi + 1 * D, mbs, L, act, M);
    };
    bool done = false;
    LnParams nl = entry_ln(0, x0);
    // FP8 mode: a norm1 LayerNorm (in- and mid-blocks) writes e4m3 rows, so it never runs as the bf16 tail of the GEMM before it
    EZB_TRY(embed(st, x, gt, gt_mask, nullptr, Be, L, fc, fp8 ? nullptr : &nl, &done));
    const float* xc = x0;
    fc.st_x = st_x0;
    for (int i = 0; i < half; ++i) {
      const bool entry = done;
      done = false;
      nl = entry_ln(i + 1, skips[i]);
      EZB_TRY(block(st, i, xc, skips[i], nullptr, nullptr, modr, mbs, Be, L, fc, entry, fp8 ? nullptr : &nl, &done));
      xc = skips[i];
      fc.st_x = blk[i].st_out;
    }
    {
      const bool entry = done;
      done = false;
      nl = entry_ln(half + 1, xa);
      EZB_TRY(block(st, half, xc, xa, nullptr, nullptr, modr, mbs, Be, L, fc, entry, &nl, &done));
    }
    xc = xa;
    fc.st_x = blk[half].st_out;
    for (int j = 0; j < half; ++j) {
      const int si = half - 1 - j;  // skips.pop()
      const bool entry = done;
      done = false;
      if (j + 1 < half) nl = entry_ln(half + 2 + j, xb);
      else nl = ln_params(xb, D, nullptr, nullptr, 0, fn_w, fn_b, modf, modf + D, mbsf, L, act, M);   // FinalBlock norm
      EZB_TRY(block(st, half + 1 + j, xc, xb, skips[si], cskips ? cskips[si] : nullptr, modr, mbs, Be, L, fc, entry, &nl, &done));
      xc = xb;
      fc.st_x = blk[half + 1 + j].st_out;
    }
    // FinalBlock (blocks.py:199-211): shift, scale = time_ada_final.chunk(2)
    if (!fc.on && !done) EZB_TRY(ln(st, xc, D, nullptr, nullptr, 0, fn_w, fn_b, modf, modf + D, mbsf, L, act, M));
    EpiLinearParams e = epi();
    e.bias = b_final; e.out_f32 = ybuf; e.ld32 = C;
    if (fc.on) e.fin = fold_in(fc.st_x, nullptr, D, uF + (size_t)fc.t * C, vF + (size_t)fc.t * C);
    EZB_TRY(lin(st, act, D, w_final, M, C, e));
    EZB_TRY(final_conv_launch(*dev, st, ybuf, fc_w, fc_b, out, Be, C, L, lens));
    ws.ok = true;
    return EZB_OK;
  }

  int controlnet_forward(const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall, const float* cond, float cscale,
                         float* const* skips_out, int Be, int L, cudaStream_t st);
  int controlnet_forward_tdev(const float* x, const int32_t* tdev, const float* scale_dev, float* const* skips_out, int Be, int L, cudaStream_t st);
  int controlnet_forward_cached(const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall, float cscale,
                                float* const* skips_out, int Be, int L, cudaStream_t st);
  int set_condition(const float* cond, int Be, int L, cudaStream_t st);
  int set_condition_rows(const float* cond, int row0, int n, int L, cudaStream_t st);
  int controlnet_stem(const float* cond, float* out, int Be, int L, cudaStream_t st);
  int controlnet_trunk(const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall, const int32_t* tdev, const float* cond,
                       float cscale, const float* scale_dev, float* const* skips_out, int Be, int L, cudaStream_t st);
};

}  // namespace ezb

namespace ezb {
// DiTControlNet.forward (controlnet.py:252-315) with the eval-time stem (controlnet.py:65-84: cond_mask_infer = zeros,
// so mask_embed is never written and the appended mask channel is all-zero).
inline int Dit::controlnet_forward(const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall, const float* cond, float cscale,
                                   float* const* skips_out, int Be, int L, cudaStream_t st) {
  if (!d.is_controlnet) return fail(EZB_ERR_STATE, "ezb_controlnet_forward called on a DiT handle");
  EZB_TRY(check_call(Be, L));
  return controlnet_trunk(x, gt, gt_mask, tidx, tall, nullptr, cond, cscale, nullptr, skips_out, Be, L, st);
}

// The four convolutions of the stem (controlnet_pre, controlnet.py:65-84) for conditions of 2L samples, as conv1d_direct_kernel takes them.
struct StemConv { int Cin, cin_real, Tin, Cout, Tout, K, stride, pad, act, transposed; };
inline StemConv stem_conv(int stage, int c0, int c1, int D, int L) {
  const int T = 2 * L;
  switch (stage) {
    case 0: return {1, 1, T, c0, T, 1, 1, 0, 0, 0};                 // conv_in
    case 1: return {c0 + 1, c0, T, c0 + 1, T, 3, 1, 1, 1, 0};       // conv3 + SiLU (mask channel == 0)
    case 2: return {c0 + 1, c0 + 1, T, c1, L, 3, 2, 1, 1, 0};       // conv3 stride 2 + SiLU
    default: return {c1, c1, L, D, L, 1, 1, 0, 0, 1};               // conv_out -> (B,L,D)
  }
}
inline int stem_conv_launch(cudaStream_t st, const StemConv& c, const float* in, const float* w, const float* bias, float* out, int B) {
  const size_t n = (size_t)B * c.Cout * c.Tout;
  ++launch_counter();
  conv1d_direct_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, w, bias, out, B, c.Cin, c.cin_real, c.Tin, c.Cout, c.Tout, c.K, c.stride, c.pad,
                                                                     c.act, c.transposed);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}

// The stem of Be conditions (Be,1,2L) into out (Be,L,D).  It depends on the condition only, and every kernel computes each output element on its
// own, so a clip's rows do not depend on the batch.
inline int Dit::controlnet_stem(const float* cond, float* out, int Be, int L, cudaStream_t st) {
  const float* const ins[4] = {cond, cs_t0, cs_t1, cs_t2};
  const float* const ws[4] = {cs_in_w, cs_c0_w, cs_c1_w, cs_out_w};
  const float* const bs[4] = {cs_in_b, cs_c0_b, cs_c1_b, cs_out_b};
  float* const outs[4] = {cs_t0, cs_t1, cs_t2, out};
  for (int s = 0; s < 4; ++s) EZB_TRY(stem_conv_launch(st, stem_conv(s, d.cond_c0, d.cond_c1, D, L), ins[s], ws[s], bs[s], outs[s], Be));
  return EZB_OK;
}

inline int Dit::set_condition(const float* cond, int Be, int L, cudaStream_t st) {
  if (!d.is_controlnet) return fail(EZB_ERR_STATE, "ezb_controlnet_set_condition called on a DiT handle");
  if (!finalized) return fail(EZB_ERR_STATE, "weights not finalized");
  if (Be < 1 || Be > d.max_batch || L < 1 || L > d.max_len) return fail(EZB_ERR_SHAPE, "set_condition: Be %d / L %d exceed workspace (%d, %d)", Be, L, d.max_batch, d.max_len);
  cond_Be = Be; cond_L = L;
  return controlnet_stem(cond, cond_cache, Be, L, st);
}

// rows [row0, row0 + n) of the layout the last set_condition established (ezb_controlnet_set_condition_rows)
inline int Dit::set_condition_rows(const float* cond, int row0, int n, int L, cudaStream_t st) {
  if (!d.is_controlnet) return fail(EZB_ERR_STATE, "ezb_controlnet_set_condition_rows called on a DiT handle");
  if (!finalized) return fail(EZB_ERR_STATE, "weights not finalized");
  if (cond_Be < 1) return fail(EZB_ERR_STATE, "set_condition_rows: no ezb_controlnet_set_condition call established the condition layout");
  if (L != cond_L) return fail(EZB_ERR_STATE, "set_condition_rows: L %d differs from the condition layout (L %d)", L, cond_L);
  if (row0 < 0 || n < 1 || row0 + n > cond_Be) return fail(EZB_ERR_SHAPE, "set_condition_rows: rows [%d, %d) outside the batch of %d", row0, row0 + n, cond_Be);
  return controlnet_stem(cond, cond_cache + (size_t)row0 * L * D, n, L, st);
}

// The trunk with device timestep indices, the cached condition and per-sample scales.  Device indices always gather per-sample modulation
// rows (no fold mode), as non-uniform host indices do, and the zero-linears run EpiLinearScaled on the tiles EpiLinear<128> takes with a
// non-zero uniform scale: each sample comes out as ezb_controlnet_forward with its scale and such host indices computes it.
inline int Dit::controlnet_forward_tdev(const float* x, const int32_t* tdev, const float* scale_dev, float* const* skips_out, int Be, int L, cudaStream_t st) {
  if (!d.is_controlnet) return fail(EZB_ERR_STATE, "ezb_controlnet_forward_tdev called on a DiT handle");
  EZB_TRY(check_call(Be, L));
  if (Be != cond_Be || L != cond_L)
    return fail(EZB_ERR_STATE, "controlnet_forward_tdev: Be %d / L %d differ from the condition set by ezb_controlnet_set_condition (%d, %d)", Be, L, cond_Be, cond_L);
  return controlnet_trunk(x, nullptr, nullptr, nullptr, 0, tdev, nullptr, 0.f, scale_dev, skips_out, Be, L, st);
}

// controlnet_forward on the condition cache: the stem computes each row on its own, so the cached rows hold the bits controlnet_forward
// writes into cond_emb, and everything after the stem takes the same path (host indices, uniform scale, fold mode).
inline int Dit::controlnet_forward_cached(const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall, float cscale,
                                          float* const* skips_out, int Be, int L, cudaStream_t st) {
  if (!d.is_controlnet) return fail(EZB_ERR_STATE, "ezb_controlnet_forward_cached called on a DiT handle");
  EZB_TRY(check_call(Be, L));
  if (Be != cond_Be || L != cond_L)
    return fail(EZB_ERR_STATE, "controlnet_forward_cached: Be %d / L %d differ from the condition set by ezb_controlnet_set_condition (%d, %d)", Be, L, cond_Be,
                cond_L);
  return controlnet_trunk(x, gt, gt_mask, tidx, tall, nullptr, nullptr, cscale, nullptr, skips_out, Be, L, st);
}

// cond: the raw condition, run through the stem into cond_emb here, or null for the condition cache.  scale_dev (device [Be]) or, when null,
// the uniform cscale.  A uniform scale of 0 writes zero skips without running the trunk: the zero-linears' out_scale reads 0 as 1.
inline int Dit::controlnet_trunk(const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall, const int32_t* tdev,
                                 const float* cond, float cscale, const float* scale_dev, float* const* skips_out, int Be, int L, cudaStream_t st) {
  if (scale_dev == nullptr && cscale == 0.f) {
    for (int i = 0; i < half; ++i) EZB_CUDA(cudaMemsetAsync(skips_out[i], 0, (size_t)Be * L * D * sizeof(float), st));
    return EZB_OK;
  }
  lens = nullptr;   // the stem convs cross clip ends: ControlNet batches are uniform in length
  dev->tmaps.trim();
  WeightSeqScope ws(dev, this, 2, ((long long)Be << 32) | (unsigned)L);
  const float *modr, *modf;
  int mbs, mbsf;
  EZB_TRY(select_mod(st, tidx, tall, tdev, Be, &modr, &modf, &mbs, &mbsf));
  const float* cemb = cond_cache;
  if (cond != nullptr) {
    EZB_TRY(controlnet_stem(cond, cond_emb, Be, L, st));
    cemb = cond_emb;
  }
  FoldCtx fc = fold_ctx(mbs, modr, L);
  const int M = Be * L;
  auto entry_ln = [&](int i, const float* xin) -> LnParams {
    const float* mi = modr + (size_t)i * 6 * D;
    return ln_params(xin, D, nullptr, nullptr, 0, blk[i].n1w, blk[i].n1b, mi + 0 * D, mi + 1 * D, mbs, L, act, M);
  };
  bool done = false;
  LnParams nl = entry_ln(0, x0);
  EZB_TRY(embed(st, x, gt, gt_mask, cemb, Be, L, fc, fp8 ? nullptr : &nl, &done));           // x = patch_embed(x) + condition
  const float* xc = x0;
  fc.st_x = st_x0;
  for (int i = 0; i < half; ++i) {
    const bool entry = done;
    done = false;
    if (i + 1 < half) nl = entry_ln(i + 1, skips[i]);
    EZB_TRY(block(st, i, xc, skips[i], nullptr, nullptr, modr, mbs, Be, L, fc, entry, i + 1 < half && !fp8 ? &nl : nullptr, &done));
    xc = skips[i];
    fc.st_x = blk[i].st_out;
  }
  for (int i = 0; i < half; ++i) {  // zero-linears * conditioning_scale (controlnet.py:311-313)
    const bf16* A = act;
    if (fc.on) A = cat[i];          // plain bf16 cast of the block output, written by its MLP-out epilogue
    else EZB_TRY(ln(st, skips[i], D, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr, 0, L, act, M));
    EpiLinearParams e = epi();
    e.bias = blk[i].zero_b; e.out_scale = cscale; e.out_f32 = skips_out[i]; e.ld32 = D;
    if (scale_dev == nullptr) {
      EZB_TRY(lin(st, A, D, blk[i].zero_w, M, D, e));
    } else if (!(opt_skip() & 8)) {
      const EpiLinearScaledParams es{e, scale_dev, L};
      if (pair) EZB_TRY((gemm2<128, EpiLinearScaled<128>>(*dev, st, A, kmul * D, blk[i].zero_w, kmul * D, M, D, kmul * D, es)));
      else EZB_TRY((gemm<128, EpiLinearScaled<128>>(*dev, st, A, kmul * D, blk[i].zero_w, kmul * D, M, D, kmul * D, es)));
    }
  }
  ws.ok = true;
  return EZB_OK;
}
}  // namespace ezb
