// C-ABI entry points of libezb200.so (declared in include/ezb200.h).
#include "../../include/ezb200.h"

#include <algorithm>
#include "dit.cuh"
#include "vae.cuh"
#include "t5.cuh"
#include "host.cuh"
#include "longform.cuh"
#include "timeline.cuh"

using namespace ezb;

namespace {
Device& device_ctx(int device) {
  static Device devs[16];
  Device& d = devs[device & 15];
  if (!d.queried && device >= 0) {
    d.queried = true;
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0) d.num_sms = sms;
    d.id = device;
  }
  return d;
}
EpiLinearParams to_epi(const ezb_test_epilogue* e) {
  EpiLinearParams p;
  memset(&p, 0, sizeof p);
  p.bias = e->bias; p.bias_mod = e->bias_mod; p.resid = e->resid; p.ldr = e->ldr; p.gate = e->gate;
  p.gate_bstride = e->gate_bstride; p.rows_per_batch = e->rows_per_batch; p.out_f32 = e->out_f32; p.ld32 = e->ld32;
  p.out_bf16 = reinterpret_cast<__nv_bfloat16*>(e->out_bf16); p.ld16 = e->ld16; p.split_stride = e->split_stride;
  p.act = e->act; p.act_a = e->act_a; p.act_b = e->act_b; p.out_scale = 0.f; p.phase_cols = 0; p.phase_ld16 = 0;
  if (e->fin_u) {
    p.fin.st0 = static_cast<const float2*>(e->fin_st); p.fin.slots0 = e->fin_slots; p.fin.ld_st = e->fin_ld_st; p.fin.inv_dim = e->fin_inv_dim;
    p.fin.u = e->fin_u; p.fin.v = e->fin_v;
    p.fin.st1 = static_cast<const float2*>(e->fin_st1); p.fin.slots1 = e->fin_st1 ? e->fin_slots1 : 0;
  }
  if (e->fout_st) {
    p.fout.st = static_cast<float2*>(e->fout_st); p.fout.ld_st = e->fout_ld_st;
    p.fout.a0 = static_cast<__nv_bfloat16*>(e->fout_a0); p.fout.ld0 = e->fout_ld0; p.fout.g0 = e->fout_g0;
    p.fout.a1 = static_cast<__nv_bfloat16*>(e->fout_a1); p.fout.ld1 = e->fout_ld1; p.fout.g1 = e->fout_g1;
  }
  return p;
}
}  // namespace

extern "C" {

__attribute__((visibility("default"))) int ezb_version(void) { return 2; }
__attribute__((visibility("default"))) const char* ezb_last_error(void) { return last_error().c_str(); }

__attribute__((visibility("default"))) int ezb_test_gemm(int device, const void* A, int lda, const void* W, int ldw, int M, int N, int K, int bn, int epi_kind,
                  const ezb_test_epilogue* e, int conv_taps, int conv_center, int conv_dil, int conv_cin_pad, int conv_T, int conv_B,
                  void* stream) {
  if (!A || !W || !e) return fail(EZB_ERR_ARG, "ezb_test_gemm: null pointer");
  EZB_CUDA(cudaSetDevice(device));
  Device& dev = device_ctx(device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const __nv_bfloat16* a = reinterpret_cast<const __nv_bfloat16*>(A);
  const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(W);
  ConvAddr conv;
  conv.taps = conv_taps; conv.center = conv_center; conv.dilation = conv_dil; conv.cin_pad = conv_cin_pad; conv.T = conv_T; conv.B = conv_B;
  const ConvAddr* cp = conv_taps > 0 ? &conv : nullptr;
  if (epi_kind == 20 || epi_kind == 21) {  // swap-AB: tiles of 128 features x 256 / 288 tokens, fp32 output
    if (cp) return fail(EZB_ERR_UNSUPPORTED, "swap-AB GEMM has no conv addressing");
    EpiLinearParams p = to_epi(e);
    if ((p.fin.u && (!p.fin.st0 || !p.fin.v)) || (p.fout.st && !p.fout.a0))
      return fail(EZB_ERR_ARG, "ezb_test_gemm: fold-in needs its partials and v, fold-out its first operand");
    if (p.fin.u && (p.fin.slots0 < 1 || (p.fin.st1 != nullptr && p.fin.slots1 < 1)))
      return fail(EZB_ERR_ARG, "ezb_test_gemm: fold-in with %d + %d partial slots", p.fin.slots0, p.fin.slots1);
    const bool fold = p.fin.u || p.fout.st;
    if (epi_kind == 20) {   // what Dit::lin dispatches
      if (fold) return gemm_swapped<EpiLinearTF>(dev, st, a, lda, w, ldw, M, N, K, p);
      if (opt_swap_mc()) return gemm_swapped_mc<EpiLinearT, 3>(dev, st, a, lda, w, ldw, M, N, K, p);
      return gemm_swapped<EpiLinearT>(dev, st, a, lda, w, ldw, M, N, K, p);
    }
    if (bn == 256) return fold ? gemm_swapped_at<256, EpiLinearTF<256>>(dev, st, a, lda, w, ldw, M, N, K, p)
                               : gemm_swapped_at<256, EpiLinearT<256>>(dev, st, a, lda, w, ldw, M, N, K, p);
    if (bn == 288) return fold ? gemm_swapped_at<288, EpiLinearTF<288>>(dev, st, a, lda, w, ldw, M, N, K, p)
                               : gemm_swapped_at<288, EpiLinearT<288>>(dev, st, a, lda, w, ldw, M, N, K, p);
    return fail(EZB_ERR_UNSUPPORTED, "ezb_test_gemm swap-AB: bn=%d (256 or 288)", bn);
  }
  if (epi_kind == 10 || epi_kind == 11) {  // 2-CTA cluster kernel with the W tile multicast (bn is the tile's N)
    if (cp) return fail(EZB_ERR_UNSUPPORTED, "cluster GEMM has no conv addressing");
    if (epi_kind == 10) {
      EpiLinearParams p = to_epi(e);
      if (bn == 128) return gemm2<128, EpiLinear<128>>(dev, st, a, lda, w, ldw, M, N, K, p);
      if (bn == 256) return gemm2<256, EpiLinear<256>>(dev, st, a, lda, w, ldw, M, N, K, p);
    } else {
      EpiGegluParams p;
      memset(&p, 0, sizeof p);
      p.bias = e->bias; p.out_bf16 = reinterpret_cast<__nv_bfloat16*>(e->out_bf16); p.ld16 = e->ld16; p.split_stride = e->split_stride;
      if (bn == 256) return gemm2_geglu(dev, st, a, lda, w, ldw, M, N, K, p);   // what Dit::block dispatches
    }
    return fail(EZB_ERR_UNSUPPORTED, "ezb_test_gemm pair: bn=%d", bn);
  }
  if (epi_kind == 12) {  // the parked-tile cluster GEGLU, which bf16x3 and outputs not 16-byte aligned run
    if (cp || bn != 256) return fail(EZB_ERR_UNSUPPORTED, "ezb_test_gemm: the parked cluster GEGLU is the plain bn=256 kernel");
    EpiGegluParams p;
    memset(&p, 0, sizeof p);
    p.bias = e->bias; p.out_bf16 = reinterpret_cast<__nv_bfloat16*>(e->out_bf16); p.ld16 = e->ld16; p.split_stride = e->split_stride;
    return gemm2<256, EpiGeglu<256>>(dev, st, a, lda, w, ldw, M, N, K, p);
  }
  if (epi_kind == 0) {
    EpiLinearParams p = to_epi(e);
    if (bn == 64) return gemm<64, EpiLinear<64>>(dev, st, a, lda, w, ldw, M, N, K, p, cp);
    if (bn == 128) return gemm<128, EpiLinear<128>>(dev, st, a, lda, w, ldw, M, N, K, p, cp);
    if (bn == 256) return gemm<256, EpiLinear<256>>(dev, st, a, lda, w, ldw, M, N, K, p, cp);
  } else if (epi_kind == 1) {
    EpiGegluParams p;
    memset(&p, 0, sizeof p);
    p.bias = e->bias; p.out_bf16 = reinterpret_cast<__nv_bfloat16*>(e->out_bf16); p.ld16 = e->ld16; p.split_stride = e->split_stride;
    if (bn == 128) return gemm<128, EpiGeglu<128>>(dev, st, a, lda, w, ldw, M, N, K, p, cp);
    if (bn == 256) return gemm<256, EpiGeglu<256>>(dev, st, a, lda, w, ldw, M, N, K, p, cp);
  }
  return fail(EZB_ERR_UNSUPPORTED, "ezb_test_gemm: bn=%d epi=%d", bn, epi_kind);
}

}  // extern "C"

namespace {
bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }
int test_linear_check(const ezb_test_linear_args* a) {
  const int M = a->M, N = a->N, K = a->K, km = a->kmul;
  if (!a->A || !a->W) return fail(EZB_ERR_ARG, "ezb_test_linear: null A or W");
  if (!a->out_f32 && !a->out_bf16) return fail(EZB_ERR_ARG, "ezb_test_linear: no output");
  if (km != 1 && km != 3) return fail(EZB_ERR_ARG, "ezb_test_linear: kmul %d (1 or 3)", km);
  if (a->kernel < 0 || a->kernel > 4) return fail(EZB_ERR_ARG, "ezb_test_linear: kernel %d (0 to 4)", a->kernel);
  if ((a->kernel == 1 || a->kernel == 2) && a->scale) return fail(EZB_ERR_ARG, "ezb_test_linear: kernel %d is EpiLinear, scale selects EpiLinearScaled", a->kernel);
  if (a->kernel >= 3 && !a->scale) return fail(EZB_ERR_ARG, "ezb_test_linear: kernel %d (EpiLinearScaled) needs scale", a->kernel);
  if (a->act != ACT_NONE && a->act != ACT_SILU) return fail(EZB_ERR_ARG, "ezb_test_linear: act %d (0 none, 1 SiLU)", a->act);
  if (a->split && (km != 3 || !a->out_bf16)) return fail(EZB_ERR_ARG, "ezb_test_linear: the split bf16 output needs kmul 3 and out_bf16");
  if (a->gate && !a->resid) return fail(EZB_ERR_ARG, "ezb_test_linear: a gate needs the residual it gates into");
  if (a->scale && (a->resid || a->gate || a->out_bf16 || !a->out_f32 || a->out_scale != 0.f))
    return fail(EZB_ERR_UNSUPPORTED, "ezb_test_linear: EpiLinearScaled reads bias and writes out_f32 only");
  if (M < 1 || M > (1 << 24) || N < 8 || N % 8 || K < 8 || K % 8 || (long long)N * K > (1LL << 28))
    return fail(EZB_ERR_SHAPE, "ezb_test_linear: M %d N %d K %d (N, K multiples of 8)", M, N, K);
  if (a->lda < km * K || a->lda % 8) return fail(EZB_ERR_SHAPE, "ezb_test_linear: A pitch %d (>= %d, a multiple of 8)", a->lda, km * K);
  if ((a->gate || a->scale) && a->rows_per_batch < 1) return fail(EZB_ERR_SHAPE, "ezb_test_linear: %d rows per clip", a->rows_per_batch);
  // the epilogue reads and writes column pairs: fp32 as float2, bf16 as 4-byte pairs
  if ((a->resid && (a->ldr < N || a->ldr % 2)) || (a->gate && (a->gate_bstride < 0 || a->gate_bstride % 2)) ||
      (a->out_f32 && (a->ld32 < N || a->ld32 % 2)) || (a->out_bf16 && (a->ld16 < (a->split ? 3 * N : N) || a->ld16 % 2)))
    return fail(EZB_ERR_SHAPE, "ezb_test_linear: row pitches ldr %d gate %d ld32 %d ld16 %d for N %d", a->ldr, a->gate_bstride, a->ld32, a->ld16, N);
  if (!aligned(a->A, 16) || !aligned(a->resid, 8) || !aligned(a->gate, 8) || !aligned(a->out_f32, 8) || !aligned(a->out_bf16, 4) || !aligned(a->bias, 4))
    return fail(EZB_ERR_ARG, "ezb_test_linear: A must be 16-byte aligned, resid / gate / out_f32 8-byte, out_bf16 and bias 4-byte");
  return EZB_OK;
}
int test_linear_run(Device& dev, cudaStream_t st, const ezb_test_linear_args* a, int kernel, __nv_bfloat16* Wp) {
  const int M = a->M, N = a->N, K = a->K, km = a->kmul;
  pack_weight_kernel<<<(unsigned)(((size_t)N * K + 255) / 256), 256, 0, st>>>(a->W, N, K, Wp, K, km, 0, 0, 0, 0, 0, 0);
  EZB_CUDA(cudaGetLastError());
  if (a->w_packed) EZB_CUDA(cudaMemcpyAsync(a->w_packed, Wp, (size_t)N * km * K * sizeof(__nv_bfloat16), cudaMemcpyDeviceToDevice, st));
  const __nv_bfloat16* A = static_cast<const __nv_bfloat16*>(a->A);
  EpiLinearParams e;
  memset(&e, 0, sizeof e);
  e.bias = a->bias; e.resid = a->resid; e.ldr = a->ldr; e.gate = a->gate; e.gate_bstride = a->gate_bstride; e.rows_per_batch = a->rows_per_batch;
  e.out_f32 = a->out_f32; e.ld32 = a->ld32; e.out_bf16 = static_cast<__nv_bfloat16*>(a->out_bf16); e.ld16 = a->ld16;
  e.split_stride = a->split ? N : 0; e.act = a->act; e.out_scale = a->out_scale;
  const EpiLinearScaledParams es{e, a->scale, a->rows_per_batch};
  if (kernel == 0) {   // Dit::lin, or the ControlNet trunk's zero-linears for per-sample scales
    if (a->scale) kernel = a->pair ? 4 : 3;
    else if (!lin_takes_swap_ab(e, M, a->m_select, a->pair != 0, a->swap_ab != 0, km)) kernel = a->pair ? 2 : 1;
    else {
      if (a->ran) *a->ran = swapped_bn(dev, M, N);
      return opt_swap_mc() ? gemm_swapped_mc<EpiLinearT, 3>(dev, st, A, a->lda, Wp, K, M, N, K, e) : gemm_swapped<EpiLinearT>(dev, st, A, a->lda, Wp, K, M, N, K, e);
    }
  }
  if (a->ran) *a->ran = kernel;
  const int ldw = km * K;
  switch (kernel) {
    case 1: return gemm<128, EpiLinear<128>>(dev, st, A, a->lda, Wp, ldw, M, N, ldw, e);
    case 2: return gemm2<128, EpiLinear<128>>(dev, st, A, a->lda, Wp, ldw, M, N, ldw, e);
    case 3: return gemm<128, EpiLinearScaled<128>>(dev, st, A, a->lda, Wp, ldw, M, N, ldw, es);
    default: return gemm2<128, EpiLinearScaled<128>>(dev, st, A, a->lda, Wp, ldw, M, N, ldw, es);
  }
}
}  // namespace

extern "C" {

__attribute__((visibility("default"))) int ezb_test_linear(int device, const ezb_test_linear_args* a, void* stream) {
  if (!a) return fail(EZB_ERR_ARG, "ezb_test_linear: null arguments");
  EZB_TRY(test_linear_check(a));
  EZB_CUDA(cudaSetDevice(device));
  Device& dev = device_ctx(device);
  dev.tmaps.trim();
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  __nv_bfloat16* Wp = nullptr;
  EZB_CUDA(cudaMallocAsync(&Wp, (size_t)a->N * a->kmul * a->K * sizeof(__nv_bfloat16), st));
  const int rc = test_linear_run(dev, st, a, a->kernel, Wp);
  EZB_CUDA(cudaFreeAsync(Wp, st));
  return rc;
}

__attribute__((visibility("default"))) int ezb_test_heads(int device, const void* A, const float* W, const ezb_test_heads_args* a, void* stream) {
  if (!A || !W || !a) return fail(EZB_ERR_ARG, "ezb_test_heads: null pointer");
  const int B = a->B, L = a->L, D = a->D, H = a->H, dh = a->dh, nsec = a->nsec;
  const int variant = a->variant == 2 ? HEADS_PACKED3_PARKED : a->variant;   // 2: the retired 128-deep-slot id runs the parked packed-3 kernel
  if (dh != 64 && dh != 72) return fail(EZB_ERR_SHAPE, "ezb_test_heads: head dimension %d (64 or 72)", dh);
  if (H < 2 || H % 2) return fail(EZB_ERR_SHAPE, "ezb_test_heads: %d heads (a positive even count)", H);
  if (D != H * dh) return fail(EZB_ERR_SHAPE, "ezb_test_heads: D %d != H %d x dh %d", D, H, dh);
  if (B < 1 || L < 1 || (long long)B * L > (1 << 24)) return fail(EZB_ERR_SHAPE, "ezb_test_heads: B %d L %d", B, L);
  if (nsec < 1 || nsec > 3) return fail(EZB_ERR_SHAPE, "ezb_test_heads: %d sections", nsec);
  if (a->ld_qk < dh || a->ld_qk % 8) return fail(EZB_ERR_SHAPE, "ezb_test_heads: q / k pitch %d (>= dh %d, a multiple of 8)", a->ld_qk, dh);
  if (a->Lpad < L) return fail(EZB_ERR_SHAPE, "ezb_test_heads: V^T pitch %d < L %d", a->Lpad, L);
  if (a->dvp < dh) return fail(EZB_ERR_SHAPE, "ezb_test_heads: V^T rows %d < dh %d", a->dvp, dh);
  if (a->variant < HEADS_PACKED3 || a->variant > HEADS_SINGLE) return fail(EZB_ERR_ARG, "ezb_test_heads: variant %d", a->variant);
  const bool packed = variant == HEADS_PACKED3 || variant == HEADS_PACKED3_PARKED;
  if (packed && nsec != 3) return fail(EZB_ERR_SHAPE, "ezb_test_heads: the packed-3 layout needs q, k and v sections");
  for (int s = 0; s < nsec; ++s) {
    const int kd = a->kinds[s];
    if (kd < 0 || kd > 2) return fail(EZB_ERR_ARG, "ezb_test_heads: section %d kind %d", s, kd);
    if ((kd == 0 && (!a->q || !a->norm_q)) || (kd == 1 && (!a->k || !a->norm_k)) || (kd == 2 && !a->vt))
      return fail(EZB_ERR_ARG, "ezb_test_heads: section %d (kind %d) without its output or LayerNorm parameters", s, kd);
  }
  if (a->rope < 0 || a->rope > 2 || (a->rope && !a->inv_freq)) return fail(EZB_ERR_ARG, "ezb_test_heads: rope mode %d", a->rope);
  const int M = B * L, N = nsec * D, bn3 = dh == 72 ? 224 : 192;
  if (a->fold_st && (!a->fold_u || !a->fold_v || a->fold_slots < 1 || a->fold_ld_st < M))
    return fail(EZB_ERR_ARG, "ezb_test_heads: fold needs u, v and %d-row partials", M);
  EZB_CUDA(cudaSetDevice(device));
  Device& dev = device_ctx(device);
  dev.tmaps.trim();
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  EpiHeadsParams e;
  memset(&e, 0, sizeof e);
  // by-value parameters (the model copies them to the host once, at finalize)
  EZB_CUDA(cudaStreamSynchronize(st));
  if (a->norm_q) { EZB_CUDA(cudaMemcpy(e.nw[0], a->norm_q, dh * sizeof(float), cudaMemcpyDeviceToHost)); EZB_CUDA(cudaMemcpy(e.nb[0], a->norm_q + dh, dh * sizeof(float), cudaMemcpyDeviceToHost)); }
  if (a->norm_k) { EZB_CUDA(cudaMemcpy(e.nw[1], a->norm_k, dh * sizeof(float), cudaMemcpyDeviceToHost)); EZB_CUDA(cudaMemcpy(e.nb[1], a->norm_k + dh, dh * sizeof(float), cudaMemcpyDeviceToHost)); }
  if (a->rope) EZB_CUDA(cudaMemcpy(e.inv_freq, a->inv_freq, (dh / 2) * sizeof(float), cudaMemcpyDeviceToHost));
  e.D = D; e.H = H; e.L = L;
  for (int s = 0; s < 3; ++s) e.kind[s] = s < nsec ? a->kinds[s] : 0;
  e.rope_kinds = 3; e.rope_ld = L; e.rope_mufu = a->rope == 2;
  e.out[0] = reinterpret_cast<__nv_bfloat16*>(a->q); e.out[1] = reinterpret_cast<__nv_bfloat16*>(a->k); e.out[2] = reinterpret_cast<__nv_bfloat16*>(a->vt);
  e.ld_qk = a->ld_qk; e.dvp = a->dvp; e.Lpad = a->Lpad;
  if (a->fold_st) {
    e.fin.st0 = reinterpret_cast<const float2*>(a->fold_st); e.fin.slots0 = a->fold_slots; e.fin.ld_st = a->fold_ld_st;
    e.fin.inv_dim = 1.0f / (float)D; e.fin.u = a->fold_u; e.fin.v = a->fold_v;
  }
  // the weight packed as Dit::init packs it (packed-3: zero-filled pad rows), the RoPE table as Dit::finalize fills it
  const int rows = packed ? H * bn3 : N;
  __nv_bfloat16* Wp = nullptr;
  float2* cs = nullptr;
  EZB_CUDA(cudaMallocAsync(&Wp, (size_t)rows * D * sizeof(__nv_bfloat16), st));
  EZB_CUDA(cudaMemsetAsync(Wp, 0, (size_t)rows * D * sizeof(__nv_bfloat16), st));
  const unsigned grid_w = (unsigned)(((size_t)D * D + 255) / 256);
  if (packed) {
    for (int s = 0; s < 3; ++s) pack_weight_kernel<<<grid_w, 256, 0, st>>>(W + (size_t)s * D * D, D, D, Wp, D, 1, 0, 0, 0, dh, s * H, bn3);
  } else {
    pack_weight_kernel<<<grid_w * nsec, 256, 0, st>>>(W, N, D, Wp, D, 1, 0, 0, 0, 0, 0, 0);
  }
  EZB_CUDA(cudaGetLastError());
  if (a->rope) {
    EZB_CUDA(cudaMallocAsync(&cs, (size_t)L * (dh / 2) * sizeof(float2), st));
    rope_table_kernel<<<(L * (dh / 2) + 255) / 256, 256, 0, st>>>(a->inv_freq, cs, L, dh / 2);
    EZB_CUDA(cudaGetLastError());
    e.rope = cs;
  }
  const int rc = heads_gemm(dev, st, reinterpret_cast<const __nv_bfloat16*>(A), Wp, M, N, dh, variant, e);
  EZB_CUDA(cudaFreeAsync(Wp, st));
  if (cs) EZB_CUDA(cudaFreeAsync(cs, st));
  return rc;
}

__attribute__((visibility("default"))) int ezb_test_mlp(int device, const void* A, const float* W1, const float* b1, const void* W2, const float* b2, float* x,
                                                        const float* gate, int gate_bstride, int rows_per_batch, void* mid, void* bar, int M, int D, int inner,
                                                        int variant, void* stream) {
  if (!A || !W1 || !b1 || !W2 || !b2 || !x || !mid || !bar) return fail(EZB_ERR_ARG, "ezb_test_mlp: null pointer");
  if (M < 1 || D < 64 || D % 8 || inner < 128 || inner % 128) return fail(EZB_ERR_SHAPE, "ezb_test_mlp: M %d D %d inner %d", M, D, inner);
  // the swap-AB epilogue looks up the gates of at most two clips per 32-token chunk (the model takes this path for clips of >= 32 tokens)
  if (gate && rows_per_batch < 32) return fail(EZB_ERR_SHAPE, "ezb_test_mlp: %d rows per clip (>= 32)", rows_per_batch);
  if (variant < 0 || variant > 2) return fail(EZB_ERR_ARG, "ezb_test_mlp: variant %d", variant);
  EZB_CUDA(cudaSetDevice(device));
  Device& dev = device_ctx(device);
  dev.tmaps.trim();
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  constexpr int half = 128;   // GEGLU packing group of the 256-wide N-tiles
  __nv_bfloat16* W1p = nullptr;
  float* b1p = nullptr;
  EZB_CUDA(cudaMallocAsync(&W1p, (size_t)2 * inner * D * sizeof(__nv_bfloat16), st));
  EZB_CUDA(cudaMallocAsync(&b1p, (size_t)2 * inner * sizeof(float), st));
  pack_weight_kernel<<<(unsigned)(((size_t)2 * inner * D + 255) / 256), 256, 0, st>>>(W1, 2 * inner, D, W1p, D, 1, 0, inner, half, 0, 0, 0);
  pack_geglu_bias_kernel<<<(2 * inner + 255) / 256, 256, 0, st>>>(b1, b1p, inner, half);
  EZB_CUDA(cudaGetLastError());
  EpiGegluParams g;
  memset(&g, 0, sizeof g);
  g.bias = b1p; g.out_bf16 = reinterpret_cast<__nv_bfloat16*>(mid); g.ld16 = inner;
  EpiLinearParams p;
  memset(&p, 0, sizeof p);
  p.bias = b2; p.resid = x; p.ldr = D; p.gate = gate; p.gate_bstride = gate_bstride; p.rows_per_batch = rows_per_batch > 0 ? rows_per_batch : 1;
  p.out_f32 = x; p.ld32 = D;
  const __nv_bfloat16* a16 = reinterpret_cast<const __nv_bfloat16*>(A);
  const __nv_bfloat16* w2 = reinterpret_cast<const __nv_bfloat16*>(W2);
  const __nv_bfloat16* m16 = reinterpret_cast<const __nv_bfloat16*>(mid);
  int rc;
  if (variant == 0) {
    rc = mlp_fused<EpiGeglu<256>, EpiLinearT<256>>(dev, st, a16, W1p, M, 2 * inner, D, g, m16, w2, D, inner, p, reinterpret_cast<GridBarrier*>(bar));
  } else {
    rc = variant == 2 ? gemm2<256, EpiGeglu<256>>(dev, st, a16, D, W1p, D, M, 2 * inner, D, g) : gemm2_geglu(dev, st, a16, D, W1p, D, M, 2 * inner, D, g);
    if (rc == EZB_OK) rc = gemm_swapped<EpiLinearT>(dev, st, m16, inner, w2, inner, M, D, inner, p);
  }
  EZB_CUDA(cudaFreeAsync(W1p, st));
  EZB_CUDA(cudaFreeAsync(b1p, st));
  return rc;
}

}  // extern "C"

namespace {
int test_fold_check(const ezb_test_fold_args* a) {
  const int kind = a->kind, M = a->M, N = a->N, K = a->K;
  if (kind < 0 || kind > 3) return fail(EZB_ERR_ARG, "ezb_test_fold: kind %d", kind);
  if (!a->shift != !a->scale) return fail(EZB_ERR_ARG, "ezb_test_fold: shift and scale come in pairs");
  if (kind <= 2) {
    if (!a->W || !a->w || !a->b || !a->G || !a->Cc || !a->u || !a->v) return fail(EZB_ERR_ARG, "ezb_test_fold: the tables need W, w, b, G, Cc, u and v");
    if (K > FOLD_MAX_K) return fail(EZB_ERR_UNSUPPORTED, "ezb_test_fold: K %d (the tables take at most %d)", K, FOLD_MAX_K);
    if (K < 8 || K % 8) return fail(EZB_ERR_SHAPE, "ezb_test_fold: K %d (a multiple of 8)", K);
    if (a->shift && a->R > 1 && a->ld_mod < K) return fail(EZB_ERR_SHAPE, "ezb_test_fold: modulation rows %d apart, narrower than K %d", a->ld_mod, K);
  }
  if (kind == 0) {
    if (!a->w_packed) return fail(EZB_ERR_ARG, "ezb_test_fold: the tables write the packed weight");
    if (N < 1 || a->R < 1 || a->R > 128 || (long long)N * K > (1LL << 28)) return fail(EZB_ERR_SHAPE, "ezb_test_fold: tables N %d R %d", N, a->R);
    return EZB_OK;
  }
  if (kind <= 2) {
    const int inner = a->inner, bn = kind == 2 ? 256 : a->geglu_bn;
    if (!a->A || !a->st || !a->bias || !a->out) return fail(EZB_ERR_ARG, "ezb_test_fold: the GEGLU needs A, st, bias and out");
    if (a->R != 1) return fail(EZB_ERR_ARG, "ezb_test_fold: the GEGLU tables take one modulation row (R 1, not %d)", a->R);
    if (M < 1 || M > (1 << 24) || inner < 64 || inner % 64) return fail(EZB_ERR_SHAPE, "ezb_test_fold: M %d inner %d (a multiple of 64)", M, inner);
    if (bn != 0 && bn != 128 && bn != 256) return fail(EZB_ERR_ARG, "ezb_test_fold: geglu_bn %d (0, 128 or 256)", bn);
    if (bn == 256 && inner % 128) return fail(EZB_ERR_UNSUPPORTED, "ezb_test_fold: 256-wide GEGLU tiles need inner %d to be a multiple of 128", inner);
    if (a->slots < 1 || a->ld_st < M) return fail(EZB_ERR_SHAPE, "ezb_test_fold: %d partial slots of pitch %d for %d rows", a->slots, a->ld_st, M);
  }
  if (kind == 2) {
    if (!a->W2 || !a->b2 || !a->x || !a->fout_st || !a->a0 || !a->g0 || !a->grid_barrier)
      return fail(EZB_ERR_ARG, "ezb_test_fold: the fused MLP needs W2, b2, x, fout_st, a0, g0 and grid_barrier");
    if (K % 32) return fail(EZB_ERR_SHAPE, "ezb_test_fold: the folded-out partials need K %d to be a multiple of 32", K);
    if (a->gate && a->rows_per_batch < 32) return fail(EZB_ERR_SHAPE, "ezb_test_fold: %d rows per clip (>= 32)", a->rows_per_batch);
    if (a->variant < 0 || a->variant > 1) return fail(EZB_ERR_ARG, "ezb_test_fold: variant %d", a->variant);
  }
  if (kind == 3) {
    if (!a->A || !a->W16 || !a->out_f32 || !a->ln_out || !a->w || !a->b || !a->grid_barrier)
      return fail(EZB_ERR_ARG, "ezb_test_fold: the LayerNorm tail needs A, W16, out_f32, ln_out, w, b and grid_barrier");
    if (M < 1 || M > (1 << 24) || N < 4 || N % 4 || K < 8 || K % 8 || a->D2 < 0 || a->D2 % 4)
      return fail(EZB_ERR_SHAPE, "ezb_test_fold: tail M %d N %d K %d D2 %d", M, N, K, a->D2);
    if ((a->D2 > 0) != (a->x2 != nullptr) || (a->x3 && !a->x2)) return fail(EZB_ERR_ARG, "ezb_test_fold: x2 must come with D2 > 0, x3 with x2");
    if (a->shift && (a->x2 || a->rows_per_batch < 1 || a->ld_mod < 0 || a->ld_mod % 4))
      return fail(EZB_ERR_ARG, "ezb_test_fold: modulation needs one source, rows_per_batch >= 1 and ld_mod a multiple of 4");
    if (a->gate && (!a->resid || a->rows_per_batch < 32)) return fail(EZB_ERR_ARG, "ezb_test_fold: a gate needs a residual and clips of >= 32 rows");
    if (a->bn != 0 && a->bn != 256 && a->bn != 288) return fail(EZB_ERR_ARG, "ezb_test_fold: bn %d (0, 256 or 288)", a->bn);
    const void* ps[] = {a->out_f32, a->x2, a->x3, a->w, a->b, a->shift, a->scale, a->ln_out, a->A};
    for (const void* q : ps)
      if (!aligned(q, 16)) return fail(EZB_ERR_ARG, "ezb_test_fold: LayerNorm pointers and A must be 16-byte aligned");
  }
  return EZB_OK;
}
// kinds 1 / 2: W and its bias packed as Dit::init packs them, the site-3 tables as Dit::build_fold_tables builds them, then the GEMM(s)
int test_fold_run(Device& dev, cudaStream_t st, ezb_test_fold_args* a, __nv_bfloat16* Wp, float* bp) {
  const int M = a->M, D = a->K, inner = a->inner;
  const int bn = a->kind == 2 ? 256 : a->geglu_bn ? a->geglu_bn : (inner % 128 == 0 ? 256 : 128), gh = bn / 2;
  pack_weight_kernel<<<(unsigned)(((size_t)2 * inner * D + 255) / 256), 256, 0, st>>>(a->W, 2 * inner, D, Wp, D, 1, 0, inner, gh, 0, 0, 0);
  pack_geglu_bias_kernel<<<(2 * inner + 255) / 256, 256, 0, st>>>(a->bias, bp, inner, gh);
  EZB_CUDA(cudaGetLastError());
  if (a->w_packed) EZB_CUDA(cudaMemcpyAsync(a->w_packed, Wp, (size_t)2 * inner * D * sizeof(__nv_bfloat16), cudaMemcpyDeviceToDevice, st));
  EZB_TRY(fold_gc_launch(st, a->w, a->b, a->shift, a->scale, a->ld_mod, a->G, a->Cc, 1, D));
  EZB_TRY(fold_uv_launch(st, Wp, D, a->G, a->Cc, bp, a->u, a->v, 2 * inner, D, 1));   // v carries the packed GEGLU bias
  EpiGegluParams g;
  memset(&g, 0, sizeof g);
  g.bias = bp; g.out_bf16 = static_cast<__nv_bfloat16*>(a->out); g.ld16 = inner;
  g.fin.st0 = static_cast<const float2*>(a->st); g.fin.slots0 = a->slots; g.fin.ld_st = a->ld_st; g.fin.inv_dim = 1.0f / (float)D;
  g.fin.u = a->u; g.fin.v = a->v;
  const __nv_bfloat16* A = static_cast<const __nv_bfloat16*>(a->A);
  if (a->kind == 1) {
    if (bn == 256) return gemm2<256, EpiGeglu<256, true>>(dev, st, A, D, Wp, D, M, 2 * inner, D, g);
    return gemm<128, EpiGeglu<128, true>>(dev, st, A, D, Wp, D, M, 2 * inner, D, g);
  }
  EpiLinearParams e;
  memset(&e, 0, sizeof e);
  e.bias = a->b2; e.resid = a->x; e.ldr = D; e.gate = a->gate; e.gate_bstride = a->gate_bstride; e.rows_per_batch = a->gate ? a->rows_per_batch : 1;
  e.out_f32 = a->x; e.ld32 = D;
  e.fout.st = static_cast<float2*>(a->fout_st); e.fout.ld_st = a->ld_st; e.fout.a0 = static_cast<__nv_bfloat16*>(a->a0); e.fout.ld0 = D; e.fout.g0 = a->g0;
  const __nv_bfloat16* mid = static_cast<const __nv_bfloat16*>(a->out);
  const __nv_bfloat16* W2 = static_cast<const __nv_bfloat16*>(a->W2);
  if (a->variant == 0)
    return mlp_fused<EpiGeglu<256, true>, EpiLinearTF<256>>(dev, st, A, Wp, M, 2 * inner, D, g, mid, W2, D, inner, e, static_cast<GridBarrier*>(a->grid_barrier));
  EZB_TRY((gemm2<256, EpiGeglu<256, true>>(dev, st, A, D, Wp, D, M, 2 * inner, D, g)));
  return gemm_swapped<EpiLinearTF>(dev, st, mid, inner, W2, inner, M, D, inner, e);
}
}  // namespace

extern "C" {

__attribute__((visibility("default"))) int ezb_test_fold(int device, ezb_test_fold_args* a, void* stream) {
  if (!a) return fail(EZB_ERR_ARG, "ezb_test_fold: null arguments");
  EZB_TRY(test_fold_check(a));
  EZB_CUDA(cudaSetDevice(device));
  Device& dev = device_ctx(device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int M = a->M, N = a->N, K = a->K;
  if (a->kind == 0) {   // Dit::build_fold_tables / Dit::finalize
    __nv_bfloat16* Wp = static_cast<__nv_bfloat16*>(a->w_packed);
    pack_weight_kernel<<<(unsigned)(((size_t)N * K + 255) / 256), 256, 0, st>>>(a->W, N, K, Wp, K, 1, 0, 0, 0, 0, 0, 0);
    EZB_CUDA(cudaGetLastError());
    EZB_TRY(fold_gc_launch(st, a->w, a->b, a->shift, a->scale, a->ld_mod, a->G, a->Cc, a->R, K));
    return fold_uv_launch(st, Wp, K, a->G, a->Cc, a->add_v, a->u, a->v, N, K, a->R);
  }
  if (a->kind == 3) {   // Dit::lin with a LayerNorm tail (gemm_swapped_ln)
    LnParams lp;
    memset(&lp, 0, sizeof lp);
    lp.x = a->out_f32; lp.x2 = a->x2; lp.x3 = a->x3; lp.D1 = N; lp.D2 = a->D2; lp.w = a->w; lp.b = a->b; lp.shift = a->shift; lp.scale = a->scale;
    lp.mod_bstride = a->ld_mod; lp.rows_per_batch = a->shift ? a->rows_per_batch : 1; lp.out = static_cast<__nv_bfloat16*>(a->ln_out); lp.kmul = 1;
    lp.M = M;
    EpiLinearParams e;
    memset(&e, 0, sizeof e);
    e.bias = a->bias; e.resid = a->resid; e.ldr = N; e.gate = a->gate; e.gate_bstride = a->gate_bstride; e.rows_per_batch = a->gate ? a->rows_per_batch : 1;
    e.out_f32 = a->out_f32; e.ld32 = N;
    const __nv_bfloat16* A = static_cast<const __nv_bfloat16*>(a->A);
    const __nv_bfloat16* W = static_cast<const __nv_bfloat16*>(a->W16);
    GridBarrier* bar = static_cast<GridBarrier*>(a->grid_barrier);
    const int bn = a->bn ? a->bn : swapped_bn(dev, M, N);
    bool fused = false;
    const int rc = bn == 288 ? gemm_swapped_ln_at<288, EpiLinearT<288>>(dev, st, A, K, W, K, M, N, K, e, lp, bar, &fused)
                             : gemm_swapped_ln_at<256, EpiLinearT<256>>(dev, st, A, K, W, K, M, N, K, e, lp, bar, &fused);
    a->ran_bn = bn;
    a->ran_fused = fused ? 1 : 0;
    return rc;
  }
  dev.tmaps.trim();
  __nv_bfloat16* Wp = nullptr;
  float* bp = nullptr;
  EZB_CUDA(cudaMallocAsync(&Wp, (size_t)2 * a->inner * K * sizeof(__nv_bfloat16), st));
  EZB_CUDA(cudaMallocAsync(&bp, (size_t)2 * a->inner * sizeof(float), st));
  const int rc = test_fold_run(dev, st, a, Wp, bp);
  EZB_CUDA(cudaFreeAsync(Wp, st));
  EZB_CUDA(cudaFreeAsync(bp, st));
  return rc;
}

namespace {
// packs W (reference layout fp32) as Dit::init does, quantises it as Dit::finalize does, runs the kernel
int test_fp8_gemm(Device& dev, cudaStream_t st, const ezb_test_fp8_args* a, __nv_bfloat16* Wp, uint8_t* Wq, float* Ws, float* bp) {
  const int D = a->D, M = a->M;
  const uint8_t* A = static_cast<const uint8_t*>(a->q);
  if (a->kind == 1) {
    constexpr int half = 128;   // GEGLU packing group of the 256-wide N-tiles
    const int inner = a->inner, N = 2 * inner;
    pack_weight_kernel<<<(unsigned)(((size_t)N * D + 255) / 256), 256, 0, st>>>(a->w, N, D, Wp, D, 1, 0, inner, half, 0, 0, 0);
    pack_geglu_bias_kernel<<<(N + 255) / 256, 256, 0, st>>>(a->b, bp, inner, half);
    quant_rows_e4m3_kernel<<<(N + 7) / 8, 256, 0, st>>>(Wp, N, D, Wq, Ws);
    EZB_CUDA(cudaGetLastError());
    if (a->w_q) EZB_CUDA(cudaMemcpyAsync(a->w_q, Wq, (size_t)N * D, cudaMemcpyDeviceToDevice, st));
    if (a->w_s) EZB_CUDA(cudaMemcpyAsync(a->w_s, Ws, (size_t)N * sizeof(float), cudaMemcpyDeviceToDevice, st));
    EpiGegluParams g;
    memset(&g, 0, sizeof g);
    g.bias = bp; g.out_bf16 = static_cast<__nv_bfloat16*>(a->out); g.ld16 = inner;
    return gemm2_fp8<256, EpiGeglu<256>>(dev, st, A, a->s, Wq, Ws, M, N, D, g);
  }
  const int H = a->H, dh = a->dh, bn3 = dh == 72 ? 224 : 192, rows = H * bn3;
  const unsigned grid_w = (unsigned)(((size_t)D * D + 255) / 256);
  for (int s = 0; s < 3; ++s) pack_weight_kernel<<<grid_w, 256, 0, st>>>(a->w + (size_t)s * D * D, D, D, Wp, D, 1, 0, 0, 0, dh, s * H, bn3);
  quant_rows_e4m3_kernel<<<(rows + 7) / 8, 256, 0, st>>>(Wp, rows, D, Wq, Ws);
  EZB_CUDA(cudaGetLastError());
  if (a->w_q) EZB_CUDA(cudaMemcpyAsync(a->w_q, Wq, (size_t)rows * D, cudaMemcpyDeviceToDevice, st));
  if (a->w_s) EZB_CUDA(cudaMemcpyAsync(a->w_s, Ws, (size_t)rows * sizeof(float), cudaMemcpyDeviceToDevice, st));
  EpiHeadsParams e;
  memset(&e, 0, sizeof e);
  EZB_CUDA(cudaStreamSynchronize(st));   // by-value parameters, as ezb_test_heads
  EZB_CUDA(cudaMemcpy(e.nw[0], a->norm_q, dh * sizeof(float), cudaMemcpyDeviceToHost)); EZB_CUDA(cudaMemcpy(e.nb[0], a->norm_q + dh, dh * sizeof(float), cudaMemcpyDeviceToHost));
  EZB_CUDA(cudaMemcpy(e.nw[1], a->norm_k, dh * sizeof(float), cudaMemcpyDeviceToHost)); EZB_CUDA(cudaMemcpy(e.nb[1], a->norm_k + dh, dh * sizeof(float), cudaMemcpyDeviceToHost));
  if (a->rope) EZB_CUDA(cudaMemcpy(e.inv_freq, a->inv_freq, (dh / 2) * sizeof(float), cudaMemcpyDeviceToHost));
  e.D = D; e.H = H; e.L = a->L;
  for (int s = 0; s < 3; ++s) e.kind[s] = s;
  e.rope_kinds = 3; e.rope_ld = a->L; e.rope_mufu = a->rope == 2;
  e.out[0] = static_cast<__nv_bfloat16*>(a->q_out); e.out[1] = static_cast<__nv_bfloat16*>(a->k_out); e.out[2] = static_cast<__nv_bfloat16*>(a->vt_out);
  e.ld_qk = a->ld_qk; e.dvp = a->dvp; e.Lpad = a->Lpad;
  float2* cs = nullptr;
  if (a->rope) {
    EZB_CUDA(cudaMallocAsync(&cs, (size_t)a->L * (dh / 2) * sizeof(float2), st));
    rope_table_kernel<<<(a->L * (dh / 2) + 255) / 256, 256, 0, st>>>(a->inv_freq, cs, a->L, dh / 2);
    EZB_CUDA(cudaGetLastError());
    e.rope = cs;
  }
  const int rc = heads_gemm_fp8(dev, st, A, a->s, Wq, Ws, M, dh, e);
  if (cs) EZB_CUDA(cudaFreeAsync(cs, st));
  return rc;
}
int test_vae_run(Device& dev, cudaStream_t st, const ezb_test_vae_args* a, int kmul, float* scratch, size_t part, __nv_bfloat16** wp) {
  float *norms = scratch, *wfold = scratch + part;
  const VaeSnake sn{scratch + 2 * part, scratch + 3 * part};
  const VaeSnake* snake = a->act ? &sn : nullptr;
  const int kind = a->kind, C = kind == 3 || kind == 6 ? a->cin : a->cout;
  if (a->act && kind != 6) EZB_TRY(vae_snake_prep(st, a->alpha, a->beta, sn, a->cout));
  if (kind <= 2) {
    VaeConv c = kind == 0 ? vae_conv_geom(a->cin, a->cout, a->taps, a->dil, kmul)
              : kind == 1 ? vae_convT_geom(a->cin, a->cout, a->stride, kmul) : vae_conv_strided_geom(a->cin, a->cout, a->stride, kmul);
    c.bias = a->bias;
    const size_t bytes = c.w_elems() * sizeof(__nv_bfloat16);
    EZB_CUDA(cudaMallocAsync(wp, bytes, st));
    EZB_CUDA(cudaMemsetAsync(*wp, 0, bytes, st));   // the pad columns, as Vae::alloc zeroes them
    c.w = *wp;
    EZB_TRY(kind == 1 ? vae_pack_convT_w(st, c, a->weight_v, a->weight_g, norms, kmul) : vae_pack_conv_w(st, c, a->weight_v, a->weight_g, norms, kmul));
    EZB_TRY(vae_conv(dev, st, c, kmul, static_cast<const __nv_bfloat16*>(a->x), a->B, a->T, a->resid, a->raw,
                     static_cast<__nv_bfloat16*>(a->act), snake));
    if (a->w_packed) EZB_CUDA(cudaMemcpyAsync(a->w_packed, c.w, bytes, cudaMemcpyDeviceToDevice, st));
    return EZB_OK;
  }
  const float* x = static_cast<const float*>(a->x);
  if (kind == 3) {
    EZB_TRY(vae_fold_wave_w(st, a->weight_v, a->weight_g, norms, wfold, C));
    EZB_TRY(vae_wave_out(st, static_cast<const __nv_bfloat16*>(a->x), wfold, a->out, a->B, C, a->T, kmul));
  } else if (kind == 4) {
    EZB_TRY(vae_fold_conv_in_w(st, a->weight_v, a->weight_g, norms, wfold, C));
    EZB_TRY(vae_enc_conv_in(st, x, wfold, a->bias, sn, a->raw, static_cast<__nv_bfloat16*>(a->act), a->B, C, a->T, kmul));
  } else if (kind == 5) {
    return vae_sample(st, x, a->noise, a->out, a->B, C, a->T);
  } else {
    return vae_latent_pack(st, x, static_cast<__nv_bfloat16*>(a->act), a->B, C, a->T, kmul);
  }
  if (a->w_packed) EZB_CUDA(cudaMemcpyAsync(a->w_packed, wfold, (size_t)7 * C * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return EZB_OK;
}
}  // namespace

__attribute__((visibility("default"))) int ezb_test_vae(int device, const ezb_test_vae_args* a, void* stream) {
  if (!a) return fail(EZB_ERR_ARG, "ezb_test_vae: null arguments");
  const int kind = a->kind, B = a->B, T = a->T, cin = a->cin, cout = a->cout, s = a->stride;
  if (kind < 0 || kind > 6) return fail(EZB_ERR_ARG, "ezb_test_vae: kind %d", kind);
  if (a->precision != 0 && a->precision != 1) return fail(EZB_ERR_ARG, "ezb_test_vae: precision %d", a->precision);
  if (!a->x) return fail(EZB_ERR_ARG, "ezb_test_vae: null input");
  const long long rows = (long long)B * T * (kind == 1 || kind == 2 ? (s > 1 ? s : 1) : 1);
  if (B < 1 || T < 1 || rows > (1 << 26)) return fail(EZB_ERR_SHAPE, "ezb_test_vae: B %d T %d", B, T);
  if (kind <= 4 && kind != 3 && (!a->weight_v || !a->weight_g || !a->bias)) return fail(EZB_ERR_ARG, "ezb_test_vae: kind %d needs weight_v, weight_g and bias", kind);
  if (a->act && kind != 6 && (!a->alpha || !a->beta)) return fail(EZB_ERR_ARG, "ezb_test_vae: an activated output needs the snake's alpha and beta");
  if (kind <= 2) {
    if (cin < 8 || cin % 8 || cout < 8 || cout % 8 || cin > 8192 || cout > 8192)
      return fail(EZB_ERR_SHAPE, "ezb_test_vae: cin %d cout %d (multiples of 8, at most 8192)", cin, cout);
    if (!a->raw && !a->act) return fail(EZB_ERR_ARG, "ezb_test_vae: conv without an output");
    if (kind == 0 && (a->taps < 1 || a->taps % 2 == 0 || a->dil < 1)) return fail(EZB_ERR_SHAPE, "ezb_test_vae: conv taps %d dilation %d (odd taps)", a->taps, a->dil);
    if (kind == 1 && (s < 2 || s % 2)) return fail(EZB_ERR_UNSUPPORTED, "ezb_test_vae: conv-transpose stride %d (even, >= 2)", s);
    if (kind == 2 && s < 2) return fail(EZB_ERR_SHAPE, "ezb_test_vae: strided conv stride %d (>= 2)", s);
  } else if (kind == 3) {
    if (cin < 4 || cin % 4 || !a->weight_v || !a->weight_g || !a->out) return fail(EZB_ERR_SHAPE, "ezb_test_vae: wave out over %d channels (multiple of 4) needs weights and out", cin);
  } else if (kind == 4) {
    if (cout < 1 || !a->raw || !a->act) return fail(EZB_ERR_ARG, "ezb_test_vae: the stem over %d channels writes raw and act", cout);
  } else if (kind == 5) {
    if (cout < 1 || !a->out) return fail(EZB_ERR_ARG, "ezb_test_vae: sample over %d channels needs out", cout);
  } else if (cin < 1 || !a->act) {
    return fail(EZB_ERR_ARG, "ezb_test_vae: latent pack over %d channels needs act", cin);
  }
  const int C = kind <= 2 ? (cin > cout ? cin : cout) : (kind == 3 || kind == 6 ? cin : cout);
  if (C > 8192) return fail(EZB_ERR_SHAPE, "ezb_test_vae: %d channels (at most 8192)", C);
  EZB_CUDA(cudaSetDevice(device));
  Device& dev = device_ctx(device);
  dev.tmaps.trim();
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t part = ((size_t)7 * C + 63) / 64 * 64;   // norms, folded weights, snake a, snake 1/b
  float* scratch = nullptr;
  __nv_bfloat16* wp = nullptr;
  EZB_CUDA(cudaMallocAsync(&scratch, 4 * part * sizeof(float), st));
  const int rc = test_vae_run(dev, st, a, a->precision == 1 ? 3 : 1, scratch, part, &wp);
  EZB_CUDA(cudaFreeAsync(scratch, st));
  if (wp) EZB_CUDA(cudaFreeAsync(wp, st));
  return rc;
}

__attribute__((visibility("default"))) int ezb_test_fp8(int device, const ezb_test_fp8_args* a, void* stream) {
  if (!a) return fail(EZB_ERR_ARG, "ezb_test_fp8: null arguments");
  const int kind = a->kind, M = a->M, D = a->D;
  if (kind < 0 || kind > 2) return fail(EZB_ERR_ARG, "ezb_test_fp8: kind %d", kind);
  if (M < 1 || M > (1 << 24) || D < 16 || D % 16 || D > 1152) return fail(EZB_ERR_SHAPE, "ezb_test_fp8: M %d D %d (D a multiple of 16, at most 1152)", M, D);
  if (!a->q || !a->s) return fail(EZB_ERR_ARG, "ezb_test_fp8: null operand q / s");
  if (kind == 0 && (!a->x || !a->weight || !a->bias || (!a->shift != !a->scale))) return fail(EZB_ERR_ARG, "ezb_test_fp8: LayerNorm needs x, weight, bias");
  if (kind == 1 && (!a->w || !a->b || !a->out || a->inner < 128 || a->inner % 128))
    return fail(EZB_ERR_ARG, "ezb_test_fp8: GEGLU needs w, b, out and inner (a multiple of 128), inner %d", a->inner);
  if (kind == 2) {
    const int H = a->H, dh = a->dh;
    if ((dh != 64 && dh != 72) || H < 2 || H % 2 || D != H * dh) return fail(EZB_ERR_SHAPE, "ezb_test_fp8: heads H %d dh %d D %d", H, dh, D);
    if (a->B < 1 || a->L < 1 || (long long)a->B * a->L != M) return fail(EZB_ERR_SHAPE, "ezb_test_fp8: B %d L %d M %d", a->B, a->L, M);
    if (!a->w || !a->norm_q || !a->norm_k || !a->q_out || !a->k_out || !a->vt_out) return fail(EZB_ERR_ARG, "ezb_test_fp8: heads needs w, norms and outputs");
    if (a->ld_qk < dh || a->ld_qk % 8 || a->Lpad < a->L || a->dvp < dh) return fail(EZB_ERR_SHAPE, "ezb_test_fp8: output pitches");
    if (a->rope < 0 || a->rope > 2 || (a->rope && !a->inv_freq)) return fail(EZB_ERR_ARG, "ezb_test_fp8: rope mode %d", a->rope);
  }
  EZB_CUDA(cudaSetDevice(device));
  Device& dev = device_ctx(device);
  dev.tmaps.trim();
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (kind == 0) {
    LnParams p;
    memset(&p, 0, sizeof p);
    p.x = a->x; p.D1 = D; p.w = a->weight; p.b = a->bias; p.shift = a->shift; p.scale = a->scale; p.mod_bstride = 0; p.rows_per_batch = 1;
    p.kmul = 1; p.M = M;
    const LnFp8Out o{static_cast<uint8_t*>(a->q), a->s};
    const int grid = dev.num_sms * 4 < (M + 3) / 4 ? dev.num_sms * 4 : (M + 3) / 4;   // as Dit::ln8
    if (D == 1152) return launch_k(ln_fp8_kernel<9, true>, dim3(grid), dim3(128), 0, st, 1, p, o);
    if (D == 1024) return launch_k(ln_fp8_kernel<8, true>, dim3(grid), dim3(128), 0, st, 1, p, o);
    return launch_k(ln_fp8_kernel<9, false>, dim3(grid), dim3(128), 0, st, 1, p, o);
  }
  const size_t rows = kind == 1 ? (size_t)2 * a->inner : (size_t)a->H * (a->dh == 72 ? 224 : 192);
  __nv_bfloat16* Wp = nullptr;
  uint8_t* Wq = nullptr;
  float *Ws = nullptr, *bp = nullptr;
  EZB_CUDA(cudaMallocAsync(&Wp, rows * D * sizeof(__nv_bfloat16), st));
  EZB_CUDA(cudaMemsetAsync(Wp, 0, rows * D * sizeof(__nv_bfloat16), st));   // packed-3 pad rows stay 0, as Dit::alloc leaves them
  EZB_CUDA(cudaMallocAsync(&Wq, rows * D, st));
  EZB_CUDA(cudaMallocAsync(&Ws, rows * sizeof(float), st));
  EZB_CUDA(cudaMallocAsync(&bp, rows * sizeof(float), st));
  const int rc = test_fp8_gemm(dev, st, a, Wp, Wq, Ws, bp);
  EZB_CUDA(cudaFreeAsync(Wp, st));
  EZB_CUDA(cudaFreeAsync(Wq, st));
  EZB_CUDA(cudaFreeAsync(Ws, st));
  EZB_CUDA(cudaFreeAsync(bp, st));
  return rc;
}
}  // extern "C"

namespace {
// can LayerNorm kernel `variant` (LnVariant) take these parameters?
bool ln_variant_fits(const LnParams& p, int variant) {
  const bool reg_width = p.D1 == 1152 || p.D1 == 1024;
  switch (variant) {
    case LN_AUTO: case LN_GENERIC: return true;
    case LN_REG1: case LN_REG8: return p.kmul == 1 && !p.x2 && p.w && reg_width;
    case LN_GC: return p.kmul == 1 && !p.x2 && p.G && reg_width;
    case LN_CAT: return p.kmul == 1 && p.x2 && p.w && !p.shift && p.D2 == p.D1 && reg_width;
  }
  return false;
}
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
int test_step_check(const ezb_test_step_args* a) {
  const int kind = a->kind;
  if (kind < 0 || kind > 5) return fail(EZB_ERR_ARG, "ezb_test_step: kind %d", kind);
  if (!a->x || !a->out) return fail(EZB_ERR_ARG, "ezb_test_step: null input or output");
  if (kind == 0) {
    if (a->M < 1 || a->M > (1 << 26)) return fail(EZB_ERR_SHAPE, "ezb_test_step: LayerNorm over %d rows", a->M);
    if (a->kmul != 1 && a->kmul != 3) return fail(EZB_ERR_ARG, "ezb_test_step: kmul %d (1 or 3)", a->kmul);
    if (a->D1 < 4 || a->D1 % 4 || a->D2 < 0 || a->D2 % 4) return fail(EZB_ERR_SHAPE, "ezb_test_step: LayerNorm widths %d + %d (multiples of 4)", a->D1, a->D2);
    if ((a->D2 > 0) != (a->x2 != nullptr) || (a->x3 && !a->x2)) return fail(EZB_ERR_ARG, "ezb_test_step: x2 must come with D2 > 0, x3 with x2");
    if (!a->w != !a->b || !a->shift != !a->scale || !a->G != !a->Cc) return fail(EZB_ERR_ARG, "ezb_test_step: w / b, shift / scale and G / Cc come in pairs");
    if (a->shift && (a->x2 || a->rows_per_batch < 1 || a->mod_bstride < 0))
      return fail(EZB_ERR_ARG, "ezb_test_step: modulation needs one source, rows_per_batch >= 1 and mod_bstride >= 0");
    if (a->G && (a->x2 || (a->D1 != 1152 && a->D1 != 1024))) return fail(EZB_ERR_ARG, "ezb_test_step: a precombined affine is for one source of 1024 or 1152");
    if (a->variant < LN_AUTO || a->variant > LN_CAT) return fail(EZB_ERR_ARG, "ezb_test_step: LayerNorm variant %d", a->variant);
    // the kernels read every input as float4 and the register variants store 8-byte groups of the output
    const void* ps[] = {a->x, a->x2, a->x3, a->w, a->b, a->shift, a->scale, a->G, a->Cc, a->out};
    for (const void* q : ps)
      if (!aligned16(q)) return fail(EZB_ERR_ARG, "ezb_test_step: LayerNorm pointers must be 16-byte aligned");
    if (a->shift && a->mod_bstride % 4) return fail(EZB_ERR_ARG, "ezb_test_step: mod_bstride %d (a multiple of 4)", a->mod_bstride);
    return EZB_OK;
  }
  if (kind == 1) {
    const int B = a->B, L = a->L, H = a->H, dh = a->dh, nsec = a->nsec;
    if (B < 1 || L < 1 || H < 1 || dh < 2 || dh > 96 || dh % 2) return fail(EZB_ERR_SHAPE, "ezb_test_step: qk_prep B %d L %d H %d dh %d (even, <= 96)", B, L, H, dh);
    if (nsec < 1 || nsec > 3 || (long long)B * L * H * nsec > (1 << 26)) return fail(EZB_ERR_SHAPE, "ezb_test_step: qk_prep %d sections", nsec);
    if (a->in_bf16 != 0 && a->in_bf16 != 1) return fail(EZB_ERR_ARG, "ezb_test_step: in_bf16 %d", a->in_bf16);
    for (int s = 0; s < nsec; ++s) {
      const int kd = a->kinds[s];
      if (kd < 0 || kd > 2) return fail(EZB_ERR_ARG, "ezb_test_step: section %d kind %d", s, kd);
      if (a->col_off[s] < 0 || a->col_off[s] + H * dh > a->ld_in) return fail(EZB_ERR_SHAPE, "ezb_test_step: section %d at column %d past the row of %d", s, a->col_off[s], a->ld_in);
      if ((kd == 0 && !a->norm_q) || (kd == 1 && !a->norm_k)) return fail(EZB_ERR_ARG, "ezb_test_step: section %d without its LayerNorm parameters", s);
      if (!a->f32_out[s] && !a->bf_out[s]) return fail(EZB_ERR_ARG, "ezb_test_step: section %d has no output", s);
      if (a->bf_out[s] && kd < 2 && a->ld_qk < dh) return fail(EZB_ERR_SHAPE, "ezb_test_step: q / k pitch %d < dh %d", a->ld_qk, dh);
      if (a->bf_out[s] && kd == 2 && (a->Lpad < L || a->dv_pad < dh)) return fail(EZB_ERR_SHAPE, "ezb_test_step: V^T %d x %d for dh %d L %d", a->dv_pad, a->Lpad, dh, L);
    }
    return EZB_OK;
  }
  if (kind == 2) {
    if (a->B < 1 || a->B > 65535 || a->L < 1 || a->C < 16 || a->C % 16 || a->Kp < 2 * a->C + 1) return fail(EZB_ERR_SHAPE, "ezb_test_step: patch_pack B %d C %d L %d Kp %d", a->B, a->C, a->L, a->Kp);
    if (a->kmul != 1 && a->kmul != 3) return fail(EZB_ERR_ARG, "ezb_test_step: kmul %d (1 or 3)", a->kmul);
    if (!a->mask_embed || (a->gt_mask && !a->gt)) return fail(EZB_ERR_ARG, "ezb_test_step: patch_pack needs mask_embed, a gt_mask needs gt");
    return EZB_OK;
  }
  if (kind == 3) {
    if (a->B < 1 || a->B > 65535 || a->L < 1 || a->C < 4 || a->C % 4 || a->C > 512) return fail(EZB_ERR_SHAPE, "ezb_test_step: final_conv B %d C %d L %d", a->B, a->C, a->L);
    if (!a->w || !a->b) return fail(EZB_ERR_ARG, "ezb_test_step: final_conv needs w and b");
    if (!aligned16(a->w) || !aligned16(a->b)) return fail(EZB_ERR_ARG, "ezb_test_step: final_conv reads w and b as float4 (16-byte aligned)");
    return EZB_OK;
  }
  if (kind == 4) {
    if (a->R < 1 || a->N < 1 || a->K < 1 || a->ld_in < a->K || a->ld_out < a->N || (a->add && a->ld_add < a->N))
      return fail(EZB_ERR_SHAPE, "ezb_test_step: small_linear R %d N %d K %d pitches %d / %d / %d", a->R, a->N, a->K, a->ld_in, a->ld_add, a->ld_out);
    if (!a->w || (a->act != 0 && a->act != 1)) return fail(EZB_ERR_ARG, "ezb_test_step: small_linear needs w; act %d (0 or 1)", a->act);
    return EZB_OK;
  }
  if (a->M < 1 || a->M > (1 << 20)) return fail(EZB_ERR_SHAPE, "ezb_test_step: %d timesteps", a->M);
  return EZB_OK;
}
// qk_prep parameters as Dit::qk_prep fills them (p.in set by the caller)
template <typename Params>
void test_qk_params(Params& p, const ezb_test_step_args* a) {
  p.ld_in = a->ld_in; p.n_sections = a->nsec;
  for (int s = 0; s < 3; ++s) {
    p.col_off[s] = s < a->nsec ? a->col_off[s] : 0; p.sec_kind[s] = s < a->nsec ? a->kinds[s] : 0;
    p.f32_out[s] = s < a->nsec ? a->f32_out[s] : nullptr; p.bf_out[s] = s < a->nsec ? static_cast<__nv_bfloat16*>(a->bf_out[s]) : nullptr;
  }
  if (a->norm_q) { p.nw[0] = a->norm_q; p.nb[0] = a->norm_q + a->dh; }
  if (a->norm_k) { p.nw[1] = a->norm_k; p.nb[1] = a->norm_k + a->dh; }
  p.use_rope = a->inv_freq != nullptr; p.inv_freq = a->inv_freq;
  p.B = a->B; p.L = a->L; p.H = a->H; p.dh = a->dh; p.ld_qk = a->ld_qk; p.Lpad = a->Lpad; p.dv_pad = a->dv_pad;
}
}  // namespace

extern "C" {

__attribute__((visibility("default"))) int ezb_test_step(int device, const ezb_test_step_args* a, void* stream) {
  if (!a) return fail(EZB_ERR_ARG, "ezb_test_step: null arguments");
  EZB_TRY(test_step_check(a));
  LnParams p;
  memset(&p, 0, sizeof p);
  if (a->kind == 0) {
    p.x = static_cast<const float*>(a->x); p.x2 = a->x2; p.x3 = a->x3; p.D1 = a->D1; p.D2 = a->D2; p.w = a->w; p.b = a->b;
    p.shift = a->shift; p.scale = a->scale; p.mod_bstride = a->mod_bstride; p.rows_per_batch = a->shift ? a->rows_per_batch : 1;
    p.out = static_cast<__nv_bfloat16*>(a->out); p.kmul = a->kmul; p.M = a->M; p.G = a->G; p.C = a->Cc;
    if (!ln_variant_fits(p, a->variant)) return fail(EZB_ERR_UNSUPPORTED, "ezb_test_step: LayerNorm variant %d cannot take D1 %d D2 %d kmul %d", a->variant, a->D1, a->D2, a->kmul);
  }
  EZB_CUDA(cudaSetDevice(device));
  Device& dev = device_ctx(device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const float* x = static_cast<const float*>(a->x);
  switch (a->kind) {
    case 0: return ln_launch(dev, st, p, a->variant);
    case 1: {
      if (a->in_bf16) {
        QkPrepParams<__nv_bfloat16> q;
        memset(&q, 0, sizeof q);
        q.in = static_cast<const __nv_bfloat16*>(a->x);
        test_qk_params(q, a);
        return qk_prep_launch(st, q);
      }
      QkPrepParams<float> q;
      memset(&q, 0, sizeof q);
      q.in = x;
      test_qk_params(q, a);
      return qk_prep_launch(st, q);
    }
    case 2: return patch_pack_launch(st, x, a->gt, a->gt_mask, a->mask_embed, static_cast<__nv_bfloat16*>(a->out), a->B, a->C, a->L, a->Kp, a->kmul);
    case 3: return final_conv_launch(dev, st, x, a->w, a->b, static_cast<float*>(a->out), a->B, a->C, a->L, a->lens);
    case 4: return small_linear_launch(st, x, a->ld_in, a->w, a->b, a->add, a->ld_add, static_cast<float*>(a->out), a->ld_out, a->R, a->N, a->K, a->act, a->out_scale);
    default: return timestep_embed_launch(st, x, static_cast<float*>(a->out), a->M);
  }
}

}  // extern "C"

namespace {
int test_cond_check(const ezb_test_cond_args* a) {
  const int kind = a->kind;
  if (kind < 0 || kind > 6) return fail(EZB_ERR_ARG, "ezb_test_cond: kind %d", kind);
  if (!a->in || (!a->out && !(kind == 1 && a->out32))) return fail(EZB_ERR_ARG, "ezb_test_cond: null input or output");
  if ((kind == 1 || kind == 4 || kind == 5) && a->kmul != 1 && a->kmul != 3)
    return fail(EZB_ERR_ARG, "ezb_test_cond: kmul %d (1 or 3)", a->kmul);
  if (kind <= 1) {
    if (a->M < 1 || a->M > (1 << 24) || a->D < 4 || a->D % 4 || (long long)a->M * a->D > (1LL << 30))
      return fail(EZB_ERR_SHAPE, "ezb_test_cond: M %d D %d (D a multiple of 4)", a->M, a->D);
    if (!a->w) return fail(EZB_ERR_ARG, "ezb_test_cond: kind %d needs w", kind);
    if (kind == 0 && a->vocab < 1) return fail(EZB_ERR_SHAPE, "ezb_test_cond: vocabulary of %d", a->vocab);
    if (kind == 1 && !(a->eps >= 0.f)) return fail(EZB_ERR_ARG, "ezb_test_cond: eps %g", a->eps);
    // t5_embed / t5_rms read their rows and write the fp32 output as float4
    const void* ps[] = {a->in, a->w, kind == 0 ? a->out : nullptr, a->out32};
    for (const void* p : ps)
      if (reinterpret_cast<uintptr_t>(p) & 15) return fail(EZB_ERR_ARG, "ezb_test_cond: kind %d pointers must be 16-byte aligned", kind);
    return EZB_OK;
  }
  if (kind == 2 || kind == 3 || kind == 5) {
    const bool per_head = kind != 3;   // t5_bias has no batch and no head dimension
    if (a->L < 1 || a->H < 1 || (long long)a->H * a->L * a->L > (1LL << 28) ||
        (per_head && (a->B < 1 || a->dk < 1 || (long long)a->B * a->L * a->H * a->dk > (1LL << 28) || (long long)a->B * a->H > 65535)))
      return fail(EZB_ERR_SHAPE, "ezb_test_cond: B %d L %d H %d dk %d", a->B, a->L, a->H, a->dk);
    if (kind == 2 && (!a->out32 || !a->out_v)) return fail(EZB_ERR_ARG, "ezb_test_cond: t5_heads writes q (out), k (out32) and v (out_v)");
    if (kind == 3 && !a->w) return fail(EZB_ERR_ARG, "ezb_test_cond: t5_bias needs the bucket table w");
    if (kind == 5) {
      if (a->dk % 4 || a->dk > 96) return fail(EZB_ERR_UNSUPPORTED, "ezb_test_cond: T5 attention head dimension %d (a multiple of 4, at most 96)", a->dk);
      if (!a->k || !a->v || !a->b) return fail(EZB_ERR_ARG, "ezb_test_cond: T5 attention needs k, v and the position bias b");
      const void* ps[] = {a->in, a->k, a->v};
      for (const void* p : ps)
        if (reinterpret_cast<uintptr_t>(p) & 15) return fail(EZB_ERR_ARG, "ezb_test_cond: q, k and v must be 16-byte aligned");
    }
    return EZB_OK;
  }
  if (kind == 4) {
    if (a->M < 1 || a->F < 1 || (long long)a->M * a->F > (1LL << 30)) return fail(EZB_ERR_SHAPE, "ezb_test_cond: gated GELU M %d F %d", a->M, a->F);
    return EZB_OK;
  }
  if (a->stage < 0 || a->stage > 3) return fail(EZB_ERR_ARG, "ezb_test_cond: stem stage %d", a->stage);
  if (a->B < 1 || a->L < 1 || a->c0 < 1 || a->c1 < 1 || a->D < 1 || (long long)a->B * 2 * a->L * (a->c0 + 1 > a->c1 ? a->c0 + 1 : a->c1) > (1LL << 30) ||
      (long long)a->B * a->L * a->D > (1LL << 30))
    return fail(EZB_ERR_SHAPE, "ezb_test_cond: stem B %d L %d widths %d, %d, %d", a->B, a->L, a->c0, a->c1, a->D);
  if (!a->w || !a->b) return fail(EZB_ERR_ARG, "ezb_test_cond: the stem convolution needs w and b");
  return EZB_OK;
}
}  // namespace

extern "C" {

__attribute__((visibility("default"))) int ezb_test_cond(int device, const ezb_test_cond_args* a, void* stream) {
  if (!a) return fail(EZB_ERR_ARG, "ezb_test_cond: null arguments");
  EZB_TRY(test_cond_check(a));
  EZB_CUDA(cudaSetDevice(device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  __nv_bfloat16* o16 = static_cast<__nv_bfloat16*>(a->out);
  float* o32 = static_cast<float*>(a->out);
  const float* x = static_cast<const float*>(a->in);
  switch (a->kind) {
    case 0: return t5_embed_launch(st, static_cast<const int32_t*>(a->in), a->w, o32, a->M, a->D, a->vocab);
    case 1: return t5_rms_launch(st, x, a->w, o16, a->out32, a->M, a->D, a->kmul, a->eps);
    case 2: return t5_heads_launch(st, x, o32, a->out32, a->out_v, a->B, a->L, a->H, a->dk);
    case 3: return t5_bias_launch(st, static_cast<const int32_t*>(a->in), a->w, o32, a->H, a->L);
    case 4: return t5_gated_gelu_launch(st, x, o16, a->M, a->F, a->kmul);
    case 5:
      EZB_CUDA(cudaFuncSetAttribute(attn_simt_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
      return t5_attention_launch(st, x, a->k, a->v, a->key_mask, a->b, o16, a->B, a->H, a->L, a->dk, a->kmul);
    default: return stem_conv_launch(st, stem_conv(a->stage, a->c0, a->c1, a->D, a->L), x, a->w, a->b, o32, a->B);
  }
}

#define EZB_API __attribute__((visibility("default")))
#define ST(s) reinterpret_cast<cudaStream_t>(s)

EZB_API int ezb_dit_create(ezb_dit** out, const ezb_dit_desc* desc, int device) {
  if (!out || !desc) return fail(EZB_ERR_ARG, "ezb_dit_create: null argument");
  EZB_CUDA(cudaSetDevice(device));
  Dit* h = new Dit();
  int rc = h->init(*desc, &device_ctx(device));
  if (rc != 0) { delete h; return rc; }
  *out = reinterpret_cast<ezb_dit*>(h);
  return EZB_OK;
}
EZB_API int ezb_dit_destroy(ezb_dit* h) {
  delete reinterpret_cast<Dit*>(h);
  return EZB_OK;
}
EZB_API int ezb_dit_load_weight(ezb_dit* h, const char* key, const float* data, const int64_t* shape, int ndim, void* stream) {
  if (!h || !key || !data || !shape) return fail(EZB_ERR_ARG, "ezb_dit_load_weight: null argument");
  return reinterpret_cast<Dit*>(h)->load_weight(key, data, shape, ndim, ST(stream));
}
EZB_API int ezb_dit_finalize_weights(ezb_dit* h, void* stream) {
  if (!h) return fail(EZB_ERR_ARG, "null handle");
  (void)stream;
  return reinterpret_cast<Dit*>(h)->finalize();
}
EZB_API int ezb_dit_set_context(ezb_dit* h, const float* ctx, const uint8_t* ctx_mask, int Be, int Lc, void* stream) {
  if (!h || !ctx || !ctx_mask) return fail(EZB_ERR_ARG, "ezb_dit_set_context: null argument");
  return reinterpret_cast<Dit*>(h)->set_context(ctx, ctx_mask, Be, Lc, ST(stream));
}
EZB_API int ezb_dit_set_timesteps(ezb_dit* h, const int64_t* ts, int n, void* stream) {
  if (!h || !ts) return fail(EZB_ERR_ARG, "ezb_dit_set_timesteps: null argument");
  return reinterpret_cast<Dit*>(h)->set_timesteps(ts, n, ST(stream));
}
EZB_API int ezb_dit_forward(ezb_dit* h, const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall,
                            const float* const* cskips, float* out, int Be, int L, void* stream, const int32_t* lens) {
  if (!h || !x || !out) return fail(EZB_ERR_ARG, "ezb_dit_forward: null argument");
  return reinterpret_cast<Dit*>(h)->forward(x, gt, gt_mask, tidx, tall, cskips, out, Be, L, lens, ST(stream));
}
EZB_API int ezb_controlnet_forward(ezb_dit* h, const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall,
                                   const float* condition, float scale, float* const* skips_out, int Be, int L, void* stream) {
  if (!h || !x || !condition || !skips_out) return fail(EZB_ERR_ARG, "ezb_controlnet_forward: null argument");
  return reinterpret_cast<Dit*>(h)->controlnet_forward(x, gt, gt_mask, tidx, tall, condition, scale, skips_out, Be, L, ST(stream));
}
EZB_API int ezb_cfg_ddim_step(int device, const float* model_out, float* latents, const float* noise, int B, int C, int L, float gs, float gr,
                              const float* coef, void* stream, const int32_t* lens) {
  if (!model_out || !latents || !coef || B < 1 || C < 1 || L < 1) return fail(EZB_ERR_ARG, "ezb_cfg_ddim_step: bad argument");
  if (coef[4] != 0.f && !noise) return fail(EZB_ERR_ARG, "ezb_cfg_ddim_step: sigma != 0 needs a noise tensor");
  EZB_CUDA(cudaSetDevice(device));
  const float* uncond = gs != 0.f ? model_out + (size_t)B * C * L : nullptr;
  return launch_k(cfg_ddim_kernel, dim3(B * CFG_CLUSTER), dim3(1024), 0, ST(stream), CFG_CLUSTER, model_out, uncond, latents,
                  coef[4] != 0.f ? noise : (const float*)nullptr, lens, C, L, gs, gr, coef[0], coef[1], coef[2], coef[3], coef[4]);
}
EZB_API int ezb_dit_set_context_rows(ezb_dit* h, const float* ctx, const uint8_t* ctx_mask, int row0, int n, int Lc, void* stream) {
  if (!h || !ctx || !ctx_mask) return fail(EZB_ERR_ARG, "ezb_dit_set_context_rows: null argument");
  return reinterpret_cast<Dit*>(h)->set_context_rows(ctx, ctx_mask, row0, n, Lc, ST(stream));
}
EZB_API int ezb_dit_forward_tdev(ezb_dit* h, const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* t_index_dev,
                                 const float* const* cskips, float* out, int Be, int L, void* stream, const int32_t* lens) {
  if (!h || !x || !out || !t_index_dev) return fail(EZB_ERR_ARG, "ezb_dit_forward_tdev: null argument");
  return reinterpret_cast<Dit*>(h)->forward(x, gt, gt_mask, nullptr, 0, cskips, out, Be, L, lens, ST(stream), t_index_dev);
}
EZB_API int ezb_controlnet_set_condition(ezb_dit* h, const float* condition, int Be, int L, void* stream) {
  if (!h || !condition) return fail(EZB_ERR_ARG, "ezb_controlnet_set_condition: null argument");
  return reinterpret_cast<Dit*>(h)->set_condition(condition, Be, L, ST(stream));
}
EZB_API int ezb_controlnet_set_condition_rows(ezb_dit* h, const float* condition, int row0, int n, int L, void* stream) {
  if (!h || !condition) return fail(EZB_ERR_ARG, "ezb_controlnet_set_condition_rows: null argument");
  return reinterpret_cast<Dit*>(h)->set_condition_rows(condition, row0, n, L, ST(stream));
}
EZB_API int ezb_controlnet_forward_tdev(ezb_dit* h, const float* x, const int32_t* t_index_dev, const float* scale_dev, float* const* skips_out, int Be,
                                        int L, void* stream) {
  if (!h || !x || !t_index_dev || !scale_dev || !skips_out) return fail(EZB_ERR_ARG, "ezb_controlnet_forward_tdev: null argument");
  return reinterpret_cast<Dit*>(h)->controlnet_forward_tdev(x, t_index_dev, scale_dev, skips_out, Be, L, ST(stream));
}
EZB_API int ezb_controlnet_forward_cached(ezb_dit* h, const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* tidx, int tall,
                                          float scale, float* const* skips_out, int Be, int L, void* stream) {
  if (!h || !x || !skips_out) return fail(EZB_ERR_ARG, "ezb_controlnet_forward_cached: null argument");
  return reinterpret_cast<Dit*>(h)->controlnet_forward_cached(x, gt, gt_mask, tidx, tall, scale, skips_out, Be, L, ST(stream));
}
EZB_API int ezb_cfg_ddim_step_slots(int device, const float* model_out, float* latents, const float* noise, const ezb_ddim_slot* slots, int B, int C,
                                    int L, void* stream, const int32_t* lens) {
  if (!model_out || !latents || !slots || B < 1 || C < 1 || L < 1) return fail(EZB_ERR_ARG, "ezb_cfg_ddim_step_slots: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  return launch_k(cfg_ddim_slots_kernel, dim3(B * CFG_CLUSTER), dim3(1024), 0, ST(stream), CFG_CLUSTER, model_out, model_out + (size_t)B * C * L,
                  latents, noise, lens, slots, C, L);
}
EZB_API int ezb_cfg_dpm_step(int device, const float* model_out, float* latents, float* history, const float* noise, int B, int C, int L, float gs,
                             float gr, const float* coef, int order, void* stream, const int32_t* lens) {
  if (!model_out || !latents || !history || !coef || B < 1 || C < 1 || L < 1 || (order != 1 && order != 2))
    return fail(EZB_ERR_ARG, "ezb_cfg_dpm_step: bad argument");
  if (coef[6] != 0.f && !noise) return fail(EZB_ERR_ARG, "ezb_cfg_dpm_step: kz != 0 needs a noise tensor");
  EZB_CUDA(cudaSetDevice(device));
  ezb_dpm_slot s;
  s.guidance_scale = gs;
  s.guidance_rescale = gr;
  for (int i = 0; i < 7; ++i) s.coef[i] = coef[i];
  s.flags = EZB_SLOT_ACTIVE | (gs != 0.f ? EZB_SLOT_CFG : 0) | (order == 2 ? EZB_SLOT_ORDER2 : 0);
  const float* uncond = gs != 0.f ? model_out + (size_t)B * C * L : nullptr;
  return launch_k(cfg_dpm_kernel, dim3(B * CFG_CLUSTER), dim3(1024), 0, ST(stream), CFG_CLUSTER, model_out, uncond, latents, history,
                  coef[6] != 0.f ? noise : (const float*)nullptr, lens, C, L, s);
}
EZB_API int ezb_cfg_dpm_step_slots(int device, const float* model_out, float* latents, float* history, const float* noise, const ezb_dpm_slot* slots,
                                   int B, int C, int L, void* stream, const int32_t* lens) {
  if (!model_out || !latents || !history || !slots || B < 1 || C < 1 || L < 1) return fail(EZB_ERR_ARG, "ezb_cfg_dpm_step_slots: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  return launch_k(cfg_dpm_slots_kernel, dim3(B * CFG_CLUSTER), dim3(1024), 0, ST(stream), CFG_CLUSTER, model_out, model_out + (size_t)B * C * L,
                  latents, history, noise, lens, slots, C, L);
}
EZB_API int ezb_window_gather(int device, const float* latents, float* windows, const int32_t* plan_dev, int B, int C, int Nmax, int W, int Lw,
                              int overlap, int copies, void* stream) {
  if (!latents || !windows || !plan_dev || B < 1 || C < 1 || Nmax < 1 || W < B || Lw < 2 || overlap < 1 || overlap > Lw / 2 ||
      (copies != 1 && copies != 2))
    return fail(EZB_ERR_ARG, "ezb_window_gather: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  EZB_CUDA(window_gather_launch(ST(stream), WindowPlan{plan_dev, B, C, Nmax, W, Lw, overlap}, latents, windows, copies));
  return EZB_OK;
}
EZB_API int ezb_window_blend(int device, const float* windows, float* out, const int32_t* plan_dev, int B, int C, int Nmax, int W, int Lw, int overlap,
                             void* stream) {
  if (!windows || !out || !plan_dev || B < 1 || C < 1 || Nmax < 1 || W < B || Lw < 2 || overlap < 1 || overlap > Lw / 2)
    return fail(EZB_ERR_ARG, "ezb_window_blend: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  EZB_CUDA(window_blend_launch(ST(stream), WindowPlan{plan_dev, B, C, Nmax, W, Lw, overlap}, windows, out));
  return EZB_OK;
}
EZB_API int ezb_vae_create(ezb_vae** out, const ezb_vae_desc* desc, int device) {
  if (!out || !desc) return fail(EZB_ERR_ARG, "ezb_vae_create: null argument");
  EZB_CUDA(cudaSetDevice(device));
  Vae* h = new Vae();
  int rc = h->init(*desc, &device_ctx(device));
  if (rc != 0) { delete h; return rc; }
  *out = reinterpret_cast<ezb_vae*>(h);
  return EZB_OK;
}
EZB_API int ezb_vae_destroy(ezb_vae* h) {
  delete reinterpret_cast<Vae*>(h);
  return EZB_OK;
}
EZB_API int ezb_vae_load_weight(ezb_vae* h, const char* key, const float* data, const int64_t* shape, int ndim, void* stream) {
  if (!h || !key || !data || !shape) return fail(EZB_ERR_ARG, "ezb_vae_load_weight: null argument");
  return reinterpret_cast<Vae*>(h)->load_weight(key, data, shape, ndim, ST(stream));
}
EZB_API int ezb_vae_finalize_weights(ezb_vae* h, void* stream) {
  if (!h) return fail(EZB_ERR_ARG, "null handle");
  return reinterpret_cast<Vae*>(h)->finalize(ST(stream));
}
EZB_API int ezb_vae_encode(ezb_vae* h, const float* audio, const float* noise, float* z, int B, int T, void* stream) {
  if (!h || !audio || !z) return fail(EZB_ERR_ARG, "ezb_vae_encode: null argument");
  return reinterpret_cast<Vae*>(h)->encode(audio, noise, z, B, T, ST(stream));
}
EZB_API int ezb_t5_create(ezb_t5** out, const ezb_t5_desc* desc, int device) {
  if (!out || !desc) return fail(EZB_ERR_ARG, "ezb_t5_create: null argument");
  EZB_CUDA(cudaSetDevice(device));
  T5* h = new T5();
  int rc = h->init(*desc, &device_ctx(device));
  if (rc != 0) { delete h; return rc; }
  *out = reinterpret_cast<ezb_t5*>(h);
  return EZB_OK;
}
EZB_API int ezb_t5_destroy(ezb_t5* h) {
  delete reinterpret_cast<T5*>(h);
  return EZB_OK;
}
EZB_API int ezb_t5_load_weight(ezb_t5* h, const char* key, const float* data, const int64_t* shape, int ndim, void* stream) {
  if (!h || !key || !data || !shape) return fail(EZB_ERR_ARG, "ezb_t5_load_weight: null argument");
  return reinterpret_cast<T5*>(h)->load_weight(key, data, shape, ndim, ST(stream));
}
EZB_API int ezb_t5_finalize_weights(ezb_t5* h, void* stream) {
  if (!h) return fail(EZB_ERR_ARG, "null handle");
  (void)stream;
  return reinterpret_cast<T5*>(h)->finalize();
}
EZB_API int ezb_t5_forward(ezb_t5* h, const int32_t* ids, const uint8_t* mask, const int32_t* buckets, float* out, int B, int L, void* stream) {
  if (!h || !ids || !mask || !out) return fail(EZB_ERR_ARG, "ezb_t5_forward: null argument");
  return reinterpret_cast<T5*>(h)->forward(ids, mask, buckets, out, B, L, ST(stream));
}
EZB_API int ezb_energy_condition(int device, const float* audio, float* out, int B, int T, int hop, int win, float min_db, int norm, int qlevels,
                                 void* stream) {
  if (!audio || !out) return fail(EZB_ERR_ARG, "ezb_energy_condition: null pointer");
  if (B < 1 || hop < 1 || win < hop || T < hop) return fail(EZB_ERR_SHAPE, "ezb_energy_condition: B=%d T=%d hop=%d window=%d", B, T, hop, win);
  // an odd window - hop: the reference pads (win - hop - 1) / 2 samples per side and returns (T - 1) / hop frames, not the T / hop computed here
  if ((win - hop) % 2) return fail(EZB_ERR_UNSUPPORTED, "ezb_energy_condition: window %d - hop %d is odd", win, hop);
  const int pad = (win - hop) / 2, n_frames = T / hop;
  if (pad >= T) return fail(EZB_ERR_SHAPE, "ezb_energy_condition: reflect padding %d needs more than %d samples", pad, T);
  if ((size_t)n_frames * sizeof(float) > 200 * 1024) return fail(EZB_ERR_SHAPE, "ezb_energy_condition: %d frames exceed the shared-memory table", n_frames);
  EZB_CUDA(cudaSetDevice(device));
  EZB_CUDA(cudaFuncSetAttribute(energy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  ++launch_counter();
  energy_kernel<<<B, 1024, n_frames * sizeof(float), ST(stream)>>>(audio, out, T, n_frames, hop, win, min_db, powf(10.f, min_db / 10.f), norm, qlevels);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
EZB_API int ezb_wave_prepare(int device, const float* in, float* out, int B, int T_in, int T_out, int normalize, float gate, void* stream) {
  if (!in || !out || B < 1 || T_in < 1 || T_out < 1) return fail(EZB_ERR_ARG, "ezb_wave_prepare: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  wave_prepare_kernel<<<B, 1024, 0, ST(stream)>>>(in, out, T_in, T_out, 1e-9f, gate, normalize);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
EZB_API int ezb_wave_splice(int device, float* dst, long long dst_len, const float* src, long long start, long long n, void* stream) {
  if (!dst || !src) return fail(EZB_ERR_ARG, "ezb_wave_splice: null pointer");
  if (start < 0 || n < 0 || start + n > dst_len) return fail(EZB_ERR_SHAPE, "ezb_wave_splice: [%lld, %lld) outside a clip of %lld samples", start, start + n, dst_len);
  if (n == 0) return EZB_OK;
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  wave_splice_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(dst, src, start, n);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
EZB_API int ezb_wave_to_pcm16(int device, const float* in, int16_t* out, long long n, void* stream) {
  if (!in || !out || n < 0) return fail(EZB_ERR_ARG, "ezb_wave_to_pcm16: bad argument");
  if (n == 0) return EZB_OK;
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  wave_to_pcm16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(in, out, n);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
EZB_API int ezb_vae_decode(ezb_vae* h, const float* z, float* wav, int B, int L, void* stream) {
  if (!h || !z || !wav) return fail(EZB_ERR_ARG, "ezb_vae_decode: null argument");
  return reinterpret_cast<Vae*>(h)->decode(z, wav, B, L, ST(stream));
}
EZB_API int ezb_vae_decode_lens(ezb_vae* h, const float* z, float* wav, int B, int L, const int32_t* lens, void* stream) {
  if (!h || !z || !wav || !lens) return fail(EZB_ERR_ARG, "ezb_vae_decode_lens: null argument");
  return reinterpret_cast<Vae*>(h)->decode(z, wav, B, L, ST(stream), lens);
}
EZB_API int ezb_vae_encode_lens(ezb_vae* h, const float* audio, const float* noise, float* z, int B, int T, const int32_t* lens, void* stream) {
  if (!h || !audio || !z || !lens) return fail(EZB_ERR_ARG, "ezb_vae_encode_lens: null argument");
  return reinterpret_cast<Vae*>(h)->encode(audio, noise, z, B, T, ST(stream), lens);
}
EZB_API int ezb_vae_encode_noised(ezb_vae* h, const float* audio, const float* vae_noise, const float* eps, const float* ab_dev, float scale,
                                  float shift, float* x_t, int B, int T, const int32_t* lens, void* stream) {
  if (!h || !audio || !eps || !ab_dev || !x_t) return fail(EZB_ERR_ARG, "ezb_vae_encode_noised: null argument");
  const VaeNoised nd{eps, ab_dev, scale, shift};
  return reinterpret_cast<Vae*>(h)->encode(audio, vae_noise, x_t, B, T, ST(stream), lens, &nd);
}
}  // extern "C"

namespace {
// impl 0 / 3: fp32 CUDA-core kernel (q,k,v fp32 [B,H,L,dh]; 3 writes bf16x3 rows); impl 1/4/6/7/8 (+100): tensor-core kernel (q,k bf16
// [B*H,L,DHP], vt bf16 [B*H,DVP,Lkpad]).  Every argument is checked before any device work.
int test_attention(int device, const void* q, const void* k, const void* v, const uint8_t* key_mask, const int32_t* lens, void* out, int B, int H,
                   int Lq, int Lk, int dh, int impl, void* stream) {
  if (!q || !k || !v || !out) return fail(EZB_ERR_ARG, "ezb_test_attention: null pointer");
  const bool simt = impl == 0 || impl == 3;
  const int variant = impl % 100;
  if (!simt && (impl < 0 || impl >= 200 || (variant != 1 && variant != 4 && variant != 6 && variant != 7 && variant != 8)))
    return fail(EZB_ERR_ARG, "ezb_test_attention: impl %d", impl);
  if (simt && (dh < 4 || dh % 4 || dh > 96)) return fail(EZB_ERR_UNSUPPORTED, "fp32 attention: head dimension %d (multiples of 4 up to 96)", dh);
  if (!simt && (dh < 8 || dh % 8 || dh > 80)) return fail(EZB_ERR_UNSUPPORTED, "attention: head dimension %d (multiples of 8 up to 80)", dh);
  if (variant == 8 && dh != 64 && dh != 72) return fail(EZB_ERR_UNSUPPORTED, "attention generation 8: head dimension %d (64 or 72)", dh);
  if (B < 1 || H < 1 || Lq < 1 || Lk < 1 || (long long)B * H > 65535)
    return fail(EZB_ERR_SHAPE, "ezb_test_attention: B %d H %d Lq %d Lk %d", B, H, Lq, Lk);
  const float scale = 1.0f / sqrtf((float)dh);
  if (simt) {
    EZB_CUDA(cudaSetDevice(device));
    auto kern = lens ? attn_simt_kernel<true> : attn_simt_kernel<false>;
    EZB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    dim3 grid((Lq + SA_WARPS * SA_QW - 1) / (SA_WARPS * SA_QW), B * H);
    ++launch_counter();
    kern<<<grid, SA_WARPS * 32, attn_simt_smem(dh), ST(stream)>>>(reinterpret_cast<const float*>(q), reinterpret_cast<const float*>(k),
                                                                            reinterpret_cast<const float*>(v), key_mask,
                                                                            reinterpret_cast<__nv_bfloat16*>(out), H, Lq, Lk, dh, scale,
                                                                            impl == 3 ? 3 : 1, lens, nullptr);
    EZB_CUDA(cudaGetLastError());
    return EZB_OK;
  }
  // impl 1: the variant the options select; 4 / 6 / 7 / 8: that generation forced; +100: q / k rows of 80 elements for dh = 72 (the product's
  // layout) instead of a 64-multiple
  const int row80 = impl >= 100;
  EZB_CUDA(cudaSetDevice(device));
  const int dhp = (row80 && dh == 72) ? 80 : (dh + 63) / 64 * 64;
  const int dvp = (dh + 15) / 16 * 16, lkpad = (Lk + 7) / 8 * 8;
  device_ctx(device).tmaps.trim();
  return attention_mma(device_ctx(device), ST(stream), reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k),
                       reinterpret_cast<const __nv_bfloat16*>(v), key_mask, reinterpret_cast<__nv_bfloat16*>(out), B, H, Lq, Lk, lkpad, dh, dhp, dvp, scale, variant == 1 ? 0 : variant,
                       lens);
}
}  // namespace

extern "C" {
EZB_API int ezb_test_attention(int device, const void* q, const void* k, const void* v, const uint8_t* key_mask, void* out, int B, int H, int Lq,
                               int Lk, int dh, int impl, void* stream) {
  return test_attention(device, q, k, v, key_mask, nullptr, out, B, H, Lq, Lk, dh, impl, stream);
}
EZB_API int ezb_test_attention_lens(int device, const void* q, const void* k, const void* v, const int32_t* lens, void* out, int B, int H, int L, int dh,
                                    int impl, void* stream) {
  if (!lens) return fail(EZB_ERR_ARG, "ezb_test_attention_lens: null lengths");
  return test_attention(device, q, k, v, nullptr, lens, out, B, H, L, L, dh, impl, stream);
}


// runtime switches (A/B testing): "pair_gemm" 0/1 -- read when a handle is created
EZB_API unsigned long long ezb_option_epoch(void) { return option_epoch(); }
EZB_API int ezb_set_option(const char* name, int value) {
  ++option_epoch();   // captured CUDA graphs bake the kernel selection in: the host layer keys its graph cache on this counter
  if (name && !strcmp(name, "pair_gemm")) { opt_pair_gemm() = value; return EZB_OK; }
  if (name && !strcmp(name, "pdl")) { opt_pdl() = value; return EZB_OK; }
  if (name && !strcmp(name, "swap_ab")) { opt_swap_ab() = value; return EZB_OK; }
  if (name && !strcmp(name, "qkv3")) { opt_qkv3() = value; return EZB_OK; }
  if (name && !strcmp(name, "ln_tail")) { opt_ln_tail() = value; return EZB_OK; }
  if (name && !strcmp(name, "heads_dbg")) { opt_heads_dbg() = value; return EZB_OK; }
  if (name && !strcmp(name, "mlp2_pair")) { opt_mlp2_pair() = value; return EZB_OK; }
  if (name && !strcmp(name, "cq_single")) { opt_cq_single() = value; return EZB_OK; }
  if (name && !strcmp(name, "attn6")) { opt_attn6() = value; return EZB_OK; }
  if (name && !strcmp(name, "attn7")) { opt_attn7() = value; return EZB_OK; }
  if (name && !strcmp(name, "attn8")) { opt_attn8() = value; return EZB_OK; }
  if (name && !strcmp(name, "attn_res")) { opt_attn_res() = value; return EZB_OK; }
  if (name && !strcmp(name, "attn_pp")) { opt_attn_pp() = value; return EZB_OK; }
  if (name && !strcmp(name, "gemm_debug")) {  // cycle counters of CTA 0 of every 2-CTA cluster GEMM launch (accumulated; needs -DEZB_GEMM_DEBUG)
    if (value && !gemm_dbg_buf()) { EZB_CUDA(cudaMalloc(&gemm_dbg_buf(), 64)); EZB_CUDA(cudaMemset(gemm_dbg_buf(), 0, 64)); }
    if (!value && gemm_dbg_buf()) { cudaFree(gemm_dbg_buf()); gemm_dbg_buf() = nullptr; }
    return EZB_OK;
  }
  if (name && !strcmp(name, "attn_poly")) { opt_attn_poly() = value; return EZB_OK; }
  if (name && !strcmp(name, "attn_dbg")) { opt_attn_dbg() = value; return EZB_OK; }
  if (name && !strcmp(name, "w_prefetch")) { opt_w_prefetch() = value; return EZB_OK; }
  if (name && !strcmp(name, "ln_variant")) { opt_ln_variant() = value; return EZB_OK; }
  if (name && !strcmp(name, "mlp_fused")) { opt_mlp_fused() = value; return EZB_OK; }
  if (name && !strcmp(name, "dhp80")) { opt_dhp80() = value; return EZB_OK; }
  if (name && !strcmp(name, "ln_fold")) { opt_fold() = value; return EZB_OK; }
  if (name && !strcmp(name, "skip")) { opt_skip() = value; return EZB_OK; }
  if (name && !strcmp(name, "swap_mc")) { opt_swap_mc() = value; return EZB_OK; }
  if (name && !strcmp(name, "rope_mufu")) { opt_rope_mufu() = value; return EZB_OK; }
  return fail(EZB_ERR_ARG, "unknown option");
}
EZB_API int ezb_debug_read(unsigned long long* out8) {
  if (!gemm_dbg_buf() || !out8) return fail(EZB_ERR_STATE, "gemm_debug is off");
  EZB_CUDA(cudaDeviceSynchronize());
  EZB_CUDA(cudaMemcpy(out8, gemm_dbg_buf(), 64, cudaMemcpyDeviceToHost));
  EZB_CUDA(cudaMemset(gemm_dbg_buf(), 0, 64));
  return EZB_OK;
}
// ---- accounting / profiling hooks (bench.py)
EZB_API unsigned long long ezb_launch_count(void) { return launch_counter(); }
// kernels replayed through a captured CUDA graph never pass the launch helpers: the host layer reports them here
EZB_API void ezb_launch_count_add(unsigned long long n) { launch_counter() += n; }
EZB_API unsigned long long ezb_attn_launch_count(int generation) { return generation >= 0 && generation <= 8 ? attn_launch_counts()[generation] : 0; }
EZB_API unsigned long long ezb_ln_launch_count(int variant) { return variant >= LN_GENERIC && variant <= LN_CAT ? ln_launch_counts()[variant] : 0; }
EZB_API int ezb_prof_gemm_begin(void) {
  GemmProf& gp = gemm_prof();
  gp.on = true; gp.used = 0; gp.flops.clear();
  return EZB_OK;
}
// Synchronises the device; returns the number of GEMM launches recorded since begin, their total algorithmic FLOPs and the
// sum of their CUDA-event durations (ms).
EZB_API int ezb_prof_gemm_end(int* launches, double* flops, double* ms) {
  GemmProf& gp = gemm_prof();
  gp.on = false;
  EZB_CUDA(cudaDeviceSynchronize());
  double f = 0, t = 0;
  for (size_t i = 0; i < gp.flops.size(); ++i) {
    float m = 0.f;
    EZB_CUDA(cudaEventElapsedTime(&m, gp.ev[2 * i], gp.ev[2 * i + 1]));
    f += gp.flops[i]; t += m;
  }
  if (launches) *launches = (int)gp.flops.size();
  if (flops) *flops = f;
  if (ms) *ms = t;
  return EZB_OK;
}

// After ezb_prof_gemm_end: the same statistics restricted to launches with at least `min_flops` algorithmic FLOPs (the dominant
// GEMM of the step is the GEGLU MLP-in projection, the largest single launch).
EZB_API int ezb_prof_gemm_stats(double min_flops, int* launches, double* flops, double* ms) {
  GemmProf& gp = gemm_prof();
  double f = 0, t = 0;
  int n = 0;
  for (size_t i = 0; i < gp.flops.size(); ++i) {
    if (gp.flops[i] < min_flops) continue;
    float m = 0.f;
    EZB_CUDA(cudaEventElapsedTime(&m, gp.ev[2 * i], gp.ev[2 * i + 1]));
    f += gp.flops[i]; t += m; ++n;
  }
  if (launches) *launches = n;
  if (flops) *flops = f;
  if (ms) *ms = t;
  return EZB_OK;
}

EZB_API int ezb_loop_gather(int device, const float* latents, float* windows, const int32_t* plan_dev, const int32_t* offsets_dev, int B, int C,
                            int Nmax, int W, int Lw, int overlap, int copies, void* stream) {
  if (!latents || !windows || !plan_dev || !offsets_dev || B < 1 || C < 1 || Nmax < 1 || W < B || Lw < 2 || overlap < 1 || overlap > Lw / 2 ||
      (copies != 1 && copies != 2))
    return fail(EZB_ERR_ARG, "ezb_loop_gather: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  EZB_CUDA(loop_gather_launch(ST(stream), LoopPlan{plan_dev, offsets_dev, B, C, Nmax, W, Lw, overlap}, latents, windows, copies));
  return EZB_OK;
}
EZB_API int ezb_loop_blend(int device, const float* windows, float* out, const int32_t* plan_dev, const int32_t* offsets_dev, int B, int C, int Nmax,
                           int W, int Lw, int overlap, void* stream) {
  if (!windows || !out || !plan_dev || !offsets_dev || B < 1 || C < 1 || Nmax < 1 || W < B || Lw < 2 || overlap < 1 || overlap > Lw / 2)
    return fail(EZB_ERR_ARG, "ezb_loop_blend: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  EZB_CUDA(loop_blend_launch(ST(stream), LoopPlan{plan_dev, offsets_dev, B, C, Nmax, W, Lw, overlap}, windows, out));
  return EZB_OK;
}

EZB_API int ezb_timeline_gather(int device, const float* latents, float* windows, const int32_t* plan_dev, const int32_t* rows_dev, int B, int C,
                                int Nmax, int W, int R, int Lw, int overlap, int uncond, void* stream) {
  if (!latents || !windows || !plan_dev || !rows_dev || !aligned16(rows_dev) || B < 1 || C < 1 || Nmax < 1 || W < B || R < W || Lw < 2 ||
      overlap < 1 || overlap > Lw / 2 || (uncond != 0 && uncond != 1))
    return fail(EZB_ERR_ARG, "ezb_timeline_gather: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  EZB_CUDA(timeline_gather_launch(ST(stream), TimelinePlan{WindowPlan{plan_dev, B, C, Nmax, W, Lw, overlap}, rows_dev, nullptr, R}, latents, windows,
                                  uncond));
  return EZB_OK;
}
EZB_API int ezb_timeline_guide(int device, const float* model_out, float* guided, const int32_t* rows_dev, const int32_t* lens_dev, int R, int W, int C,
                               int Lw, float gs, float gr, void* stream) {
  if (!model_out || !guided || !rows_dev || !lens_dev || !aligned16(rows_dev) || W < 1 || R < W || C < 1 || Lw < 1)
    return fail(EZB_ERR_ARG, "ezb_timeline_guide: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  EZB_CUDA(timeline_guide_launch(ST(stream), model_out, guided, rows_dev, lens_dev, R, W, C, Lw, gs, gr));
  return EZB_OK;
}
EZB_API int ezb_timeline_blend(int device, const float* windows, float* out, const int32_t* plan_dev, const int32_t* rows_dev, const int32_t* spans_dev,
                               int B, int C, int Nmax, int W, int R, int Lw, int overlap, void* stream) {
  if (!windows || !out || !plan_dev || !rows_dev || !spans_dev || !aligned16(rows_dev) || B < 1 || C < 1 || Nmax < 1 || W < B || R < W ||
      Lw < 2 || overlap < 1 || overlap > Lw / 2)
    return fail(EZB_ERR_ARG, "ezb_timeline_blend: bad argument");
  EZB_CUDA(cudaSetDevice(device));
  ++launch_counter();
  EZB_CUDA(timeline_blend_launch(ST(stream), TimelinePlan{WindowPlan{plan_dev, B, C, Nmax, W, Lw, overlap}, rows_dev, spans_dev, R}, windows, out));
  return EZB_OK;
}

}  // extern "C"
