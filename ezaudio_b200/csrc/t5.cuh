// T5 (v1.1 / flan-T5, gated-GELU) text encoder: the step BEFORE the denoiser path (SURVEY 8(f) row 3).
// Reference call site: src/inference.py:38-50 (`text_encoder(input_ids=, attention_mask=).last_hidden_state`), model class
// transformers.T5EncoderModel (api/ezaudio.py:78-79).  Runs once per generate call on <= 100 tokens per prompt, so it is weight-bandwidth
// bound (2.4 GB of bf16 weights for flan-T5-XL); the linears reuse the wgmma 2-CTA cluster GEMM of the DiT, everything else is small fp32 kernels:
//   ids -> embedding gather -> 24 x [ RMSNorm+cast -> QKV GEMM -> head permute -> fp32 attention (unscaled, + relative-position bias,
//   + key mask) -> O GEMM (+ residual) -> RMSNorm+cast -> [wi_1 | wi_0] GEMM -> gelu_new(g) * h -> wo GEMM (+ residual) ] -> RMSNorm.
#pragma once
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "attention_simt.cuh"
#include "host.cuh"

namespace ezb {

// x fp32 [M, D] <- table[ids[m]]
__global__ void t5_embed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ table, float* __restrict__ x, int M, int D, int vocab) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * (D / 4)) return;
  const int m = i / (D / 4), c = i - (size_t)m * (D / 4);
  int id = ids[m];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  reinterpret_cast<float4*>(x)[i] = reinterpret_cast<const float4*>(table + (size_t)id * D)[c];
}
// T5LayerNorm: y = w * x * rsqrt(mean(x^2) + eps); bf16 A operand [M, kmul*D] and / or fp32 out.  One warp per row.
__global__ void __launch_bounds__(256) t5_rms_kernel(const float* __restrict__ x, const float* __restrict__ w, __nv_bfloat16* __restrict__ out16,
                                                     float* __restrict__ out32, int M, int D, int kmul, float eps) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (size_t)row * D;
  float q = 0.f;
  for (int c = lane * 4; c < D; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + c);
    q += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  const float r = rsqrtf(warp_sum(q) / D + eps);
  for (int c = lane * 4; c < D; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + c), g = *reinterpret_cast<const float4*>(w + c);
    const float y[4] = {g.x * (v.x * r), g.y * (v.y * r), g.z * (v.z * r), g.w * (v.w * r)};
    if (out32) *reinterpret_cast<float4*>(out32 + (size_t)row * D + c) = make_float4(y[0], y[1], y[2], y[3]);
    if (out16) {
#pragma unroll
      for (int e = 0; e < 4; ++e) store_act(out16 + (size_t)row * kmul * D, c + e, D, kmul, y[e]);
    }
  }
}
// qkv fp32 [B*L, 3*inner] -> q, k, v fp32 [B, H, L, dk]
__global__ void t5_heads_kernel(const float* __restrict__ qkv, float* __restrict__ q, float* __restrict__ k, float* __restrict__ v, int B, int L, int H, int dk) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int inner = H * dk;
  if (i >= (size_t)B * L * 3 * inner) return;
  const int c = i % (3 * inner);
  const size_t m = i / (3 * inner);
  const int b = m / L, l = m - (size_t)b * L;
  const int sec = c / inner, cc = c - sec * inner, h = cc / dk, d = cc - h * dk;
  float* dst = sec == 0 ? q : (sec == 1 ? k : v);
  dst[(((size_t)b * H + h) * L + l) * dk + d] = qkv[i];
}
// position bias [H, L, L] = relative_attention_bias[bucket[q, k], h]  (compute_bias of T5Attention; block 0's table serves every block)
__global__ void t5_bias_kernel(const int32_t* __restrict__ bucket, const float* __restrict__ table, float* __restrict__ bias, int H, int L) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)H * L * L) return;
  const int h = i / ((size_t)L * L);
  const size_t qk = i - (size_t)h * L * L;
  bias[i] = table[(size_t)bucket[qk] * H + h];
}
// gated GELU (T5DenseGatedActDense with NewGELUActivation): u fp32 [M, 2F] = [wi_1 x | wi_0 x] -> bf16 [M, kmul*F] = gelu_new(g) * h
__global__ void t5_gated_gelu_kernel(const float* __restrict__ u, __nv_bfloat16* __restrict__ out, int M, int F, int kmul) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * F) return;
  const int m = i / F, c = i - (size_t)m * F;
  const float h = u[(size_t)m * 2 * F + c], g = u[(size_t)m * 2 * F + F + c];
  const float t = tanhf(0.7978845608028654f * (g + 0.044715f * g * g * g));
  store_act(out + (size_t)m * kmul * F, c, F, kmul, 0.5f * g * (1.0f + t) * h);
}

// The launches of T5::forward (grids and shared memory), shared with the ezb_test_cond hook.
inline unsigned t5_grid(size_t n) { return (unsigned)((n + 255) / 256); }
inline int t5_embed_launch(cudaStream_t st, const int32_t* ids, const float* table, float* x, int M, int D, int vocab) {
  ++launch_counter();
  t5_embed_kernel<<<t5_grid((size_t)M * (D / 4)), 256, 0, st>>>(ids, table, x, M, D, vocab);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
inline int t5_rms_launch(cudaStream_t st, const float* x, const float* w, __nv_bfloat16* out16, float* out32, int M, int D, int kmul, float eps) {
  ++launch_counter();
  t5_rms_kernel<<<(M + 7) / 8, 256, 0, st>>>(x, w, out16, out32, M, D, kmul, eps);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
inline int t5_heads_launch(cudaStream_t st, const float* qkv, float* q, float* k, float* v, int B, int L, int H, int dk) {
  ++launch_counter();
  t5_heads_kernel<<<t5_grid((size_t)B * L * 3 * H * dk), 256, 0, st>>>(qkv, q, k, v, B, L, H, dk);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
inline int t5_bias_launch(cudaStream_t st, const int32_t* bucket, const float* table, float* bias, int H, int L) {
  ++launch_counter();
  t5_bias_kernel<<<t5_grid((size_t)H * L * L), 256, 0, st>>>(bucket, table, bias, H, L);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
inline int t5_gated_gelu_launch(cudaStream_t st, const float* u, __nv_bfloat16* out, int M, int F, int kmul) {
  ++launch_counter();
  t5_gated_gelu_kernel<<<t5_grid((size_t)M * F), 256, 0, st>>>(u, out, M, F, kmul);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}
// unscaled attention with the position bias [H, L, L] and the key mask [B, L]; the caller has raised the kernel's shared-memory limit to 100 KB
inline int t5_attention_launch(cudaStream_t st, const float* q, const float* k, const float* v, const uint8_t* mask, const float* bias, __nv_bfloat16* out,
                               int B, int H, int L, int dk, int kmul) {
  dim3 ga((L + SA_WARPS * SA_QW - 1) / (SA_WARPS * SA_QW), B * H);
  ++launch_counter();
  attn_simt_kernel<false><<<ga, SA_WARPS * 32, attn_simt_smem(dk), st>>>(q, k, v, mask, out, H, L, L, dk, 1.0f /* T5: no 1/sqrt(d) */, kmul, nullptr, bias);
  EZB_CUDA(cudaGetLastError());
  return EZB_OK;
}

struct T5 {
  ezb_t5_desc d;
  Device* dev = nullptr;
  int D, H, dk, inner, F, nl, kmul;
  std::vector<void*> allocs;
  struct Spec {
    std::vector<int64_t> shape;
    std::function<int(const float*, cudaStream_t)> load;
    bool loaded = false;
  };
  std::map<std::string, Spec> specs;
  struct Layer {
    __nv_bfloat16 *qkv = nullptr, *o = nullptr, *wi = nullptr, *wo = nullptr;
    float *ln0 = nullptr, *ln1 = nullptr;
  };
  std::vector<Layer> layers;
  float *emb = nullptr, *rel = nullptr, *lnf = nullptr;
  // workspace
  float *x = nullptr, *qkv32 = nullptr, *q32 = nullptr, *k32 = nullptr, *v32 = nullptr, *u32 = nullptr, *bias = nullptr;
  __nv_bfloat16 *act = nullptr, *attn = nullptr, *mid = nullptr;
  int32_t *ids_d = nullptr, *bucket_d = nullptr;
  int bucket_L = -1;                 // length the device bucket table currently holds
  std::vector<int32_t> bucket_h;     // its host staging copy
  bool finalized = false;

  ~T5() {
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
  int reg_f32(const std::string& key, std::vector<int64_t> shape, float** dst) {
    size_t n = 1;
    for (auto v : shape) n *= v;
    EZB_TRY(alloc(dst, n));
    float* p = *dst;
    Spec s;
    s.shape = shape;
    s.load = [p, n](const float* src, cudaStream_t st) -> int {
      EZB_CUDA(cudaMemcpyAsync(p, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
      return EZB_OK;
    };
    specs[key] = std::move(s);
    return EZB_OK;
  }
  // fp32 [N, K] (nn.Linear layout) -> rows [row_off, row_off + N) of the packed bf16 [Ntot, kmul*K] operand
  void reg_linear(const std::string& key, int N, int K, __nv_bfloat16* dst, int row_off) {
    const int km = kmul;
    Spec s;
    s.shape = {N, K};
    s.load = [=](const float* src, cudaStream_t st) -> int {
      const size_t n = (size_t)N * K;
      ++launch_counter();
      pack_weight_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, N, K, dst, K, km, row_off, 0, 1, 0, 0, 0);
      EZB_CUDA(cudaGetLastError());
      return EZB_OK;
    };
    specs[key] = std::move(s);
  }

  int init(const ezb_t5_desc& desc, Device* device) {
    d = desc;
    dev = device;
    D = d.d_model; H = d.num_heads; dk = d.d_kv; inner = H * dk; F = d.d_ff; nl = d.num_layers;
    kmul = d.precision == 1 ? 3 : 1;
    if (d.precision != 0 && d.precision != 1) return fail(EZB_ERR_UNSUPPORTED, "t5: precision %d", d.precision);
    if (D <= 0 || D % 8 || inner % 8 || F % 8 || dk <= 0 || dk > 96 || dk % 4 || nl <= 0 || d.vocab_size <= 0 || d.num_buckets <= 1 || d.max_batch <= 0 || d.max_len <= 0)
      return fail(EZB_ERR_UNSUPPORTED, "t5: d_model %d d_kv %d heads %d d_ff %d layers %d", D, dk, H, F, nl);
    EZB_TRY(reg_f32("shared.weight", {d.vocab_size, D}, &emb));
    EZB_TRY(reg_f32("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", {d.num_buckets, H}, &rel));
    EZB_TRY(reg_f32("encoder.final_layer_norm.weight", {D}, &lnf));
    layers.resize(nl);
    for (int i = 0; i < nl; ++i) {
      Layer& w = layers[i];
      const std::string a = "encoder.block." + std::to_string(i) + ".layer.0.", f = "encoder.block." + std::to_string(i) + ".layer.1.";
      EZB_TRY(alloc(&w.qkv, (size_t)3 * inner * kmul * D));
      EZB_TRY(alloc(&w.o, (size_t)D * kmul * inner));
      EZB_TRY(alloc(&w.wi, (size_t)2 * F * kmul * D));
      EZB_TRY(alloc(&w.wo, (size_t)D * kmul * F));
      reg_linear(a + "SelfAttention.q.weight", inner, D, w.qkv, 0);
      reg_linear(a + "SelfAttention.k.weight", inner, D, w.qkv, inner);
      reg_linear(a + "SelfAttention.v.weight", inner, D, w.qkv, 2 * inner);
      reg_linear(a + "SelfAttention.o.weight", D, inner, w.o, 0);
      reg_linear(f + "DenseReluDense.wi_1.weight", F, D, w.wi, 0);      // h (linear branch) first, g (gelu branch) second
      reg_linear(f + "DenseReluDense.wi_0.weight", F, D, w.wi, F);
      reg_linear(f + "DenseReluDense.wo.weight", D, F, w.wo, 0);
      EZB_TRY(reg_f32(a + "layer_norm.weight", {D}, &w.ln0));
      EZB_TRY(reg_f32(f + "layer_norm.weight", {D}, &w.ln1));
    }
    const size_t Mx = (size_t)d.max_batch * d.max_len;
    EZB_TRY(alloc(&x, Mx * D));
    EZB_TRY(alloc(&qkv32, Mx * 3 * inner));
    EZB_TRY(alloc(&q32, Mx * inner));
    EZB_TRY(alloc(&k32, Mx * inner));
    EZB_TRY(alloc(&v32, Mx * inner));
    EZB_TRY(alloc(&u32, Mx * 2 * F));
    EZB_TRY(alloc(&bias, (size_t)H * d.max_len * d.max_len));
    EZB_TRY(alloc(&act, Mx * kmul * D));
    EZB_TRY(alloc(&attn, Mx * kmul * inner));
    EZB_TRY(alloc(&mid, Mx * kmul * F));
    EZB_TRY(alloc(&ids_d, Mx));
    EZB_TRY(alloc(&bucket_d, (size_t)d.max_len * d.max_len));
    return EZB_OK;
  }
  int load_weight(const char* key, const float* data, const int64_t* shape, int ndim, cudaStream_t st) {
    std::string k(key);
    if (k == "encoder.embed_tokens.weight") return EZB_OK;  // alias of shared.weight in T5EncoderModel.state_dict()
    auto it = specs.find(k);
    if (it == specs.end()) return fail(EZB_ERR_WEIGHT, "t5: unexpected state-dict key '%s'", key);
    Spec& s = it->second;
    bool ok = (int)s.shape.size() == ndim;
    for (int i = 0; ok && i < ndim; ++i) ok = s.shape[i] == shape[i];
    if (!ok) return fail(EZB_ERR_WEIGHT, "t5: shape mismatch for '%s'", key);
    EZB_TRY(s.load(data, st));
    s.loaded = true;
    return EZB_OK;
  }
  int finalize() {
    for (auto& kv : specs)
      if (!kv.second.loaded) return fail(EZB_ERR_WEIGHT, "t5: missing state-dict key '%s'", kv.first.c_str());
    EZB_CUDA(cudaDeviceSynchronize());
    finalized = true;
    return EZB_OK;
  }
  // T5Attention._relative_position_bucket (bidirectional) in float32, the caller may pass the table computed by the reference's own torch ops
  void host_buckets(int L, std::vector<int32_t>& out) const {
    const int nb = d.num_buckets / 2, max_exact = nb / 2;
    out.resize((size_t)L * L);
    for (int q = 0; q < L; ++q)
      for (int k = 0; k < L; ++k) {
        const int rp = k - q, n = rp < 0 ? -rp : rp;
        int v = rp > 0 ? nb : 0;
        if (n < max_exact) v += n;
        else {
          const float t = logf((float)n / (float)max_exact) / (float)log((double)d.max_distance / max_exact) * (float)(nb - max_exact);
          int large = max_exact + (int)t;
          v += large < nb - 1 ? large : nb - 1;
        }
        out[(size_t)q * L + k] = v;
      }
  }
  int lin(cudaStream_t st, const __nv_bfloat16* A, int K, const __nv_bfloat16* W, int M, int N, const EpiLinearParams& e) {
    return gemm2<128, EpiLinear<128>>(*dev, st, A, kmul * K, W, kmul * K, M, N, kmul * K, e);
  }
  int forward(const int32_t* ids, const uint8_t* mask, const int32_t* buckets, float* out, int B, int L, cudaStream_t st) {
    if (!finalized) return fail(EZB_ERR_STATE, "t5: weights not finalized");
    if (B < 1 || L < 1 || B > d.max_batch || L > d.max_len) return fail(EZB_ERR_SHAPE, "t5: B=%d L=%d (max %d, %d)", B, L, d.max_batch, d.max_len);
    const int M = B * L;
    if (buckets == nullptr) {
      if (bucket_L != L) {  // the table depends on L only: built on the host in float32 (bit-compatible with the reference's torch ops) once per length;
        host_buckets(L, bucket_h);  // the staging vector lives in the handle, so the copy needs no synchronisation
        EZB_CUDA(cudaMemcpyAsync(bucket_d, bucket_h.data(), bucket_h.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        bucket_L = L;
      }
      buckets = bucket_d;
    }
    EZB_TRY(t5_embed_launch(st, ids, emb, x, M, D, d.vocab_size));
    EZB_TRY(t5_bias_launch(st, buckets, rel, bias, H, L));
    EpiLinearParams z;
    memset(&z, 0, sizeof z);
    static bool attr[16] = {};  // function attributes are per device
    if (!attr[dev->id & 15]) { EZB_CUDA(cudaFuncSetAttribute(attn_simt_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024)); attr[dev->id & 15] = true; }
    for (int i = 0; i < nl; ++i) {
      const Layer& w = layers[i];
      EZB_TRY(t5_rms_launch(st, x, w.ln0, act, nullptr, M, D, kmul, d.eps));
      EpiLinearParams e = z;
      e.out_f32 = qkv32; e.ld32 = 3 * inner;
      EZB_TRY(lin(st, act, D, w.qkv, M, 3 * inner, e));
      EZB_TRY(t5_heads_launch(st, qkv32, q32, k32, v32, B, L, H, dk));
      EZB_TRY(t5_attention_launch(st, q32, k32, v32, mask, bias, attn, B, H, L, dk, kmul));
      e = z;
      e.resid = x; e.ldr = D; e.out_f32 = x; e.ld32 = D;
      EZB_TRY(lin(st, attn, inner, w.o, M, D, e));
      EZB_TRY(t5_rms_launch(st, x, w.ln1, act, nullptr, M, D, kmul, d.eps));
      e = z;
      e.out_f32 = u32; e.ld32 = 2 * F;
      EZB_TRY(lin(st, act, D, w.wi, M, 2 * F, e));
      EZB_TRY(t5_gated_gelu_launch(st, u32, mid, M, F, kmul));
      e = z;
      e.resid = x; e.ldr = D; e.out_f32 = x; e.ld32 = D;
      EZB_TRY(lin(st, mid, F, w.wo, M, D, e));
    }
    return t5_rms_launch(st, x, lnf, nullptr, out, M, D, kmul, d.eps);
  }
};

}  // namespace ezb
