// vae_sample_noised_kernel: see vae_noised.cuh for why it lives in a translation unit of its own.
#include "vae_noised.cuh"

namespace ezb {

// z as vae_sample_body (vae.cuh) computes it -- the same expression, so the same bits -- then scale_shift (src/utils/utils.py:20-21) and
// diffusers' add_noise with the sample's (a, s) = ab[b]:  x_t = a * ((z + shift) * scale) + s * eps.  The products and the sum are rounded
// one by one (no FMA contraction), as PyTorch computes the three ops.  LENS: frames at or past the clip's end (lens[b] clamped to [1, L],
// as clip_frames does) are written as zeros, and the encoder rows, the noise and eps there are not read.
template <bool LENS>
__global__ void vae_sample_noised_kernel(const float* __restrict__ enc, const float* __restrict__ noise, float* __restrict__ x_t, int Cz, int L,
                                         const int32_t* __restrict__ lens, VaeNoised nd) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= (size_t)Cz * L) return;
  const int c = i / L, l = i - (size_t)c * L;
  const size_t o = ((size_t)b * Cz + c) * L + l;
  if (LENS && l >= min(max(lens[b], 1), L)) { x_t[o] = 0.f; return; }
  const float* row = enc + ((size_t)b * L + l) * 2 * Cz;
  const float mean = row[c], sc = row[Cz + c];
  const float sp = sc > 20.f ? sc : log1pf(expf(sc));  // F.softplus (threshold 20)
  const float nz = noise ? noise[o] : 0.f;
  const float z = nz * (sp + 1e-4f) + mean;
  const float x0 = __fmul_rn(__fadd_rn(z, nd.shift), nd.scale);
  x_t[o] = __fadd_rn(__fmul_rn(nd.ab[2 * b], x0), __fmul_rn(nd.ab[2 * b + 1], nd.eps[o]));
}

cudaError_t vae_sample_noised_launch(cudaStream_t st, const float* enc, const float* noise, const VaeNoised& n, float* x_t, int B, int Cz, int L,
                                     const int32_t* lens) {
  dim3 g2((unsigned)(((size_t)Cz * L + 255) / 256), B);
  if (lens != nullptr) vae_sample_noised_kernel<true><<<g2, 256, 0, st>>>(enc, noise, x_t, Cz, L, lens, n);
  else vae_sample_noised_kernel<false><<<g2, 256, 0, st>>>(enc, noise, x_t, Cz, L, nullptr, n);
  return cudaGetLastError();
}

}  // namespace ezb
