// The start latent of an audio-to-audio variation (ezb_vae_encode_noised): the VAE bottleneck sample, scale_shift and diffusers' add_noise
// in one pass over the encoder's output.  The kernel is compiled in a translation unit of its own (vae_noised.cu): adding it to ezb.cu's
// module changes the code NVVM emits for an unrelated kernel there (attn_simt_kernel<true>), and every kernel of that module keeps its
// code this way.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ezb {

// eps (B, Cz, L) fp32; ab: device fp32 [B][2], (a_b, s_b) per clip, read when the kernel runs; scale / shift: the autoencoder's
struct VaeNoised { const float* eps; const float* ab; float scale, shift; };

// enc [B*L, 2*Cz] channels-last (mean | scale), noise (B, Cz, L) or null (-> the mean), lens (device int32 [B]) or null -> x_t (B, Cz, L)
cudaError_t vae_sample_noised_launch(cudaStream_t st, const float* enc, const float* noise, const VaeNoised& n, float* x_t, int B, int Cz, int L,
                                     const int32_t* lens);

}  // namespace ezb
