/* libezb200 -- C ABI of the H100-native (sm_90a) EzAudio hot path (DiT denoiser step + Oobleck VAE decode).
 *
 * The reference (haidog-yaqub/EzAudio) is pure Python/PyTorch and has no FFI of its own; its drop-in boundary is the
 * Python call surface (SURVEY.md section 8b).  Each entry point below names the reference interface it replaces
 * (paths relative to the reference root).  Python binds these with ctypes (ezaudio_b200/_lib.py); INTEGRATION.md
 * shows the stub a reference maintainer would add.
 *
 * Conventions: plain pointers and sizes, no torch types.  Every device pointer is owned by the caller (PyTorch) and
 * must stay valid until the stream-ordered call has executed.  All work is enqueued on the cudaStream_t passed as
 * `stream` (void*).  The per-step entry points (set_context, set_context_rows, set_timesteps, forward, forward_tdev, controlnet_forward,
 * controlnet_set_condition, controlnet_set_condition_rows, controlnet_forward_tdev, controlnet_forward_cached,
 * cfg_ddim_step, cfg_ddim_step_slots, cfg_dpm_step, cfg_dpm_step_slots, window_gather, window_blend, loop_gather, loop_blend,
 * timeline_gather, timeline_guide, timeline_blend, decode, encode, encode_noised, energy_condition, t5_forward) never synchronise and are safe inside CUDA-graph capture; the load-time ones (create,
 * load_weight, finalize_weights) may synchronise the device.  A handle is not re-entrant.  Returns 0 on success,
 * a negative ezb_status otherwise; ezb_last_error() gives the message of the calling thread's last failure.
 */
#ifndef EZB200_H
#define EZB200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  EZB_OK = 0, EZB_ERR_ARG = -1, EZB_ERR_SHAPE = -2, EZB_ERR_UNSUPPORTED = -3, EZB_ERR_CUDA = -4, EZB_ERR_STATE = -5,
  EZB_ERR_WEIGHT = -6
} ezb_status;

typedef struct ezb_dit ezb_dit; /* one MaskDiT/UDiT or DiTControlNet instance on one device */
typedef struct ezb_vae ezb_vae; /* one OobleckDecoder instance on one device */

/* Hyper-parameters of `MaskDiT(**params['model'])` (api/ezaudio.py:83; ckpts/ezaudio-xl.yml:5-37).  Only the shipped
 * switch combination is implemented (1d, ada_sola_bias, cross, rope shared, qk layernorm, geglu, skip+skip_norm). */
typedef struct {
  int32_t embed_dim, num_heads, depth, context_dim, inner_dim, ada_rank;
  float ada_scaling;          /* ada_sola_alpha / ada_sola_rank (src/models/blocks.py:25) */
  int32_t latent_chans;       /* 128: x / gt channels; in_chans = 2*latent_chans + 1 */
  int32_t is_controlnet;      /* 1: DiTControlNet (src/models/controlnet.py:87) -- first half + stem + zero linears */
  int32_t cond_c0, cond_c1;   /* controlnet stem widths (cond_blocks, ckpts/controlnet/energy_l.yml:40) */
  int32_t max_batch, max_len, max_ctx_len, max_timesteps; /* workspace bounds (effective batch incl. CFG doubling) */
  int32_t precision;          /* 0: bf16 operands / fp32 accumulate; 1: bf16x3 split operands (fp32-grade parity mode);
                                 2: FP8 -- the self-attention QKV and GEGLU up-projections of every block take e4m3 operands (one fp32 scale
                                 per token row and per weight row, amax / 448) on fp32-accumulating wgmma, everything else as in mode 0.
                                 Needs head dim 64 or 72 with an even head count and embed_dim <= 1152. */
} ezb_dit_desc;

int ezb_version(void); /* 2: ezb_dit_forward / ezb_cfg_ddim_step take per-sample lengths */
const char* ezb_last_error(void);

/* --- model lifetime / weights: replaces MaskDiT(...).load_state_dict(torch.load(ckpt)['model']) (api/ezaudio.py:83-85) */
int ezb_dit_create(ezb_dit** out, const ezb_dit_desc* desc, int device);
int ezb_dit_destroy(ezb_dit* h);
/* One call per state-dict entry, reference key names and layouts (SURVEY Appendix D); `data` is a DEVICE fp32 pointer.
 * The library repacks into its own layouts (QKV concat, GEGLU interleave, bf16 / split-bf16 cast) and keeps no
 * reference to `data`. */
int ezb_dit_load_weight(ezb_dit* h, const char* ref_key, const float* data, const int64_t* shape, int ndim, void* stream);
int ezb_dit_finalize_weights(ezb_dit* h, void* stream); /* fails listing the first missing key */

/* --- step-invariant precompute.
 * context path: udit.py:94-97,295 (context_embed) + blocks.py:150 (norm_context) + attention.py:128-129,142 (to_k,to_v,norm_k)
 * for every block; ctx (Be,Lc,context_dim) fp32, ctx_mask (Be,Lc) uint8 (1 = keep; attention.py:30-37). */
int ezb_dit_set_context(ezb_dit* h, const float* ctx, const uint8_t* ctx_mask, int Be, int Lc, void* stream);
/* time path: modules.py:19-61 (TimestepEmbedder), udit.py:313-316 (time_act, time_ada, time_ada_final), blocks.py:39-45
 * (AdaLN) evaluated for n distinct timestep values (HOST array); forward calls then refer to them by index. */
int ezb_dit_set_timesteps(ezb_dit* h, const int64_t* timesteps_host, int n, void* stream);

/* --- one denoiser forward: MaskDiT.forward (conditioners.py:156-183) + UDiT.forward (udit.py:281-362).
 * x (Be,C,L) fp32; gt (Be,C,L) fp32 or NULL (mask_embed everywhere, conditioners.py:174-175); gt_mask (Be,L) uint8 or
 * NULL: 1 = position is regenerated (gt replaced by mask_embed there, mask channel = 1; conditioners.py:150-153,176);
 * t_index_host[Be]: index into the table of ezb_dit_set_timesteps per sample (NULL = all use `t_index_all`);
 * controlnet_skips: NULL or depth/2 device pointers (Be,L,D) fp32 in in-block order (udit.py:345-348);
 * out (Be,C,L) fp32.
 * lens: NULL (every sample is L frames long) or a DEVICE int32 [Be]: sample b is a clip of lens[b] frames padded to L.  Its frames
 * < lens[b] come out as a forward of that clip alone at L = lens[b] computes them, whatever the padded frames hold (NaN included); its
 * frames >= lens[b] of `out` are not written.  Kernels read the lengths when they run (a captured graph replays with new lengths) and
 * clamp them to [1, L]; validating them is the caller's job.  gt / gt_mask are padded like x (the Python layer marks the
 * padded frames as regenerated); not combined with ControlNet skips by the Python layer. */
int ezb_dit_forward(ezb_dit* h, const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* t_index_host,
                    int t_index_all, const float* const* controlnet_skips, float* out, int Be, int L, void* stream,
                    const int32_t* lens);
/* DiTControlNet.forward (controlnet.py:252-315): condition (Be,1,2L) fp32; writes depth/2 skips (Be,L,D) fp32, already
 * multiplied by conditioning_scale, into skips_out[i] (conditioning_scale 0: zeros, without running the network). */
int ezb_controlnet_forward(ezb_dit* h, const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* t_index_host,
                           int t_index_all, const float* condition, float conditioning_scale, float* const* skips_out, int Be,
                           int L, void* stream);

/* --- step-level scheduling: samples of one batch at different points of different schedules (continuous batching).
 * ezb_dit_set_context_rows: the context path of ezb_dit_set_context for rows [row0, row0 + n) of the batch only -- context_embed,
 * norm_context, and per block the cross-attention K / V^T caches and the key-mask bytes of those rows; the other rows keep what they hold.
 * ctx (n,Lc,context_dim) fp32 and ctx_mask (n,Lc) uint8 are DEVICE pointers to the new rows.  It writes into the layout (Be, Lc) of the last
 * ezb_dit_set_context call and fails with EZB_ERR_STATE when there was none or when Lc differs from it; the rows come out bit-identical to a
 * ezb_dit_set_context of the whole updated batch (the kernels are chosen for the whole batch).  Graph-safe, no synchronisation. */
int ezb_dit_set_context_rows(ezb_dit* h, const float* ctx, const uint8_t* ctx_mask, int row0, int n, int Lc, void* stream);
/* ezb_dit_forward with the per-sample timestep indices in DEVICE memory: t_index_dev int32 [Be], indices into the table of
 * ezb_dit_set_timesteps.  The indices are read when the kernels run (a captured graph replays with new indices); out-of-range values are
 * clamped to the table, validating them is the caller's job.  The output is bit-identical to ezb_dit_forward with the same indices in
 * t_index_host when they are not all equal (a batch that shares one timestep may take other kernels there). */
int ezb_dit_forward_tdev(ezb_dit* h, const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* t_index_dev,
                         const float* const* controlnet_skips, float* out, int Be, int L, void* stream, const int32_t* lens);
/* ControlNet handles.  ezb_controlnet_set_condition: runs the stem (controlnet_pre, which does not depend on the timestep) of condition
 * (Be,1,2L) fp32 DEVICE once, into a condition cache [Be, L, embed_dim] the handle owns; ezb_controlnet_forward neither reads nor writes it.
 * The call fixes the cache layout (Be, L).  ezb_controlnet_set_condition_rows: rows [row0, row0 + n) of that layout from condition (n,1,2L);
 * the other rows keep what they hold.  It fails with EZB_ERR_STATE when there is no layout or L differs from it, with EZB_ERR_SHAPE when the
 * rows fall outside the batch; the rows come out bit-identical to ezb_controlnet_set_condition of the whole updated batch.
 * ezb_controlnet_forward_tdev: ezb_controlnet_forward with the per-sample timestep indices t_index_dev int32 [Be] and conditioning scales
 * scale_dev fp32 [Be] in DEVICE memory (read when the kernels run, like ezb_dit_forward_tdev's indices) and the condition from the cache;
 * Be must match the context batch and the condition layout, L the layout.  Sample b's skips are the zero-linear outputs times scale_dev[b]
 * (0 gives zeros).  For host indices that are not all equal, each sample whose scale s != 0 comes out bit-identical to
 * ezb_controlnet_forward with those indices, the same condition and conditioning_scale s.  All three are graph-safe, no synchronisation. */
int ezb_controlnet_set_condition(ezb_dit* h, const float* condition, int Be, int L, void* stream);
int ezb_controlnet_set_condition_rows(ezb_dit* h, const float* condition, int row0, int n, int L, void* stream);
int ezb_controlnet_forward_tdev(ezb_dit* h, const float* x, const int32_t* t_index_dev, const float* scale_dev, float* const* skips_out, int Be,
                                int L, void* stream);
/* ezb_controlnet_forward with the stem's output taken from the condition cache instead of a condition argument: for any host indices
 * (all equal or not) and any conditioning_scale, the skips are bit-identical to ezb_controlnet_forward with the condition that was cached
 * (the stem computes each row on its own; everything after it takes the same kernels, fold mode included).  conditioning_scale 0 gives zeros
 * without running the network.  Be must match the context batch and the condition layout, L the layout (EZB_ERR_STATE otherwise).  A
 * sampling loop that repeats one condition at every step runs the stem once (ezb_controlnet_set_condition) instead of once per step.
 * Graph-safe, no synchronisation. */
int ezb_controlnet_forward_cached(ezb_dit* h, const float* x, const float* gt, const uint8_t* gt_mask, const int32_t* t_index_host,
                                  int t_index_all, float conditioning_scale, float* const* skips_out, int Be, int L, void* stream);

/* --- fused classifier-free guidance + rescale + DDIM update (src/inference.py:12-23,88-100; diffusers DDIMScheduler.step
 * restated, SURVEY Appendix B).  model_out holds B text rows followed by B uncond rows when guidance_scale != 0, else B
 * rows.  coef = {sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-sigma^2), sigma}; noise (B,C,L) may be NULL when
 * sigma == 0.  latents updated in place.  `device`: the CUDA device the pointers live on (the call makes it current).
 * lens: NULL or a DEVICE int32 [B] (clamped to [1, L]): sample b covers frames < lens[b] of every channel.  The rescale statistics and
 * the update run over exactly those C * lens[b] elements, in the order of a call on that clip alone (bit-identical to it); the padded
 * frames of latents are left untouched. */
int ezb_cfg_ddim_step(int device, const float* model_out, float* latents, const float* noise, int B, int C, int L, float guidance_scale,
                      float guidance_rescale, const float* coef5_host, void* stream, const int32_t* lens);
/* ezb_cfg_ddim_step with the constants of each sample in a DEVICE array slots_dev[B], read when the kernel runs (a captured graph replays
 * with new slots).  model_out always holds B text rows followed by B uncond rows.  Sample b with flags & EZB_SLOT_ACTIVE is updated as
 * ezb_cfg_ddim_step on that sample alone with its slot's guidance_scale (when flags & EZB_SLOT_CFG; without it only the text row is used,
 * as with guidance_scale 0), guidance_rescale and coef computes it, bit for bit; an inactive sample's latents are not touched.  noise
 * (B,C,L) is read only by samples whose sigma (coef[4]) is non-zero; it may be NULL when no active slot has one -- checking that is the
 * caller's job, as is validating lens (clamped to [1, L] as in ezb_cfg_ddim_step). */
typedef struct {
  float guidance_scale, guidance_rescale;
  float coef[5];   /* as coef5_host of ezb_cfg_ddim_step */
  int32_t flags;   /* EZB_SLOT_ACTIVE | EZB_SLOT_CFG */
} ezb_ddim_slot;
enum { EZB_SLOT_ACTIVE = 1, EZB_SLOT_CFG = 2 };
int ezb_cfg_ddim_step_slots(int device, const float* model_out, float* latents, const float* noise, const ezb_ddim_slot* slots_dev, int B,
                            int C, int L, void* stream, const int32_t* lens);

/* --- fused classifier-free guidance + rescale + DPM-Solver++ multistep update (diffusers DPMSolverMultistepScheduler.step restated for
 * dpmsolver++ / sde-dpmsolver++, midpoint; ezaudio_b200/scheduler.py).  Guidance, rescale, model_out, lens and `device` as in
 * ezb_cfg_ddim_step: the same reduction, element order and padded frames left untouched.  coef = {alpha_s, sigma_s, kx, k0, k1, r, kz};
 * with v the guided output, each element computes m0 = alpha_s x - sigma_s v and x <- kx x + k0 m0 + k1 (r (m0 - m1)) + kz z.
 * history (B,C,L) fp32 holds m1, the previous step's m0: it is read only at order 2 (order 1 drops the k1 term), and this step's m0 is
 * written into it.  noise (B,C,L) is read only when kz != 0 and may be NULL otherwise.  latents updated in place. */
int ezb_cfg_dpm_step(int device, const float* model_out, float* latents, float* history, const float* noise, int B, int C, int L,
                     float guidance_scale, float guidance_rescale, const float* coef7_host, int order, void* stream, const int32_t* lens);
/* ezb_cfg_dpm_step with the constants of each sample in a DEVICE array slots_dev[B], read when the kernel runs, as ezb_cfg_ddim_step_slots:
 * model_out always holds B text rows followed by B uncond rows; a sample with flags & EZB_SLOT_ACTIVE is updated as ezb_cfg_dpm_step on that
 * sample alone (order 2 when flags & EZB_SLOT_ORDER2) computes it, bit for bit; an inactive sample's latents and history are not touched.
 * noise is read only by samples whose kz (coef[6]) is non-zero; checking that it is there, and validating lens, is the caller's job.
 * A batch whose samples run different samplers launches ezb_cfg_ddim_step_slots and this call on the same buffers, each with the other
 * kind's slots inactive. */
typedef struct {
  float guidance_scale, guidance_rescale;
  float coef[7];   /* as coef7_host of ezb_cfg_dpm_step */
  int32_t flags;   /* EZB_SLOT_ACTIVE | EZB_SLOT_CFG | EZB_SLOT_ORDER2 */
} ezb_dpm_slot;
enum { EZB_SLOT_ORDER2 = 4 };
int ezb_cfg_dpm_step_slots(int device, const float* model_out, float* latents, float* history, const float* noise, const ezb_dpm_slot* slots_dev,
                           int B, int C, int L, void* stream, const int32_t* lens);

/* Windowed denoising of clips longer than the denoiser's trained window (MultiDiffusion, Bar-Tal et al. 2023).  Clip b of N_b frames is
 * cut into windows of Lw frames overlapping by `overlap` frames (1 <= overlap <= Lw / 2, hop H = Lw - overlap): N_b <= Lw is one window
 * [0, N_b); otherwise n_b = ceil((N_b - Lw) / H) + 1 windows start at k * H for k < n_b - 1, and the last at N_b - Lw.  Window k weighs its
 * local frame j by min(1, left, right): left = (j + 1) / (overlap + 1) when k > 0, else 1; right = (Lw - j) / (overlap + 1) when
 * k < n_b - 1, else 1.  plan_dev: DEVICE int32 [B][3] = (first window row, n_b, N_b) per clip, the clips' windows laid out clip by clip as
 * consecutive rows 0 .. W - 1; it is read when the kernels run (a captured graph follows a new plan of the same W) and validating it is
 * the caller's job (ezaudio_b200.inference.window_plan builds it).  latents / out (B, C, Nmax) fp32, windows (rows, C, Lw) fp32.
 * ezb_window_gather: window row r gets its frames of the long latents and zeros past its length (N_b when N_b < Lw); copies 2 writes the
 *   same rows again at row offset W (the uncond half of a CFG batch).
 * ezb_window_blend: frame f < N_b of clip b gets sum_k w_k v_k / sum_k w_k over the windows covering it, in increasing k, in fp32, the
 *   division IEEE-rounded; one covering window of weight 1 gives its value bit for bit.  Window frames past a window's length and long
 *   frames at or past N_b are neither read nor written. */
int ezb_window_gather(int device, const float* latents, float* windows, const int32_t* plan_dev, int B, int C, int Nmax, int W, int Lw,
                      int overlap, int copies, void* stream);
int ezb_window_blend(int device, const float* windows, float* out, const int32_t* plan_dev, int B, int C, int Nmax, int W, int Lw, int overlap,
                     void* stream);

/* Seamless loops: windowed denoising on a circle, where frame N_b - 1 of loop b is followed by frame 0.  plan_dev is the table above, with
 * the windows of loop b: N_b <= Lw is one window of Lw_b = N_b frames, otherwise n_b = ceil(N_b / (Lw - overlap)) windows of Lw_b = Lw
 * frames.  offsets_dev: DEVICE int32 [B], the step's shift r_b, read when the kernels run (a captured schedule passes each step's row of a
 * [steps][B] table).  Window k of loop b starts at s_k = (floor(k * N_b / n_b) + r_b) mod N_b and holds frames (s_k + j) mod N_b, j < Lw_b;
 * its weight at j is 1 when n_b == 1, else min(1, (j + 1) / (overlap + 1), (Lw_b - j) / (overlap + 1)).  ezaudio_b200.inference.loop_plan
 * builds the table.
 * ezb_loop_gather: window row r gets its frames and zeros past Lw_b; copies 2 writes the same rows again at row offset W.
 * ezb_loop_blend: frame f < N_b gets sum w v / sum w over the windows covering it, summed in decreasing local index j (the first term
 *   starting both sums), in fp32, the division IEEE-rounded.  The order depends only on where f sits in each window, so adding d to every
 *   offset (with the latents rolled by d) rolls the result by d exactly; one covering window of weight 1 gives its value bit for bit.  Window
 *   frames past Lw_b and frames at or past N_b are neither read nor written. */
int ezb_loop_gather(int device, const float* latents, float* windows, const int32_t* plan_dev, const int32_t* offsets_dev, int B, int C, int Nmax,
                    int W, int Lw, int overlap, int copies, void* stream);
int ezb_loop_blend(int device, const float* windows, float* out, const int32_t* plan_dev, const int32_t* offsets_dev, int B, int C, int Nmax, int W,
                   int Lw, int overlap, void* stream);

/* Timelines of prompts over long clips (MultiDiffusion's region-based generation on the time axis).  The clips are windowed as for
 * ezb_window_gather (plan_dev: the same DEVICE int32 [B][3] table, W windows).  Every window carries one conditioned row per segment
 * active in it, and under guidance all of them share the window's one unconditional row.
 * rows_dev: DEVICE int32 [R][4], 16-byte aligned, = (window, s, e, T) per conditioned row, laid out clip by clip, window by window, then in
 *   timeline order.  [s, e) are the segment's frames and T >= 0 its transition in frames.  Segment [s, e) weighs frame f by
 *   a(f) = min(1, (f - s + T + 1) / (T + 1), (e + T - f) / (T + 1)) on [s - T, e + T) and 0 elsewhere, each ratio an IEEE fp32 division;
 *   a segment is active in a window when [s - T, e + T) meets it.
 * spans_dev: DEVICE int32 [B][2] = (first row, row count) per clip.
 * The tables are read when the kernels run, so a captured graph follows new segment boundaries, transitions and clip lengths with the
 * same R and W; validating them is the caller's job (ezaudio_b200.inference.timeline_plan builds them).
 * ezb_timeline_gather: row r < R gets its window's frames of the long latents and zeros past the window's length; with uncond 1, row R + k
 *   gets window k's the same way (the DiT input is then R + W rows).
 * ezb_timeline_guide: model_out (R + W, C, Lw) -> guided (R, C, Lw).  Row r is guided against row R + window(r) over lens_dev[r] frames:
 *   the bits ezb_cfg_ddim_step computes with coefficients (1, 0, 0, 1, 0), no noise and lens {lens_dev[r]} on the pair laid out as
 *   [row r | row R + window(r)] (the same clusters, slices and double-precision reduction).  guided is that call's "latents" and must hold
 *   finite values.  A row whose window lies outside 0 .. W - 1 is left untouched.
 * ezb_timeline_blend: windows (R, C, Lw) -> out (B, C, Nmax).  Frame f < N_b of clip b gets sum w_k(j) a(f) v_r(j) / sum w_k(j) a(f) over
 *   the rows of its span whose window k covers f (at local frame j, weight w_k as for ezb_window_blend) and whose a(f) > 0, in row order,
 *   in fp32: the product w_k(j) * a(f) is rounded first, the first term starts both sums, the rest are fused multiply-adds and sums, and
 *   the division is IEEE-rounded.  One covering row of weight 1 gives its value bit for bit, and a single segment covering the clip gives
 *   ezb_window_blend's bits.  Row frames past a window's length and frames at or past N_b are neither read nor written. */
int ezb_timeline_gather(int device, const float* latents, float* windows, const int32_t* plan_dev, const int32_t* rows_dev, int B, int C, int Nmax,
                        int W, int R, int Lw, int overlap, int uncond, void* stream);
int ezb_timeline_guide(int device, const float* model_out, float* guided, const int32_t* rows_dev, const int32_t* lens_dev, int R, int W, int C, int Lw,
                       float gs, float gr, void* stream);
int ezb_timeline_blend(int device, const float* windows, float* out, const int32_t* plan_dev, const int32_t* rows_dev, const int32_t* spans_dev,
                       int B, int C, int Nmax, int W, int R, int Lw, int overlap, void* stream);

/* --- VAE decoder: OobleckDecoder.forward (stable_vae/models/autoencoders.py:149-190) behind
 * Autoencoder(embedding=z) (src/modules/autoencoder_wrapper.py:74-77). */
typedef struct {
  int32_t latent_dim, channels, out_channels;
  int32_t n_stages;
  int32_t c_mults[8];  /* config c_mults (without the leading 1) */
  int32_t strides[8];
  int32_t max_batch, max_latent_len;
  int32_t precision;
  int32_t with_encoder;    /* 1: also hold OobleckEncoder + VAE bottleneck (editing_audio, api/ezaudio.py:175) */
  int32_t in_channels;     /* 1 */
  int32_t enc_latent_dim;  /* 2 * latent_dim (mean | scale) */
} ezb_vae_desc;
int ezb_vae_create(ezb_vae** out, const ezb_vae_desc* desc, int device);
int ezb_vae_destroy(ezb_vae* h);
/* keys: "decoder.layers...." with weight_g / weight_v / bias / alpha / beta (stable_vae/__init__.py:25-31 after prefix strip) */
int ezb_vae_load_weight(ezb_vae* h, const char* ref_key, const float* data, const int64_t* shape, int ndim, void* stream);
int ezb_vae_finalize_weights(ezb_vae* h, void* stream);
int ezb_vae_decode(ezb_vae* h, const float* z /*(B,latent,L)*/, float* wav /*(B,out_channels,L*prod(strides))*/, int B, int L,
                   void* stream);
/* Autoencoder(audio=x) (src/modules/autoencoder_wrapper.py:69-73): OobleckEncoder (stable_vae/models/autoencoders.py:115-146) +
 * VAEBottleneck.encode (bottleneck.py:66-87): z = mean + (softplus(scale) + 1e-4) * noise.  audio (B,1,T) fp32, T a multiple of the
 * hop (480); noise (B,latent,L) fp32 drawn by the caller (the reference uses torch.randn_like), NULL -> z = mean. */
int ezb_vae_encode(ezb_vae* h, const float* audio, const float* noise, float* z, int B, int T, void* stream);
/* Decode / encode of a padded batch of clips of different lengths.  lens: DEVICE int32 [B], latent frames per clip, read when the kernels
 * run (a captured graph replays with new lengths) and clamped to [1, L]; validating them is the caller's job.
 * ezb_vae_decode_lens: samples < hop * lens[b] of clip b come out bit-identical to ezb_vae_decode of z[b, :, :lens[b]] alone, the samples
 *   past them as zeros, whatever the padded frames of z hold (NaN included).
 * ezb_vae_encode_lens: clip b is the first hop * lens[b] samples of audio[b] (T = hop * L); frames < lens[b] of z[b] come out bit-identical
 *   to ezb_vae_encode of that clip alone with noise[b, :, :lens[b]], the frames past them as zeros, whatever audio and noise hold past
 *   the clip's end. */
int ezb_vae_decode_lens(ezb_vae* h, const float* z, float* wav, int B, int L, const int32_t* lens, void* stream);
int ezb_vae_encode_lens(ezb_vae* h, const float* audio, const float* noise, float* z, int B, int T, const int32_t* lens, void* stream);
/* ezb_vae_encode_noised: the start latent of an audio-to-audio variation (SDEdit) in the encode's last pass.  With z of ezb_vae_encode
 *   (vae_noise as its noise, NULL -> the mean), x_t = a_b * ((z + shift) * scale) + s_b * eps_b: scale_shift (src/utils/utils.py:20-21,
 *   the latent the denoiser was trained on, src/train.py:275-284) then diffusers' add_noise, each product and the sum rounded in fp32 as
 *   PyTorch rounds them.  ab_dev: DEVICE fp32 [B][2], (a_b, s_b) per clip, read when the kernel runs (one captured graph serves any mix);
 *   eps (B,latent,L) fp32; scale and shift are the autoencoder's.  lens (DEVICE int32 [B], or NULL) as in ezb_vae_encode_lens: frames at or
 *   past lens[b] are written as zeros, and the encoder rows, vae_noise and eps there are not read.  With a = 1, s = 0, scale = 1 and
 *   shift = 0, x_t equals z of ezb_vae_encode / ezb_vae_encode_lens bit for bit. */
int ezb_vae_encode_noised(ezb_vae* h, const float* audio, const float* vae_noise, const float* eps, const float* ab_dev, float scale, float shift,
                          float* x_t, int B, int T, const int32_t* lens, void* stream);

/* EnergyExtractor.forward (src/models/conditions/energy.py:19-56) as wrapped by Conditioner (condition_wrapper.py:26-42): audio (B,T) fp32
 * -> (B, T/hop) fp32 frame energies in dB, normalised per clip when norm != 0; quantize_levels <= 1 disables quantisation. Only the shipped
 * padding mode ('reflect') exists.  Refused (EZB_ERR_UNSUPPORTED): an odd window_size - hop_size.  Refused (EZB_ERR_SHAPE): T < hop_size,
 * window_size < hop_size, a reflect padding (window_size - hop_size) / 2 >= T, more than 51200 frames (the per-clip shared-memory table). */
int ezb_energy_condition(int device, const float* audio, float* out, int B, int T, int hop_size, int window_size, float min_db, int norm,
                         int quantize_levels, void* stream);

/* --- waveform pre / post-processing around the path (SURVEY 8(f) row 4), device pointers, fp32 mono clips.
 * ezb_wave_prepare: per clip  x <- x / (max|x| + 1e-9) when normalize != 0 (api/ezaudio.py:147, api/controlnet.py:119), samples with
 *   |x| <= gate zeroed when gate > 0 (`surpass_noise`, api/controlnet.py:121-124), then zero-padded or cropped from T_in to T_out samples
 *   (api/controlnet.py:131-136).  in (B,T_in), out (B,T_out).
 * ezb_wave_splice: dst[start : start+n] = src[0 : n] -- the paste of the regenerated chunk into the original clip (api/ezaudio.py:198-203).
 * ezb_wave_to_pcm16: round(x * 32768) saturated to int16 -- the sample format soundfile.write(path, audio, sr) produces by default for
 *   WAV (t2a_demo.py:13,20). */
int ezb_wave_prepare(int device, const float* in, float* out, int B, int T_in, int T_out, int normalize, float gate, void* stream);
int ezb_wave_splice(int device, float* dst, long long dst_len, const float* src, long long start, long long n, void* stream);
int ezb_wave_to_pcm16(int device, const float* in, int16_t* out, long long n, void* stream);

/* --- T5 (v1.1 / flan-T5, gated-GELU) text encoder: `text_encoder(input_ids=, attention_mask=).last_hidden_state`, src/inference.py:38-50;
 * model class transformers.T5EncoderModel loaded at api/ezaudio.py:78-79 (SURVEY 8(f) row 3: the step before the denoiser path). */
typedef struct ezb_t5 ezb_t5;
typedef struct {
  int32_t vocab_size, d_model, d_kv, num_heads, d_ff, num_layers;
  int32_t num_buckets;   /* relative_attention_num_buckets (32) */
  int32_t max_distance;  /* relative_attention_max_distance (128) */
  float eps;             /* layer_norm_epsilon (1e-6) */
  int32_t max_batch, max_len;
  int32_t precision;     /* 0 = bf16 operands, 1 = bf16x3 (parity mode), as in ezb_dit_desc */
} ezb_t5_desc;
int ezb_t5_create(ezb_t5** out, const ezb_t5_desc* desc, int device);
int ezb_t5_destroy(ezb_t5* h);
/* keys of T5EncoderModel.state_dict(): shared.weight, encoder.block.{i}.layer.0.SelfAttention.{q,k,v,o}.weight, ...relative_attention_bias.weight
 * (block 0), encoder.block.{i}.layer.{0,1}.layer_norm.weight, ...DenseReluDense.{wi_0,wi_1,wo}.weight, encoder.final_layer_norm.weight */
int ezb_t5_load_weight(ezb_t5* h, const char* ref_key, const float* data, const int64_t* shape, int ndim, void* stream);
int ezb_t5_finalize_weights(ezb_t5* h, void* stream);
/* ids (B, L) int32, attention mask (B, L) uint8 (1 = token), out (B, L, d_model) fp32, all device pointers.  `buckets` (L, L) int32 device
 * pointer = T5Attention._relative_position_bucket(key - query) as computed by the caller with the reference's own torch ops, or NULL to let
 * the library compute it on the host in float32. */
int ezb_t5_forward(ezb_t5* h, const int32_t* ids, const uint8_t* mask, const int32_t* buckets, float* out, int B, int L, void* stream);

/* --- kernel-level hooks used by tests/ and profiling only (not part of the drop-in surface). */
typedef struct {
  const float* bias; int32_t bias_mod;
  const float* resid; int32_t ldr;
  const float* gate; int32_t gate_bstride; int32_t rows_per_batch;
  float* out_f32; int32_t ld32;
  void* out_bf16; int32_t ld16; int32_t split_stride;
  int32_t act; const float* act_a; const float* act_b;
  /* swap-AB kinds only: LayerNorm folded into the epilogue (gemm.cuh FoldIn / FoldOut), null fin_u and fout_st: none.  fin_st / fout_st
     are float2 (sum, sum of squares) partials, slot-major with pitch fin_ld_st / fout_ld_st. */
  const void* fin_st; int32_t fin_slots; int32_t fin_ld_st; float fin_inv_dim; const float* fin_u; const float* fin_v;
  void* fout_st; int32_t fout_ld_st; void* fout_a0; int32_t fout_ld0; const float* fout_g0; void* fout_a1; int32_t fout_ld1; const float* fout_g1;
  /* second fold-in source (the out-blocks' skip_norm over [x | skip]): its partials follow fin_st's in the row statistics; NULL: none */
  const void* fin_st1; int32_t fin_slots1;
} ezb_test_epilogue;
/* C = A[M,K] W[N,K]^T through the wgmma GEMM; epi_kind 0 = linear epilogue, 1 = GEGLU (packed W); 10 / 11 = the same on 2-CTA
   clusters (11: the GEGLU kernel the model dispatches); 12 = the parked-tile cluster GEGLU; 20 = swap-AB as the model dispatches it
   (token width chosen from the shape, fold epilogue when a fold is set); 21 = the same with the token width bn (256 or 288).
   conv_* = 0 for plain. */
int ezb_test_gemm(int device, const void* A_bf16, int lda, const void* W_bf16, int ldw, int M, int N, int K, int bn, int epi_kind,
                  const ezb_test_epilogue* e, int conv_taps, int conv_center, int conv_dil, int conv_cin_pad, int conv_T,
                  int conv_B, void* stream);
/* The DiT's linears on 128-wide N-tiles (csrc/gemm.cuh EpiLinear, EpiLinearScaled), launched as Dit::lin and the ControlNet zero-linears
   launch them, from a reference-layout weight.  Device pointers unless noted.
   W fp32 [N, K], packed by the library as Dit::init packs it into W' bf16 [N, kmul*K]: kmul 1 bf16(W); kmul 3 (bf16x3) [hi | hi | lo] with
   hi = bf16(W), lo = bf16(W - hi).  w_packed (optional) receives W'.  A bf16 [M, kmul*K], row pitch lda >= kmul*K ([hi | lo | hi] in bf16x3).
   Epilogue of EpiLinear, per row r and column c < N:  v = (A W'^T + bias)[r, c] * out_scale (out_scale 0 reads as 1; bias optional);
   with resid (pitch ldr)  v = resid[r, c] + v, or with gate too  v = resid[r, c] + (1 - gate[b * gate_bstride + c]) v,  b = r / rows_per_batch;
   out_f32 (pitch ld32) receives v; out_bf16 (pitch ld16) receives bf16(act(v)) (act 0 none, 1 SiLU), and when split (kmul 3 only) also the
   remainder bf16(act(v) - hi) at column c + N and hi again at c + 2N.  scale, fp32 [B], selects EpiLinearScaled instead:
   out_f32 = (A W'^T + bias) * scale[r / rows_per_batch] (bias and out_f32 only; a scale of 0 gives zeros).
   kernel: 1 single-CTA gemm<128, EpiLinear<128>>; 2 2-CTA cluster gemm2<128, EpiLinear<128>>; 3 / 4 the same two with EpiLinearScaled (scale
   set); 0 the kernel Dit::lin runs for these pair / swap_ab (the model's runtime switches), kmul, m_select (the token count the kernel is
   chosen for, 0: M) and epilogue -- which can be the swap-AB kernel -- or, with scale, the one the ControlNet trunk runs for pair.
   ran (optional HOST pointer) receives the kernel that ran: 1 to 4, or 256 / 288, the token width of the swap-AB tiles.
   Every argument is checked before any device work. */
typedef struct {
  int32_t M, N, K, kmul, lda;
  const void* A; const float* W; void* w_packed;
  const float* bias;
  const float* resid; int32_t ldr;
  const float* gate; int32_t gate_bstride; int32_t rows_per_batch;
  float* out_f32; int32_t ld32;
  void* out_bf16; int32_t ld16; int32_t split; int32_t act;
  float out_scale;
  const float* scale;
  int32_t kernel, pair, swap_ab, m_select;
  int32_t* ran;
} ezb_test_linear_args;
int ezb_test_linear(int device, const ezb_test_linear_args* args, void* stream);
/* Q/K/V-type projection with the fused per-head LayerNorm(dh) + RoPE + attention-layout epilogue (the fast mode's Q/K/V, cross-Q and
   cross-K/V GEMMs).  Device pointers.  A [B*L, D] bf16; W [nsec*D, D] fp32 in the reference layout (section s = rows s*D ..), packed and
   rounded to bf16 by the library as the model packs it.  Section s has kind kinds[s]: 0 q, 1 k (both LayerNorm(dh) -> optional RoPE at the
   position within the clip -> bf16 rows [b*H + h, l, 0..dh) of pitch ld_qk), 2 v (bf16 V^T [b*H + h, 0..dvp, 0..Lpad): rows dh..dvp written
   as zeros, columns L..Lpad not written). */
typedef struct {
  int32_t B, L, D, H, dh, nsec;
  int32_t kinds[3];
  const float* norm_q;        /* [2][dh] LayerNorm weight | bias of kind 0 (NULL when no section is kind 0) */
  const float* norm_k;        /* the same for kind 1 */
  const float* inv_freq;      /* [dh/2] RoPE frequencies */
  int32_t rope;               /* 0 none, 1 (cos, sin) table filled by the library, 2 __sincosf from inv_freq */
  void* q; void* k; void* vt;
  int32_t ld_qk, dvp, Lpad;
  /* LayerNorm folded in (NULL fold_st: off): float2 [fold_slots][fold_ld_st] per-row (sum x, sum x^2) partials of the D-wide x, and u, v
     in the packed output-column order (packed-3: H * N-tile entries, 0 in the pad columns) */
  const void* fold_st; int32_t fold_slots, fold_ld_st;
  const float* fold_u; const float* fold_v;
  /* 0 / 1: three heads per N-tile (nsec 3) on the register-fragment schedule / on the parked tile with staged q, k stores (2: as 1);
     3 / 4: two heads per N-tile on 2-CTA clusters, fragment / parked; 5: two heads per N-tile on the single-CTA kernel.  The fold and
     q / k outputs that are not 16-byte aligned run the parked tile under every variant. */
  int32_t variant;
} ezb_test_heads_args;
int ezb_test_heads(int device, const void* A_bf16, const float* W_f32, const ezb_test_heads_args* args, void* stream);
/* MLP of a DiT block: x += (1 - gate[b]) * (bf16(GEGLU(A W1^T + b1)) W2^T + b2), b = row / rows_per_batch (gate NULL: plain residual).
   Device pointers.  A [M, D] bf16; W1 [2*inner, D] and b1 [2*inner] fp32 in the reference layout ([hidden; gate] rows), packed by the
   library; W2 [D, inner] bf16; b2 [D]; x [M, D] fp32 updated in place; gate row stride gate_bstride; mid [M, inner] bf16 receives the GEGLU
   output; grid_barrier: two zeroed uint32 (count, generation), left with count 0.  variant 0: one persistent launch (GEGLU, grid barrier,
   swap-AB output projection); 1: the same two GEMMs as two launches; 2: as 1 with the parked-tile GEGLU kernel (the one bf16x3 and
   outputs without 16-byte alignment run). */
int ezb_test_mlp(int device, const void* A_bf16, const float* W1_f32, const float* b1_f32, const void* W2_bf16, const float* b2, float* x,
                 const float* gate, int gate_bstride, int rows_per_batch, void* mid_bf16, void* grid_barrier, int M, int D, int inner,
                 int variant, void* stream);
/* The folded LayerNorm (csrc/gemm.cuh FoldIn / FoldOut, csrc/dit.cuh build_fold_tables) and the LayerNorm tail of a swap-AB GEMM
   (csrc/gemm_ln.cuh), launched as Dit launches them.  Device pointers unless noted; every argument is checked before any device work.
   Tables (kinds 0-2): G = w (1 + scale), Cc = b (1 + scale) + shift for R modulation rows (row r of shift / scale at r * ld_mod; both NULL:
   G = w, Cc = b) -> G, Cc fp32 [R, K]; then U = G W'^T, V = Cc W'^T (+ add_v) -> u, v fp32 [R, N], W' the packed bf16 weight.
   kind 0 tables:        W fp32 [N, K] in the reference layout, packed plainly (bf16(W)) into w_packed [N, K]; add_v [N] optional.  K at most
                         2304 (a larger K is refused with EZB_ERR_UNSUPPORTED).
   kind 1 FoldIn GEGLU:  W fp32 [2 inner, K] ([hidden; gate] rows) and bias [2 inner], packed as Dit::init packs them for GEGLU N-tiles of
                         geglu_bn columns (0: what Dit picks, 256 when inner % 128 == 0, else 128); the tables with R = 1, N = 2 inner and
                         add_v = the packed bias (u, v in the packed order); then the GEGLU GEMM with the LayerNorm folded in: A bf16 [M, K]
                         = bf16(x G) of the rows x whose (sum, sum of squares) partials are st, float2 [slots][ld_st] -> out bf16 [M, inner].
                         w_packed (optional) receives W'.
   kind 2 fused MLP:     kind 1 with geglu_bn 256 into out = mid bf16 [M, inner], then x += (1 - gate[b]) (mid W2^T + b2) in place, x fp32
                         [M, K], W2 bf16 [K, inner], b = row / rows_per_batch (gate NULL: plain residual), folded out: a0 bf16 [M, K] =
                         bf16(x g0) and fout_st float2 [K / 32][ld_st] partials of the new x.  variant 0: one persistent launch on
                         grid_barrier (two zeroed uint32, left with count 0); 1: the same two GEMMs as two launches.
   kind 3 LayerNorm tail: x = A W16^T + bias (+ resid, gated as kind 2) -> out_f32 fp32 [M, N] (A bf16 [M, K], W16 bf16 [N, K], resid pitch
                         N), on swap-AB tiles of bn tokens (0: the width gemm_swapped_ln picks; 256 or 288), and the LayerNorm of the row
                         [x | x2 (+ x3)] (x2 / x3 fp32 [M, D2], optional) with w / b, optional modulation shift / scale (row
                         (row / rows_per_batch) * ld_mod) -> ln_out bf16 [M, N + D2]: as the tail phase of the same launch behind
                         grid_barrier when the tiles fit one wave, else not at all (the caller launches it).  ran_bn and ran_fused receive
                         the token width and whether the tail ran.  LayerNorm pointers 16-byte aligned, N, D2 and ld_mod multiples of 4. */
typedef struct {
  int32_t kind, variant;
  int32_t M, N, K, R, inner, geglu_bn, bn;
  const float* w; const float* b; const float* shift; const float* scale; int32_t ld_mod, rows_per_batch;
  const float* W; const float* bias; const float* add_v;
  void* w_packed; float* G; float* Cc; float* u; float* v;
  const void* A; const void* st; int32_t slots, ld_st;
  void* out;
  const void* W2; const float* b2; float* x; const float* gate; int32_t gate_bstride;
  void* fout_st; void* a0; const float* g0;
  void* grid_barrier;
  const void* W16; const float* resid; float* out_f32; const float* x2; const float* x3; int32_t D2; void* ln_out;
  int32_t ran_bn, ran_fused;
} ezb_test_fold_args;
int ezb_test_fold(int device, ezb_test_fold_args* args, void* stream);
/* One layer of the Oobleck VAE, launched as Vae::decode / Vae::encode launch it (csrc/vae.cuh vae_conv and friends), from reference-layout
   fp32 weights that the library weight-norms and packs.  Device pointers; kmul = 3 when precision is 1 (bf16x3), else 1.
   kind 0 conv:       Conv1d(cin -> cout, taps, dilation dil, padding dil * (taps - 1) / 2), taps odd.  x: bf16 A [B, T, kmul*cin];
                      weight_v [cout, cin, taps], weight_g [cout].  raw: fp32 [B, T, cout] (+ resid [B, T, cout], which may alias raw);
                      act: bf16 SnakeBeta(alpha, beta)(raw) [B, T, kmul*cout] ([hi | lo | hi] in bf16x3).
   kind 1 conv-T:     ConvTranspose1d(cin -> cout, k = 2 stride, stride (even), padding stride / 2).  weight_v [cin, cout, 2 stride],
                      weight_g [cin]; raw [B, T*stride, cout], act [B, T*stride, kmul*cout].
   kind 2 strided:    Conv1d(cin -> cout, k = 2 stride, stride, padding ceil(stride / 2)).  x [B, T*stride, kmul*cin]; T output rows.
   kind 3 wave out:   Conv1d(cin -> 1, k = 7, padding 3, no bias) of x [B, T, kmul*cin]; weight_v [1, cin, 7], weight_g [1]; out fp32 [B, T].
   kind 4 stem:       Conv1d(1 -> cout, k = 7, padding 3) of fp32 audio x [B, T]; weight_v [cout, 1, 7]; raw and act (both required).
   kind 5 sample:     x fp32 enc [B*T, 2*cout] (mean | scale), noise fp32 [B, cout, T] or NULL -> out z [B, cout, T].
   kind 6 latent:     x fp32 z [B, cin, T] -> act bf16 [B, T, kmul*cin].
   bias [cout] (kinds 0, 1, 2, 4).  act needs alpha and beta ([cout], SnakeBeta's log-scale parameters).  w_packed (optional, kinds 0-4)
   receives the weights the kernel read: kinds 0-2 bf16 [N, taps', cin_pad] with N = stride*cout for kind 1 (row r*cout + co: phase r),
   cout otherwise, taps' = 3 for kind 1, 2*stride for kind 2, cin_pad = kmul*cin rounded up to 64, each tap [hi(cin) | hi | lo | 0];
   kinds 3 and 4 fp32 [7][C]. */
typedef struct {
  int32_t kind, precision;
  int32_t B, T, cin, cout, taps, dil, stride;
  const float* weight_v; const float* weight_g; const float* bias;
  const float* alpha; const float* beta;
  const void* x; const float* resid; const float* noise;
  float* raw; void* act; float* out;
  void* w_packed;
} ezb_test_vae_args;
int ezb_test_vae(int device, const ezb_test_vae_args* args, void* stream);
/* The FP8 mode's kernels (precision 2), launched as the model launches them.  Device pointers.
   kind 0: LayerNorm (eps 1e-5, weight / bias [D]) + AdaLN modulate (shift / scale [D], one row for all rows; NULL: none) of x [M, D] fp32
           -> q [M, D] e4m3 and row scales s [M] (s = amax / 448 of the row, q = e4m3(y * 448 / amax)).
   kind 1: GEGLU projection of A = q [M, D] e4m3 with row scales s: W [2*inner, D], b [2*inner] fp32 in the reference layout ([hidden; gate]
           rows), packed and quantised by the library; out [M, inner] bf16.
   kind 2: packed self-attention QKV projection of A = (q, s) with the heads epilogue: W [3D, D] fp32 reference layout ([q; k; v]); outputs and
           their layout as ezb_test_heads with nsec 3, kinds {0, 1, 2} and the staged packed-3 variant.
   w_q / w_s (optional, kinds 1 and 2): receive the e4m3 weight and its row scales as the GEMM read them (packed row order). */
typedef struct {
  int32_t kind, M, D;
  const float* x; const float* weight; const float* bias; const float* shift; const float* scale;
  void* q; float* s;
  int32_t inner; const float* w; const float* b; void* out;
  int32_t B, L, H, dh;
  const float* norm_q; const float* norm_k; const float* inv_freq; int32_t rope;
  void* q_out; void* k_out; void* vt_out; int32_t ld_qk, dvp, Lpad;
  void* w_q; float* w_s;
} ezb_test_fp8_args;
int ezb_test_fp8(int device, const ezb_test_fp8_args* args, void* stream);
/* The bandwidth kernels of a DiT step (csrc/elementwise.cuh), launched with the grid and shared memory the model uses (csrc/dit.cuh
   ln_launch and friends).  Device pointers; those of kind 0 and final_conv's w and b are read as float4 and must be 16-byte aligned
   (kind 0: mod_bstride a multiple of 4).  Every argument, alignment included, is checked before any device work.
   kind 0 LayerNorm (eps 1e-5) of the row [x | x2 (+ x3)] (x fp32 [M, D1], x2 / x3 optional fp32 [M, D2]) with affine w / b [D1 + D2]
          (both NULL: cast only), optional AdaLN modulate y (1 + scale) + shift (shift / scale rows at (row / rows_per_batch) * mod_bstride,
          single source only), optional precombined affine G / Cc [D1] (the ln_gc kernel: y = (x - mu) rstd G + Cc) -> out bf16
          [M, kmul (D1 + D2)] ([hi | lo | hi] when kmul is 3).  variant: 0 the kernel Dit::ln selects under the current option "ln_variant";
          1 generic, 2 / 3 register-resident with 1 / 8 CTAs per SM minimum, 4 precombined affine (G, Cc), 5 register-resident concat
          (D1 == D2): 2-5 take D1 = 1024 or 1152 and kmul 1 only.
   kind 1 per-head LayerNorm + RoPE + attention layout (qk_prep) of x [B*L, ld_in] (fp32, or bf16 when in_bf16): nsec sections of kinds
          kinds[s] (0 q, 1 k, 2 v) at column offsets col_off[s]; norm_q / norm_k [2][dh] weight | bias; inv_freq [dh/2] (NULL: no RoPE);
          f32_out[s] fp32 [B, H, L, dh] and / or bf_out[s] bf16 (q, k: [B, H, L, ld_qk]; v: V^T [B, H, dv_pad, Lpad], rows dh..dv_pad zeroed).
   kind 2 patch_pack: x [B, C, L], gt [B, C, L] or NULL, gt_mask [B, L] uint8 or NULL, mask_embed [C] -> out bf16 [B*L, kmul Kp].
   kind 3 final_conv: x = y fp32 [B*L, C], w [3][C][C] (tap, in, out), b [C], lens [B] or NULL -> out fp32 [B, C, L] (frames < lens[b]).
   kind 4 small_linear: out[r, n] = act(out_scale (x[r, :] . w[n, :]) + b[n]) + add[r, n], r < R, n < N, over K; act 0 none, 1 SiLU; b and
          add optional; row pitches ld_in, ld_add, ld_out.
   kind 5 timestep_embed: x = t fp32 [M] -> out fp32 [M, 256] = [cos | sin]. */
typedef struct {
  int32_t kind, variant;
  int32_t M, D1, D2, kmul, mod_bstride, rows_per_batch;
  int32_t B, L, C, Kp, H, dh, nsec, in_bf16;
  int32_t kinds[3], col_off[3];
  int32_t ld_in, ld_qk, Lpad, dv_pad;
  int32_t R, N, K, ld_add, ld_out, act;
  float out_scale;
  const void* x; const float* x2; const float* x3; const float* w; const float* b;
  const float* shift; const float* scale; const float* G; const float* Cc;
  const float* gt; const uint8_t* gt_mask; const float* mask_embed; const float* add; const int32_t* lens;
  const float* norm_q; const float* norm_k; const float* inv_freq;
  void* out; float* f32_out[3]; void* bf_out[3];
} ezb_test_step_args;
int ezb_test_step(int device, const ezb_test_step_args* args, void* stream);
/* The kernels that turn the prompt and the reference audio into DiT inputs (csrc/t5.cuh, the ControlNet stem's conv1d_direct_kernel),
   launched one at a time with the grid and shared memory T5::forward and Dit::controlnet_stem use.  Device pointers; in, w and the fp32
   outputs of kinds 0 and 1, and q, k, v of kind 5, are read / written as float4 and must be 16-byte aligned.  Every argument is checked
   before any device work.
   kind 0 t5_embed:      in int32 ids [M] (clamped to [0, vocab)), w table fp32 [vocab, D] -> out fp32 [M, D].  D a multiple of 4.
   kind 1 t5_rms:        in x fp32 [M, D], w [D], eps -> out bf16 [M, kmul D] ([hi | lo | hi] when kmul is 3) and / or out32 fp32 [M, D].
                         D a multiple of 4.
   kind 2 t5_heads:      in qkv fp32 [B*L, 3*H*dk] -> out q, out32 k, out_v v, fp32 [B, H, L, dk] each.
   kind 3 t5_bias:       in int32 buckets [L, L] (each < the rows of w), w relative_attention_bias fp32 [num_buckets, H] -> out fp32 [H, L, L].
   kind 4 t5_gated_gelu: in u fp32 [M, 2F] = [h | g] -> out bf16 [M, kmul F] = gelu_new(g) h.
   kind 5 T5 attention:  attn_simt_kernel with scale 1: in q, k, v fp32 [B, H, L, dk] (dk a multiple of 4, at most 96), b position bias fp32
                         [H, L, L], key_mask uint8 [B, L] (NULL: every key) -> out bf16 [B, L, kmul H dk].
   kind 6 conv1d_direct: convolution `stage` of the ControlNet stem (widths c0, c1 = cond_blocks, D = embed_dim) for conditions of 2L samples,
                         w [Cout, Cin, K], b [Cout]:
                         0 conv_in         Conv1d(1 -> c0, 1) of in [B, 1, 2L] -> out [B, c0, 2L];
                         1 conv3 + SiLU    Conv1d(c0 + 1 -> c0 + 1, 3, padding 1) of [in | 0], in [B, c0, 2L] (the all-zero mask channel is
                                           not read) -> out [B, c0 + 1, 2L];
                         2 conv3 s2 + SiLU Conv1d(c0 + 1 -> c1, 3, stride 2, padding 1) of in [B, c0 + 1, 2L] -> out [B, c1, L];
                         3 conv_out        Conv1d(c1 -> D, 1) of in [B, c1, L] -> out transposed, [B, L, D]. */
typedef struct {
  int32_t kind, M, D, F, kmul, vocab;
  float eps;
  int32_t B, L, H, dk;
  int32_t c0, c1, stage;
  const void* in; const float* w; const float* b; const float* k; const float* v; const uint8_t* key_mask;
  void* out; float* out32; float* out_v;
} ezb_test_cond_args;
int ezb_test_cond(int device, const ezb_test_cond_args* args, void* stream);
/* impl 0: fp32 CUDA-core kernel (q, k, v fp32 [B,H,L,dh]; dh a multiple of 4 up to 96) writing out [B, Lq, H dh]; 3: the same kernel writing
   bf16x3 rows [B, Lq, 3 H dh] = [hi | lo | hi], as the bf16x3 parity mode runs it; 1: the tensor-core kernel variant the options select
   (dh a multiple of 8 up to 80); 4 / 6 / 7 / 8: that generation forced (8 takes dh 64 or 72 only); +100: q / k rows of 80 elements for
   dh = 72 (the product's layout) instead of a 64-multiple.  B, H, Lq, Lk >= 1 and B H <= 65535.  Bad arguments are refused before any
   device work. */
int ezb_test_attention(int device, const void* q, const void* k, const void* vt, const uint8_t* key_mask, void* out_bf16,
                       int B, int H, int Lq, int Lk, int dh, int impl, void* stream);
/* Self-attention (Lq = Lk = L, no key mask) of a padded batch, as ezb_test_attention with the same impl codes: lens DEVICE int32 [B],
   sample b attends over its first lens[b] tokens; output rows >= lens[b] are written as zeros. */
int ezb_test_attention_lens(int device, const void* q, const void* k, const void* vt, const int32_t* lens, void* out_bf16, int B, int H,
                            int L, int dh, int impl, void* stream);

/* runtime switches for A/B measurements and profiling (csrc/host.cuh, csrc/ezb.cu list them): e.g. "pair_gemm" (1 = 2-CTA cluster tiles
   sharing the weight tile, default), "attn6" / "attn7" / "attn8" / "attn_res" (attention variant), "ln_variant", "skip" (profiling: kernel classes not launched).  Products never need to call this. */
int ezb_set_option(const char* name, int value);
/* incremented by every ezb_set_option call: hosts that cache captured CUDA graphs key them on it (options change kernel selection) */
unsigned long long ezb_option_epoch(void);
/* debugging aid: with option "gemm_debug"=1 (library built with EZB_DEBUG=1), CTA 0 of each 2-CTA cluster GEMM accumulates cycle
   counters (gemm.cuh GemmShape::dbg); this reads and resets them */
int ezb_debug_read(unsigned long long* out8);
/* accounting: kernels launched by this library so far (process-wide); per-GEMM CUDA-event timing for bench.py's roofline leg */
unsigned long long ezb_launch_count(void);
void ezb_launch_count_add(unsigned long long n); /* launches replayed from a captured CUDA graph */
/* stand-alone LayerNorm launches of one kernel (the variant numbers of ezb_test_step: 1 generic, 2 / 3 register-resident, 4 precombined
   affine, 5 register-resident concat) so far, process-wide; a captured CUDA graph counts once, at capture */
unsigned long long ezb_ln_launch_count(int variant);
/* tensor-core attention launches of one generation (4, 6, 7 or 8) so far, process-wide; a captured CUDA graph counts once, at capture */
unsigned long long ezb_attn_launch_count(int generation);
int ezb_prof_gemm_begin(void);
int ezb_prof_gemm_end(int* launches, double* flops, double* ms);
int ezb_prof_gemm_stats(double min_flops, int* launches, double* flops, double* ms); /* subset of the last profile */

#ifdef __cplusplus
}
#endif
#endif
