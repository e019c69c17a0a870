"""Sampling loop: src/inference.py:26-107 and src/inference_controlnet.py:27-128 re-hosted on the CUDA library.

Differences from the reference loop, all additive:
  * batched prompts (the reference hard-codes batch 1, src/inference.py:67; SURVEY 0.8): prompt i gets its own
    torch.Generator(seed + i), so prompt 0 of a batch reproduces the reference's B=1 run with the same seed;
  * step-invariant work (context embedding, cross-attention K/V, timestep/AdaLN tables) is computed once per clip;
  * CFG + rescale + DDIM update is one fused kernel (ezb_cfg_ddim_step); so is CFG + rescale + DPM-Solver++ (ezb_cfg_dpm_step) when the
    scheduler is a `scheduler.DPMSolverMultistepScheduler` -- the swap a diffusers user makes with `noise_scheduler`; eta is then ignored;
  * clips of different lengths in one batch (`lengths=`): the batch is padded to `audio_frames` and every prompt's frames come out as
    that prompt run alone at its own length computes them (same seed, same bits); one length-aware VAE decode turns the padded batch into
    waveforms.  Inpainting joins in with `padded_gt=True`: gt / gt_mask padded like the batch, ignored past each clip's end.
The call still accepts `tokenizer` / `text_encoder` like the reference; pass `text_embeds=(emb, mask, uncond_emb,
uncond_mask)` to use cached T5 outputs instead (BASELINE configs use cached embeddings).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib


def scale_shift_re(x, scale, shift):
    """src/utils/utils.py:24-25."""
    return (x / scale) - shift


def encode_text(tokenizer, text_encoder, params, text_raw, neg_text, device):
    """src/inference.py:38-50."""
    ml = params["text_encoder"]["max_length"]
    tb = tokenizer(text_raw, max_length=ml, padding="max_length", truncation=True, return_tensors="pt")
    text, mask = tb.input_ids.to(device), tb.attention_mask.to(device).bool()
    text = text_encoder(input_ids=text, attention_mask=mask).last_hidden_state
    ub = tokenizer(neg_text, max_length=ml, padding="max_length", truncation=True, return_tensors="pt")
    utext, umask = ub.input_ids.to(device), ub.attention_mask.to(device).bool()
    utext = text_encoder(input_ids=utext, attention_mask=umask).last_hidden_state
    return text, mask, utext, umask


def _ddim_step(model_out, latents, noise, B, Cc, L, gs, gr, coef, lens=None):
    arr = (C.c_float * 5)(*coef)
    _lib.check(_lib.lib().ezb_cfg_ddim_step(latents.device.index, _lib.ptr(model_out), _lib.ptr(latents), _lib.ptr(noise), B, Cc, L, float(gs or 0.0), float(gr or 0.0),
                                            arr, _lib.stream_ptr(), _lib.ptr(lens)))


def _dpm_step(model_out, latents, history, noise, B, Cc, L, gs, gr, coef, order, lens=None):
    arr = (C.c_float * 7)(*coef)
    _lib.check(_lib.lib().ezb_cfg_dpm_step(latents.device.index, _lib.ptr(model_out), _lib.ptr(latents), _lib.ptr(history), _lib.ptr(noise), B, Cc, L,
                                           float(gs or 0.0), float(gr or 0.0), arr, int(order), _lib.stream_ptr(), _lib.ptr(lens)))


def check_lengths(lengths, B: int, L: int, gt=None, controlnet=None, padded_gt=False):
    """Validates per-prompt clip lengths (frames) against the batch size and the padded length L, on the host, before any device work.
    Inpainting goes with lengths only when the caller states, with `padded_gt=True`, that `gt` (and its mask) is the padded (B,C,L) batch
    whose frames past each clip's end are to be ignored; a ControlNet never does."""
    if gt is not None and not padded_gt:
        raise NotImplementedError("per-prompt lengths with inpainting (gt) need padded_gt=True: gt / gt_mask padded to the batch's length, "
                                  "ignored past each clip's end")
    if controlnet is not None:
        raise NotImplementedError("per-prompt lengths with a ControlNet are not supported: its stem convolutions cross the clip ends")
    lens = [int(v) for v in lengths]
    if any(v != w for v, w in zip(lens, lengths)):
        raise ValueError(f"lengths must be whole frame counts, got {list(lengths)}")
    if len(lens) != B:
        raise ValueError(f"lengths lists one length per prompt: got {len(lens)} for {B} prompts")
    if any(v < 1 or v > L for v in lens):
        raise ValueError(f"every length must lie in 1..{L} (the padded length), got {lens}")
    if gt is not None and (tuple(gt.shape[:1]) + tuple(gt.shape[2:])) != (B, L):
        raise ValueError(f"gt must be the padded batch ({B}, C, {L}), got {tuple(gt.shape)}")
    return lens


@torch.no_grad()
def sample_latents(unet, noise_scheduler, text, text_mask, uncond_text=None, uncond_mask=None, gt=None, gt_mask=None,
                   audio_frames=500, guidance_scale=3, guidance_rescale=0.0, ddim_steps=50, eta=1, random_seed=2024,
                   controlnet=None, condition=None, conditioning_scale=1.0, init_noise=None, step_noise=None, device=None,
                   use_graphs=True, paste_gt=True, lengths=None, padded_gt=False):
    """Denoising loop on cached text embeddings.  text (B,Lc,ctx) / text_mask (B,Lc); uncond_* (1 or B rows) when
    guidance_scale is truthy.  gt / gt_mask (B,C,L) for inpainting.  Returns the final latents (B,C,L) fp32 on device.
    `init_noise` / `step_noise` inject the RNG draws (parity tests); otherwise per-prompt generators are used.
    `paste_gt`: apply the final `pred[~gt_mask] = gt[~gt_mask]` here (standalone use); `inference()` passes False and pastes after
    scale_shift_re like src/inference.py:102-105.
    `lengths`: one clip length (frames, 1..audio_frames) per prompt, or None.  The batch is padded to `audio_frames`; prompt b's initial
    noise and per-step draws are made at its own shape (1, C, lengths[b]), so its frames < lengths[b] of the result equal a run of that
    prompt alone at audio_frames = lengths[b] with the same seed (random_seed must then be per-prompt or None; injected noise is not
    accepted).  Frames past a prompt's length are zero.  One captured graph serves every mix of lengths at the same padded length.
    gt / gt_mask go with lengths under `padded_gt=True` (refused without it): both are padded to audio_frames like the batch, the solo run
    is the one with gt[b:b+1, :, :lengths[b]] and the same slice of
    the mask; what gt and gt_mask hold past a clip's end is ignored."""
    if lengths is not None:
        lengths = check_lengths(lengths, text.shape[0], int(audio_frames), gt, controlnet, padded_gt)
        if init_noise is not None or step_noise is not None:
            raise ValueError("lengths draws the noise per prompt: init_noise / step_noise cannot be injected")
    dev_index = unet._h.dev_index   # the loop runs where the denoiser's weights live
    if device is not None:
        d = torch.device(device)
        if d.type != "cuda" or (d.index is not None and d.index != dev_index):
            raise ValueError(f"sample_latents(device={d}) but the denoiser lives on cuda:{dev_index}")
    device = torch.device("cuda", dev_index)
    if lengths is not None and gt is not None:   # past a clip's end nothing of gt is used: those frames count as regenerated
        gt, gt_mask = gt.to(device=device, dtype=torch.float32).clone(), gt_mask.to(device).bool().clone()
        for b, n in enumerate(lengths):
            gt[b, :, n:] = 0
            gt_mask[b, ..., n:] = True
    # every launch below (noise draws, the C-ABI calls, graph capture and replay) targets `device`, whatever the caller's current device is
    with torch.cuda.device(device):
        lat = _sample_latents_on_device(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, gt, gt_mask, audio_frames, guidance_scale,
                                        guidance_rescale, ddim_steps, eta, random_seed, controlnet, condition, conditioning_scale, init_noise,
                                        step_noise, device, use_graphs, lengths)
        if gt is not None and paste_gt:
            lat = torch.where(gt_mask.to(device).bool().expand_as(lat), lat, gt.to(device=device, dtype=lat.dtype))
        return lat


def _sample_latents_on_device(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, gt, gt_mask, audio_frames, guidance_scale,
                              guidance_rescale, ddim_steps, eta, random_seed, controlnet, condition, conditioning_scale, init_noise, step_noise,
                              device, use_graphs, lengths=None):
    B = text.shape[0]
    Cc = unet.cfg["out_chans"]
    L = int(audio_frames)
    use_cfg = bool(guidance_scale)
    dpm = getattr(noise_scheduler, "kind", "ddim") == "dpm"   # DPM-Solver++: multistep, keeps the previous x0 prediction per sample
    noise_scheduler.set_timesteps(ddim_steps)
    timesteps = [int(t) for t in noise_scheduler.timesteps]

    gens = None
    if init_noise is None:
        gens = []
        per_prompt = isinstance(random_seed, (list, tuple))   # one seed per prompt (batching front-end): prompt i ~ Generator(seed_i)
        if per_prompt and len(random_seed) != B:
            raise ValueError(f"random_seed lists one seed per prompt: got {len(random_seed)} for {B} prompts")
        for i in range(B):
            g = torch.Generator(device=device)
            if per_prompt:
                g.manual_seed(int(random_seed[i]))
            elif random_seed is not None:
                g.manual_seed(int(random_seed) + i)
            else:
                g.seed()
            gens.append(g)
        if lengths is None:
            latents = torch.cat([torch.randn((1, Cc, L), generator=g, device=device) for g in gens], 0)
        else:   # each prompt's draw at its own shape, placed into the zeroed padded batch
            latents = torch.zeros((B, Cc, L), device=device)
            for b, g in enumerate(gens):
                latents[b, :, :lengths[b]] = torch.randn((1, Cc, lengths[b]), generator=g, device=device)[0]
    else:
        latents = init_noise.to(device=device, dtype=torch.float32).clone()
    latents = latents.contiguous()

    text = text.to(device=device, dtype=torch.float32)
    text_mask = text_mask.to(device).bool()
    if use_cfg:
        if uncond_text.shape[0] == 1 and B > 1:
            uncond_text, uncond_mask = uncond_text.expand(B, -1, -1), uncond_mask.expand(B, -1)
        ctx = torch.cat([text, uncond_text.to(device=device, dtype=torch.float32)], 0).contiguous()
        cmask = torch.cat([text_mask, uncond_mask.to(device).bool()], 0).contiguous()
    else:
        ctx, cmask = text.contiguous(), text_mask.contiguous()
    Be = ctx.shape[0]

    gt_c = m8 = None
    if gt is not None:
        gt = gt.to(device=device, dtype=torch.float32).contiguous()
        gm = gt_mask.to(device)
        gt_c = torch.cat([gt, gt], 0).contiguous() if use_cfg else gt
        m1 = unet._h._mask_u8(gm, B, L, device)
        m8 = torch.cat([m1, m1], 0).contiguous() if use_cfg else m1

    unet.set_context(ctx, cmask)
    unet.set_timesteps(timesteps)
    if controlnet is not None:
        controlnet.set_context(ctx, cmask)
        controlnet.set_timesteps(timesteps)
        cond = condition.to(device=device, dtype=torch.float32)
        cond_c = torch.cat([cond, cond], 0).contiguous() if use_cfg else cond.contiguous()
        skips = [torch.empty(Be, L, unet.cfg["embed_dim"], device=device, dtype=torch.float32) for _ in range(controlnet.half)]

    # ---- the loop.  Every step is the same launch sequence on static buffers, so the WHOLE schedule (all steps: ~365 kernels each) is captured
    # once into one CUDA graph per shape / schedule and replayed with a single launch; the per-step Gaussian draws of DDIM (eta > 0; and of
    # sde-dpmsolver++) stay in
    # PyTorch -- same generators, same order, same per-step tensor shapes as the step-by-step loop -- and are simply made up front into one
    # [steps, B, C, L] buffer (one graph per step would interleave 50 launches and 200 RNG kernels).
    # Everything a captured launch sequence bakes in is in the key: shapes (incl. the context length, which fixes the cross-attention K/V layout and
    # tensor maps), the schedule, the guidance constants, which ControlNet handle (its serial, not id(): ids are recycled) and the
    # library's option epoch (ezb_set_option changes kernel selection).
    nsteps = len(timesteps)
    draw = noise_scheduler.draws_noise if dpm else bool(eta and eta > 0)
    sampler = (noise_scheduler.algorithm_type, noise_scheduler.solver_order) if dpm else ("ddim", float(eta or 0.0))
    key = (B, Be, L, lengths is not None, int(ctx.shape[1]), tuple(timesteps), use_cfg, float(guidance_scale or 0.0), float(guidance_rescale or 0.0), sampler,
           gt is not None, controlnet._h.serial if controlnet is not None else 0, float(conditioning_scale), int(_lib.lib().ezb_option_epoch()))
    cache = unet.__dict__.setdefault("_loop_cache", {})
    st = cache.get(key) if use_graphs else None
    if st is None:
        st = dict(lat=torch.empty(B, Cc, L, device=device, dtype=torch.float32),
                  x_in=torch.empty(Be, Cc, L, device=device, dtype=torch.float32) if use_cfg else None,
                  out=torch.empty(Be, Cc, L, device=device, dtype=torch.float32),
                  noise=torch.empty(nsteps, B, Cc, L, device=device, dtype=torch.float32) if draw else None,
                  hist=torch.empty(B, Cc, L, device=device, dtype=torch.float32) if dpm else None,   # the previous step's x0 prediction
                  gt=None if gt_c is None else torch.empty_like(gt_c), m8=None if m8 is None else torch.empty_like(m8),
                  cond=None, skips=None, graph=None, launches=0,
                  lens=torch.empty(Be, device=device, dtype=torch.int32) if lengths is not None else None)   # [lengths | lengths] under CFG
        if st["noise"] is not None and lengths is not None:
            st["noise"].zero_()   # the padded frames are never read; keep them finite
        if controlnet is not None:
            st["cond"] = torch.empty_like(cond_c)
            st["skips"] = skips
        if use_graphs:
            if len(cache) >= 4:
                cache.clear()
            cache[key] = st
    st["lat"].copy_(latents)
    if gt_c is not None:
        st["gt"].copy_(gt_c)
        st["m8"].copy_(m8)
    if controlnet is not None:
        st["cond"].copy_(cond_c)
    lens = st["lens"]
    if lens is not None:   # read by the kernels when they run: a replayed graph follows the new lengths
        lens.copy_(torch.tensor(lengths * (Be // B), dtype=torch.int32))
    lat, x_in, out, noise_all = st["lat"], st["x_in"], st["out"], st["noise"]
    if noise_all is not None:  # RNG stays in PyTorch, outside the graph: step i, prompt b draws (1, C, L) from prompt b's generator, in step order
        for i in range(nsteps):
            if step_noise is not None:
                noise_all[i].copy_(step_noise[i])
            elif lengths is None:
                for b, g in enumerate(gens):
                    noise_all[i, b:b + 1].normal_(generator=g)
            else:   # the draw a solo run makes: a contiguous (1, C, lengths[b]) tensor
                for b, g in enumerate(gens):
                    noise_all[i, b, :, :lengths[b]] = torch.empty((1, Cc, lengths[b]), device=device).normal_(generator=g)[0]

    # DPM-Solver++: every step's coefficients and order, computed once, before any capture
    dpm_coef = [noise_scheduler.step_coefficients(i) for i in range(nsteps)] if dpm else None

    def one_step(i, t):
        if use_cfg:
            x_in[:B].copy_(lat)
            x_in[B:].copy_(lat)
            xi = x_in
        else:
            xi = lat
        sk = None
        if controlnet is not None:
            sk = controlnet.forward_step(xi, i, st["cond"], conditioning_scale, gt=st["gt"], gt_mask_u8=st["m8"], outs=st["skips"])
        unet.forward_step(xi, i, gt=st["gt"], gt_mask_u8=st["m8"], controlnet_skips=sk, out=out, lengths=lens)
        if dpm:
            coef, order = dpm_coef[i]
            _dpm_step(out, lat, st["hist"], None if noise_all is None else noise_all[i], B, Cc, L, guidance_scale if use_cfg else 0.0, guidance_rescale,
                      coef, order, None if lens is None else lens[:B])
            return
        coef = noise_scheduler.step_coefficients(t, float(eta or 0.0))
        _ddim_step(out, lat, None if noise_all is None else noise_all[i], B, Cc, L, guidance_scale if use_cfg else 0.0, guidance_rescale, coef,
                   None if lens is None else lens[:B])

    L_ = _lib.lib()
    if use_graphs and st["graph"] is not None:
        st["graph"].replay()
        L_.ezb_launch_count_add(st["launches"])
    else:
        for i, t in enumerate(timesteps):   # eager pass: warms caches (tensor maps, function attributes) and IS this call's result
            one_step(i, t)
        if use_graphs:
            snap = lat.clone()
            g = torch.cuda.CUDAGraph()
            n0 = L_.ezb_launch_count()
            with torch.cuda.graph(g):
                for i, t in enumerate(timesteps):
                    one_step(i, t)
            st["launches"] = int(L_.ezb_launch_count() - n0)
            st["graph"] = g
            lat.copy_(snap)  # capture does not execute; keep the eager result
    return lat.clone()   # the inpainting paste happens after scale_shift_re, in inference() (src/inference.py:102-105)


@torch.no_grad()
def inference(autoencoder, unet, gt, gt_mask, tokenizer, text_encoder, params, noise_scheduler, text_raw, neg_text=None,
              audio_frames=500, guidance_scale=3, guidance_rescale=0.0, ddim_steps=50, eta=1, random_seed=2024, device="cuda",
              text_embeds=None, controlnet=None, condition=None, conditioning_scale=1.0, lengths=None, padded_gt=False):
    """Signature of src/inference.py:26-37 (+ keyword-only extensions).  Returns the waveform tensor (B,1,480*L).
    With `lengths` (one clip length in frames per prompt, batch padded to audio_frames; see sample_latents) it returns a list of B
    waveforms (1, 480*lengths[b]) from one length-aware VAE decode of the padded batch (each equal to the decode of that clip alone).
    gt / gt_mask go with lengths under `padded_gt=True`, as in sample_latents: padded to audio_frames, ignored past each clip's end."""
    if lengths is not None:
        lengths = check_lengths(lengths, len(text_raw) if text_embeds is None else text_embeds[0].shape[0], int(audio_frames), gt, controlnet,
                                padded_gt)
    if neg_text is None:
        neg_text = [""]
    if text_embeds is not None:
        text, text_mask, uncond_text, uncond_mask = text_embeds
    elif tokenizer is not None:
        text, text_mask, uncond_text, uncond_mask = encode_text(tokenizer, text_encoder, params, text_raw, neg_text, device)
    else:  # src/inference.py:51-53
        raise ValueError("either tokenizer/text_encoder or text_embeds is required (the denoiser is text-conditioned)")
    latents = sample_latents(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, gt, gt_mask, audio_frames, guidance_scale,
                             guidance_rescale, ddim_steps, eta, random_seed, controlnet, condition, conditioning_scale, device=device, paste_gt=False,
                             lengths=lengths, padded_gt=padded_gt)
    pred = scale_shift_re(latents, params["autoencoder"]["scale"], params["autoencoder"]["shift"])
    if gt is not None:  # src/inference.py:104-105: pred[~gt_mask] = gt[~gt_mask], with the raw gt, after the rescale
        pred = torch.where(gt_mask.to(pred.device).bool().expand_as(pred), pred, gt.to(device=pred.device, dtype=pred.dtype))
    if lengths is not None:   # what the paste put past a clip's end is never read by the decode
        w = autoencoder(embedding=pred, lengths=lengths)
        hop = w.shape[-1] // pred.shape[-1]
        return [w[b, :, :hop * n] for b, n in enumerate(lengths)]
    return autoencoder(embedding=pred)
