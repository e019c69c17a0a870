"""Sampling loop: src/inference.py:26-107 and src/inference_controlnet.py:27-128 re-hosted on the CUDA library.

Differences from the reference loop, all additive:
  * batched prompts (the reference hard-codes batch 1, src/inference.py:67; SURVEY 0.8): prompt i gets its own
    torch.Generator(seed + i), so prompt 0 of a batch reproduces the reference's B=1 run with the same seed;
  * step-invariant work (context embedding, cross-attention K/V, timestep/AdaLN tables) is computed once per clip;
  * CFG + rescale + DDIM update is one fused kernel (ezb_cfg_ddim_step); so is CFG + rescale + DPM-Solver++ (ezb_cfg_dpm_step) when the
    scheduler is a `scheduler.DPMSolverMultistepScheduler` -- the swap a diffusers user makes with `noise_scheduler`; eta is then ignored;
  * audio-to-audio variations (SDEdit): `start_index=` / `init_latents=` start sample b at its own schedule index from a noised latent
    (`OobleckDecoder.encode_noised`); the batch runs the steps from the smallest start on, each sample's update switched on from its own;
  * clips of different lengths in one batch (`lengths=`): the batch is padded to `audio_frames` and every prompt's frames come out as
    that prompt run alone at its own length computes them (same seed, same bits); one length-aware VAE decode turns the padded batch into
    waveforms.  Inpainting joins in with `padded_gt=True`: gt / gt_mask padded like the batch, ignored past each clip's end.
  * clips longer than the denoiser's window (`sample_long_latents`): overlapping windows denoised as one batch, guided per window and
    crossfaded on the device into one long prediction at every step (MultiDiffusion; ezb_window_gather / ezb_window_blend), with or
    without a ControlNet whose per-window conditions are cached once per call (ezb_controlnet_forward_cached), or with inpainting
    operands (gt / gt_mask) whose window rows are cut once per call;
  * seamless loops (`sample_loop_latents`): the same windowed loop on a circle, the windows wrapping around the loop's end and shifting
    by a golden-ratio stride at every step (ezb_loop_gather / ezb_loop_blend).
  * timelines of prompts (`sample_timeline_latents`): the windowed loop with one row per (window, prompt segment active in it), the rows of a
    window sharing one unconditional row, each row's prediction weighted by its segment's weight (ezb_timeline_gather / _guide / _blend).
The call still accepts `tokenizer` / `text_encoder` like the reference; pass `text_embeds=(emb, mask, uncond_emb,
uncond_mask)` to use cached T5 outputs instead (BASELINE configs use cached embeddings).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
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


def make_generators(random_seed, B: int, device):
    """One torch.Generator per prompt: seed_i of a list, seed + i of an int, a random seed for None."""
    per_prompt = isinstance(random_seed, (list, tuple))   # one seed per prompt (batching front-end): prompt i ~ Generator(seed_i)
    if per_prompt and len(random_seed) != B:
        raise ValueError(f"random_seed lists one seed per prompt: got {len(random_seed)} for {B} prompts")
    gens = []
    for i in range(B):
        g = torch.Generator(device=device)
        if per_prompt:
            g.manual_seed(int(random_seed[i]))
        elif random_seed is not None:
            g.manual_seed(int(random_seed) + i)
        else:
            g.seed()
        gens.append(g)
    return gens


def _slot_table(struct, rows):
    """rows [steps][B] of (guidance_scale, guidance_rescale, coef, flags) -> a device int32 block of `struct` (ezb_ddim_slot / ezb_dpm_slot)."""
    arr = (struct * sum(len(r) for r in rows))()
    for a, (gs, gr, coef, flags) in zip(arr, (e for r in rows for e in r)):
        a.guidance_scale, a.guidance_rescale, a.flags = gs, gr, flags
        a.coef[:] = coef
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.int32)


@torch.no_grad()
def sample_latents(unet, noise_scheduler, text, text_mask, uncond_text=None, uncond_mask=None, gt=None, gt_mask=None,
                   audio_frames=500, guidance_scale=3, guidance_rescale=0.0, ddim_steps=50, eta=1, random_seed=2024,
                   controlnet=None, condition=None, conditioning_scale=1.0, init_noise=None, step_noise=None, device=None,
                   use_graphs=True, paste_gt=True, lengths=None, padded_gt=False, *, start_index=None, init_latents=None, generators=None):
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
    the mask; what gt and gt_mask hold past a clip's end is ignored.
    `start_index` (one schedule index per prompt, 0..ddim_steps-1) with `init_latents` (B, C, audio_frames), the noised start of an
    audio-to-audio variation: the loop runs schedule indices min(start_index) .. ddim_steps-1, the DiT on the whole batch at every step,
    and sample b is updated from its own start_index[b] on (DPM-Solver++: with begin_index = start_index[b]); before that its latents stay
    as given.  `generators` (one per prompt, already past the initial draw) make the per-step draws, in step order, for the steps each
    sample runs; `step_noise[i]` (when injected) is the draw of schedule step i.  Each sample's bits do not depend on the other samples'
    starts, and a batch of one start equals a run of the truncated schedule."""
    if start_index is not None:
        start_index = _check_start(start_index, text.shape[0], int(ddim_steps), int(audio_frames), init_latents, controlnet, gt)
        if init_noise is not None:
            raise ValueError("a variation starts from init_latents: init_noise cannot be given with start_index")
    elif init_latents is not None or generators is not None:
        raise ValueError("init_latents / generators go with start_index")
    if lengths is not None:
        lengths = check_lengths(lengths, text.shape[0], int(audio_frames), gt, controlnet, padded_gt)
        if init_noise is not None or (step_noise is not None and start_index is None):
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
                                        step_noise, device, use_graphs, lengths, start_index, init_latents, generators)
        if gt is not None and paste_gt:
            lat = torch.where(gt_mask.to(device).bool().expand_as(lat), lat, gt.to(device=device, dtype=lat.dtype))
        return lat


def _check_start(start_index, B: int, steps: int, L: int, init_latents, controlnet, gt):
    """Validates a variation's per-prompt start indices and start latents on the host."""
    if controlnet is not None or gt is not None:
        raise NotImplementedError("a variation (start_index) runs without a ControlNet and without inpainting")
    ks = [int(k) for k in start_index]
    if len(ks) != B or any(k != v for k, v in zip(ks, start_index)) or any(k < 0 or k >= steps for k in ks):
        raise ValueError(f"start_index lists one schedule index in 0..{steps - 1} per prompt ({B} prompts), got {list(start_index)}")
    if init_latents is None or init_latents.dim() != 3 or init_latents.shape[0] != B or init_latents.shape[2] != L:
        raise ValueError(f"start_index needs init_latents of shape ({B}, C, {L})")
    return ks


def _sample_latents_on_device(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, gt, gt_mask, audio_frames, guidance_scale,
                              guidance_rescale, ddim_steps, eta, random_seed, controlnet, condition, conditioning_scale, init_noise, step_noise,
                              device, use_graphs, lengths=None, start=None, init_latents=None, generators=None):
    B = text.shape[0]
    Cc = unet.cfg["out_chans"]
    L = int(audio_frames)
    use_cfg = bool(guidance_scale)
    dpm = getattr(noise_scheduler, "kind", "ddim") == "dpm"   # DPM-Solver++: multistep, keeps the previous x0 prediction per sample
    noise_scheduler.set_timesteps(ddim_steps)
    timesteps = [int(t) for t in noise_scheduler.timesteps]

    gens = None
    if start is not None:   # a variation: the start latents are given, the generators are past their initial draw
        gens = generators
        latents = init_latents.to(device=device, dtype=torch.float32).clone()
    elif init_noise is None:
        gens = make_generators(random_seed, B, device)
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
    k0 = 0 if start is None else min(start)   # the first schedule index the loop runs
    nsteps = len(timesteps) - k0
    draw = noise_scheduler.draws_noise if dpm else bool(eta and eta > 0)
    if draw and start is not None and step_noise is None and (gens is None or len(gens) != B):
        raise ValueError("a variation that draws step noise needs one generator per prompt (generators=) or step_noise")
    sampler = (noise_scheduler.algorithm_type, noise_scheduler.solver_order) if dpm else ("ddim", float(eta or 0.0))
    key = (B, Be, L, lengths is not None, int(ctx.shape[1]), tuple(timesteps), use_cfg, float(guidance_scale or 0.0), float(guidance_rescale or 0.0), sampler,
           gt is not None, controlnet._h.serial if controlnet is not None else 0, float(conditioning_scale), int(_lib.lib().ezb_option_epoch()))
    if start is not None:
        key = key + (("start", k0),)
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
                  lens=torch.empty(Be, device=device, dtype=torch.int32) if lengths is not None else None,   # [lengths | lengths] under CFG
                  slots=None)   # a variation: the per-step slot table [steps, B] of the slots kernels
        if st["noise"] is not None and (lengths is not None or start is not None):
            st["noise"].zero_()   # the padded frames, and the draws of samples that have not started, are never read; keep them finite
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
    if noise_all is not None and start is not None:   # a variation: sample b draws at the steps it runs, at its own shape
        for i in range(nsteps):
            for b in range(B):
                if k0 + i < start[b]:
                    continue
                n = L if lengths is None else lengths[b]
                if step_noise is not None:
                    noise_all[i, b, :, :n] = step_noise[k0 + i][b, :, :n]
                else:
                    noise_all[i, b, :, :n] = torch.empty((1, Cc, n), device=device).normal_(generator=gens[b])[0]
    elif noise_all is not None:  # RNG stays in PyTorch, outside the graph: step i, prompt b draws (1, C, L) from prompt b's generator, in step order
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
    dpm_coef = [noise_scheduler.step_coefficients(i) for i in range(nsteps)] if dpm and start is None else None
    if start is not None:   # the slots kernels' constants of every step, in device memory before any capture: sample b is active from start[b]
        gs_, gr_ = float(guidance_scale) if use_cfg else 0.0, float(guidance_rescale or 0.0)
        cfg_flag = _lib.SLOT_ACTIVE | (_lib.SLOT_CFG if use_cfg else 0)
        rows = []
        for i in range(k0, len(timesteps)):
            row = []
            for b in range(B):
                if i < start[b]:
                    row.append((0.0, 0.0, (0.0,) * (7 if dpm else 5), 0))
                elif dpm:
                    coef, order = noise_scheduler.step_coefficients(i, begin_index=start[b])
                    row.append((gs_, gr_, coef, cfg_flag | (_lib.SLOT_ORDER2 if order == 2 else 0)))
                else:
                    row.append((gs_, gr_, noise_scheduler.step_coefficients(timesteps[i], float(eta or 0.0)), cfg_flag))
            rows.append(row)
        table = _slot_table(_lib.DpmSlot if dpm else _lib.DdimSlot, rows).to(device)
        if st["slots"] is None:
            st["slots"] = table
        else:   # read when the kernels run: a replayed graph follows the new starts
            st["slots"].copy_(table)
        words = (10 if dpm else 8) * B

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
        if start is not None:
            j = i - k0
            sl = st["slots"][j * words:(j + 1) * words]
            nz = None if noise_all is None else noise_all[j]
            lb = None if lens is None else lens[:B]
            if dpm:
                _lib.check(_lib.lib().ezb_cfg_dpm_step_slots(device.index, _lib.ptr(out), _lib.ptr(lat), _lib.ptr(st["hist"]), _lib.ptr(nz), _lib.ptr(sl),
                                                             B, Cc, L, _lib.stream_ptr(), _lib.ptr(lb)))
            else:
                _lib.check(_lib.lib().ezb_cfg_ddim_step_slots(device.index, _lib.ptr(out), _lib.ptr(lat), _lib.ptr(nz), _lib.ptr(sl), B, Cc, L,
                                                              _lib.stream_ptr(), _lib.ptr(lb)))
            return
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
        for i in range(k0, len(timesteps)):   # eager pass: warms caches (tensor maps, function attributes) and IS this call's result
            one_step(i, timesteps[i])
        if use_graphs:
            snap = lat.clone()
            g = torch.cuda.CUDAGraph()
            n0 = L_.ezb_launch_count()
            with torch.cuda.graph(g):
                for i in range(k0, len(timesteps)):
                    one_step(i, timesteps[i])
            st["launches"] = int(L_.ezb_launch_count() - n0)
            st["graph"] = g
            lat.copy_(snap)  # capture does not execute; keep the eager result
    return lat.clone()   # the inpainting paste happens after scale_shift_re, in inference() (src/inference.py:102-105)


def window_plan(n: int, window: int, overlap: int):
    """The windows (start, length) of a clip of n frames for windowed denoising (include/ezb200.h, ezb_window_gather): n <= window is one
    window [0, n); otherwise windows of `window` frames start every window - overlap frames, and the last one ends at the clip's end."""
    if not 1 <= overlap <= window // 2:
        raise ValueError(f"overlap must lie in 1..{window // 2} frames (half the window of {window}), got {overlap}")
    if n <= window:
        return [(0, n)]
    hop = window - overlap
    count = -(-(n - window) // hop) + 1
    return [(k * hop, window) for k in range(count - 1)] + [(n - window, window)]


def window_weights(k: int, count: int, length: int, window: int, overlap: int):
    """fp32 crossfade weights of window k of count over its `length` frames: min(1, (j + 1) / (overlap + 1) after the first window,
    (window - j) / (overlap + 1) before the last), as the blend kernel computes them."""
    j = np.arange(length)
    w = np.ones(length, dtype=np.float32)
    o1 = np.float32(overlap + 1)
    if k > 0:
        w = np.minimum(w, (j + 1).astype(np.float32) / o1)
    if k < count - 1:
        w = np.minimum(w, (window - j).astype(np.float32) / o1)
    return w


def long_plan(lengths, window: int, overlap: int):
    """Windows of a batch of long clips, laid out clip by clip as consecutive DiT rows: (the plan table [(first row, count, N)] per clip,
    the windows [(clip, start, length)] in row order)."""
    table, windows = [], []
    for b, n in enumerate(lengths):
        ws = window_plan(n, window, overlap)
        table.append((len(windows), len(ws), n))
        windows += [(b, s, ln) for s, ln in ws]
    return table, windows


def check_long(lengths, B: int, window: int, overlap: int, use_cfg: bool, max_rows: int, max_len: int):
    """Validates a windowed run on the host before any device work; returns (lengths, plan table, windows)."""
    lens = [int(v) for v in lengths]
    if len(lens) != B or any(v != w for v, w in zip(lens, lengths)) or any(v < 1 for v in lens):
        raise ValueError(f"lengths lists one positive whole frame count per prompt ({B} prompts), got {list(lengths)}")
    if not 2 <= int(window) <= max_len:
        raise ValueError(f"window must lie in 2..{max_len} frames (the denoiser's max_len), got {window}")
    table, windows = long_plan(lens, int(window), int(overlap))
    rows = len(windows) * (2 if use_cfg else 1)
    if rows > max_rows:
        raise ValueError(f"{len(windows)} windows{' x 2 (CFG)' if use_cfg else ''} = {rows} DiT rows exceed the row capacity {max_rows} "
                         f"(2 * max_batch): needs max_batch >= {-(-rows // 2)}")
    return lens, table, windows


GOLDEN_STRIDE = 0.3819660112501051   # 2 - phi: the per-step shift of a loop's windows, as a fraction of the loop


def loop_plan(n: int, window: int, overlap: int):
    """The windows of a seamless loop of n frames (frame n - 1 followed by frame 0; include/ezb200.h, ezb_loop_gather): (count, length).
    n <= window is one window of n frames, the whole circle; otherwise ceil(n / (window - overlap)) windows of `window` frames, window k
    starting at floor(k * n / count) (plus the step's offset, mod n, loop_starts), so neighbours overlap by at least `overlap` frames."""
    if not 1 <= overlap <= window // 2:
        raise ValueError(f"overlap must lie in 1..{window // 2} frames (half the window of {window}), got {overlap}")
    if n < 2:
        raise ValueError(f"a loop needs at least 2 frames, got {n}")
    if n <= window:
        return 1, n
    return -(-n // (window - overlap)), window


def loop_starts(n: int, count: int, offset: int):
    """Start frames of a loop's windows at a step with offset r: ((k * n) // count + r) mod n."""
    return [((k * n) // count + offset) % n for k in range(count)]


def loop_stride(n: int) -> int:
    """R = floor(n * (2 - phi) + 0.5): the golden-ratio stride by which a loop's windows move from one step to the next."""
    return int(np.floor(n * GOLDEN_STRIDE + 0.5))


def loop_offsets(lengths, nsteps: int):
    """The shift schedule [steps][B]: r_{i,b} = (i * R_b) mod N_b.  It moves the seam between windows, and the DiT input edges, to a
    different place at every step; for a one-window loop it is what denoises the wrap-around in context."""
    return [[(i * loop_stride(n)) % n for n in lengths] for i in range(nsteps)]


def loop_weights(count: int, length: int, overlap: int):
    """fp32 weights of a loop window over its `length` frames: 1 for a one-window loop, else min(1, (j + 1) / (overlap + 1),
    (length - j) / (overlap + 1)) -- both ends taper, since on a circle every window has two neighbours -- as the blend kernel computes them."""
    if count == 1:
        return np.ones(length, dtype=np.float32)
    j = np.arange(length)
    o1 = np.float32(overlap + 1)
    return np.minimum(np.float32(1), np.minimum((j + 1).astype(np.float32) / o1, (length - j).astype(np.float32) / o1))


def check_loop(lengths, B: int, window: int, overlap: int, use_cfg: bool, max_rows: int, max_len: int):
    """Validates a seamless-loop run on the host before any device work; returns (lengths, plan table [(first row, count, N)] per loop,
    the windows [(loop, 0, length)] in row order -- their starts move with every step's offset)."""
    lens = [int(v) for v in lengths]
    if len(lens) != B or any(v != w for v, w in zip(lens, lengths)) or any(v < 2 for v in lens):
        raise ValueError(f"lengths lists one whole frame count >= 2 per loop ({B} loops), got {list(lengths)}")
    if not 2 <= int(window) <= max_len:
        raise ValueError(f"window must lie in 2..{max_len} frames (the denoiser's max_len), got {window}")
    table, windows = [], []
    for b, n in enumerate(lens):
        count, ln = loop_plan(n, int(window), int(overlap))
        table.append((len(windows), count, n))
        windows += [(b, 0, ln)] * count
    rows = len(windows) * (2 if use_cfg else 1)
    if rows > max_rows:
        raise ValueError(f"{len(windows)} windows{' x 2 (CFG)' if use_cfg else ''} = {rows} DiT rows exceed the row capacity {max_rows} "
                         f"(2 * max_batch): needs max_batch >= {-(-rows // 2)}")
    return lens, table, windows


def segment_weights(s: int, e: int, n: int, transition: int):
    """fp32 weights of a timeline segment [s, e) over a clip of n frames with a transition of T frames: min(1, (f - s + T + 1) / (T + 1),
    (e + T - f) / (T + 1)) on [s - T, e + T), 0 elsewhere, each ratio an IEEE fp32 division, as ezb_timeline_blend computes them.  1 inside
    the segment, tapering over T frames on either side: abutting segments crossfade over 2T frames centred on their boundary."""
    f = np.arange(n, dtype=np.int64)
    t1 = np.float32(transition + 1)
    a = np.minimum(np.float32(1), np.minimum((f - s + transition + 1).astype(np.float32) / t1, (e + transition - f).astype(np.float32) / t1))
    a[(f < s - transition) | (f >= e + transition)] = 0
    return a


def timeline_plan(segments, lengths, window: int, overlap: int, transition: int):
    """Rows of a batch of timelines: segments[b] lists clip b's [(s, e)] frame ranges in timeline order.  The windows are long_plan's; a
    segment is active in a window when [s - T, e + T) meets it, and each (window, active segment) is one conditioned DiT row, clip by clip,
    window by window, then in timeline order.  Returns (the plan table and windows of long_plan, the rows [(window, clip, segment index)],
    the spans [(first row, row count)] per clip)."""
    table, windows = long_plan(lengths, window, overlap)
    rows, spans = [], []
    for b, (first, count, _) in enumerate(table):
        r0 = len(rows)
        for k in range(first, first + count):
            _, ws, ln = windows[k]
            rows += [(k, b, q) for q, (s, e) in enumerate(segments[b]) if s - transition < ws + ln and e + transition > ws]
        spans.append((r0, len(rows) - r0))
    return table, windows, rows, spans


def check_timeline(segments, lengths, B: int, window: int, overlap: int, transition: int, use_cfg: bool, max_rows: int, max_len: int):
    """Validates a timeline run on the host before any device work: every segment non-empty and inside its clip, the segments of a clip
    covering all of its frames, T >= 0, the window rules of check_long and the row capacity (the conditioned rows, plus one unconditional
    row per window under CFG).  Returns (lengths, plan table, windows, rows, spans) as timeline_plan gives them."""
    lens, _, _ = check_long(lengths, B, window, overlap, False, 1 << 62, max_len)   # the window rules; the capacity is checked below
    if len(segments) != B:
        raise ValueError(f"segments lists one timeline per clip: got {len(segments)} for {B} clips")
    T = int(transition)
    if T != transition or T < 0:
        raise ValueError(f"transition must be a whole frame count >= 0, got {transition}")
    segs = []
    for b, (clip, n) in enumerate(zip(segments, lens)):
        if len(clip) < 1:
            raise ValueError(f"timeline {b} has no segment")
        cover = np.zeros(n + 1, dtype=np.int64)
        out = []
        for s, e in clip:
            if int(s) != s or int(e) != e or not 0 <= s < e <= n:
                raise ValueError(f"timeline {b}: segment frames [{s}, {e}) must be whole, non-empty and inside the clip's {n} frames")
            cover[int(s)] += 1
            cover[int(e)] -= 1
            out.append((int(s), int(e)))
        gap = np.flatnonzero(np.cumsum(cover)[:n] == 0)
        if gap.size:
            raise ValueError(f"timeline {b}: no segment covers frame {int(gap[0])} (the segments must cover all {n} frames)")
        segs.append(out)
    table, windows, rows, spans = timeline_plan(segs, lens, int(window), int(overlap), T)
    n_rows = len(rows) + (len(windows) if use_cfg else 0)
    if n_rows > max_rows:
        uncond = f" + {len(windows)} unconditional rows (CFG)" if use_cfg else ""
        raise ValueError(f"{len(rows)} timeline rows{uncond} = {n_rows} DiT rows exceed the row capacity {max_rows} (2 * max_batch): "
                         f"needs max_batch >= {-(-n_rows // 2)}")
    return lens, table, windows, rows, spans


@torch.no_grad()
def sample_timeline_latents(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, segments, lengths, window, overlap, transition,
                            guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, *, device=None, use_graphs=True):
    """Long clips from a timeline of prompts: the windowed loop of sample_long_latents where window k of clip b carries one conditioned row
    per segment active in it (timeline_plan) and, under guidance, all of them share the window's one unconditional row.  segments[b] lists
    clip b's [(prompt, s, e)]: `prompt` a row of text (P, Lc, ctx) / text_mask (P, Lc), [s, e) its frames; `transition` (frames) the
    taper T of segment_weights.  uncond_text / uncond_mask have one row, or one per clip.  At every step ezb_timeline_gather cuts the rows,
    the DiT runs them as one batch, ezb_timeline_guide guides each conditioned row against its window's uncond row (the rescale's std over
    one window), and ezb_timeline_blend weighs row r's prediction by its window's crossfade weight times its segment's weight, driving the
    DDIM or DPM-Solver++ update of the long latent.  Returns the latents (B, C, max(lengths)) fp32 on the device, zero past each clip's end.
    Seeds as in sample_long_latents.  The whole schedule is one captured graph; its tables are read on the device, so a replay follows new
    boundaries, prompts and lengths with the same row layout.  A one-segment timeline is sample_long_latents with that prompt, bit for bit."""
    B = len(segments)
    use_cfg = bool(guidance_scale)
    desc = unet._h.desc
    frames = [[(s, e) for _, s, e in clip] for clip in segments]
    lens, table, windows, rows, spans = check_timeline(frames, lengths, B, window, overlap, transition, use_cfg, int(desc.max_batch),
                                                       int(desc.max_len))
    P = text.shape[0]
    prompt = [segments[b][q][0] for _, b, q in rows]
    if any(int(p) != p or not 0 <= p < P for p in prompt):
        raise ValueError(f"every segment's prompt must be a row index of text (0..{P - 1})")
    T = int(transition)
    tl = dict(rows=[(k, *frames[b][q], T) for k, b, q in rows], spans=spans, prompt=[int(p) for p in prompt])
    dev_index = unet._h.dev_index
    if device is not None:
        d = torch.device(device)
        if d.type != "cuda" or (d.index is not None and d.index != dev_index):
            raise ValueError(f"sample_timeline_latents(device={d}) but the denoiser lives on cuda:{dev_index}")
    device = torch.device("cuda", dev_index)
    with torch.cuda.device(device):
        return _sample_long_on_device(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, lens, table, windows, int(window),
                                      int(overlap), guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, device, use_graphs,
                                      timeline=tl)


@torch.no_grad()
def sample_loop_latents(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, lengths, window, overlap, guidance_scale,
                        guidance_rescale, ddim_steps, eta, random_seed, *, offsets=None, init_noise=None, step_noise=None, device=None,
                        use_graphs=True):
    """Seamless loops: windowed denoising (as sample_long_latents) on a circle, where frame lengths[b] - 1 of loop b is followed by its
    frame 0.  At step i the windows of loop b (loop_plan) start at ((k * N_b) // count + r_{i,b}) mod N_b, with the golden-ratio shift
    schedule r = loop_offsets(lengths, steps); the gather (ezb_loop_gather) wraps around, the DiT denoises every window of every loop as
    one batch, each window is guided on its own, and the blend (ezb_loop_blend, weights loop_weights) drives the DDIM or DPM-Solver++ update
    of the loop latent.  Returns the latents (B, C, max(lengths)) fp32 on the device, zero past each loop's end.  Loop b's generator
    (random_seed as in sample_latents) draws the initial and per-step noise at (1, C, lengths[b]).  The whole schedule is one captured
    graph; the plan and every step's offsets are read on the device.
    `offsets` ([steps][B] ints) replaces the shift schedule; `init_noise` (B, C, max(lengths)) and `step_noise` (one (B, C, max(lengths))
    per step) replace the generator draws; frames past a loop's end are not read.  With all offsets 0, a loop that fits one window is
    sample_latents at that length, bit for bit; adding d to every offset with the noise rolled by d rolls the result by d, bit for bit."""
    B = text.shape[0]
    use_cfg = bool(guidance_scale)
    desc = unet._h.desc
    lens, table, windows = check_loop(lengths, B, window, overlap, use_cfg, int(desc.max_batch), int(desc.max_len))
    noise_scheduler.set_timesteps(ddim_steps)
    nsteps, N, Cc = len(noise_scheduler.timesteps), max(lens), unet.cfg["out_chans"]
    if offsets is None:
        offsets = loop_offsets(lens, nsteps)
    offs = [[int(v) for v in row] for row in offsets]
    if len(offs) != nsteps or any(len(row) != B for row in offs):
        raise ValueError(f"offsets lists {B} ints per step for {nsteps} steps")
    if init_noise is not None and tuple(init_noise.shape) != (B, Cc, N):
        raise ValueError(f"init_noise must be {(B, Cc, N)}, got {tuple(init_noise.shape)}")
    if step_noise is not None and (len(step_noise) != nsteps or any(tuple(s.shape) != (B, Cc, N) for s in step_noise)):
        raise ValueError(f"step_noise lists one {(B, Cc, N)} tensor per step ({nsteps} steps)")
    dev_index = unet._h.dev_index
    if device is not None:
        d = torch.device(device)
        if d.type != "cuda" or (d.index is not None and d.index != dev_index):
            raise ValueError(f"sample_loop_latents(device={d}) but the denoiser lives on cuda:{dev_index}")
    device = torch.device("cuda", dev_index)
    with torch.cuda.device(device):
        return _sample_long_on_device(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, lens, table, windows, int(window),
                                      int(overlap), guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, device, use_graphs,
                                      offsets=offs, init_noise=init_noise, step_noise=step_noise)


@torch.no_grad()
def sample_long_latents(unet, noise_scheduler, text, text_mask, uncond_text=None, uncond_mask=None, lengths=(), window=500, overlap=100,
                        guidance_scale=3, guidance_rescale=0.0, ddim_steps=50, eta=1, random_seed=2024, device=None, use_graphs=True, *,
                        controlnet=None, condition=None, conditioning_scale=1.0, gt=None, gt_mask=None):
    """Windowed denoising (MultiDiffusion) of clips longer than the denoiser's window: clip b has lengths[b] frames; at every step its
    latent is cut into overlapping windows of `window` frames (`overlap` frames of overlap, window_plan), the DiT denoises every window
    of every clip as one batch, each window's prediction is guided and rescaled on its own (the rescale's std is over one window, as over one
    trained-length clip), and the blend of the windows' predictions (crossfade weights, window_weights) drives the DDIM or DPM-Solver++
    update of the long latent.  Returns the latents (B, C, max(lengths)) fp32 on the device, zero past each clip's end.
    Prompt b's generator (random_seed as in sample_latents) draws the initial noise and each step's noise at (1, C, lengths[b]): the draws
    a solo sample_latents at that length makes, so a clip that fits one window comes out as that call computes it, bit for bit.
    The windows (x 2 under CFG) must fit the DiT's row capacity: one forward per step.  The whole schedule is one captured graph.
    `controlnet` (a DiTControlNet with the DiT's rows) with `condition` (B, 1, 2 * max(lengths)) fp32: clip b's condition frames are valid
    up to 2 * lengths[b], and every clip must be at least one window long, so that every window is full-length.  Window [s, s + window) of
    clip b is conditioned on condition[b, :, 2s:2s + 2 * window]; those rows go through the ControlNet's stem once per call, into its
    condition cache (DiTControlNet.set_condition), and every step reads the cache at its timestep with `conditioning_scale`.
    `gt` (B, C, max(lengths)) fp32 with `gt_mask` (B, max(lengths)) or (B, C, max(lengths)) bool, identical across channels, True =
    regenerate: inpainting over long clips.  gt is the raw VAE latent of each clip, as sample_latents takes it; neither is read past clip
    b's lengths[b] frames.  Once per call every window row's slice of gt (ezb_window_gather, zeros past a window's length) and of the mask
    (ones past a window's length) is cut into static buffers that every step's DiT forward reads, so a replayed graph follows new clips and
    masks.  The latents are returned without the paste: the caller applies pred[~mask] = gt[~mask] after scale_shift_re, as inference()
    does.  A clip that fits one window comes out as sample_latents with that gt and mask computes it, bit for bit."""
    B = text.shape[0]
    use_cfg = bool(guidance_scale)
    desc = unet._h.desc
    max_rows, max_len = int(desc.max_batch), int(desc.max_len)
    if gt is not None and (controlnet is not None or condition is not None):
        raise NotImplementedError("inpainting (gt) over long clips runs without a ControlNet")
    if (gt is None) != (gt_mask is None):
        raise ValueError("gt and gt_mask go together")
    if controlnet is not None or condition is not None:
        if controlnet is None or condition is None:
            raise ValueError("controlnet and condition go together")
        cdesc = controlnet._h.desc
        max_rows, max_len = min(max_rows, int(cdesc.max_batch)), min(max_len, int(cdesc.max_len))
    lens, table, windows = check_long(lengths, B, window, overlap, use_cfg, max_rows, max_len)
    if controlnet is not None:
        if tuple(condition.shape) != (B, 1, 2 * max(lens)):
            raise ValueError(f"condition must be (B, 1, 2 * max(lengths)) = {(B, 1, 2 * max(lens))}, got {tuple(condition.shape)}")
        if min(lens) < int(window):
            raise ValueError(f"with a ControlNet every clip must be at least one window ({int(window)} frames) long, got {lens}: its stem "
                             "convolutions cross a shorter window's end")
    if gt is not None:
        N, Cc = max(lens), unet.cfg["out_chans"]
        if tuple(gt.shape) != (B, Cc, N) or tuple(gt_mask.shape) not in ((B, N), (B, Cc, N)):
            raise ValueError(f"gt must be (B, C, max(lengths)) = {(B, Cc, N)} and gt_mask (B, max(lengths)) or (B, C, max(lengths)), got "
                             f"{tuple(gt.shape)} and {tuple(gt_mask.shape)}")
    dev_index = unet._h.dev_index
    if device is not None:
        d = torch.device(device)
        if d.type != "cuda" or (d.index is not None and d.index != dev_index):
            raise ValueError(f"sample_long_latents(device={d}) but the denoiser lives on cuda:{dev_index}")
    device = torch.device("cuda", dev_index)
    with torch.cuda.device(device):
        return _sample_long_on_device(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, lens, table, windows, int(window),
                                      int(overlap), guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, device, use_graphs,
                                      controlnet, condition, conditioning_scale, gt, gt_mask)


def _guide_windows(out, guided, W, Cc, Lw, gs, gr, wlens):
    """The guided, rescaled v of every window: ezb_cfg_ddim_step on the window rows with coefficients (1, 0, 0, 1, 0) and no noise writes
    0 * x0 + 1 * (1 * v + 0 * x) = v into `guided`, exactly the v that kernel computes for its own update (same cluster reduction, same
    rescale ratio bits).  `guided` (W, C, Lw) plays the latents and must hold finite values (0 * x must be 0)."""
    _ddim_step(out, guided, None, W, Cc, Lw, gs, gr, (1.0, 0.0, 0.0, 1.0, 0.0), wlens)


def _sample_long_on_device(unet, noise_scheduler, text, text_mask, uncond_text, uncond_mask, lens, table, windows, Lw, O, guidance_scale,
                           guidance_rescale, ddim_steps, eta, random_seed, device, use_graphs, controlnet=None, condition=None,
                           conditioning_scale=1.0, gt=None, gt_mask=None, offsets=None, init_noise=None, step_noise=None, timeline=None):
    """The windowed loop of sample_long_latents, and of sample_loop_latents when `offsets` ([steps][B] ints, the loops' shifts) is given:
    then the circular gather and blend (ezb_loop_gather / ezb_loop_blend) read step i's row of a device offsets table in place of the
    linear ones, and the schedule is captured into a cache of its own.  init_noise / step_noise (loops only) replace the draws.
    `timeline` (sample_timeline_latents: the rows [(window, s, e, T)], the spans [(first row, count)] per clip and the text row of every
    conditioned row) switches the gather, the guidance and the blend to ezb_timeline_gather / _guide / _blend, with R conditioned rows and
    one unconditional row per window under CFG, and a cache of its own."""
    B, W, N = len(lens), len(windows), max(lens)
    loop, tl = offsets is not None, timeline is not None
    R = len(timeline["rows"]) if tl else W   # conditioned DiT rows
    Cc = unet.cfg["out_chans"]
    use_cfg = bool(guidance_scale)
    if gt is not None:   # the mask as one byte per frame (B, N); checked before any RNG draw
        m1 = unet._h._mask_u8(gt_mask, B, N, device)
    dpm = getattr(noise_scheduler, "kind", "ddim") == "dpm"
    noise_scheduler.set_timesteps(ddim_steps)
    timesteps = [int(t) for t in noise_scheduler.timesteps]
    nsteps = len(timesteps)
    gens = make_generators(random_seed, B, device)
    latents = torch.zeros((B, Cc, N), device=device)
    for b, g in enumerate(gens):
        if init_noise is None:
            latents[b, :, :lens[b]] = torch.randn((1, Cc, lens[b]), generator=g, device=device)[0]
        else:
            latents[b, :, :lens[b]] = init_noise[b, :, :lens[b]].to(device=device, dtype=torch.float32)

    # the T5 context of every window row: [text of each window | "" of each window]; a timeline's rows take their segment's prompt
    clip_of = torch.tensor([b for b, _, _ in windows], device=device)
    text_of = torch.tensor(timeline["prompt"], device=device) if tl else clip_of
    text = text.to(device=device, dtype=torch.float32)[text_of]
    text_mask = text_mask.to(device).bool()[text_of]
    if use_cfg:
        if uncond_text.shape[0] == 1:
            uncond_text, uncond_mask = uncond_text.expand(B, -1, -1), uncond_mask.expand(B, -1)
        ctx = torch.cat([text, uncond_text.to(device=device, dtype=torch.float32)[clip_of]], 0).contiguous()
        cmask = torch.cat([text_mask, uncond_mask.to(device).bool()[clip_of]], 0).contiguous()
    else:
        ctx, cmask = text.contiguous(), text_mask.contiguous()
    Be = ctx.shape[0]
    unet.set_context(ctx, cmask)
    unet.set_timesteps(timesteps)
    if controlnet is not None:   # every window row's condition, [cond | cond] under CFG, through the stem once into the condition cache
        cond = condition.to(device=device, dtype=torch.float32)
        rows = torch.stack([cond[b, :, 2 * s:2 * (s + Lw)] for b, s, _ in windows])
        controlnet.set_condition(torch.cat([rows] * (Be // W), 0))
        controlnet.set_context(ctx, cmask)
        controlnet.set_timesteps(timesteps)

    # Everything the captured launches bake in is in the key: shapes (B, window rows, the longest clip, window, overlap, context length), the
    # schedule, the guidance constants, the sampler, the ControlNet handle (its serial) and scale, and the library's option epoch.  The plan
    # table, the lengths and the ControlNet's condition cache are read on the device.
    draw = noise_scheduler.draws_noise if dpm else bool(eta and eta > 0)
    sampler = (noise_scheduler.algorithm_type, noise_scheduler.solver_order) if dpm else ("ddim", float(eta or 0.0))
    key = (B, W, N, Lw, O, int(ctx.shape[1]), tuple(timesteps), use_cfg, float(guidance_scale or 0.0), float(guidance_rescale or 0.0), sampler,
           controlnet._h.serial if controlnet is not None else 0, float(conditioning_scale), int(_lib.lib().ezb_option_epoch()), gt is not None)
    if tl:   # the row layout; the row and span tables are read on the device
        key = key + (("timeline", R),)
    cache = unet.__dict__.setdefault("_loop_long_cache" if loop else "_timeline_cache" if tl else "_long_cache", {})
    st = cache.get(key) if use_graphs else None
    if st is None:
        st = dict(lat=torch.empty(B, Cc, N, device=device), x_in=torch.empty(Be, Cc, Lw, device=device), out=torch.empty(Be, Cc, Lw, device=device),
                  guided=torch.zeros(R, Cc, Lw, device=device) if use_cfg else None, v=torch.empty(B, Cc, N, device=device),
                  noise=torch.zeros(nsteps, B, Cc, N, device=device) if draw else None,
                  hist=torch.empty(B, Cc, N, device=device) if dpm else None,
                  plan=torch.empty(B * 3, device=device, dtype=torch.int32), wlens=torch.empty(Be, device=device, dtype=torch.int32),
                  lens=torch.empty(B, device=device, dtype=torch.int32), graph=None, launches=0,
                  skips=None if controlnet is None else [torch.empty(Be, Lw, unet.cfg["embed_dim"], device=device) for _ in range(controlnet.half)],
                  gt=None if gt is None else torch.empty(Be, Cc, Lw, device=device),
                  m8=None if gt is None else torch.empty(Be, Lw, device=device, dtype=torch.uint8),
                  offs=torch.empty(nsteps, B, device=device, dtype=torch.int32) if loop else None,
                  rows=torch.empty(R * 4, device=device, dtype=torch.int32) if tl else None,
                  spans=torch.empty(B * 2, device=device, dtype=torch.int32) if tl else None)
        if use_graphs:
            if len(cache) >= 2:
                cache.clear()
            cache[key] = st
    st["lat"].copy_(latents)
    st["plan"].copy_(torch.tensor([e for row in table for e in row], dtype=torch.int32))
    if gt is not None:   # constant over the schedule: every window row's gt and mask bytes, cut once per call into the static buffers
        gsrc = gt.to(device=device, dtype=torch.float32).contiguous()
        _lib.check(_lib.lib().ezb_window_gather(device.index, _lib.ptr(gsrc), _lib.ptr(st["gt"]), _lib.ptr(st["plan"]), B, Cc, N, W, Lw, O, Be // W,
                                                _lib.stream_ptr()))
        j = np.arange(Lw)   # window frame j of row (b, s, ln) is clip frame s + j of b; past ln it reads the trailing 1 (regenerate)
        idx = np.stack([np.where(j < ln, b * N + s + j, B * N) for b, s, ln in windows])
        src = torch.cat([m1.reshape(-1), torch.ones(1, device=device, dtype=torch.uint8)])
        st["m8"].copy_(src[torch.from_numpy(np.tile(idx, (Be // W, 1))).to(device)])
    if tl:   # read when the kernels run: a replayed graph follows new boundaries, transitions and prompts with the same rows
        st["rows"].copy_(torch.tensor([e for row in timeline["rows"] for e in row], dtype=torch.int32))
        st["spans"].copy_(torch.tensor([e for row in timeline["spans"] for e in row], dtype=torch.int32))
        st["wlens"].copy_(torch.tensor([windows[row[0]][2] for row in timeline["rows"]] + ([ln for _, _, ln in windows] if use_cfg else []),
                                       dtype=torch.int32))
    else:
        st["wlens"].copy_(torch.tensor([ln for _, _, ln in windows] * (Be // W), dtype=torch.int32))
    st["lens"].copy_(torch.tensor(lens, dtype=torch.int32))
    if loop:   # read when the kernels run: a replayed graph follows new offsets
        st["offs"].copy_(torch.tensor(offsets, dtype=torch.int32))
    lat, x_in, out, v, noise_all, plan = st["lat"], st["x_in"], st["out"], st["v"], st["noise"], st["plan"]
    if noise_all is not None:   # step i, prompt b: the (1, C, lengths[b]) draw of a solo run, in step order
        for i in range(nsteps):
            for b, g in enumerate(gens):
                if step_noise is None:
                    noise_all[i, b, :, :lens[b]] = torch.empty((1, Cc, lens[b]), device=device).normal_(generator=g)[0]
                else:
                    noise_all[i, b, :, :lens[b]] = step_noise[i][b, :, :lens[b]].to(device=device, dtype=torch.float32)
    dpm_coef = [noise_scheduler.step_coefficients(i) for i in range(nsteps)] if dpm else None
    gs, gr = (float(guidance_scale), float(guidance_rescale or 0.0)) if use_cfg else (0.0, 0.0)
    L_ = _lib.lib()

    def one_step(i, t):
        if loop:
            _lib.check(L_.ezb_loop_gather(device.index, _lib.ptr(lat), _lib.ptr(x_in), _lib.ptr(plan), _lib.ptr(st["offs"][i]), B, Cc, N, W, Lw, O,
                                          Be // W, _lib.stream_ptr()))
        elif tl:
            _lib.check(L_.ezb_timeline_gather(device.index, _lib.ptr(lat), _lib.ptr(x_in), _lib.ptr(plan), _lib.ptr(st["rows"]), B, Cc, N, W, R, Lw, O,
                                              int(use_cfg), _lib.stream_ptr()))
        else:
            _lib.check(L_.ezb_window_gather(device.index, _lib.ptr(lat), _lib.ptr(x_in), _lib.ptr(plan), B, Cc, N, W, Lw, O, Be // W,
                                            _lib.stream_ptr()))
        if controlnet is None:
            unet.forward_step(x_in, i, gt=st["gt"], gt_mask_u8=st["m8"], out=out, lengths=st["wlens"])
        else:   # every window is full-length: no lengths, which the DiT does not combine with ControlNet skips
            sk = controlnet.forward_step(x_in, i, conditioning_scale=conditioning_scale, outs=st["skips"])
            unet.forward_step(x_in, i, controlnet_skips=sk, out=out)
        src = out
        if use_cfg and tl:
            _lib.check(L_.ezb_timeline_guide(device.index, _lib.ptr(out), _lib.ptr(st["guided"]), _lib.ptr(st["rows"]), _lib.ptr(st["wlens"]), R, W,
                                             Cc, Lw, gs, gr, _lib.stream_ptr()))
            src = st["guided"]
        elif use_cfg:
            _guide_windows(out, st["guided"], W, Cc, Lw, gs, gr, st["wlens"][:W])
            src = st["guided"]
        if loop:
            _lib.check(L_.ezb_loop_blend(device.index, _lib.ptr(src), _lib.ptr(v), _lib.ptr(plan), _lib.ptr(st["offs"][i]), B, Cc, N, W, Lw, O,
                                         _lib.stream_ptr()))
        elif tl:
            _lib.check(L_.ezb_timeline_blend(device.index, _lib.ptr(src), _lib.ptr(v), _lib.ptr(plan), _lib.ptr(st["rows"]), _lib.ptr(st["spans"]),
                                             B, Cc, N, W, R, Lw, O, _lib.stream_ptr()))
        else:
            _lib.check(L_.ezb_window_blend(device.index, _lib.ptr(src), _lib.ptr(v), _lib.ptr(plan), B, Cc, N, W, Lw, O, _lib.stream_ptr()))
        nz = None if noise_all is None else noise_all[i]
        if dpm:
            coef, order = dpm_coef[i]
            _dpm_step(v, lat, st["hist"], nz, B, Cc, N, 0.0, 0.0, coef, order, st["lens"])
        else:
            _ddim_step(v, lat, nz, B, Cc, N, 0.0, 0.0, noise_scheduler.step_coefficients(t, float(eta or 0.0)), st["lens"])

    if use_graphs and st["graph"] is not None:
        st["graph"].replay()
        L_.ezb_launch_count_add(st["launches"])
    else:
        for i, t in enumerate(timesteps):   # eager pass: warms caches and IS this call's result
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
            lat.copy_(snap)
    return lat.clone()


@torch.no_grad()
def inference(autoencoder, unet, gt, gt_mask, tokenizer, text_encoder, params, noise_scheduler, text_raw, neg_text=None,
              audio_frames=500, guidance_scale=3, guidance_rescale=0.0, ddim_steps=50, eta=1, random_seed=2024, device="cuda",
              text_embeds=None, controlnet=None, condition=None, conditioning_scale=1.0, lengths=None, padded_gt=False, *, start_index=None,
              init_latents=None, generators=None):
    """Signature of src/inference.py:26-37 (+ keyword-only extensions).  Returns the waveform tensor (B,1,480*L).
    With `lengths` (one clip length in frames per prompt, batch padded to audio_frames; see sample_latents) it returns a list of B
    waveforms (1, 480*lengths[b]) from one length-aware VAE decode of the padded batch (each equal to the decode of that clip alone).
    gt / gt_mask go with lengths under `padded_gt=True`, as in sample_latents: padded to audio_frames, ignored past each clip's end.
    start_index / init_latents / generators: an audio-to-audio variation, as in sample_latents."""
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
                             lengths=lengths, padded_gt=padded_gt, start_index=start_index, init_latents=init_latents, generators=generators)
    pred = scale_shift_re(latents, params["autoencoder"]["scale"], params["autoencoder"]["shift"])
    if gt is not None:  # src/inference.py:104-105: pred[~gt_mask] = gt[~gt_mask], with the raw gt, after the rescale
        pred = torch.where(gt_mask.to(pred.device).bool().expand_as(pred), pred, gt.to(device=pred.device, dtype=pred.dtype))
    if lengths is not None:   # what the paste put past a clip's end is never read by the decode
        w = autoencoder(embedding=pred, lengths=lengths)
        hop = w.shape[-1] // pred.shape[-1]
        return [w[b, :, :hop * n] for b, n in enumerate(lengths)]
    return autoencoder(embedding=pred)
