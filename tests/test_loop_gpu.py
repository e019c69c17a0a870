"""Sampling loop (set_context / set_timesteps / forward_step / fused CFG+DDIM kernel) vs the CPU oracle loop on the same
weights, latents and injected noise.  Parity precision (bf16x3): tolerance 5e-3 max-abs on latents of std ~1 after N steps
(per-step DiT error < 1e-3 compounds through the DDIM recursion)."""
import pytest
import torch

from ezaudio_b200 import synth, weights
from oracle import ezaudio_oracle as O

pytestmark = pytest.mark.gpu


def _setup(B=2, L=40, Lc=12):
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    ctx, mask = synth.synth_context(B, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    noise = synth.synth_latents(B, L, seed=5)
    return cfg, sd, ctx, mask, uctx, umask, noise


@pytest.mark.parametrize("eta,gs,gr,inpaint", [(0.0, 3.0, 0.5, False), (1.0, 5.0, 0.75, False), (1.0, None, 0.0, False), (1.0, 3.5, 0.0, True)])
def test_loop_matches_oracle(eta, gs, gr, inpaint):
    from ezaudio_b200.dit import MaskDiT
    from ezaudio_b200.inference import sample_latents
    from ezaudio_b200.scheduler import DDIMScheduler
    B, L, Lc, steps = 2, 40, 12, 4
    cfg, sd, ctx, mask, uctx, umask, noise = _setup(B, L, Lc)
    g = torch.Generator().manual_seed(9)
    step_noise = [torch.randn(B, 128, L, generator=g) for _ in range(steps)]
    gt, gm = synth.synth_gt(B, L) if inpaint else (None, None)
    with torch.no_grad():
        ref = O.sample_loop(sd, cfg, noise, ctx, mask, uctx.expand(B, -1, -1), umask.expand(B, -1), gt=gt, gt_mask=gm, guidance_scale=gs,
                            guidance_rescale=gr, ddim_steps=steps, eta=eta, step_noise=step_noise)
    m = MaskDiT(precision="bf16x3", max_batch=2 * B, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    lat = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, gt, gm, audio_frames=L, guidance_scale=gs, guidance_rescale=gr, ddim_steps=steps,
                         eta=eta, init_noise=noise, step_noise=[s.cuda() for s in step_noise])
    err = float((lat.cpu() - ref).abs().max())
    assert err < 5e-3, err


@pytest.mark.parametrize("name,precision,tol", [("controlnet_tiny72", "bf16x3", 1e-3), ("controlnet_XL", "bf16x3", 1e-3), ("controlnet_XL", "bf16", 6e-2)])
def test_controlnet_matches_reference_golden(name, precision, tol):
    """DiTControlNet skips + UDiT(controlnet_skips) vs the UNMODIFIED reference (tests/golden/controlnet_*.npz; controlnet_XL =
    BASELINE config C4 shapes at effective batch 2: EzAudio-XL + energy ControlNet, L = 500, Lc = 100)."""
    from ezaudio_b200.dit import DiTControlNet, MaskDiT
    from tests import helpers
    xl = name.endswith("XL")
    cfg, cn = (synth.model_cfg("xl") if xl else synth.tiny_model(72)), synth.CONTROLNET
    g = helpers.load_golden(name)
    seed = int(g["seed"])
    stride = int(g["skip_stride"]) if "skip_stride" in g.files else 1
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), seed)
    sd_cn = weights.synthetic_state_dict(weights.controlnet_param_shapes(cfg, cn), seed + 1)
    B, L, Lc = 2, int(g["L"]), int(g["Lc"])
    x = synth.synth_latents(B, L).cuda()
    ctx, mask = synth.synth_context(B, Lc, cfg["context_dim"])
    ctx, mask = ctx.cuda(), mask.cuda()
    cond = torch.rand(B, 1, 2 * L, generator=torch.Generator().manual_seed(9)).cuda()
    t = torch.tensor(499)
    kw = dict(precision=precision, max_batch=B, max_len=L, max_ctx_len=Lc, max_timesteps=8)
    unet = MaskDiT(**kw, **cfg).load_state_dict(sd)
    cnet = DiTControlNet(**kw, **cfg, **cn).load_state_dict(sd_cn, mask_embed=sd["mask_embed"])
    x257, _ = unet(x, t, ctx, context_mask=mask, forward_model=False)
    skips = cnet(x257, t, ctx, context_mask=mask, condition=cond, conditioning_scale=0.8)
    out = unet.model(x257, t, ctx, context_mask=mask, controlnet_skips=list(skips))
    torch.cuda.synchronize()
    s0, s1 = torch.from_numpy(g["skip0"]), torch.from_numpy(g["skip_last"])
    e0 = float((skips[0][:, ::stride].cpu() - s0).abs().max())
    e1 = float((skips[-1][:, ::stride].cpu() - s1).abs().max())
    eo = float((helpers.golden_view(g, out.cpu()) - torch.from_numpy(g["out"])).abs().max())
    print(f"[parity] {name} [{precision}]: skip0 {e0:.3e} (std {float(s0.std()):.2f}) skip_last {e1:.3e} (std {float(s1.std()):.2f}) out {eo:.3e}")
    # the tolerances are stated for tensors of std ~ 1 (the DiT output); the deepest ControlNet skip of the XL model has std ~ 1.9
    assert e0 < tol * max(1.0, float(s0.std())) and e1 < tol * max(1.0, float(s1.std())) and eo < tol, (e0, e1, eo)


def test_graph_replay_equals_eager():
    """Second call replays the captured per-step CUDA graphs: must reproduce the eager (first) call bit for bit, and the
    non-graph path must agree too."""
    from ezaudio_b200.dit import MaskDiT
    from ezaudio_b200.inference import sample_latents
    from ezaudio_b200.scheduler import DDIMScheduler
    B, L, Lc, steps = 2, 40, 12, 3
    cfg, sd, ctx, mask, uctx, umask, noise = _setup(B, L, Lc)
    g = torch.Generator().manual_seed(9)
    step_noise = [torch.randn(B, 128, L, generator=g).cuda() for _ in range(steps)]
    m = MaskDiT(precision="bf16", max_batch=2 * B, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    kw = dict(audio_frames=L, guidance_scale=5.0, guidance_rescale=0.75, ddim_steps=steps, eta=1.0, init_noise=noise, step_noise=step_noise)
    a = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, **kw)
    b = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, **kw)
    c = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, use_graphs=False, **kw)
    assert torch.equal(a, b)
    assert torch.equal(a, c)


def test_50_step_bf16_loop_drift_vs_oracle():
    """The loop bench.py times is 50 DDIM steps in bf16 with CFG 5 / rescale 0.75 / eta 1: per-step DiT error (bf16 floor, a few 1e-2)
    compounds through the recursion.  Measured here on the tiny dh=72 model against the fp32 oracle loop with the same injected
    noise; printed so that the drift is on record, bounded so that a regression (e.g. a wrong coefficient at one step) fails."""
    from ezaudio_b200.dit import MaskDiT
    from ezaudio_b200.inference import sample_latents
    from ezaudio_b200.scheduler import DDIMScheduler
    B, L, Lc, steps = 2, 40, 12, 50
    cfg, sd, ctx, mask, uctx, umask, noise = _setup(B, L, Lc)
    g = torch.Generator().manual_seed(9)
    step_noise = [torch.randn(B, 128, L, generator=g) for _ in range(steps)]
    with torch.no_grad():
        ref = O.sample_loop(sd, cfg, noise, ctx, mask, uctx.expand(B, -1, -1), umask.expand(B, -1), guidance_scale=5.0, guidance_rescale=0.75,
                            ddim_steps=steps, eta=1.0, step_noise=step_noise)
    res = {}
    for precision in ("bf16x3", "bf16"):
        m = MaskDiT(precision=precision, max_batch=2 * B, max_len=L, max_ctx_len=Lc, max_timesteps=64, **cfg).load_state_dict(sd)
        lat = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, audio_frames=L, guidance_scale=5.0, guidance_rescale=0.75, ddim_steps=steps,
                             eta=1.0, init_noise=noise, step_noise=[s.cuda() for s in step_noise])
        err = (lat.cpu() - ref).abs()
        res[precision] = (float(err.max()), float(err.mean()))
        print(f"[parity] 50-step CFG loop [{precision}]: max-abs {res[precision][0]:.3e} mean-abs {res[precision][1]:.3e} (latent std {float(ref.std()):.3f})")
    assert res["bf16x3"][0] < 2e-2, res
    assert res["bf16"][0] < 0.5 and res["bf16"][1] < 6e-2, res
