"""ControlNet requests in the continuous-batching engine, on the GPU: the device-index ControlNet forward with per-sample scales against
ezb_controlnet_forward (bit for bit), the condition cache, engine.ContinuousEngine with an EzAudio_ControlNet end to end (co-tenant
invariance, one graph, the fp32 oracle loop) and the per-clip list form of EzAudio_ControlNet.generate_audio."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from ezaudio_b200 import _lib, config, synth, weights
from oracle import ezaudio_oracle as O

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=1)
def _xl_state_dicts():
    cfg = synth.model_cfg("xl")
    return (weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 4),
            weights.synthetic_state_dict(weights.controlnet_param_shapes(cfg, synth.CONTROLNET), 5))


def _controlnet(kind, precision, Be, L, Lc):
    from ezaudio_b200.dit import DiTControlNet
    cfg = synth.model_cfg("xl") if kind == "xl" else synth.tiny_model(72)
    if kind == "xl":
        sd, sd_cn = _xl_state_dicts()
    else:
        sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
        sd_cn = weights.synthetic_state_dict(weights.controlnet_param_shapes(cfg, synth.CONTROLNET), 4)
    net = DiTControlNet(precision=precision, max_batch=Be, max_len=L, max_ctx_len=Lc, max_timesteps=16, **cfg, **synth.CONTROLNET)
    net.load_state_dict(sd_cn, mask_embed=sd["mask_embed"])
    ctx, mask = synth.synth_context(Be, Lc, cfg["context_dim"])
    net.set_context(ctx.cuda(), mask.cuda())
    net.set_timesteps([999, 759, 479, 239, 19])
    return cfg, net


def _cond(Be, L, seed):
    return torch.rand(Be, 1, 2 * L, generator=torch.Generator().manual_seed(seed)).cuda()


def _host_index_forward(net, x, rows, cond, scale):
    """ezb_controlnet_forward with per-sample host indices and one scale."""
    Be = x.shape[0]
    return [s.clone() for s in net._run(x, None, None, (C.c_int32 * Be)(*rows), 0, cond, scale, None)]


def _tdev_forward(net, x, rows, scales):
    t = torch.tensor(rows, dtype=torch.int32, device="cuda")
    s = torch.tensor(scales, dtype=torch.float32, device="cuda")
    return [o.clone() for o in net.forward_step(x, t_index=t, scale=s)]


@pytest.mark.parametrize("kind,precision", [("tiny", "bf16"), ("tiny", "bf16x3"), ("xl", "bf16")])
def test_forward_tdev_matches_host_index_path_per_scale(kind, precision):
    Be, L, Lc = 4, (500 if kind == "xl" else 96), (100 if kind == "xl" else 12)
    cfg, net = _controlnet(kind, precision, Be, L, Lc)
    x = synth.synth_latents(Be, L).cuda()
    cond = _cond(Be, L, 9)
    net.set_condition(cond)
    rows = [0, 2, 4, 1]                         # not all equal: the host path gathers per-sample rows too
    scales = [0.5, 1.0, 1.3, 0.0]
    got = _tdev_forward(net, x, rows, scales)
    for s in (0.5, 1.0, 1.3):
        want = _host_index_forward(net, x, rows, cond, s)
        torch.cuda.synchronize()
        for b in (b for b, v in enumerate(scales) if v == s):
            for i, (g, w) in enumerate(zip(got, want)):
                assert torch.equal(g[b].view(torch.int32), w[b].view(torch.int32)), (s, b, i, float((g[b] - w[b]).abs().max()))
    for g in got:   # scale 0: the skips are exactly zero (the reference multiplies by conditioning_scale)
        assert bool((g[3] == 0).all())
        assert bool((g[:3] != 0).any())


def test_condition_cache_rows_and_isolation_from_the_per_call_path():
    from ezaudio_b200.dit import DiTControlNet
    Be, L, Lc = 4, 96, 12
    cfg, net = _controlnet("tiny", "bf16", Be, L, Lc)
    x = synth.synth_latents(Be, L).cuda()
    rows, scales = [0, 2, 4, 1], [1.0, 0.5, 1.0, 1.3]
    cond = _cond(Be, L, 9)
    new = _cond(1, L, 10)
    net.set_condition(cond)
    net.set_condition_rows(new, 2)
    got = _tdev_forward(net, x, rows, scales)
    cond2 = cond.clone()
    cond2[2] = new[0]
    net.set_condition(cond2)
    want = _tdev_forward(net, x, rows, scales)
    torch.cuda.synchronize()
    for g, w in zip(got, want):
        assert torch.equal(g.view(torch.int32), w.view(torch.int32))
    _host_index_forward(net, x, rows, _cond(Be, L, 11), 0.7)   # ezb_controlnet_forward on another condition: the cache is untouched
    again = _tdev_forward(net, x, rows, scales)
    torch.cuda.synchronize()
    for g, w in zip(again, want):
        assert torch.equal(g.view(torch.int32), w.view(torch.int32))
    with pytest.raises(_lib.EzbError, match="error -5"):
        net.set_condition_rows(_cond(1, L - 8, 12), 0)            # L differs from the layout
    with pytest.raises(_lib.EzbError, match="error -2"):
        net.set_condition_rows(new, Be)                           # row outside the batch
    with pytest.raises(_lib.EzbError, match="error -5"):
        net.forward_step(x[:, :, :L - 8].contiguous(), t_index=torch.zeros(Be, dtype=torch.int32, device="cuda"),
                         scale=torch.ones(Be, device="cuda"))     # L differs from the condition layout
    fresh = DiTControlNet(precision="bf16", max_batch=Be, max_len=L, max_ctx_len=Lc, max_timesteps=16, **cfg, **synth.CONTROLNET)
    fresh.load_state_dict(weights.synthetic_state_dict(weights.controlnet_param_shapes(cfg, synth.CONTROLNET), 4),
                          mask_embed=torch.zeros(cfg["out_chans"]))
    with pytest.raises(_lib.EzbError, match="error -5"):
        fresh.set_condition_rows(new, 0)                          # no layout yet


def _tiny_cn(precision, max_batch=3):
    from ezaudio_b200 import api
    from tests.test_api_gpu import _tiny_params
    p = _tiny_params()
    p["controlnet"] = synth.CONTROLNET
    p["conditioner"] = config.BUILTIN_CONTROLNET["energy"]["conditioner"]
    return api.EzAudio_ControlNet("energy", ckpt_path="synthetic:5", controlnet_path="synthetic:6", vae_path="synthetic:6",
                                  text_encoder=api.SyntheticTextEncoder(64, 16), max_batch=max_batch, params=p, precision=precision)


def _clip(seconds, seed, amp=0.1):
    return (amp * np.random.default_rng(seed).standard_normal(int(seconds * 24000))).astype(np.float32)


MIX = [dict(prompt="rain on a roof", audio=_clip(3, 1), surpass_noise=0.05, guidance_scale=3.5, guidance_rescale=0.0, ddim_steps=8, eta=0.0,
            conditioning_scale=0.5, random_seed=21),
       dict(prompt="", audio=_clip(12, 2), guidance_scale=5, guidance_rescale=0.75, ddim_steps=4, eta=1.0, conditioning_scale=1, random_seed=22),
       dict(prompt="wind in trees", audio=_clip(1.5, 3, 0.3), guidance_scale=5, guidance_rescale=0.75, ddim_steps=4, eta=1.0,
            conditioning_scale=0, random_seed=23)]
TARGET = dict(prompt="a siren", audio=_clip(4, 7), surpass_noise=0.02, guidance_scale=3.5, guidance_rescale=0.5, ddim_steps=8, eta=1.0,
              conditioning_scale=1.3, random_seed=7)


def test_engine_control_request_independent_of_co_tenants_and_one_graph():
    from ezaudio_b200.engine import ContinuousEngine
    from ezaudio_b200.frontend import ControlRequest
    ez = _tiny_cn("bf16")
    alone = ContinuousEngine(ez, slots=3, ddim_steps=(4, 8))
    (sr, want), = alone.run([ControlRequest(**TARGET)])
    assert sr == 24000 and want.dtype == np.float32 and want.shape == (4 * 24000,) and np.isfinite(want).all()
    eng = ContinuousEngine(ez, slots=3, ddim_steps=(4, 8))
    for r in MIX[:2]:
        eng.submit(**r)
    out = {}
    for _ in range(3):                    # the target joins at step 3, next to other clips, scales, guidance, eta and step counts
        out.update({t: w for t, _, w in eng.step()})
    t_target = eng.submit(**TARGET)
    eng.submit(**MIX[2])
    for t, _, w in eng.stream():
        out[t] = w
    assert len(out) == 4
    assert out[t_target].tobytes() == want.tobytes()
    assert out[1].shape == (10 * 24000,) and out[3].shape == (int(1.5 * 24000),)   # trimmed to each clip's length, capped at 10 s
    # a generate_audio call in between replaces both handles' context and table; the engine restores them
    ez.generate_audio("a cat", _clip(2, 9), ddim_steps=3, random_seed=1)
    (_, again), = eng.run([ControlRequest(**TARGET)])
    assert again.tobytes() == want.tobytes()
    assert eng.backend.captures == 1 and alone.backend.captures == 1


def test_engine_control_latents_match_oracle_loop():
    from ezaudio_b200 import post
    from ezaudio_b200.api import energy_condition
    from ezaudio_b200.engine import ContinuousEngine
    ez = _tiny_cn("bf16x3")
    cfg = ez.params["model"]
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 5)
    sd_cn = weights.synthetic_state_dict(weights.controlnet_param_shapes(cfg, synth.CONTROLNET), 6)
    eng = ContinuousEngine(ez, slots=2, ddim_steps=(4, 8))
    lat, slot_of = {}, {}
    finish, admit = eng.backend.finish, eng.backend.admit

    def keep(k, frames):
        lat[k] = eng.backend.lat[k].cpu()
        return finish(k, frames)

    def rec(k, prompt, seed, frames, **kw):
        slot_of[seed] = k
        return admit(k, prompt, seed, frames, **kw)

    eng.backend.finish, eng.backend.admit = keep, rec
    reqs = MIX + [TARGET]
    got = {}
    for r in reqs:
        eng.submit(**r)
    while eng.pending():
        for t, _, _ in eng.step():
            got[t] = lat[slot_of[reqs[t]["random_seed"]]]
    enc = ez.encode_text
    uctx, umask = enc([""])
    ckw = {k: v for k, v in ez.params["conditioner"].items() if k != "condition_type"}
    for t, r in enumerate(reqs):
        g = torch.Generator(device="cuda").manual_seed(r["random_seed"])
        noise = torch.randn((1, 128, 500), generator=g, device="cuda").cpu()
        steps = [torch.empty((1, 128, 500), device="cuda").normal_(generator=g).cpu() for _ in range(r["ddim_steps"])] if r["eta"] > 0 else None
        wave = post.prepare_wave(torch.from_numpy(r["audio"]).cuda().unsqueeze(0), 240000, normalize=True, gate=r.get("surpass_noise", 0))
        cond = energy_condition(wave, **ckw).cpu()
        ctx, mask = enc([r["prompt"]])
        use_cfg = r["prompt"] != ""
        with torch.no_grad():
            ref = O.sample_loop(sd, cfg, noise, ctx.cpu(), mask.cpu(), uctx.cpu(), umask.cpu(), guidance_scale=r["guidance_scale"] if use_cfg else None,
                                guidance_rescale=r["guidance_rescale"], ddim_steps=r["ddim_steps"], eta=r["eta"], step_noise=steps,
                                controlnet=(sd_cn, cfg, cond, r["conditioning_scale"]))
        err = float((got[t] - ref[0]).abs().max())
        assert err < 5e-3, (t, err)


def test_generate_audio_per_clip_list(monkeypatch):
    from ezaudio_b200 import api, post
    ez = _tiny_cn("bf16", max_batch=2)
    clips, gates, seeds = [_clip(3, 11), _clip(12, 12)], [0.0, 0.05], [5, 6]
    seen = {}
    real = api.inference

    def spy(*a, **kw):
        seen["condition"] = kw["condition"].clone()
        return real(*a, **kw)

    monkeypatch.setattr(api, "inference", spy)
    sr, wavs = ez.generate_audio(["a siren", "rain"], clips, surpass_noise=gates, ddim_steps=3, random_seed=seeds)
    monkeypatch.setattr(api, "inference", real)
    ckw = {k: v for k, v in ez.params["conditioner"].items() if k != "condition_type"}
    assert tuple(seen["condition"].shape) == (2, 1, 1000)
    for b, (c, g) in enumerate(zip(clips, gates)):
        alone = api.energy_condition(post.prepare_wave(torch.from_numpy(c).cuda().unsqueeze(0), 240000, normalize=True, gate=g), **ckw)
        assert torch.equal(seen["condition"][b:b + 1].view(torch.int32), alone.view(torch.int32)), b
    assert sr == 24000 and [w.shape for w in wavs] == [(3 * 24000,), (10 * 24000,)]
    for b, (p, c, g, s) in enumerate(zip(["a siren", "rain"], clips, gates, seeds)):
        _, want = ez.generate_audio(p, c, surpass_noise=g, ddim_steps=3, random_seed=s)
        assert want.shape == wavs[b].shape
        assert np.allclose(wavs[b], want, atol=2e-2), (b, float(np.abs(wavs[b] - want).max()))
