"""Continuous batching on the GPU: the per-slot CFG / DDIM kernel, the device-index DiT forward and context-row replacement against the
paths they stand in for (bit for bit), and engine.ContinuousEngine end to end (co-tenant invariance, the fp32 oracle loop, one graph)."""
import functools

import numpy as np
import pytest
import torch

from ezaudio_b200 import _lib, synth, weights
from oracle import ezaudio_oracle as O

pytestmark = pytest.mark.gpu


def _slot_array(slots):
    arr = (_lib.DdimSlot * len(slots))()
    for a, (gs, gr, coef, flags) in zip(arr, slots):
        a.guidance_scale, a.guidance_rescale, a.flags = gs, gr, flags
        a.coef[:] = coef
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.int32).cuda()


def test_cfg_ddim_step_slots_matches_per_sample_calls():
    from ezaudio_b200.inference import _ddim_step
    B, Cc, L = 6, 128, 100
    lens = [100, 37, 1, 64, 100, 50]
    A, G = _lib.SLOT_ACTIVE, _lib.SLOT_CFG
    # (guidance_scale, guidance_rescale, coef, flags): CFG with / without rescale, no CFG, eta 0 (sigma 0) and 1, one inactive slot
    slots = [(5.0, 0.75, (0.8, 0.6, 0.9, 0.3, 0.25), A | G), (3.5, 0.0, (0.7, 0.71, 0.8, 0.6, 0.0), A | G),
             (0.0, 0.75, (0.8, 0.6, 0.9, 0.3, 0.25), A), (5.0, 0.75, (0.5, 0.86, 0.6, 0.8, 0.0), A | G),
             (5.0, 0.5, (0.8, 0.6, 0.9, 0.3, 0.25), 0), (0.0, 0.0, (0.9, 0.43, 0.95, 0.31, 0.0), A)]
    g = torch.Generator(device="cuda").manual_seed(5)
    mo = torch.randn(2 * B, Cc, L, device="cuda", generator=g)
    lat = torch.randn(B, Cc, L, device="cuda", generator=g)
    nz = torch.randn(B, Cc, L, device="cuda", generator=g)
    mo_p, lat_p, nz_p = mo.clone(), lat.clone(), nz.clone()
    for b, n in enumerate(lens):
        mo_p[b, :, n:] = float("nan"); mo_p[B + b, :, n:] = float("nan"); nz_p[b, :, n:] = float("nan"); lat_p[b, :, n:] = 7.0
    for b, s in enumerate(slots):
        if s[2][4] == 0:
            nz_p[b] = float("nan")   # sigma 0: the slot must not read its noise
    before = lat_p.clone()
    lens_d = torch.tensor(lens, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().ezb_cfg_ddim_step_slots(0, _lib.ptr(mo_p), _lib.ptr(lat_p), _lib.ptr(nz_p), _lib.ptr(_slot_array(slots)), B, Cc, L,
                                                  _lib.stream_ptr(), _lib.ptr(lens_d)))
    torch.cuda.synchronize()
    for b, ((gs, gr, coef, flags), n) in enumerate(zip(slots, lens)):
        if not flags & A:
            assert torch.equal(lat_p[b].view(torch.int32), before[b].view(torch.int32)), b   # byte for byte untouched
            continue
        ls = lat[b:b + 1, :, :n].contiguous()
        rows = [mo[b:b + 1, :, :n]] + ([mo[B + b:B + b + 1, :, :n]] if flags & G else [])
        _ddim_step(torch.cat(rows).contiguous(), ls, nz[b:b + 1, :, :n].contiguous() if coef[4] else None, 1, Cc, n, gs if flags & G else 0.0,
                   gr, coef)
        torch.cuda.synchronize()
        assert torch.equal(lat_p[b, :, :n], ls[0]), (b, n)
        assert bool((lat_p[b, :, n:] == 7.0).all()), (b, n)


@functools.lru_cache(maxsize=1)
def _xl_state_dict():
    return weights.synthetic_state_dict(weights.dit_param_shapes(synth.model_cfg("xl")), 4)


def _model(kind, precision, Be, L, Lc):
    from ezaudio_b200.dit import MaskDiT
    cfg = synth.model_cfg("xl") if kind == "xl" else synth.tiny_model(72)
    sd = _xl_state_dict() if kind == "xl" else weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    return cfg, MaskDiT(precision=precision, max_batch=Be, max_len=L, max_ctx_len=Lc, max_timesteps=16, **cfg).load_state_dict(sd)


@pytest.mark.parametrize("kind,precision", [("tiny", "bf16"), ("tiny", "bf16x3"), ("xl", "bf16")])
def test_forward_device_t_index_matches_host_index_path(kind, precision):
    Be, L, Lc = 4, (500 if kind == "xl" else 96), (100 if kind == "xl" else 12)
    cfg, m = _model(kind, precision, Be, L, Lc)
    ts = [999, 759, 479, 239, 19]
    m.set_timesteps(ts)
    x = synth.synth_latents(Be, L).cuda()
    ctx, mask = synth.synth_context(Be, Lc, cfg["context_dim"])
    ctx, mask = ctx.cuda(), mask.cuda()
    for rows in ([0, 2, 4, 1], [3, 3, 0, 3]):   # per-sample timesteps (not all equal: the host path gathers too)
        want, _ = m(x, torch.tensor([ts[r] for r in rows]), ctx, context_mask=mask)   # module path: host indices (ezb_dit_forward)
        got = m.forward_step(x, 0, t_index=torch.tensor(rows, dtype=torch.int32, device="cuda"))
        torch.cuda.synchronize()
        assert torch.equal(got, want), (rows, float((got - want).abs().max()))


@pytest.mark.parametrize("kind,precision", [("tiny", "bf16"), ("tiny", "bf16x3"), ("xl", "bf16")])
def test_set_context_rows_matches_set_context_of_the_batch(kind, precision):
    # tiny: Be * Lc = 512 tokens, so the whole batch takes the swap-AB kernel for context_embed's second linear and one row alone would not
    Be, L, Lc = 4, (500 if kind == "xl" else 64), (100 if kind == "xl" else 128)
    cfg, m = _model(kind, precision, Be, L, Lc)
    m.set_timesteps([999, 479])
    x = synth.synth_latents(Be, L).cuda()
    ctx, mask = synth.synth_context(Be, Lc, cfg["context_dim"])
    new, nmask = synth.synth_context(1, Lc, cfg["context_dim"], seed=21)
    tix = torch.tensor([0, 1, 1, 0], dtype=torch.int32, device="cuda")
    m.set_context(ctx.cuda(), mask.cuda())
    m.set_context_rows(new.cuda(), nmask.cuda(), 2)
    got = m.forward_step(x, 0, t_index=tix).clone()
    ctx2, mask2 = ctx.clone(), mask.clone()
    ctx2[2], mask2[2] = new[0], nmask[0]
    m.set_context(ctx2.cuda(), mask2.cuda())
    want = m.forward_step(x, 0, t_index=tix)
    torch.cuda.synchronize()
    assert torch.equal(got, want), float((got - want).abs().max())
    with pytest.raises(_lib.EzbError):
        m.set_context_rows(new[:, :Lc - 1].cuda(), nmask[:, :Lc - 1].cuda(), 0)   # Lc differs from the layout
    with pytest.raises(_lib.EzbError):
        m.set_context_rows(new.cuda(), nmask.cuda(), Be)                           # row outside the batch


def _tiny_ez(precision, monkeypatch):
    from ezaudio_b200 import api, config
    from tests.test_api_gpu import _tiny_params
    tiny = _tiny_params()
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    return api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16), max_batch=3,
                       max_length_s=2, precision=precision)


MIX = [dict(prompt="rain on a roof", length=2, guidance_scale=3.5, guidance_rescale=0.0, ddim_steps=8, eta=0.0, random_seed=21),
       dict(prompt="", length=0.7, guidance_scale=5, guidance_rescale=0.75, ddim_steps=4, eta=1.0, random_seed=22),
       dict(prompt="wind in trees", length=1.3, guidance_scale=5, guidance_rescale=0.75, ddim_steps=4, eta=1.0, random_seed=23)]
TARGET = dict(prompt="a dog barks", length=1.5, guidance_scale=5, guidance_rescale=0.75, ddim_steps=8, eta=1.0, random_seed=7)


def test_engine_request_audio_independent_of_co_tenants_and_one_graph(monkeypatch):
    from ezaudio_b200.engine import ContinuousEngine
    ez = _tiny_ez("bf16", monkeypatch)
    alone = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8))
    (sr, want), = alone.run([synth_req(TARGET)])
    assert sr == 24000 and want.dtype == np.float32 and want.shape == (int(24000 * 1.5),) and np.isfinite(want).all()
    eng = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8))
    for r in MIX[:2]:
        eng.submit(**r)
    out = {}
    for _ in range(3):                    # the target joins at step 3, in slot 2, next to other guidance, eta, step counts and lengths
        out.update({t: w for t, _, w in eng.step()})
    t_target = eng.submit(**TARGET)
    eng.submit(**MIX[2])                  # queued behind it: takes the slot of whichever finishes first
    for t, _, w in eng.stream():
        out[t] = w
    assert len(out) == 4
    assert out[t_target].tobytes() == want.tobytes()
    # a generate_audio call in between replaces the denoiser's context and table; the engine restores them
    ez.generate_audio("a cat", length=1, ddim_steps=3, random_seed=1)
    (_, again), = eng.run([synth_req(TARGET)])
    assert again.tobytes() == want.tobytes()
    assert eng.backend.captures == 1 and alone.backend.captures == 1   # every admission and step replayed the one graph of the shape


def synth_req(d):
    from ezaudio_b200.frontend import Request
    return Request(**d)


def test_engine_latents_match_oracle_loop(monkeypatch):
    from ezaudio_b200.engine import ContinuousEngine
    ez = _tiny_ez("bf16x3", monkeypatch)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(ez.params["model"]), 3)
    eng = ContinuousEngine(ez, slots=2, max_length_s=2, ddim_steps=(4, 8))
    lat = {}
    finish = eng.backend.finish

    def keep(k, frames):
        lat[k, frames] = eng.backend.lat[k, :, :frames].cpu()
        return finish(k, frames)

    eng.backend.finish = keep
    reqs = MIX + [TARGET]
    slot_of = {}
    admit = eng.backend.admit

    def rec(k, prompt, seed, frames):
        slot_of[seed] = (k, frames)
        return admit(k, prompt, seed, frames)

    eng.backend.admit = rec
    got = {}
    for r in reqs:
        eng.submit(**r)
    while eng.pending():
        for t, _, _ in eng.step():
            r = reqs[t]
            got[t] = lat[slot_of[r["random_seed"]]]
    enc = ez.encode_text
    uctx, umask = enc([""])
    for t, r in enumerate(reqs):
        n = int(r["length"] * 50)
        g = torch.Generator(device="cuda").manual_seed(r["random_seed"])
        noise = torch.randn((1, 128, n), generator=g, device="cuda").cpu()
        steps = [torch.empty((1, 128, n), device="cuda").normal_(generator=g).cpu() for _ in range(r["ddim_steps"])] if r["eta"] > 0 else None
        ctx, mask = enc([r["prompt"]])
        cfg = r["prompt"] != ""
        with torch.no_grad():
            ref = O.sample_loop(sd, ez.params["model"], noise, ctx, mask, uctx, umask, guidance_scale=r["guidance_scale"] if cfg else None,
                                guidance_rescale=r["guidance_rescale"], ddim_steps=r["ddim_steps"], eta=r["eta"], step_noise=steps)
        err = float((got[t] - ref[0]).abs().max())
        assert err < 5e-3, (t, err)
