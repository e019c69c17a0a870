"""Long ControlNet clips on the GPU: ezb_controlnet_forward_cached against ezb_controlnet_forward (bit for bit), the one-window identity of
EzAudio_ControlNet.generate_long_audio with generate_audio, the per-window conditions the loop caches, the windowed loop against the
oracle's DiT + ControlNet driven by fp64 windows, batches against solo calls and graph replay, the row capacity, and a ContinuousEngine
sharing the handles with a long call."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from ezaudio_b200 import _lib, synth, weights
from ezaudio_b200.inference import long_plan
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
from oracle import ezaudio_oracle as O
from tests.test_controlnet_engine_gpu import TARGET, _clip, _cond, _controlnet, _host_index_forward, _tiny_cn
from tests.test_longform_gpu import _blend64, _draws

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- the entry point
def _cached(net, x, rows, tall, scale):
    """ezb_controlnet_forward_cached with host indices `rows` (or all `tall`); returns (status, skips)."""
    Be, _, L = x.shape
    outs = [torch.full((Be, L, net.cfg["embed_dim"]), 7.0, device="cuda") for _ in range(net.half)]
    arr = (C.c_void_p * net.half)(*[o.data_ptr() for o in outs])
    tidx = None if rows is None else (C.c_int32 * Be)(*rows)
    rc = _lib.lib().ezb_controlnet_forward_cached(net._h.h, _lib.ptr(x), None, None, tidx, tall, float(scale), arr, Be, L, _lib.stream_ptr())
    return rc, outs


def _same(got, want):
    torch.cuda.synchronize()
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g.view(torch.int32), w.view(torch.int32)), (i, float((g - w).abs().max()))


@pytest.mark.parametrize("kind,precision", [("tiny", "bf16"), ("tiny", "bf16x3"), ("xl", "bf16")])
def test_forward_cached_equals_forward_on_the_cached_condition(kind, precision):
    gc.collect()
    Be, L, Lc = 4, (500 if kind == "xl" else 96), (100 if kind == "xl" else 12)
    cfg, net = _controlnet(kind, precision, Be, L, Lc)
    x = synth.synth_latents(Be, L).cuda()
    cond = _cond(Be, L, 9)
    net.set_condition(cond)
    for s in (0.5, 1.0, 1.3):
        for step in (0, 3):   # uniform host indices: the path generate_audio takes, folded LayerNorm included
            got = [o.clone() for o in net.forward_step(x, step, conditioning_scale=s)]
            _same(got, [o.clone() for o in net.forward_step(x, step, cond, s)])
        rows = [0, 2, 4, 1]   # non-uniform host indices
        rc, got = _cached(net, x, rows, 0, s)
        assert rc == 0
        _same(got, _host_index_forward(net, x, rows, cond, s))
    for rows, tall in ((None, 2), ([0, 2, 4, 1], 0)):   # scale 0: exact zeros, the network does not run
        rc, got = _cached(net, x, rows, tall, 0.0)
        torch.cuda.synchronize()
        assert rc == 0 and all(bool((g == 0).all()) for g in got)


def test_forward_cached_layout_and_isolation():
    gc.collect()
    Be, L, Lc = 4, 96, 12
    cfg, net = _controlnet("tiny", "bf16", Be, L, Lc)
    x = synth.synth_latents(Be, L).cuda()
    cond = _cond(Be, L, 9)
    net.set_condition(cond)
    want = [o.clone() for o in net.forward_step(x, 2, conditioning_scale=1.3)]
    net.forward_step(x, 2, _cond(Be, L, 11), 0.7)   # ezb_controlnet_forward on another condition leaves the cache as it was
    _same(net.forward_step(x, 2, conditioning_scale=1.3), want)
    rc, _ = _cached(net, x[:, :, :L - 8].contiguous(), None, 2, 1.0)   # L differs from the condition layout
    assert rc == -5
    net.set_condition(cond[:2])   # a layout of 2 rows: the context batch of 4 no longer matches it
    rc, _ = _cached(net, x, None, 2, 1.0)
    assert rc == -5
    with pytest.raises(_lib.EzbError, match="error -5"):
        net.forward_step(x, 2, conditioning_scale=1.0)


# ---------------------------------------------------------------- one window: generate_audio bit for bit
SAMPLERS = [("ddim", 0.0), ("ddim", 1.0), ("dpmsolver++", 1.0), ("sde-dpmsolver++", 1.0)]


def _set_sampler(ez, alg):
    ez.noise_scheduler = DDIMScheduler(**ez.params["diff"]) if alg == "ddim" else DPMSolverMultistepScheduler(**ez.params["diff"], algorithm_type=alg)


@pytest.mark.parametrize("alg,eta", SAMPLERS)
def test_one_window_equals_generate_audio(alg, eta):
    gc.collect()
    ez = _tiny_cn("bf16")
    _set_sampler(ez, alg)
    cases = [("a dog barks", _clip(3, 31), 0.0, 1.0, 3.5),
             ("rain on a roof", _clip(10, 32, 0.3), 0.05, 1.3, 5.0),   # exactly 10 s, noise-gated
             ("", _clip(3, 33), 0.0, 0.0, 0.0)]                        # empty prompt: no guidance; scale 0
    for prompt, clip, gate, scale, gs in cases:
        kw = dict(surpass_noise=gate, guidance_rescale=0.5, ddim_steps=5, eta=eta, conditioning_scale=scale, random_seed=17)
        sr, want = ez.generate_audio(prompt, clip, guidance_scale=gs, **kw)
        sr2, got = ez.generate_long_audio(prompt, clip, window_length=10, guidance_scale=gs if prompt else 3.5, **kw)
        assert sr2 == sr and got.dtype == want.dtype and got.shape == want.shape == clip.shape, (prompt, got.shape)
        assert got.tobytes() == want.tobytes(), (alg, eta, prompt)


# ---------------------------------------------------------------- the conditions the loop caches
def test_cached_condition_rows_are_windows_of_the_whole_clip_condition(monkeypatch):
    from ezaudio_b200 import post
    from ezaudio_b200.api import energy_condition
    gc.collect()
    ez = _tiny_cn("bf16", max_batch=6)
    seen = []
    real = ez.controlnet.set_condition
    monkeypatch.setattr(ez.controlnet, "set_condition", lambda c: (seen.append(c.clone()), real(c))[1])
    clips, gates = [_clip(4.5, 41, 0.3), _clip(1.5, 42)], [0.02, 0.0]
    Lw, O_ = 100, 20
    ez.generate_long_audio(["a siren", "rain"], clips, window_length=2, overlap=0.4, surpass_noise=gates, ddim_steps=2, random_seed=[1, 2])
    assert len(seen) == 1
    frames = [225, 100]   # 4.5 s: 225 frames; 1.5 s: padded to one 2 s window
    table, windows = long_plan(frames, Lw, O_)
    assert [t[1] for t in table] == [3, 1]
    ckw = {k: v for k, v in ez.params["conditioner"].items() if k != "condition_type"}
    whole = []
    for c, g, n in zip(clips, gates, frames):
        wave = post.prepare_wave(torch.from_numpy(c).cuda().unsqueeze(0), n * 480, normalize=True, gate=g)
        ec = energy_condition(wave, **ckw)
        assert tuple(ec.shape) == (1, 1, 2 * n)
        want = O.energy_extract(wave.cpu(), 240, 1920, -60.0, True)
        assert float((ec.cpu()[:, 0] - want[..., 0]).abs().max()) < 2e-5
        whole.append(ec)
    rows = torch.stack([whole[b][0, :, 2 * s:2 * (s + Lw)] for b, s, _ in windows])
    want = torch.cat([rows, rows])   # the uncond half repeats the rows
    assert tuple(seen[0].shape) == tuple(want.shape) == (2 * len(windows), 1, 2 * Lw)
    assert torch.equal(seen[0].view(torch.int32), want.view(torch.int32))


# ---------------------------------------------------------------- the loop against the oracle
@pytest.mark.parametrize("sampler", ["ddim", "dpmsolver++"])
def test_long_controlnet_loop_matches_oracle_with_fp64_windows(sampler):
    from ezaudio_b200.dit import DiTControlNet, MaskDiT
    from ezaudio_b200.inference import sample_long_latents
    gc.collect()
    lens, Lw, O_, gs, gr, steps, eta, seed, scale, Lc = [73, 61], 40, 8, 3.0, 0.5, 4, 1.0, 11, 1.3, 12
    table, windows = long_plan(lens, Lw, O_)
    assert table[0][1] == 3   # three windows, the last overlapping both others
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    sd_cn = weights.synthetic_state_dict(weights.controlnet_param_shapes(cfg, synth.CONTROLNET), 4)
    ctx, mask = synth.synth_context(2, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    kw = dict(precision="bf16x3", max_batch=12, max_len=Lw, max_ctx_len=Lc, max_timesteps=8)
    m = MaskDiT(**kw, **cfg).load_state_dict(sd)
    cn = DiTControlNet(**kw, **cfg, **synth.CONTROLNET).load_state_dict(sd_cn, mask_embed=sd["mask_embed"])
    cond = torch.rand(2, 1, 2 * max(lens), generator=torch.Generator().manual_seed(5))
    cond[1, :, 2 * lens[1]:] = float("nan")   # past clip 1's end: never read
    sched = DDIMScheduler() if sampler == "ddim" else DPMSolverMultistepScheduler(algorithm_type=sampler)
    lat = sample_long_latents(m, sched, ctx, mask, uctx, umask, lens, Lw, O_, gs, gr, steps, eta, seed, controlnet=cn, condition=cond.cuda(),
                              conditioning_scale=scale).cpu()
    init, step_noise = _draws(seed, lens, steps, sampler == "ddim")
    sched.set_timesteps(steps)
    clip = [b for b, _, _ in windows]
    wctx = torch.cat([ctx[clip], uctx.expand(len(windows), -1, -1)])
    wmask = torch.cat([mask[clip], umask.expand(len(windows), -1)])
    wcond = torch.stack([cond[b, :, 2 * s:2 * (s + Lw)] for b, s, _ in windows])
    wcond = torch.cat([wcond, wcond])
    x = [v.double() for v in init]
    m1 = [None] * len(lens)
    with torch.no_grad():
        for i, t in enumerate(sched.timesteps.tolist()):
            xw = torch.stack([x[b][:, s:s + ln] for b, s, ln in windows]).float()
            x257, _ = O.maskdit_concat(sd, torch.cat([xw, xw]))
            sk = O.controlnet_forward(sd_cn, cfg, x257, torch.tensor(t), wctx, wmask, wcond, scale)
            out = O.udit_forward(sd, cfg, x257, torch.tensor(t), wctx, wmask, controlnet_skips=sk)
            o_t, o_u = out.chunk(2, 0)
            vw = O.cfg_combine(o_t, o_u, gs, gr).double().numpy()
            v = [torch.from_numpy(a) for a in _blend64(vw, table, windows, lens, Lw, O_)]
            for b in range(len(lens)):
                if sampler == "ddim":
                    c = [float(e) for e in sched.step_coefficients(t, eta)]
                    x0, eps = c[0] * x[b] - c[1] * v[b], c[0] * v[b] + c[1] * x[b]
                    x[b] = c[2] * x0 + c[3] * eps + c[4] * step_noise[i][b].double()
                else:
                    c, order = sched.step_coefficients(i)
                    m0 = c[0] * x[b] - c[1] * v[b]
                    p = c[2] * x[b] + c[3] * m0
                    if order == 2:
                        p = p + c[4] * (c[5] * (m0 - m1[b]))
                    x[b], m1[b] = p, m0
    for b, n in enumerate(lens):
        err = float((lat[b, :, :n].double() - x[b]).abs().max())
        print(f"[long cn] {sampler} clip {b} ({n} frames, {table[b][1]} windows): loop vs oracle DiT + ControlNet + fp64 windows max-abs {err:.2e}")
        assert err < 5e-3, (b, err)
        assert torch.equal(lat[b, :, n:], torch.zeros(128, max(lens) - n))


# ---------------------------------------------------------------- batches, replay, capacity, the engine
def test_batch_equals_solo_and_replay():
    gc.collect()
    ez = _tiny_cn("bf16", max_batch=6)
    prompts, seeds = ["a siren", "rain on a roof", "wind in trees"], [5, 9, 13]
    clips, gates = [_clip(4.5, 51, 0.3), _clip(1.5, 52), _clip(3, 53)], [0.02, 0.0, 0.05]   # 3 + 1 + 2 windows x 2 = 12 rows
    kw = dict(window_length=2, overlap=0.4, surpass_noise=gates, guidance_scale=3.5, guidance_rescale=0.5, ddim_steps=4, eta=1.0,
              conditioning_scale=1.3)
    sr, batch = ez.generate_long_audio(prompts, clips, random_seed=seeds, **kw)
    assert sr == 24000 and [w.shape for w in batch] == [c.shape for c in clips]
    assert all(np.isfinite(w).all() for w in batch)
    _, again = ez.generate_long_audio(prompts, clips, random_seed=seeds, **kw)   # graph replay
    for a, b in zip(batch, again):
        assert a.tobytes() == b.tobytes()
    for p, c, g, s, w in zip(prompts, clips, gates, seeds, batch):
        _, solo = ez.generate_long_audio(p, c, random_seed=s, **dict(kw, surpass_noise=g))
        assert solo.tobytes() == w.tobytes(), p
    _, shifted = ez.generate_long_audio(prompts, clips, random_seed=[s + 1 for s in seeds], **kw)
    assert all(a.tobytes() != b.tobytes() for a, b in zip(batch, shifted))


def test_row_capacity_raises_and_leaves_the_handle_usable():
    gc.collect()
    ez = _tiny_cn("bf16", max_batch=3)   # 6 rows
    kw = dict(window_length=2, overlap=0.4, ddim_steps=3, random_seed=1)
    with pytest.raises(ValueError, match="max_batch >= 6"):
        ez.generate_long_audio("rain", _clip(10, 61), **kw)   # 6 windows x 2
    _, a = ez.generate_long_audio("rain", _clip(4.5, 62), **kw)   # 3 windows x 2
    _, b = ez.generate_long_audio("rain", _clip(4.5, 62), **kw)
    assert a.tobytes() == b.tobytes() and np.isfinite(a).all() and a.shape == (int(4.5 * 24000),)
    _, c = ez.generate_audio("rain", _clip(2, 63), ddim_steps=3, random_seed=1)
    assert np.isfinite(c).all()


def test_engine_sharing_the_handles_with_a_long_call():
    from ezaudio_b200.engine import ContinuousEngine
    from ezaudio_b200.frontend import ControlRequest
    gc.collect()
    ez = _tiny_cn("bf16", max_batch=4)
    eng = ContinuousEngine(ez, slots=3, ddim_steps=(4, 8))
    (_, want), = eng.run([ControlRequest(**TARGET)])
    _, long = ez.generate_long_audio("a cat", _clip(6, 71), window_length=2, overlap=0.4, ddim_steps=3, random_seed=1)   # 4 windows x 2
    assert np.isfinite(long).all()
    (_, again), = eng.run([ControlRequest(**TARGET)])
    (_, fresh), = ContinuousEngine(ez, slots=3, ddim_steps=(4, 8)).run([ControlRequest(**TARGET)])
    assert again.tobytes() == want.tobytes() and fresh.tobytes() == want.tobytes()
