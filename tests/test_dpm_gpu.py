"""DPM-Solver++ multistep on the GPU: the fused CFG + rescale + DPM-Solver++ kernels (ezb_cfg_dpm_step, ezb_cfg_dpm_step_slots) against an
fp64 restatement and against themselves (lens, slots), a 25-step schedule with an analytic Gaussian denoiser, the sampling loop against the
oracle's DiT driven with the fp64 update, graph replay, batched lengths, and the continuous engine (text-to-audio and ControlNet)."""
import gc

import numpy as np
import pytest
import torch

from ezaudio_b200 import _lib, synth, weights
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
from oracle import ezaudio_oracle as O

pytestmark = pytest.mark.gpu

ALGS = ("dpmsolver++", "sde-dpmsolver++")


def _dpm_ref(t, u, x, m1, z, n, gs, gr, c, order):
    """float64 rescale_noise_cfg + DPM-Solver++ update of one sample's first n frames -> (prev, m0, fp32 allowance of prev, of m0)."""
    t, x = t.double(), x.double()
    if u is None:
        v, V = t, t.abs()
    else:
        u = u.double()
        v = u + gs * (t - u)
        V = u.abs() + abs(gs) * (t.abs() + u.abs())
        if gr > 0:
            ratio = float(t.std() / v.std())
            v = gr * (v * ratio) + (1 - gr) * v
            V = V * (1 + ratio)
    c = [float(e) for e in c]
    m0 = c[0] * x - c[1] * v
    M0 = abs(c[0]) * x.abs() + abs(c[1]) * V
    prev = c[2] * x + c[3] * m0
    mag = abs(c[2]) * x.abs() + abs(c[3]) * M0
    if order == 2:
        prev = prev + c[4] * (c[5] * (m0 - m1.double()))
        mag = mag + abs(c[4] * c[5]) * (M0 + m1.double().abs())
    if z is not None:
        prev = prev + c[6] * z.double()
        mag = mag + abs(c[6]) * z.double().abs()
    return prev, m0, 2.0 ** -20 * mag, 2.0 ** -20 * M0


def _dpm_call(mo, lat, hist, noise, B, Cc, L, gs, gr, coef, order, lens=None):
    from ezaudio_b200.inference import _dpm_step
    _dpm_step(mo, lat, hist, noise, B, Cc, L, gs, gr, coef, order, lens)


CASES = [  # (B, C, L, guidance, rescale, lens)
    (1, 128, 1, 5.0, 0.75, None), (4, 128, 500, 5.0, 0.75, None), (4, 128, 500, 5.0, 0.0, None), (4, 128, 500, 0.0, 0.75, None),
    (4, 128, 1500, 5.0, 0.75, [1500, 1, 777, 1499]), (3, 130, 7, 3.5, 0.75, [7, 3, 1]), (2, 3, 1, 5.0, 0.75, None)]


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("B,Cc,L,gs,gr,lens", CASES)
def test_cfg_dpm_step(B, Cc, L, gs, gr, lens, alg, order):
    """Per-element bound against fp64; padded frames of latents and history keep their NaNs; unread noise (kz = 0) and unread history
    (order 1) hold NaN; each sample under lens is bit-identical to a call on that clip alone; a second call gives the same bits."""
    s = DPMSolverMultistepScheduler(algorithm_type=alg)
    s.set_timesteps(25)
    step = 7 if order == 2 else 0
    coef, o = s.step_coefficients(step)
    assert o == order
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + L)
    rows = 2 * B if gs != 0 else B
    mo = torch.randn(rows, Cc, L, device="cuda", generator=g)
    lat0 = torch.randn(B, Cc, L, device="cuda", generator=g)
    hist0 = torch.randn(B, Cc, L, device="cuda", generator=g)
    noise = torch.randn(B, Cc, L, device="cuda", generator=g) if coef[6] != 0 else None
    n = lens if lens is not None else [L] * B
    if order == 1:
        hist0.fill_(float("nan"))   # not read at order 1
    for b in range(B):
        for r in ((b, B + b) if gs != 0 else (b,)):
            mo[r, :, n[b]:] = float("nan")
        lat0[b, :, n[b]:] = float("nan")
        hist0[b, :, n[b]:] = float("nan")
        if noise is not None:
            noise[b, :, n[b]:] = float("nan")
    lens_d = None if lens is None else torch.tensor(lens, dtype=torch.int32, device="cuda")
    lat, hist = lat0.clone(), hist0.clone()
    unread = torch.full((B, Cc, L), float("nan"), device="cuda")   # the noise when kz == 0: must not be read
    _dpm_call(mo, lat, hist, noise if noise is not None else unread, B, Cc, L, gs, gr, coef, order, lens_d)
    lat2, hist2 = lat0.clone(), hist0.clone()
    _dpm_call(mo, lat2, hist2, noise if noise is not None else unread, B, Cc, L, gs, gr, coef, order, lens_d)
    torch.cuda.synchronize()
    assert torch.equal(lat.view(torch.int32), lat2.view(torch.int32)) and torch.equal(hist.view(torch.int32), hist2.view(torch.int32))
    c32 = [float(np.float32(v)) for v in coef]
    for b in range(B):
        sl = (b, slice(None), slice(0, n[b]))
        ref, m0, allow, allow_m = _dpm_ref(mo[sl], mo[(B + b,) + sl[1:]] if gs != 0 else None, lat0[sl], hist0[sl],
                                           None if noise is None else noise[sl], n[b], gs, gr, c32, order)
        err, err_m = (lat[sl].double() - ref).abs(), (hist[sl].double() - m0).abs()
        assert bool((err <= allow).all()), f"sample {b}: err {float(err.max()):.3e}"
        assert bool((err_m <= allow_m).all()), f"sample {b}: m0 err {float(err_m.max()):.3e}"
        assert bool(torch.isnan(lat[b, :, n[b]:]).all()) and bool(torch.isnan(hist[b, :, n[b]:]).all()), f"sample {b}: padded frames written"
        if lens is not None:   # the clip alone: a packed [1, C, n] call
            rows_b = [mo[b:b + 1, :, :n[b]]] + ([mo[B + b:B + b + 1, :, :n[b]]] if gs != 0 else [])
            ls, hs = lat0[b:b + 1, :, :n[b]].contiguous(), hist0[b:b + 1, :, :n[b]].contiguous()
            nz = noise[b:b + 1, :, :n[b]].contiguous() if noise is not None else None
            _dpm_call(torch.cat(rows_b).contiguous(), ls, hs, nz, 1, Cc, n[b], gs, gr, coef, order)
            torch.cuda.synchronize()
            assert torch.equal(lat[b, :, :n[b]].view(torch.int32), ls[0].view(torch.int32)), b
            assert torch.equal(hist[b, :, :n[b]].view(torch.int32), hs[0].view(torch.int32)), b


def _slot_bytes(struct, slots):
    arr = (struct * len(slots))()
    for a, (gs, gr, coef, flags) in zip(arr, slots):
        a.guidance_scale, a.guidance_rescale, a.flags = gs, gr, flags
        a.coef[:] = coef
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.int32).cuda()


def test_cfg_dpm_step_slots_matches_per_sample_calls_next_to_ddim_slots():
    """The DDIM slots kernel then the DPM one on the same buffers, as the engine launches them: every DPM slot equals ezb_cfg_dpm_step on
    that sample alone, every DDIM slot equals ezb_cfg_ddim_step, bit for bit; inactive slots keep latents and history byte for byte."""
    from ezaudio_b200.inference import _ddim_step
    B, Cc, L = 7, 128, 100
    lens = [100, 37, 1, 64, 100, 50, 80]
    A, G, O2 = _lib.SLOT_ACTIVE, _lib.SLOT_CFG, _lib.SLOT_ORDER2
    dpm = {}
    for alg in ALGS:
        s = DPMSolverMultistepScheduler(algorithm_type=alg)
        s.set_timesteps(10)
        dpm[alg] = [s.step_coefficients(i) for i in range(10)]
    ddim = DDIMScheduler()
    ddim.set_timesteps(10)
    dd = ddim.step_coefficients(int(ddim.timesteps[3]), 1.0)
    # per sample: ("dpm", gs, gr, coef, order, flags) / ("ddim", gs, gr, coef, flags) / None (free)
    plan = [("dpm", 5.0, 0.75) + dpm["dpmsolver++"][4] + (A | G | O2,), ("ddim", 5.0, 0.75, dd, A | G), ("dpm", 0.0, 0.75) + dpm["sde-dpmsolver++"][0] + (A,),
            None, ("dpm", 3.5, 0.0) + dpm["sde-dpmsolver++"][9] + (A | G,), ("dpm", 5.0, 0.5) + dpm["sde-dpmsolver++"][5] + (A | G | O2,),
            ("ddim", 0.0, 0.0, ddim.step_coefficients(int(ddim.timesteps[9]), 0.0), A)]
    zero5, zero7 = (0.0,) * 5, (0.0,) * 7
    ddim_slots = [(p[1], p[2], p[3], p[4]) if p and p[0] == "ddim" else (0.0, 0.0, zero5, 0) for p in plan]
    dpm_slots = [(p[1], p[2], p[3], p[5]) if p and p[0] == "dpm" else (0.0, 0.0, zero7, 0) for p in plan]
    g = torch.Generator(device="cuda").manual_seed(5)
    mo = torch.randn(2 * B, Cc, L, device="cuda", generator=g)
    lat = torch.randn(B, Cc, L, device="cuda", generator=g)
    hist = torch.randn(B, Cc, L, device="cuda", generator=g)
    nz = torch.randn(B, Cc, L, device="cuda", generator=g)
    lat_p, hist_p = lat.clone(), hist.clone()
    for b, n in enumerate(lens):
        lat_p[b, :, n:] = 7.0
        hist_p[b, :, n:] = 7.0
    before_l, before_h = lat_p.clone(), hist_p.clone()
    lens_d = torch.tensor(lens, dtype=torch.int32, device="cuda")
    L_ = _lib.lib()
    _lib.check(L_.ezb_cfg_ddim_step_slots(0, _lib.ptr(mo), _lib.ptr(lat_p), _lib.ptr(nz), _lib.ptr(_slot_bytes(_lib.DdimSlot, ddim_slots)), B, Cc, L,
                                          _lib.stream_ptr(), _lib.ptr(lens_d)))
    _lib.check(L_.ezb_cfg_dpm_step_slots(0, _lib.ptr(mo), _lib.ptr(lat_p), _lib.ptr(hist_p), _lib.ptr(nz), _lib.ptr(_slot_bytes(_lib.DpmSlot, dpm_slots)),
                                         B, Cc, L, _lib.stream_ptr(), _lib.ptr(lens_d)))
    torch.cuda.synchronize()
    for b, (p, n) in enumerate(zip(plan, lens)):
        if p is None:
            assert torch.equal(lat_p[b].view(torch.int32), before_l[b].view(torch.int32)) and torch.equal(hist_p[b].view(torch.int32),
                                                                                                          before_h[b].view(torch.int32)), b
            continue
        cfg = bool(p[-1] & G)
        rows = torch.cat([mo[b:b + 1, :, :n]] + ([mo[B + b:B + b + 1, :, :n]] if cfg else [])).contiguous()
        ls, hs = lat[b:b + 1, :, :n].contiguous(), hist[b:b + 1, :, :n].contiguous()
        if p[0] == "ddim":
            _ddim_step(rows, ls, nz[b:b + 1, :, :n].contiguous() if p[3][4] else None, 1, Cc, n, p[1] if cfg else 0.0, p[2], p[3])
            torch.cuda.synchronize()
            assert torch.equal(hist_p[b].view(torch.int32), before_h[b].view(torch.int32)), b   # a DDIM slot's history is untouched
        else:
            _dpm_call(rows, ls, hs, nz[b:b + 1, :, :n].contiguous() if p[3][6] else None, 1, Cc, n, p[1] if cfg else 0.0, p[2], p[3], p[4])
            torch.cuda.synchronize()
            assert torch.equal(hist_p[b, :, :n], hs[0]), b
        assert torch.equal(lat_p[b, :, :n], ls[0]), (b, p[0])
        assert bool((lat_p[b, :, n:] == 7.0).all()) and bool((hist_p[b, :, n:] == 7.0).all()), b


def test_analytic_gaussian_schedule_through_the_kernel():
    """25 DPM-Solver++ 2M steps with the exact posterior-mean denoiser of N(0.3, 0.7^2) data, evaluated on the GPU in fp32 each step and
    updated by the kernel (no guidance), end within 1e-4 max-abs of the same schedule run in fp64 on the host."""
    mu, sd, B, Cc, L = 0.3, 0.7, 2, 128, 500
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(25)
    abar = DDIMScheduler().alphas_cumprod.double().numpy()
    x = torch.randn(B, Cc, L, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    xh = x.double().cpu()
    hist = torch.empty_like(x)
    m1 = None

    def v_of(x, a, sg):
        x0 = mu + a * sd * sd / (a * a * sd * sd + sg * sg) * (x - a * mu)
        return a * (x - a * x0) / sg - sg * x0

    for i, t in enumerate(s.timesteps.tolist()):
        a, sg = float(np.sqrt(abar[t])), float(np.sqrt(1 - abar[t]))
        coef, order = s.step_coefficients(i)
        _dpm_call(v_of(x, a, sg).contiguous(), x, hist, None, B, Cc, L, 0.0, 0.0, coef, order)
        v = v_of(xh, a, sg)
        m0 = coef[0] * xh - coef[1] * v
        p = coef[2] * xh + coef[3] * m0
        if order == 2:
            p = p + coef[4] * (coef[5] * (m0 - m1))
        xh, m1 = p, m0
    torch.cuda.synchronize()
    err = float((x.cpu().double() - xh).abs().max())
    print(f"[dpm] 25-step analytic Gaussian: kernel vs fp64 host max-abs {err:.2e}")
    assert err < 1e-4, err


def _setup(B=2, L=40, Lc=12):
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    ctx, mask = synth.synth_context(B, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    noise = synth.synth_latents(B, L, seed=5)
    return cfg, sd, ctx, mask, uctx, umask, noise


def _oracle_dpm(sd, cfg, noise, ctx, mask, uctx, umask, gt, gm, gs, gr, steps, alg, step_noise):
    """The oracle's DiT forward (the one O.sample_loop calls) driven step by step with the fp64 DPM-Solver++ update."""
    s = DPMSolverMultistepScheduler(algorithm_type=alg)
    s.set_timesteps(steps)
    x, m1 = noise.double(), None
    for i, t in enumerate(O.DDIM().set_timesteps(steps)):
        assert int(t) == int(s.timesteps[i])
        xf = x.float()
        if gs:
            out, _ = O.maskdit_forward(sd, cfg, torch.cat([xf, xf]), t, torch.cat([ctx, uctx]), torch.cat([mask, umask]),
                                       None if gt is None else torch.cat([gt, gt]), None if gm is None else torch.cat([gm, gm]))
            o_t, o_u = out.chunk(2, 0)
            v = O.cfg_combine(o_t, o_u, gs, gr).double()
        else:
            out, _ = O.maskdit_forward(sd, cfg, xf, t, ctx, mask, gt, gm)
            v = out.double()
        c, order = s.step_coefficients(i)
        m0 = c[0] * x - c[1] * v
        p = c[2] * x + c[3] * m0
        if order == 2:
            p = p + c[4] * (c[5] * (m0 - m1))
        if c[6] != 0:
            p = p + c[6] * step_noise[i].double()
        x, m1 = p, m0
    x = x.float()
    return torch.where(gm, x, gt) if gt is not None else x


@pytest.mark.parametrize("alg,gs,gr,inpaint,steps", [("dpmsolver++", 3.0, 0.5, False, 4), ("dpmsolver++", None, 0.0, False, 5),
                                                     ("sde-dpmsolver++", 5.0, 0.75, False, 6), ("dpmsolver++", 3.5, 0.0, True, 5),
                                                     ("sde-dpmsolver++", 3.5, 0.75, True, 4)])
def test_loop_matches_oracle_dit_with_fp64_update(alg, gs, gr, inpaint, steps):
    from ezaudio_b200.dit import MaskDiT
    from ezaudio_b200.inference import sample_latents
    B, L, Lc = 2, 40, 12
    cfg, sd, ctx, mask, uctx, umask, noise = _setup(B, L, Lc)
    g = torch.Generator().manual_seed(9)
    step_noise = [torch.randn(B, 128, L, generator=g) for _ in range(steps)]
    gt, gm = synth.synth_gt(B, L) if inpaint else (None, None)
    with torch.no_grad():
        ref = _oracle_dpm(sd, cfg, noise, ctx, mask, uctx.expand(B, -1, -1), umask.expand(B, -1), gt, gm, gs, gr, steps, alg, step_noise)
    m = MaskDiT(precision="bf16x3", max_batch=2 * B, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    lat = sample_latents(m, DPMSolverMultistepScheduler(algorithm_type=alg), ctx, mask, uctx, umask, gt, gm, audio_frames=L, guidance_scale=gs,
                         guidance_rescale=gr, ddim_steps=steps, eta=1.0, init_noise=noise, step_noise=[s.cuda() for s in step_noise])
    err = float((lat.cpu() - ref).abs().max())
    print(f"[dpm] {alg} {steps} steps gs {gs} gr {gr} inpaint {inpaint}: loop vs oracle DiT + fp64 update max-abs {err:.2e}")
    assert err < 5e-3, err


@pytest.mark.parametrize("alg", ALGS)
def test_graph_replay_equals_eager(alg):
    from ezaudio_b200.dit import MaskDiT
    from ezaudio_b200.inference import sample_latents
    gc.collect()   # models of earlier tests (and their captured graphs) must not be finalised during this test's capture
    B, L, Lc, steps = 2, 40, 12, 5
    cfg, sd, ctx, mask, uctx, umask, noise = _setup(B, L, Lc)
    g = torch.Generator().manual_seed(9)
    step_noise = [torch.randn(B, 128, L, generator=g).cuda() for _ in range(steps)]
    m = MaskDiT(precision="bf16", max_batch=2 * B, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    kw = dict(audio_frames=L, guidance_scale=5.0, guidance_rescale=0.75, ddim_steps=steps, eta=1.0, init_noise=noise, step_noise=step_noise)
    a = sample_latents(m, DPMSolverMultistepScheduler(algorithm_type=alg), ctx, mask, uctx, umask, **kw)
    b = sample_latents(m, DPMSolverMultistepScheduler(algorithm_type=alg), ctx, mask, uctx, umask, **kw)
    c = sample_latents(m, DPMSolverMultistepScheduler(algorithm_type=alg), ctx, mask, uctx, umask, use_graphs=False, **kw)
    d = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, **kw)   # same shapes, other sampler: another graph
    assert torch.equal(a, b) and torch.equal(a, c)
    assert not torch.equal(a, d)


def _tiny_ez(precision, monkeypatch):
    from tests.test_engine_gpu import _tiny_ez as make
    return make(precision, monkeypatch)


@pytest.mark.parametrize("alg", ALGS)
def test_generate_audio_lengths_equal_solo_calls(alg, monkeypatch):
    ez = _tiny_ez("bf16", monkeypatch)
    ez.noise_scheduler = DPMSolverMultistepScheduler(**ez.params["diff"], algorithm_type=alg)
    prompts, lengths, seeds = ["rain", "a dog barks", "wind"], [1.0, 2.0, 0.6], [11, 12, 13]
    sr, wavs = ez.generate_audio(prompts, length=lengths, ddim_steps=6, random_seed=seeds)
    for p, n, s, w in zip(prompts, lengths, seeds, wavs):
        sr1, w1 = ez.generate_audio(p, length=n, ddim_steps=6, random_seed=s)
        assert sr1 == sr and np.asarray(w1).tobytes() == np.asarray(w).tobytes(), (p, n)


MIX = [dict(prompt="rain on a roof", length=2, guidance_scale=3.5, guidance_rescale=0.0, ddim_steps=8, eta=0.0, random_seed=21),
       dict(prompt="", length=0.7, guidance_scale=5, guidance_rescale=0.75, ddim_steps=4, eta=1.0, random_seed=22),
       dict(prompt="wind in trees", length=1.3, guidance_scale=5, guidance_rescale=0.75, ddim_steps=4, eta=1.0, random_seed=23)]
TARGET = dict(prompt="a dog barks", length=1.5, guidance_scale=5, guidance_rescale=0.75, ddim_steps=8, eta=1.0, random_seed=7, scheduler="dpmsolver++")
SDE = dict(prompt="a bell", length=1.1, guidance_scale=3.5, guidance_rescale=0.5, ddim_steps=4, random_seed=8, scheduler="sde-dpmsolver++")
ALL = ("ddim",) + ALGS


def test_engine_dpm_requests_next_to_ddim_requests(monkeypatch):
    from ezaudio_b200.engine import ContinuousEngine
    from ezaudio_b200.frontend import Request
    ez = _tiny_ez("bf16", monkeypatch)
    alone = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8), schedulers=ALL)
    want = {k: alone.run([Request(**d)])[0][1] for k, d in (("target", TARGET), ("sde", SDE))}
    eng = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8), schedulers=ALL)
    t_mix = [eng.submit(**MIX[0])]
    t_sde = eng.submit(**SDE)
    out = {}
    for _ in range(3):
        out.update({t: w for t, _, w in eng.step()})
    t_target = eng.submit(**TARGET)
    t_mix += [eng.submit(**MIX[1]), eng.submit(**MIX[2])]   # DDIM requests admitted mid-flight
    for t, _, w in eng.stream():
        out[t] = w
    assert out[t_target].tobytes() == want["target"].tobytes()
    assert out[t_sde].tobytes() == want["sde"].tobytes()
    assert eng.backend.captures == 1 and alone.backend.captures == 1
    # the DDIM requests come out as in a default (DDIM-only) engine
    plain = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8))
    ref = plain.run([Request(**d) for d in MIX])
    for t, (_, w) in zip(t_mix, ref):
        assert out[t].tobytes() == w.tobytes(), t
    assert plain.backend.hist is None and plain.backend.dpm_slots_dev is None


def test_engine_dpm_latents_match_solo_sample_latents(monkeypatch):
    """A DPM request's latents in the engine against sample_latents of the same request alone (same seed: the same initial and step draws);
    the batch composition picks other DiT kernels, so the bound is the bf16x3 one."""
    from ezaudio_b200.engine import ContinuousEngine
    from ezaudio_b200.inference import sample_latents
    ez = _tiny_ez("bf16x3", monkeypatch)
    eng = ContinuousEngine(ez, slots=2, max_length_s=2, ddim_steps=(4, 8), schedulers=ALL)
    lat = {}
    finish = eng.backend.finish

    def keep(k, frames):
        lat[frames] = eng.backend.lat[k, :, :frames].cpu()
        return finish(k, frames)

    eng.backend.finish = keep
    for r in (TARGET, SDE, MIX[0]):
        eng.submit(**r)
    while eng.pending():
        eng.step()
    uctx, umask = ez.encode_text([""])
    for r in (TARGET, SDE):
        n = int(r["length"] * 50)
        ctx, mask = ez.encode_text([r["prompt"]])
        ref = sample_latents(ez.unet, DPMSolverMultistepScheduler(algorithm_type=r["scheduler"]), ctx, mask, uctx, umask, audio_frames=n,
                             guidance_scale=r["guidance_scale"], guidance_rescale=r["guidance_rescale"], ddim_steps=r["ddim_steps"],
                             random_seed=r["random_seed"]).cpu()
        err = float((lat[n] - ref[0]).abs().max())
        print(f"[dpm] engine vs solo sample_latents ({r['scheduler']}): max-abs {err:.2e}")
        assert err < 5e-3, (r["scheduler"], err)


def test_engine_control_dpm_request():
    from ezaudio_b200.engine import ContinuousEngine
    from ezaudio_b200.frontend import ControlRequest
    from tests.test_controlnet_engine_gpu import MIX as CMIX, TARGET as CTARGET, _tiny_cn
    ez = _tiny_cn("bf16")
    target = dict(CTARGET, scheduler="dpmsolver++")
    alone = ContinuousEngine(ez, slots=3, ddim_steps=(4, 8), schedulers=ALL)
    (_, want), = alone.run([ControlRequest(**target)])
    eng = ContinuousEngine(ez, slots=3, ddim_steps=(4, 8), schedulers=ALL)
    for r in CMIX[:2]:
        eng.submit(**r)
    out = {}
    for _ in range(3):
        out.update({t: w for t, _, w in eng.step()})
    t_target = eng.submit(**target)
    eng.submit(**dict(CMIX[2], scheduler="sde-dpmsolver++"))
    for t, _, w in eng.stream():
        out[t] = w
    assert len(out) == 4 and out[t_target].tobytes() == want.tobytes()
    assert eng.backend.captures == 1
    plain = ContinuousEngine(ez, slots=3, ddim_steps=(4, 8))
    ref = plain.run([ControlRequest(**d) for d in CMIX[:2]])
    assert out[0].tobytes() == ref[0][1].tobytes() and out[1].tobytes() == ref[1][1].tobytes()
