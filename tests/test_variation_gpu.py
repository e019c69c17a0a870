"""Audio-to-audio variations on the GPU: the fused start latent (ezb_vae_encode_noised) against PyTorch's unfused ops and fp64, the sampling
loop started part-way against the oracle's DiT driven by the fp64 DDIM / DPM-Solver++ update, the strength-1 identity with generate_audio,
mixed batches (strengths and lengths) and the continuous engine."""
import functools
import gc

import numpy as np
import pytest
import torch

from ezaudio_b200 import synth, weights
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
from oracle import ezaudio_oracle as O

pytestmark = pytest.mark.gpu

SCALE, SHIFT = 0.18, 0.5   # a scale and shift away from 1 and 0 (the shipped autoencoder's are in params["autoencoder"])


@functools.lru_cache(maxsize=None)
def _state_dict():
    sd = dict(weights.synthetic_state_dict(weights.vae_decoder_param_shapes(synth.tiny_vae(16)), 6))
    sd.update(weights.synthetic_state_dict(weights.vae_encoder_param_shapes(synth.tiny_vae_encoder(16)), 8))
    return sd


def _codec(precision="bf16", B=4, L=60):
    from ezaudio_b200.vae import OobleckDecoder
    return OobleckDecoder(precision=precision, max_batch=B, max_latent_len=L, encoder_cfg=synth.tiny_vae_encoder(16),
                          **synth.tiny_vae(16)).load_state_dict(_state_dict())


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("lens", [None, [60, 1, 37, 59]])
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_fused_start_latent(precision, lens):
    """x_t = a_b ((z + shift) scale) + s_b eps_b against: PyTorch's three fp32 ops on z of ezb_vae_encode[_lens] (bit for bit: the kernel
    rounds each op as PyTorch does), fp64 (each op's rounding bounded), the pairs (0, 1) -> eps and (1, 0) with scale 1, shift 0 -> z, bit for
    bit.  Under lens the padded audio, bottleneck noise and eps hold NaN: nothing of them reaches the clip's frames, and the frames past the
    end come out as zeros.  (The encoder rows past a clip's end are the library's workspace, which the length-aware encoder leaves
    unwritten; that the sample kernels do not read them is shown by those zeros and by tests/test_vae_varlen_gpu.py.)"""
    B, L, hop = 4, 60, 480
    vae = _codec(precision, B, L)
    g = torch.Generator(device="cuda").manual_seed(11)
    audio = 0.3 * torch.randn(B, 1, L * hop, device="cuda", generator=g)
    noise = torch.randn(B, 128, L, device="cuda", generator=g)
    eps = torch.randn(B, 128, L, device="cuda", generator=g)
    ab = torch.tensor([[0.0, 1.0], [1.0, 0.0], [0.6, 0.8], [2.0 ** -12, 1.0]], device="cuda")
    n = lens or [L] * B
    if lens is not None:
        for b, k in enumerate(lens):
            audio[b, :, k * hop:] = float("nan")
            noise[b, :, k:] = float("nan")
            eps[b, :, k:] = float("nan")
    z = vae.encode(audio, noise=noise, lengths=lens)
    x_t = vae.encode_noised(audio, ab, eps, SCALE, SHIFT, noise=noise, lengths=lens)
    torch.cuda.synchronize()
    x0 = (z + SHIFT) * SCALE
    for b, k in enumerate(n):
        want = ab[b, 0] * x0[b, :, :k] + ab[b, 1] * eps[b, :, :k]   # PyTorch's unfused fp32 ops
        assert torch.equal(_bits(x_t[b, :, :k]), _bits(want)), b
        zd, ed = z[b, :, :k].double(), eps[b, :, :k].double()
        a, s = float(ab[b, 0]), float(ab[b, 1])
        ref = a * ((zd + SHIFT) * SCALE) + s * ed
        allow = 2.0 ** -23 * (abs(a) * (zd.abs() + SHIFT) * SCALE * 3 + abs(s) * ed.abs() * 2)
        assert bool(((x_t[b, :, :k].double() - ref).abs() <= allow).all()), b
        assert bool(torch.isfinite(x_t[b, :, :k]).all())
        if lens is not None:
            assert bool((x_t[b, :, k:] == 0).all()) and not bool(torch.signbit(x_t[b, :, k:]).any()), b
    assert torch.equal(_bits(x_t[0, :, :n[0]]), _bits(eps[0, :, :n[0]]))   # (a, s) = (0, 1): x_t is eps
    one = vae.encode_noised(audio, torch.tensor([[1.0, 0.0]] * B), eps, 1.0, 0.0, noise=noise, lengths=lens)
    torch.cuda.synchronize()
    assert torch.equal(_bits(one), _bits(z))   # a = 1, s = 0, scale 1, shift 0: ezb_vae_encode[_lens]'s z, bit for bit


def test_encode_noised_rejects_bad_shapes_before_drawing():
    vae = _codec()
    audio = torch.zeros(2, 1, 10 * 480, device="cuda")
    torch.manual_seed(4)
    before = torch.cuda.get_rng_state()
    with pytest.raises(ValueError):
        vae.encode_noised(audio, [[1.0, 0.0]], torch.zeros(2, 128, 10, device="cuda"), 1.0, 0.0)
    with pytest.raises(ValueError):
        vae.encode_noised(audio, [[1.0, 0.0]] * 2, torch.zeros(2, 128, 9, device="cuda"), 1.0, 0.0)
    assert torch.equal(torch.cuda.get_rng_state(), before)   # a rejected call draws no bottleneck noise


# ---- the sampling loop started part-way, against the oracle's DiT and the fp64 update

def _setup(B=2, L=40, Lc=12):
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    ctx, mask = synth.synth_context(B, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    x_start = synth.synth_latents(B, L, seed=5)
    return cfg, sd, ctx, mask, uctx, umask, x_start


def _oracle(sd, cfg, x_start, starts, ctx, mask, uctx, umask, gs, gr, steps, sched, eta, step_noise):
    """The oracle's DiT forward at every step from min(starts), each sample updated in fp64 from its own start."""
    sched.set_timesteps(steps)
    dpm = sched.kind == "dpm"
    x, m1 = x_start.double(), torch.zeros_like(x_start, dtype=torch.float64)
    B = x.shape[0]
    for i, t in enumerate(O.DDIM().set_timesteps(steps)):
        assert int(t) == int(sched.timesteps[i])
        if i < min(starts):
            continue
        xf = x.float()
        if gs:
            out, _ = O.maskdit_forward(sd, cfg, torch.cat([xf, xf]), t, torch.cat([ctx, uctx]), torch.cat([mask, umask]))
            o_t, o_u = out.chunk(2, 0)
            v = O.cfg_combine(o_t, o_u, gs, gr).double()
        else:
            out, _ = O.maskdit_forward(sd, cfg, xf, t, ctx, mask)
            v = out.double()
        for b in range(B):
            if i < starts[b]:
                continue
            if dpm:
                c, order = sched.step_coefficients(i, begin_index=starts[b])
                m0 = c[0] * x[b] - c[1] * v[b]
                p = c[2] * x[b] + c[3] * m0
                if order == 2:
                    p = p + c[4] * (c[5] * (m0 - m1[b]))
                if c[6] != 0:
                    p = p + c[6] * step_noise[i][b].double()
                x[b], m1[b] = p, m0
            else:
                c = sched.step_coefficients(int(t), eta)
                x0 = c[0] * x[b] - c[1] * v[b]
                e = c[0] * v[b] + c[1] * x[b]
                p = c[2] * x0 + c[3] * e
                if c[4] != 0:
                    p = p + c[4] * step_noise[i][b].double()
                x[b] = p
    return x.float()


LOOP = [("ddim", 0.0, 3.0, 0.5, [2, 2], 6), ("ddim", 1.0, 5.0, 0.75, [1, 3], 6), ("ddim", 0.0, None, 0.0, [3, 4], 6),
        ("dpmsolver++", 0.0, 3.0, 0.5, [2, 2], 7), ("dpmsolver++", 0.0, 3.5, 0.0, [1, 3], 7), ("sde-dpmsolver++", 0.0, 5.0, 0.75, [2, 4], 7)]


@pytest.mark.parametrize("kind,eta,gs,gr,starts,steps", LOOP)
def test_loop_from_a_start_matches_oracle_dit_with_fp64_update(kind, eta, gs, gr, starts, steps):
    from ezaudio_b200.dit import MaskDiT
    from ezaudio_b200.inference import sample_latents
    B, L, Lc = 2, 40, 12
    cfg, sd, ctx, mask, uctx, umask, x_start = _setup(B, L, Lc)
    g = torch.Generator().manual_seed(9)
    step_noise = [torch.randn(B, 128, L, generator=g) for _ in range(steps)]
    mk = (lambda: DDIMScheduler()) if kind == "ddim" else (lambda: DPMSolverMultistepScheduler(algorithm_type=kind))
    with torch.no_grad():
        ref = _oracle(sd, cfg, x_start, starts, ctx, mask, uctx.expand(B, -1, -1), umask.expand(B, -1), gs, gr, steps, mk(), eta, step_noise)
    m = MaskDiT(precision="bf16x3", max_batch=2 * B, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    lat = sample_latents(m, mk(), ctx, mask, uctx, umask, audio_frames=L, guidance_scale=gs, guidance_rescale=gr, ddim_steps=steps, eta=eta,
                         step_noise=[s.cuda() for s in step_noise], start_index=starts, init_latents=x_start)
    err = float((lat.cpu() - ref).abs().max())
    print(f"[variation] {kind} eta {eta} starts {starts}/{steps}: loop vs oracle DiT + fp64 update max-abs {err:.2e}")
    assert err < 5e-3, err


def test_one_start_equals_the_truncated_schedule_and_replays():
    """A batch that starts at k gives the bits of a second call (graph replay) and of an eager run; a new mix of starts with the same
    minimum replays the same graph, and each sample keeps the bits it has alone (bf16x3: the same kernels at every batch size)."""
    from ezaudio_b200.dit import MaskDiT
    from ezaudio_b200.inference import sample_latents
    gc.collect()
    B, L, Lc, steps = 2, 40, 12, 6
    cfg, sd, ctx, mask, uctx, umask, x_start = _setup(B, L, Lc)
    g = torch.Generator().manual_seed(9)
    step_noise = [torch.randn(B, 128, L, generator=g).cuda() for _ in range(steps)]
    m = MaskDiT(precision="bf16x3", max_batch=2 * B, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    kw = dict(audio_frames=L, guidance_scale=5.0, guidance_rescale=0.75, ddim_steps=steps, eta=1.0, step_noise=step_noise, init_latents=x_start)
    a = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, start_index=[2, 2], **kw)
    (entry,) = [v for k, v in m._loop_cache.items() if k[-1] == ("start", 2)]
    graph = entry["graph"]
    b = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, start_index=[2, 2], **kw)
    c = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, start_index=[2, 2], use_graphs=False, **kw)
    assert torch.equal(a, b) and torch.equal(a, c)
    n = len(m._loop_cache)
    d = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, start_index=[4, 2], **kw)
    assert len(m._loop_cache) == n and entry["graph"] is graph   # same min(start_index): replayed
    assert torch.equal(d[1], a[1]) and not torch.equal(d[0], a[0])   # sample 1 does not see sample 0's start
    e = sample_latents(m, DDIMScheduler(), ctx[:1], mask[:1], uctx, umask, start_index=[4], **dict(kw, init_latents=x_start[:1],
                                                                                                   step_noise=[s[:1] for s in step_noise]))
    assert torch.equal(d[0], e[0])


# ---- the API

def _tiny_ez(monkeypatch, precision="bf16", max_batch=3):
    from ezaudio_b200 import api, config
    tiny = config.load_params("s3_xl")
    tiny["model"] = synth.tiny_model(72)
    tiny["text_encoder"] = dict(tiny["text_encoder"], max_length=16)
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    return api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16), max_batch=max_batch,
                       max_length_s=4, precision=precision)


def _clip(seconds, f, sr=24000):
    t = np.arange(int(round(seconds * sr))) / sr
    return (0.3 * np.sin(2 * np.pi * f * t) + 0.05 * np.sin(2 * np.pi * 3 * f * t)).astype(np.float32)


def _record_latents(monkeypatch):
    from ezaudio_b200 import inference as inf
    seen = []
    real = inf.sample_latents

    def rec(*a, **k):
        lat = real(*a, **k)
        seen.append(lat.clone())
        return lat
    monkeypatch.setattr(inf, "sample_latents", rec)
    return seen


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_strength_one_is_generate_audio(monkeypatch, precision):
    """DDIM, strength 1: abar_999 = 0 so x_t = eps bit for bit, and the latents and waveform are generate_audio's for the same prompt, seed
    and frame count, bit for bit."""
    ez = _tiny_ez(monkeypatch, precision)
    seen = _record_latents(monkeypatch)
    sr, want = ez.generate_audio("rain on a roof", length=1.2, ddim_steps=5, random_seed=17)
    sr2, got = ez.variation_audio("rain on a roof", _clip(1.2, 330), strength=1.0, ddim_steps=5, random_seed=17)
    assert sr == sr2 and got.shape == want.shape == (int(1.2 * 24000),)
    assert torch.equal(_bits(seen[0]), _bits(seen[1]))
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    # DPM-Solver++ at strength 1 starts from 2**-12 * x0 + eps: close to, not equal to, generate_audio
    ez.noise_scheduler = DPMSolverMultistepScheduler(**ez.params["diff"])
    _, want = ez.generate_audio("rain on a roof", length=1.2, ddim_steps=5, random_seed=17)
    _, got = ez.variation_audio("rain on a roof", _clip(1.2, 330), strength=1.0, ddim_steps=5, random_seed=17)
    assert not np.array_equal(got, want) and np.isfinite(got).all()


VARS = dict(text=["a bell", "rain on a roof", "a dog barks"], init_audio=[_clip(2.0, 220), _clip(1.31, 330), _clip(0.7, 440)],
            strength=[0.4, 1.0, 0.7], random_seed=[3, 4, 5])


@pytest.mark.parametrize("sched", ["ddim", "dpmsolver++", "sde-dpmsolver++"])
def test_mixed_batch_members_are_independent_and_match_solo_calls(monkeypatch, sched):
    ez = _tiny_ez(monkeypatch, "bf16")
    if sched != "ddim":
        ez.noise_scheduler = DPMSolverMultistepScheduler(**ez.params["diff"], algorithm_type=sched)
    torch.manual_seed(21)
    sr, batch = ez.variation_audio(**VARS, ddim_steps=10, pad_length=2.5)
    assert [w.shape for w in batch] == [(len(c),) for c in VARS["init_audio"]] and all(np.isfinite(w).all() for w in batch)
    cache = ez.unet._loop_cache
    (entry,) = cache.values()
    graph = entry["graph"]
    # same min(start_index) (strength 1 -> 0), other strengths and clips around sample 1: replayed, and sample 1 keeps its bits.  Clip 0
    # keeps its length, so clip 1's bottleneck noise (the global RNG, drawn after clip 0's) is the same draw.
    other = dict(VARS, strength=[0.9, 1.0, 0.2], init_audio=[_clip(2.0, 550), VARS["init_audio"][1], _clip(2.4, 110)])
    torch.manual_seed(21)
    sr, mixed = ez.variation_audio(**other, ddim_steps=10, pad_length=2.5)
    assert len(cache) == 1 and entry["graph"] is graph
    assert np.array_equal(mixed[1], batch[1])
    assert not np.array_equal(mixed[0], batch[0])
    # each member against its solo call (other padding, other kernels: the bf16 bound)
    torch.manual_seed(21)
    for i, got in enumerate(batch):
        one = {k: v[i] for k, v in VARS.items()}
        _, want = ez.variation_audio(**one, ddim_steps=10)
        err = float(np.abs(got - want).max())
        print(f"[variation] {sched} batch member {i} vs solo: max-abs {err:.2e} (|max| {float(np.abs(want).max()):.2e})")
        assert err <= 6e-2 * float(np.abs(want).max()) + 1e-5, (i, err)


def test_list_form_equals_scalar_calls_in_sequence_bf16x3(monkeypatch):
    """bf16x3 takes the same GEMM kernels at every token count, so the batch reproduces the scalar calls bit for bit."""
    ez = _tiny_ez(monkeypatch, "bf16x3")
    torch.manual_seed(21)
    _, batch = ez.variation_audio(**VARS, ddim_steps=6)
    torch.manual_seed(21)   # the scalar calls draw their bottleneck noise from the global RNG in this order
    for i, got in enumerate(batch):
        _, want = ez.variation_audio(**{k: v[i] for k, v in VARS.items()}, ddim_steps=6)
        assert np.array_equal(got, want), (i, float(np.abs(got - want).max()))


def test_fp8_list_form(monkeypatch):
    ez = _tiny_ez(monkeypatch, "fp8")
    sr, w = ez.variation_audio(["a bell", "wind"], [_clip(1.0, 220), _clip(0.5, 330)], strength=[0.5, 0.8], ddim_steps=10, random_seed=[1, 2])
    assert [x.shape for x in w] == [(24000,), (12000,)] and all(np.isfinite(x).all() for x in w)


def test_list_form_is_rejected_before_device_work(monkeypatch):
    from ezaudio_b200 import _lib
    ez = _tiny_ez(monkeypatch, "bf16", 2)
    torch.cuda.synchronize()
    c0 = _lib.lib().ezb_launch_count()
    bad = [dict(text=["a", "b", "c"], init_audio=[_clip(1, 220)] * 3),                       # 3 > max_batch
           dict(text=["a", ""], init_audio=[_clip(1, 220)] * 2),                              # empty mixed with non-empty
           dict(text=["a", "b"], init_audio=[_clip(1, 220)] * 2, strength=[0.5, 0.0]),        # strength 0
           dict(text=["a", "b"], init_audio=[_clip(1, 220)] * 2, strength=0.001),             # no step runs
           dict(text=["a", "b"], init_audio=[_clip(1, 220), _clip(4.5, 220)]),                # longer than max_length_s
           dict(text=["a", "b"], init_audio=[_clip(1, 220)] * 2, pad_length=5),               # pad_length past max_length_s
           dict(text=["a", "b"], init_audio=[_clip(2, 220)] * 2, pad_length=1),               # a clip past pad_length
           dict(text=["a", "b"], init_audio=[_clip(1, 220)]),                                 # one clip for two prompts
           dict(text=["a", "b"], init_audio=[_clip(1, 220), np.zeros(0, np.float32)]),        # empty clip
           dict(text=["a", "b"], init_audio=[_clip(1, 220), np.full(480, np.inf, np.float32)]),  # non-finite clip
           dict(text=["a", "b"], init_audio=[_clip(1, 220)] * 2, random_seed=[1, 2, 3]),      # seeds
           dict(text="a", init_audio=_clip(1, 220), pad_length=2)]                            # pad_length with one prompt
    for kw in bad:
        with pytest.raises(ValueError):
            ez.variation_audio(**kw, ddim_steps=10)
    torch.cuda.synchronize()
    assert _lib.lib().ezb_launch_count() == c0


# ---- the continuous engine

def test_engine_variation_alone_equals_with_co_tenants_and_one_graph(monkeypatch):
    from ezaudio_b200.engine import ContinuousEngine
    from ezaudio_b200.frontend import EditRequest, Request, VariationRequest
    from tests.test_engine_gpu import MIX
    ez = _tiny_ez(monkeypatch, "bf16")
    scheds = ("ddim", "dpmsolver++")
    target = dict(prompt="a dog barks", init_audio=_clip(1.31, 330), strength=0.6, ddim_steps=8, random_seed=7)
    target_dpm = dict(target, prompt="a bell", strength=0.5, scheduler="dpmsolver++")
    edit = dict(prompt="wind", boundary=0.3, gt_file=_clip(1.5, 220), mask_start=0.5, mask_length=0.5, ddim_steps=4, random_seed=9)
    alone = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8), schedulers=scheds)
    want = {}
    for name, r in (("ddim", target), ("dpm", target_dpm)):
        torch.manual_seed(33)
        (_, want[name]), = alone.run([VariationRequest(**r)])
        assert want[name].shape == (len(r["init_audio"]),)
    torch.manual_seed(3)
    (_, want_edit), = alone.run([EditRequest(**edit)])
    eng = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8), schedulers=scheds)
    t_mix = eng.submit(**MIX[0])
    torch.manual_seed(3)
    t_edit = eng.submit(**edit)
    out = {}
    out.update({t: w for t, _, w in eng.step()})   # admits the text-to-audio request and the edit (the edit draws from the global RNG)
    for _ in range(2):
        out.update({t: w for t, _, w in eng.step()})
    t_var = eng.submit(**target)
    torch.manual_seed(33)
    out.update({t: w for t, _, w in eng.step()})   # admits the variation alone
    for t, _, w in eng.stream():
        out[t] = w
    t_dpm = eng.submit(**target_dpm)
    torch.manual_seed(33)
    for t, _, w in eng.stream():
        out[t] = w
    assert out[t_var].tobytes() == want["ddim"].tobytes()
    assert out[t_dpm].tobytes() == want["dpm"].tobytes()
    assert out[t_edit].tobytes() == want_edit.tobytes()
    assert eng.backend.captures == 1 and alone.backend.captures == 1
    plain = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8))
    (_, ref), = plain.run([Request(**MIX[0])])
    assert out[t_mix].tobytes() == ref.tobytes()   # the text-to-audio co-tenant is unchanged
