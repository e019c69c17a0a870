"""Windowed denoising of long clips on the GPU: the gather and blend kernels against fp64 (NaN wherever they must not read), the long loop
against generate_audio for clips that fit one window (bit for bit, DDIM and DPM-Solver++), batches against solo calls and graph replay,
the loop against the oracle's DiT driven by an fp64 restatement of gather / guidance / blend / update, and the tiled VAE decode against a
one-shot decode (bit for bit) together with the receptive field it relies on."""
import functools
import gc

import numpy as np
import pytest
import torch

from ezaudio_b200 import _lib, synth, weights
from ezaudio_b200.inference import long_plan
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
from oracle import ezaudio_oracle as O

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- kernels
def _plan_dev(table):
    return torch.tensor([e for row in table for e in row], dtype=torch.int32, device="cuda")


def _blend64(wins, table, windows, lens, Lw, O_):
    """fp64 restatement of the blend: per clip, sum_k w_k v_k / sum_k w_k over the covering windows."""
    out = []
    for b, (first, count, n) in enumerate(table):
        num, den = np.zeros((wins.shape[1], n)), np.zeros(n)
        for k in range(count):
            _, s, ln = windows[first + k]
            j = np.arange(ln, dtype=np.float64)
            w = np.ones(ln)
            if k > 0:
                w = np.minimum(w, (j + 1) / (O_ + 1))
            if k < count - 1:
                w = np.minimum(w, (Lw - j) / (O_ + 1))
            num[:, s:s + ln] += w * wins[first + k, :, :ln].astype(np.float64)
            den[s:s + ln] += w
        out.append(num / den)
    return out


@pytest.mark.parametrize("C_", [16, 128])
def test_gather_and_blend_against_fp64(C_):
    Lw, O_ = 40, 8
    lens = [73, 37, 130, 40, 1]   # three windows covering frames 33..39 of the first clip, a short single window, four windows, exactly
    table, windows = long_plan(lens, Lw, O_)   # one window, a one-frame clip
    assert table[0][1] == 3 and windows[2] == (0, 33, 40)
    B, W, N = len(lens), len(windows), max(lens)
    g = torch.Generator().manual_seed(4)
    lat = torch.randn(B, C_, N, generator=g)
    for b, n in enumerate(lens):
        lat[b, :, n:] = float("nan")   # past the clip's end: never read
    lat = lat.cuda()
    plan = _plan_dev(table)
    L = _lib.lib()
    st = _lib.stream_ptr()
    for copies in (1, 2):
        win = torch.full((copies * W + 1, C_, Lw), 7.0, device="cuda")   # one spare row: nothing past copies * W is written
        _lib.check(L.ezb_window_gather(0, _lib.ptr(lat), _lib.ptr(win), _lib.ptr(plan), B, C_, N, W, Lw, O_, copies, st))
        got = win.cpu()
        for r, (b, s, ln) in enumerate(windows):
            for c in range(copies):
                row = got[c * W + r]
                assert torch.equal(row[:, :ln], lat[b, :, s:s + ln].cpu()), (r, c)
                assert torch.equal(row[:, ln:], torch.zeros(C_, Lw - ln)), (r, c)
        assert torch.equal(got[copies * W], torch.full((C_, Lw), 7.0))
    # blend: window frames past a window's length hold NaN, the output is prefilled with a sentinel that must survive past each clip's end
    wins = torch.randn(W, C_, Lw, generator=g)
    for r, (_, _, ln) in enumerate(windows):
        wins[r, :, ln:] = float("nan")
    out = torch.full((B, C_, N), 7.0, device="cuda")
    wins_d = wins.cuda()
    _lib.check(L.ezb_window_blend(0, _lib.ptr(wins_d), _lib.ptr(out), _lib.ptr(plan), B, C_, N, W, Lw, O_, st))
    got = out.cpu()
    ref = _blend64(wins.numpy(), table, windows, lens, Lw, O_)
    for b, (first, count, n) in enumerate(table):
        assert torch.equal(got[b, :, n:], torch.full((C_, N - n), 7.0)), b
        err = np.abs(got[b, :, :n].double().numpy() - ref[b])
        bound = 8 * 2.0 ** -24 * np.nanmax(np.abs(wins.numpy()))   # three products and sums, the division and the fp32 weights, of terms <= max|v|
        assert (err <= bound).all(), (b, float(err.max()))
        if count == 1:   # one covering window of weight 1: its values bit for bit
            assert torch.equal(got[b, :, :n], wins[first, :, :n]), b
    # a frame covered by one window inside a multi-window clip (weight 1 there) is also that window's value
    assert torch.equal(got[2, :, :32], wins[table[2][0], :, :32])


def test_kernels_reject_bad_arguments():
    L = _lib.lib()
    x = torch.zeros(8, device="cuda")
    p = _plan_dev([(0, 1, 4)])
    for args in ((1, 1, 4, 1, 4, 0, 1), (1, 1, 4, 1, 4, 3, 1), (1, 1, 4, 0, 4, 1, 1), (1, 1, 4, 1, 4, 1, 3)):
        B, C_, N, W, Lw, O_, copies = args
        assert L.ezb_window_gather(0, _lib.ptr(x), _lib.ptr(x), _lib.ptr(p), B, C_, N, W, Lw, O_, copies, _lib.stream_ptr()) != 0, args
    assert L.ezb_window_blend(0, _lib.ptr(x), _lib.ptr(x), None, 1, 1, 4, 1, 4, 1, _lib.stream_ptr()) != 0


# ---------------------------------------------------------------- the loop through the API
def _ez(monkeypatch, max_batch=3, precision="bf16"):
    from ezaudio_b200 import api, config
    from tests.test_api_gpu import _tiny_params
    tiny = _tiny_params()
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    return api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16),
                       max_batch=max_batch, max_length_s=2, precision=precision)


SAMPLERS = [("ddim", 0.0), ("ddim", 1.0), ("dpmsolver++", 1.0), ("sde-dpmsolver++", 1.0)]


def _set_sampler(ez, alg):
    ez.noise_scheduler = DDIMScheduler(**ez.params["diff"]) if alg == "ddim" else DPMSolverMultistepScheduler(**ez.params["diff"], algorithm_type=alg)


@pytest.mark.parametrize("alg,eta", SAMPLERS)
def test_one_window_equals_generate_audio(alg, eta, monkeypatch):
    gc.collect()
    ez = _ez(monkeypatch)
    _set_sampler(ez, alg)
    for prompt, length, gr in (("a dog barks", 1.5, 0.75), ("rain on a roof", 2, 0.0), ("", 0.7, 0.75)):
        kw = dict(guidance_scale=5, guidance_rescale=gr, ddim_steps=6, eta=eta, random_seed=17)
        sr, want = ez.generate_audio(prompt, length=length, **kw)
        sr2, got = ez.generate_long_audio(prompt, length=length, window_length=2, overlap=0.4, **kw)
        assert sr2 == sr and got.dtype == want.dtype and got.shape == want.shape == (480 * int(length * 50),), (prompt, got.shape)
        assert got.tobytes() == want.tobytes(), (alg, eta, prompt)


@pytest.mark.parametrize("alg,eta", [("ddim", 1.0), ("sde-dpmsolver++", 1.0)])
def test_batch_equals_solo_and_replay(alg, eta, monkeypatch):
    gc.collect()
    ez = _ez(monkeypatch, max_batch=8)
    _set_sampler(ez, alg)
    prompts, lengths, seeds = ["rain on a roof", "engine hum", "crowd noise"], [3.3, 0.9, 2.5], [5, 9, 13]
    kw = dict(window_length=1, overlap=0.2, guidance_scale=5, guidance_rescale=0.75, ddim_steps=5, eta=eta)
    sr, batch = ez.generate_long_audio(prompts, length=lengths, random_seed=seeds, **kw)   # 4 + 1 + 3 windows, 16 DiT rows
    assert [w.shape for w in batch] == [(480 * int(s * 50),) for s in lengths]
    assert all(np.isfinite(w).all() for w in batch)
    _, again = ez.generate_long_audio(prompts, length=lengths, random_seed=seeds, **kw)    # graph replay
    for a, b in zip(batch, again):
        assert a.tobytes() == b.tobytes()
    for p, n, s, w in zip(prompts, lengths, seeds, batch):
        _, solo = ez.generate_long_audio(p, length=n, random_seed=s, **kw)
        assert solo.tobytes() == w.tobytes(), p
    _, shifted = ez.generate_long_audio(prompts, length=lengths, random_seed=[s + 1 for s in seeds], **kw)
    assert all(a.tobytes() != b.tobytes() for a, b in zip(batch, shifted))


def test_row_capacity_raises_and_leaves_the_handle_usable(monkeypatch):
    gc.collect()
    ez = _ez(monkeypatch, max_batch=3)   # 6 DiT rows
    with pytest.raises(ValueError, match="max_batch >= 4"):
        ez.generate_long_audio("rain", length=3.3, window_length=1, overlap=0.2, ddim_steps=3, random_seed=1)   # 4 windows x 2
    _, a = ez.generate_long_audio("rain", length=2.5, window_length=1, overlap=0.2, ddim_steps=3, random_seed=1)   # 3 windows x 2
    _, b = ez.generate_long_audio("rain", length=2.5, window_length=1, overlap=0.2, ddim_steps=3, random_seed=1)
    assert a.tobytes() == b.tobytes() and np.isfinite(a).all()
    _, c = ez.generate_audio("rain", length=1, ddim_steps=3, random_seed=1)
    assert np.isfinite(c).all()


# ---------------------------------------------------------------- the loop against the oracle
def _setup(B=2, Lw=40, Lc=12):
    from ezaudio_b200.dit import MaskDiT
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    ctx, mask = synth.synth_context(B, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    m = MaskDiT(precision="bf16x3", max_batch=12, max_len=Lw, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    return cfg, sd, m, ctx, mask, uctx, umask


def _draws(seed, lens, steps, draw):
    gens = [torch.Generator(device="cuda").manual_seed(seed + b) for b in range(len(lens))]
    init = [torch.randn((1, 128, n), generator=g, device="cuda")[0].cpu() for g, n in zip(gens, lens)]
    noise = [[torch.empty((1, 128, n), device="cuda").normal_(generator=g)[0].cpu() for g, n in zip(gens, lens)] for _ in range(steps)] if draw else None
    return init, noise


@pytest.mark.parametrize("sampler", ["ddim", "dpmsolver++"])
def test_long_loop_matches_oracle_dit_with_fp64_windows(sampler):
    from ezaudio_b200.inference import sample_long_latents
    gc.collect()
    lens, Lw, O_, gs, gr, steps, eta, seed = [73, 61], 40, 8, 3.0, 0.5, 4, 1.0, 11
    table, windows = long_plan(lens, Lw, O_)
    assert table[0][1] == 3   # three windows, the last overlapping both others
    cfg, sd, m, ctx, mask, uctx, umask = _setup()
    sched = DDIMScheduler() if sampler == "ddim" else DPMSolverMultistepScheduler(algorithm_type=sampler)
    lat = sample_long_latents(m, sched, ctx, mask, uctx, umask, lens, Lw, O_, gs, gr, steps, eta, seed).cpu()
    init, step_noise = _draws(seed, lens, steps, sampler == "ddim")
    sched.set_timesteps(steps)
    clip = [b for b, _, _ in windows]
    wctx = torch.cat([ctx[clip], uctx.expand(len(windows), -1, -1)])
    wmask = torch.cat([mask[clip], umask.expand(len(windows), -1)])
    x = [v.double() for v in init]
    m1 = [None] * len(lens)
    with torch.no_grad():
        for i, t in enumerate(sched.timesteps.tolist()):
            xw = torch.stack([x[b][:, s:s + ln] for b, s, ln in windows]).float()
            out, _ = O.maskdit_forward(sd, cfg, torch.cat([xw, xw]), torch.tensor(t), wctx, wmask)
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
        print(f"[long] {sampler} clip {b} ({n} frames, {table[b][1]} windows): loop vs oracle DiT + fp64 windows max-abs {err:.2e}")
        assert err < 5e-3, (b, err)
        assert torch.equal(lat[b, :, n:], torch.zeros(128, max(lens) - n))


def test_long_graph_replay_equals_eager():
    from ezaudio_b200.inference import sample_long_latents
    gc.collect()
    cfg, sd, m, ctx, mask, uctx, umask = _setup()
    args = (m, DDIMScheduler(), ctx, mask, uctx, umask, [73, 61], 40, 8, 3.0, 0.5, 4, 1.0, 11)
    eager = sample_long_latents(*args, use_graphs=False)
    first = sample_long_latents(*args)    # eager pass + capture
    replay = sample_long_latents(*args)   # replay
    assert torch.equal(eager, first) and torch.equal(eager, replay)
    other = sample_long_latents(*args[:6], [61, 73], *args[7:])   # same rows and longest clip: the same graph follows the new plan
    solo = sample_long_latents(*args[:6], [61, 73], *args[7:], use_graphs=False)
    assert torch.equal(other, solo)


# ---------------------------------------------------------------- tiled VAE decode
VAES = {"tiny": synth.tiny_vae(16), "full": synth.VAE_DECODER}


@functools.lru_cache(maxsize=None)
def _vae_sd(name):
    return weights.synthetic_state_dict(weights.vae_decoder_param_shapes(VAES[name]), 6)


def _dec(name, M, B, precision="bf16"):
    from ezaudio_b200.vae import OobleckDecoder
    return OobleckDecoder(precision=precision, max_batch=B, max_latent_len=M, **VAES[name]).load_state_dict(_vae_sd(name))


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("name", ["tiny", "full"])
def test_decode_tiled_equals_one_shot(name, precision):
    gc.collect()
    small, big = _dec(name, 40, 3, precision), _dec(name, 160, 3, precision)   # chunks of <= 40 frames: cores of 22 inside 9-frame halos
    z = synth.synth_latents(1, 150, seed=3).cuda()
    assert torch.equal(small.decode_tiled(z), big(z))
    lens = [150, 61, 23]
    zb = synth.synth_latents(3, 150, seed=4)
    for b, n in enumerate(lens):
        zb[b, :, n:] = float("nan")   # past a clip's end: never read
    zb = zb.cuda()
    want = big(zb, lengths=lens)
    got = small.decode_tiled(zb, lengths=lens)
    assert torch.equal(got, want)
    assert torch.equal(got[1, :, 61 * 480:], torch.zeros(1, (150 - 61) * 480, device="cuda"))


def test_receptive_field_bounds_a_perturbation():
    from ezaudio_b200.vae import decoder_receptive_field
    gc.collect()
    h = decoder_receptive_field(synth.VAE_DECODER)
    dec = _dec("full", 60, 1)
    z = synth.synth_latents(1, 60, seed=5).cuda()
    base = dec(z)
    for q in (0, 29, 59):
        zp = z.clone()
        zp[:, :, q] += 1.0
        d = (dec(zp) - base)[0, 0].abs().cpu()
        lo, hi = max(0, (q - h) * 480), min(60 * 480, (q + 1 + h) * 480)
        assert float(d[:lo].abs().max() if lo else 0) == 0 and float(d[hi:].abs().max() if hi < 60 * 480 else 0) == 0, q
        assert float(d[q * 480:(q + 1) * 480].max()) > 0
        nz = torch.nonzero(d).flatten()
        print(f"[halo] frame {q}: changed samples {int(nz.min())}..{int(nz.max())}, allowed {lo}..{hi - 1}")
