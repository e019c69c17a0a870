"""Seamless loops on the GPU: the circular gather and blend kernels against a torch index gather and fp64 (NaN wherever they must not
read, sentinels wherever they must not write), decode_loop against the middle period of a one-shot decode of the loop repeated (bit for
bit), the loop against sample_latents when it fits one window with no shift (bit for bit), exact shift-equivariance (no privileged seam),
the loop against the oracle's DiT driven by an fp64 restatement of gather / guidance / blend / update, and generate_loop_audio."""
import functools
import gc

import numpy as np
import pytest
import torch

from ezaudio_b200 import _lib, synth, weights
from ezaudio_b200.inference import check_loop, loop_starts, loop_weights
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
from oracle import ezaudio_oracle as O

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- kernels
def _dev(rows):
    return torch.tensor([e for row in rows for e in row], dtype=torch.int32, device="cuda")


def _windows(table, offs, Lw):
    """[(loop, start, length)] of every window row at the given offsets."""
    out = []
    for b, (first, count, n) in enumerate(table):
        ln = min(n, Lw)
        out += [(b, s, ln) for s in loop_starts(n, count, offs[b])]
    return out


def _blend64(wins, table, offs, Lw, O_):
    res, cover = [], []
    for b, (first, count, n) in enumerate(table):
        ln = min(n, Lw)
        num, den, cnt = np.zeros((wins.shape[1], n)), np.zeros(n), np.zeros(n, dtype=int)
        w = loop_weights(count, ln, O_).astype(np.float64)
        for k, s in enumerate(loop_starts(n, count, offs[b])):
            f = (s + np.arange(ln)) % n
            num[:, f] += w * wins[first + k, :, :ln].astype(np.float64)
            den[f] += w
            cnt[f] += 1
        res.append(num / den)
        cover.append(cnt)
    return res, cover


@pytest.mark.parametrize("C_", [16, 128])
def test_loop_gather_and_blend(C_):
    Lw, O_ = 40, 8
    lens = [89, 17, 130, 40, 2, 41]   # 3 windows, one short window, 5 windows, exactly one window, the shortest loop, 2 windows
    _, table, _ = check_loop(lens, len(lens), Lw, O_, False, 64, Lw)
    B, W, N = len(lens), sum(c for _, c, _ in table), max(lens)
    g = torch.Generator().manual_seed(4)
    lat = torch.randn(B, C_, N, generator=g)
    for b, n in enumerate(lens):
        lat[b, :, n:] = float("nan")   # past a loop's end: never read
    lat_d, plan = lat.cuda(), _dev(table)
    L, st = _lib.lib(), _lib.stream_ptr()
    rng = np.random.default_rng(7)
    for trial in range(4):
        offs = [0] * B if trial == 0 else [int(rng.integers(-3 * n, 3 * n)) for n in lens]   # any int: reduced mod N on the device
        offs_d = torch.tensor(offs, dtype=torch.int32, device="cuda")
        wl = _windows(table, [o % n for o, n in zip(offs, lens)], Lw)
        for copies in (1, 2):
            win = torch.full((copies * W + 1, C_, Lw), 7.0, device="cuda")   # one spare row: nothing past copies * W is written
            _lib.check(L.ezb_loop_gather(0, _lib.ptr(lat_d), _lib.ptr(win), _lib.ptr(plan), _lib.ptr(offs_d), B, C_, N, W, Lw, O_, copies, st))
            got = win.cpu()
            want = torch.zeros(W, C_, Lw)
            for r, (b, s, ln) in enumerate(wl):
                want[r, :, :ln] = lat[b][:, torch.remainder(torch.arange(s, s + ln), lens[b])]
            for c in range(copies):
                assert torch.equal(got[c * W:(c + 1) * W], want), (trial, copies, c)
            assert torch.equal(got[copies * W], torch.full((C_, Lw), 7.0))
        # blend: window frames past Lw_b hold NaN; the output's sentinel must survive past each loop's end
        wins = torch.randn(W, C_, Lw, generator=g)
        for r, (_, _, ln) in enumerate(wl):
            wins[r, :, ln:] = float("nan")
        out = torch.full((B, C_, N), 7.0, device="cuda")
        wins_d = wins.cuda()
        _lib.check(L.ezb_loop_blend(0, _lib.ptr(wins_d), _lib.ptr(out), _lib.ptr(plan), _lib.ptr(offs_d), B, C_, N, W, Lw, O_, st))
        got = out.cpu()
        ref, cover = _blend64(wins.numpy(), table, [o % n for o, n in zip(offs, lens)], Lw, O_)
        bound = 12 * 2.0 ** -24 * np.nanmax(np.abs(wins.numpy()))   # up to four products and sums, the division and the fp32 weights
        for b, (first, count, n) in enumerate(table):
            assert torch.equal(got[b, :, n:], torch.full((C_, N - n), 7.0)), b
            err = np.abs(got[b, :, :n].double().numpy() - ref[b])
            assert (err <= bound).all(), (trial, b, float(err.max()))
            one = cover[b] == 1   # one covering window, of weight 1 there: its value bit for bit
            assert np.array_equal(got[b, :, :n].numpy()[:, one], ref[b][:, one].astype(np.float32)), (trial, b)
            if count == 1:
                assert one.all()


def test_loop_kernels_reject_bad_arguments():
    L = _lib.lib()
    x = torch.zeros(8, device="cuda")
    p, o = _dev([(0, 1, 4)]), torch.zeros(1, dtype=torch.int32, device="cuda")
    for args in ((1, 1, 4, 1, 4, 0, 1), (1, 1, 4, 1, 4, 3, 1), (1, 1, 4, 0, 4, 1, 1), (1, 1, 4, 1, 4, 1, 3)):
        B, C_, N, W, Lw, O_, copies = args
        assert L.ezb_loop_gather(0, _lib.ptr(x), _lib.ptr(x), _lib.ptr(p), _lib.ptr(o), B, C_, N, W, Lw, O_, copies, _lib.stream_ptr()) != 0, args
    assert L.ezb_loop_gather(0, _lib.ptr(x), _lib.ptr(x), _lib.ptr(p), None, 1, 1, 4, 1, 4, 1, 1, _lib.stream_ptr()) != 0
    assert L.ezb_loop_blend(0, _lib.ptr(x), _lib.ptr(x), _lib.ptr(p), None, 1, 1, 4, 1, 4, 1, _lib.stream_ptr()) != 0
    assert L.ezb_loop_blend(0, _lib.ptr(x), _lib.ptr(x), None, _lib.ptr(o), 1, 1, 4, 1, 4, 1, _lib.stream_ptr()) != 0


# ---------------------------------------------------------------- seamless decode
VAES = {"tiny": synth.tiny_vae(16), "full": synth.VAE_DECODER}


@functools.lru_cache(maxsize=None)
def _vae_sd(name):
    return weights.synthetic_state_dict(weights.vae_decoder_param_shapes(VAES[name]), 6)


def _dec(name, M, B, precision):
    from ezaudio_b200.vae import OobleckDecoder
    return OobleckDecoder(precision=precision, max_batch=B, max_latent_len=M, **VAES[name]).load_state_dict(_vae_sd(name))


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("name", ["tiny", "full"])
def test_decode_loop_equals_the_middle_period_of_a_repeat(name, precision):
    from ezaudio_b200.vae import decoder_receptive_field
    gc.collect()
    h = decoder_receptive_field(VAES[name])
    lens = [150, 5, 30, 22]   # past max_latent_len, shorter than the halo, two cores, one core of exactly max_len - 2h frames
    M = 22 + 2 * h
    small = _dec(name, M, 3, precision)
    big = _dec(name, 470, 1, precision)
    z = synth.synth_latents(len(lens), max(lens), seed=3)
    for b, n in enumerate(lens):
        z[b, :, n:] = float("nan")   # past a loop's end: never read
    zd = z.cuda()
    got = small.decode_loop(zd, lengths=lens)
    hop = small.hop
    for b, n in enumerate(lens):
        reps = 2 * -(-h // n) + 1   # the middle period sits at least h frames from both ends
        one = big(z[b:b + 1, :, :n].repeat(1, 1, reps).cuda())
        mid = one[0, 0, (reps // 2) * n * hop:(reps // 2 + 1) * n * hop]
        assert torch.equal(got[b, 0, :n * hop], mid), (name, precision, n)
        assert torch.equal(got[b, 0, n * hop:], torch.zeros((max(lens) - n) * hop, device="cuda")), b
        solo = small.decode_loop(zd[b:b + 1, :, :n])
        assert torch.equal(solo[0, 0], got[b, 0, :n * hop]), b


# ---------------------------------------------------------------- the loop
def _setup(precision="bf16x3", Lw=40, Lc=12, B=2):
    from ezaudio_b200.dit import MaskDiT
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    ctx, mask = synth.synth_context(B, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    m = MaskDiT(precision=precision, max_batch=12, max_len=Lw, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    return cfg, sd, m, ctx, mask, uctx, umask


SAMPLERS = [("ddim", 0.0), ("ddim", 1.0), ("dpmsolver++", 1.0), ("sde-dpmsolver++", 1.0)]


def _sched(alg):
    return DDIMScheduler() if alg == "ddim" else DPMSolverMultistepScheduler(algorithm_type=alg)


@pytest.mark.parametrize("alg,eta", SAMPLERS)
def test_unshifted_one_window_loop_equals_sample_latents(alg, eta):
    from ezaudio_b200.inference import sample_latents, sample_loop_latents
    gc.collect()
    cfg, sd, m, ctx, mask, uctx, umask = _setup()
    lens, steps, seed = [40, 29], 4, 21
    lat = sample_loop_latents(m, _sched(alg), ctx, mask, uctx, umask, lens, 40, 8, 3.0, 0.5, steps, eta, seed, offsets=[[0, 0]] * steps)
    for b, n in enumerate(lens):
        want = sample_latents(m, _sched(alg), ctx[b:b + 1], mask[b:b + 1], uctx, umask, audio_frames=n, guidance_scale=3.0, guidance_rescale=0.5,
                              ddim_steps=steps, eta=eta, random_seed=seed + b)
        assert torch.equal(lat[b:b + 1, :, :n], want), (alg, eta, b)
        assert torch.equal(lat[b, :, n:], torch.zeros(128, max(lens) - n, device="cuda"))


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("alg,eta", [("ddim", 1.0), ("dpmsolver++", 1.0)])
def test_shifting_every_offset_rolls_the_loop(precision, alg, eta):
    """All windows move together, so every DiT row sees the same input; the blend's order depends only on where a frame sits in each window."""
    from ezaudio_b200.inference import sample_loop_latents
    gc.collect()
    cfg, sd, m, ctx, mask, uctx, umask = _setup(precision)
    lens, steps, N = [33, 89], 4, 89   # one window; three windows, 89 not a multiple of Lw - O = 32
    g = torch.Generator().manual_seed(5)
    init = torch.randn(2, 128, N, generator=g)
    noise = [torch.randn(2, 128, N, generator=g) for _ in range(steps)]
    rng = np.random.default_rng(3)
    offs = [[int(rng.integers(0, n)) for n in lens] for _ in range(steps)]

    def roll(x, d):
        y = x.clone()
        for b, n in enumerate(lens):
            y[b, :, :n] = torch.roll(x[b, :, :n], d, dims=-1)
        return y
    base = sample_loop_latents(m, _sched(alg), ctx, mask, uctx, umask, lens, 40, 8, 3.0, 0.5, steps, eta, 0, offsets=offs, init_noise=init,
                               step_noise=noise)
    for d in (1, 17, 60):
        got = sample_loop_latents(m, _sched(alg), ctx, mask, uctx, umask, lens, 40, 8, 3.0, 0.5, steps, eta, 0,
                                  offsets=[[o + d for o in row] for row in offs], init_noise=roll(init, d), step_noise=[roll(s, d) for s in noise])
        assert torch.equal(got, roll(base, d)), (precision, alg, d)
    other = sample_loop_latents(m, _sched(alg), ctx, mask, uctx, umask, lens, 40, 8, 3.0, 0.5, steps, eta, 0,
                                offsets=[[o + 1 for o in row] for row in offs], init_noise=init, step_noise=noise)
    assert not torch.equal(other[1], base[1])   # the shift does move the windows over the latent


@pytest.mark.parametrize("sampler", ["ddim", "dpmsolver++"])
def test_loop_matches_oracle_dit_with_fp64_windows(sampler):
    from ezaudio_b200.inference import loop_offsets, sample_loop_latents
    gc.collect()
    lens, Lw, O_, gs, gr, steps, eta, seed = [89, 70], 40, 8, 3.0, 0.5, 4, 1.0, 11
    _, table, _ = check_loop(lens, 2, Lw, O_, True, 24, Lw)
    assert [c for _, c, _ in table] == [3, 3]
    cfg, sd, m, ctx, mask, uctx, umask = _setup()
    sched = _sched(sampler)
    lat = sample_loop_latents(m, sched, ctx, mask, uctx, umask, lens, Lw, O_, gs, gr, steps, eta, seed).cpu()
    offs = loop_offsets(lens, steps)
    assert any(o != 0 for row in offs for o in row)
    gens = [torch.Generator(device="cuda").manual_seed(seed + b) for b in range(2)]
    x = [torch.randn((1, 128, n), generator=g, device="cuda")[0].cpu().double() for g, n in zip(gens, lens)]
    step_noise = [[torch.empty((1, 128, n), device="cuda").normal_(generator=g)[0].cpu() for g, n in zip(gens, lens)] for _ in range(steps)] \
        if sampler == "ddim" else None
    sched.set_timesteps(steps)
    W = sum(c for _, c, _ in table)
    clip = [b for b, (_, c, _) in enumerate(table) for _ in range(c)]
    wctx, wmask = torch.cat([ctx[clip], uctx.expand(W, -1, -1)]), torch.cat([mask[clip], umask.expand(W, -1)])
    m1 = [None] * 2
    with torch.no_grad():
        for i, t in enumerate(sched.timesteps.tolist()):
            wl = _windows(table, offs[i], Lw)
            xw = torch.stack([x[b][:, torch.remainder(torch.arange(s, s + ln), lens[b])] for b, s, ln in wl]).float()
            out, _ = O.maskdit_forward(sd, cfg, torch.cat([xw, xw]), torch.tensor(t), wctx, wmask)
            o_t, o_u = out.chunk(2, 0)
            vw = O.cfg_combine(o_t, o_u, gs, gr).double().numpy()
            v = [torch.from_numpy(a) for a in _blend64(vw, table, offs[i], Lw, O_)[0]]
            for b in range(2):
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
        print(f"[loop] {sampler} loop {b} ({n} frames, {table[b][1]} windows): loop vs oracle DiT + fp64 windows max-abs {err:.2e}")
        assert err < 5e-3, (b, err)
        assert torch.equal(lat[b, :, n:], torch.zeros(128, max(lens) - n))


# ---------------------------------------------------------------- the API
def _ez(monkeypatch, max_batch=8, precision="bf16x3"):
    from ezaudio_b200 import api, config
    from tests.test_api_gpu import _tiny_params
    tiny = _tiny_params()
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    return api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16),
                       max_batch=max_batch, max_length_s=2, precision=precision)


def test_generate_loop_audio_batch_replay_and_refusal(monkeypatch):
    gc.collect()
    ez = _ez(monkeypatch)
    prompts, lengths, seeds = ["rain on a roof", "engine hum"], [3.3, 0.9], [5, 9]   # 5 windows and 1 window: 12 DiT rows
    kw = dict(window_length=1, overlap=0.2, guidance_scale=5, guidance_rescale=0.75, ddim_steps=5, eta=1)
    sr, batch = ez.generate_loop_audio(prompts, length=lengths, random_seed=seeds, **kw)
    assert sr == 24000 and [w.shape for w in batch] == [(480 * int(s * 50),) for s in lengths]
    assert all(w.dtype == np.float32 and np.isfinite(w).all() for w in batch)
    for p, n, s, w in zip(prompts, lengths, seeds, batch):
        _, solo = ez.generate_loop_audio(p, length=n, random_seed=s, **kw)
        assert solo.tobytes() == w.tobytes(), p
    new = [s + 100 for s in seeds]
    _, replay = ez.generate_loop_audio(prompts, length=lengths, random_seed=new, **kw)   # the captured schedule, new seeds
    ez.unet.__dict__.pop("_loop_long_cache")
    _, eager = ez.generate_loop_audio(prompts, length=lengths, random_seed=new, **kw)    # an eager pass
    for a, b, c in zip(replay, eager, batch):
        assert a.tobytes() == b.tobytes() and a.tobytes() != c.tobytes()
    with pytest.raises(ValueError, match="needs max_batch >= 10"):
        ez.generate_loop_audio(["rain", "wind"], length=[4, 4], random_seed=1, **kw)   # 2 x 10 windows x 2 rows > 16
    _, again = ez.generate_loop_audio(prompts, length=lengths, random_seed=seeds, **kw)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(again, batch))
    _, empty = ez.generate_loop_audio("", length=1.5, window_length=1, overlap=0.2, ddim_steps=3, random_seed=2)   # no guidance: one row per window
    assert empty.shape == (480 * 75,) and np.isfinite(empty).all()
