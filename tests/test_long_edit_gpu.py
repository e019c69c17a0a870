"""Long edits on the GPU: the tiled VAE encode against a one-shot encode (bit for bit) with the receptive field it relies on; the windowed
inpainting loop against editing_audio for crops that fit one window (bit for bit, DDIM and DPM-Solver++), against the oracle's DiT driven
by an fp64 restatement of gather / guidance / blend / update, and under graph replay; editing_long_audio's lists against scalar calls,
its paste and splice, and its refusals."""
import functools
import gc

import numpy as np
import pytest
import torch

from ezaudio_b200 import _lib, post, synth, weights
from ezaudio_b200.inference import long_plan, sample_long_latents
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
from oracle import ezaudio_oracle as O

pytestmark = pytest.mark.gpu

HOP = 480


# ---------------------------------------------------------------- tiled VAE encode
ENCODERS = {"tiny": (synth.tiny_vae_encoder(16), synth.tiny_vae(16)), "full": (synth.VAE_ENCODER, synth.VAE_DECODER)}


@functools.lru_cache(maxsize=None)
def _vae_sd(name):
    ecfg, dcfg = ENCODERS[name]
    sd = dict(weights.synthetic_state_dict(weights.vae_decoder_param_shapes(dcfg), 6))
    sd.update(weights.synthetic_state_dict(weights.vae_encoder_param_shapes(ecfg), 8))
    return sd


def _codec(name, M, B, precision="bf16"):
    from ezaudio_b200.vae import OobleckDecoder
    ecfg, dcfg = ENCODERS[name]
    return OobleckDecoder(precision=precision, max_batch=B, max_latent_len=M, encoder_cfg=ecfg, **dcfg).load_state_dict(_vae_sd(name))


def _audio(B, T, seed):
    t = torch.arange(T) / 24000.0
    g = torch.Generator().manual_seed(seed)
    return torch.stack([0.3 * torch.sin(2 * np.pi * (110 + 70 * b) * t) + 0.05 * torch.randn(T, generator=g) for b in range(B)])[:, None]


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("name", ["tiny", "full"])
def test_encode_tiled_equals_one_shot(name, precision):
    """100-frame workspace (cores of 86 inside 7-frame halos) against a workspace that holds the whole length."""
    gc.collect()
    small, big = _codec(name, 100, 3, precision), _codec(name, 300, 3, precision)
    a = _audio(1, 280 * HOP - 123, 3).cuda()   # not a whole hop: both pad the last frame with zeros
    nz = torch.randn(1, 128, 280, generator=torch.Generator().manual_seed(4)).cuda()
    assert torch.equal(small.encode_tiled(a, noise=nz), big.encode(a, noise=nz))
    assert torch.equal(small.encode_tiled(a, noise=False), big.encode(a, noise=False))
    torch.manual_seed(9)
    want = big.encode(a)
    torch.manual_seed(9)
    assert torch.equal(small.encode_tiled(a), want)   # the same (1, C, N) bottleneck draw from the global RNG
    # a mixed-length batch: clip 1 fits one chunk, clip 2 takes two; past a clip's end the audio holds NaN and is never read
    lens = [280, 61, 150]
    ab = _audio(3, 280 * HOP, 5)
    for b, n in enumerate(lens):
        ab[b, :, n * HOP:] = float("nan")
    ab = ab.cuda()
    nzb = torch.randn(3, 128, 280, generator=torch.Generator().manual_seed(6)).cuda()
    got = small.encode_tiled(ab, noise=nzb, lengths=lens)
    assert torch.equal(got, big.encode(ab, noise=nzb, lengths=lens))
    for b, n in enumerate(lens):
        assert bool((got[b, :, n:] == 0).all()), b
    torch.manual_seed(10)
    want = big.encode(ab, lengths=lens)
    torch.manual_seed(10)
    assert torch.equal(small.encode_tiled(ab, lengths=lens), want)
    torch.manual_seed(10)   # clip order: the draws of three consecutive solo encodes
    for b, n in enumerate(lens):
        solo = big.encode(ab[b:b + 1, :, :n * HOP])
        assert torch.equal(want[b:b + 1, :, :n], solo), b


def test_encode_tiled_refuses_bad_arguments():
    gc.collect()
    codec = _codec("tiny", 100, 2)
    a = torch.zeros(2, 1, 150 * HOP, device="cuda")
    for kw in (dict(lengths=[150]), dict(lengths=[0, 10]), dict(lengths=[151, 10]), dict(noise=torch.zeros(2, 128, 149, device="cuda")),
               dict(lengths=torch.tensor([150, 10], dtype=torch.int32, device="cuda"))):
        with pytest.raises(ValueError):
            codec.encode_tiled(a, **kw)
    from ezaudio_b200.vae import OobleckDecoder
    dec_only = OobleckDecoder(precision="bf16", max_batch=1, max_latent_len=100, **synth.tiny_vae(16))
    with pytest.raises(_lib.EzbError):
        dec_only.encode_tiled(a[:1])


def test_encoder_receptive_field_bounds_a_perturbation():
    from ezaudio_b200.vae import encoder_receptive_field
    gc.collect()
    h = encoder_receptive_field(synth.VAE_ENCODER)
    codec = _codec("full", 60, 1)
    a = _audio(1, 60 * HOP, 7).cuda()
    base = codec.encode(a, noise=False)
    for i in (0, 29 * HOP, 29 * HOP + HOP - 1, 60 * HOP - 1):
        ap = a.clone()
        ap[0, 0, i] += 0.5
        d = (codec.encode(ap, noise=False) - base)[0].abs().amax(0).cpu()
        q = i // HOP
        changed = torch.nonzero(d).flatten()
        assert q - h <= int(changed.min()) and int(changed.max()) <= q + h, (i, changed)
        assert float(d[q]) > 0, i
        print(f"[halo] sample {i} (frame {q}): changed frames {int(changed.min())}..{int(changed.max())}, allowed {q - h}..{q + h}")


# ---------------------------------------------------------------- the windowed inpainting loop against the oracle
def _setup(B=2, Lw=40, Lc=12):
    from ezaudio_b200.dit import MaskDiT
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    ctx, mask = synth.synth_context(B, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    m = MaskDiT(precision="bf16x3", max_batch=12, max_len=Lw, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    return cfg, sd, m, ctx, mask, uctx, umask


def _gt(lens, seed=12, spans=((20, 50),)):
    """gt (B, 128, N) with NaN past each clip (never read) and a mask (B, N), True on `spans` of clip 0 and on [0, 10) + [45, n) of the
    others: spans that cross window edges."""
    N = max(lens)
    gt = torch.randn(len(lens), 128, N, generator=torch.Generator().manual_seed(seed))
    gm = torch.zeros(len(lens), N, dtype=torch.bool)
    for b, n in enumerate(lens):
        gt[b, :, n:] = float("nan")
        for s, e in (spans if b == 0 else ((0, 10), (45, n))):
            gm[b, s:e] = True
    return gt, gm


def _draws(seed, lens, steps, draw):
    gens = [torch.Generator(device="cuda").manual_seed(seed + b) for b in range(len(lens))]
    init = [torch.randn((1, 128, n), generator=g, device="cuda")[0].cpu() for g, n in zip(gens, lens)]
    noise = [[torch.empty((1, 128, n), device="cuda").normal_(generator=g)[0].cpu() for g, n in zip(gens, lens)] for _ in range(steps)] if draw else None
    return init, noise


def _blend64(wins, table, windows, Lw, O_):
    out = []
    for first, count, n in table:
        num, den = np.zeros((wins.shape[1], n)), np.zeros(n)
        for k in range(count):
            _, s, ln = windows[first + k]
            j = np.arange(ln, dtype=np.float64)
            w = np.ones(ln)
            if k > 0:
                w = np.minimum(w, (j + 1) / (O_ + 1))
            if k < count - 1:
                w = np.minimum(w, (Lw - j) / (O_ + 1))
            num[:, s:s + ln] += w * wins[first + k, :, :ln]
            den[s:s + ln] += w
        out.append(num / den)
    return out


@pytest.mark.parametrize("sampler", ["ddim", "dpmsolver++"])
def test_long_inpainting_loop_matches_oracle_dit_with_fp64_windows(sampler):
    gc.collect()
    lens, Lw, O_, gs, gr, steps, eta, seed = [73, 61], 40, 8, 3.0, 0.5, 4, 1.0, 11
    table, windows = long_plan(lens, Lw, O_)
    assert table[0][1] == 3 and [s for _, s, _ in windows[:3]] == [0, 32, 33]   # the last window overlaps both others
    cfg, sd, m, ctx, mask, uctx, umask = _setup()
    gt, gm = _gt(lens)
    sched = DDIMScheduler() if sampler == "ddim" else DPMSolverMultistepScheduler(algorithm_type=sampler)
    lat = sample_long_latents(m, sched, ctx, mask, uctx, umask, lens, Lw, O_, gs, gr, steps, eta, seed, gt=gt, gt_mask=gm).cpu()
    init, step_noise = _draws(seed, lens, steps, sampler == "ddim")
    sched.set_timesteps(steps)
    clip = [b for b, _, _ in windows]
    wctx = torch.cat([ctx[clip], uctx.expand(len(windows), -1, -1)])
    wmask = torch.cat([mask[clip], umask.expand(len(windows), -1)])
    wgt = torch.stack([gt[b, :, s:s + ln] for b, s, ln in windows])
    wgm = torch.stack([gm[b, s:s + ln] for b, s, ln in windows])[:, None, :].expand(-1, 128, -1)
    x = [v.double() for v in init]
    m1 = [None] * len(lens)
    with torch.no_grad():
        for i, t in enumerate(sched.timesteps.tolist()):
            xw = torch.stack([x[b][:, s:s + ln] for b, s, ln in windows]).float()
            out, _ = O.maskdit_forward(sd, cfg, torch.cat([xw, xw]), torch.tensor(t), wctx, wmask, gt=torch.cat([wgt, wgt]),
                                       mae_mask_infer=torch.cat([wgm, wgm]))
            o_t, o_u = out.chunk(2, 0)
            vw = O.cfg_combine(o_t, o_u, gs, gr).double().numpy()
            v = [torch.from_numpy(a) for a in _blend64(vw, table, windows, Lw, O_)]
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
        print(f"[long edit] {sampler} clip {b} ({n} frames, {table[b][1]} windows): loop vs oracle DiT + fp64 windows max-abs {err:.2e}")
        assert err < 5e-3, (b, err)
        assert torch.equal(lat[b, :, n:], torch.zeros(128, max(lens) - n))


def test_long_inpainting_replays_on_new_gt_and_masks():
    """A second call with other gt and masks on the same plan shape replays the captured graph and equals an eager run."""
    gc.collect()
    cfg, sd, m, ctx, mask, uctx, umask = _setup()
    lens = [73, 61]
    args = (m, DDIMScheduler(), ctx, mask, uctx, umask, lens, 40, 8, 3.0, 0.5, 4, 1.0, 11)
    gt, gm = _gt(lens)
    first = sample_long_latents(*args, gt=gt, gt_mask=gm)   # eager pass + capture
    entry = [v for k, v in m._long_cache.items() if k[-1]]
    assert len(entry) == 1 and entry[0]["graph"] is not None
    graph, launches = entry[0]["graph"], entry[0]["launches"]
    assert torch.equal(first, sample_long_latents(*args, gt=gt, gt_mask=gm, use_graphs=False))
    gt2, gm2 = _gt(lens, seed=13, spans=((0, 5), (35, 73)))
    gm2 = gm2[:, None, :].expand(-1, 128, -1)   # the (B, C, N) form
    c0 = _lib.lib().ezb_launch_count()
    replay = sample_long_latents(*args, gt=gt2, gt_mask=gm2)
    now = [v for k, v in m._long_cache.items() if k[-1]]
    assert len(now) == 1 and now[0] is entry[0] and now[0]["graph"] is graph and now[0]["launches"] == launches
    assert _lib.lib().ezb_launch_count() - c0 < 2 * launches   # one replay (plus the per-call gather), no eager pass or new capture
    eager = sample_long_latents(*args, gt=gt2, gt_mask=gm2, use_graphs=False)
    assert torch.equal(replay, eager) and not torch.equal(replay, first)
    plain = sample_long_latents(*args)   # without gt: its own graph, a different result
    assert not torch.equal(plain, first)


# ---------------------------------------------------------------- through the API
def _ez(monkeypatch, max_batch=3, precision="bf16"):
    from ezaudio_b200 import api, config
    from tests.test_api_gpu import _tiny_params
    tiny = _tiny_params()
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    return api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16),
                       max_batch=max_batch, max_length_s=2, precision=precision)


def _clip(seconds, f, sr=24000):
    t = np.arange(int(seconds * sr)) / sr
    return (0.3 * np.sin(2 * np.pi * f * t) + 0.05 * np.sin(2 * np.pi * 3 * f * t)).astype(np.float32)


def _set_sampler(ez, alg):
    ez.noise_scheduler = DDIMScheduler(**ez.params["diff"]) if alg == "ddim" else DPMSolverMultistepScheduler(**ez.params["diff"], algorithm_type=alg)


@pytest.mark.parametrize("alg,eta", [("ddim", 0.0), ("ddim", 1.0), ("dpmsolver++", 1.0), ("sde-dpmsolver++", 1.0)])
def test_one_window_equals_editing_audio(alg, eta, monkeypatch):
    gc.collect()
    ez = _ez(monkeypatch)
    _set_sampler(ez, alg)
    edits = (dict(text="a dog barks", gt_file=_clip(1.5, 220), mask_start=0.5, mask_length=0.5, boundary=0.3),   # mid-clip, 1.1-s crop
             dict(text="rain on a roof", gt_file=_clip(1.0, 330), mask_start=1.0, mask_length=0.6, boundary=0.3),   # outpainting
             dict(text="", gt_file=_clip(1.2, 440), mask_start=0.2, mask_length=0.4, boundary=0.5))           # no guidance
    for e in edits:
        kw = dict(guidance_scale=3.5, guidance_rescale=0.5, ddim_steps=5, eta=eta, random_seed=17)
        torch.manual_seed(31)
        sr, want = ez.editing_audio(**e, **kw)
        torch.manual_seed(31)
        sr2, got = ez.editing_long_audio(**e, window_length=2, overlap=0.4, **kw)
        assert sr2 == sr and got.dtype == want.dtype and got.shape == want.shape, (e["text"], got.shape, want.shape)
        assert got.tobytes() == want.tobytes(), (alg, eta, e["text"], float(np.abs(got - want).max()))


# crops of 6 s (4 windows of 2 s with 0.4 s overlap; two VAE chunks), 5 s (3 windows, outpainting 2 s past the clip's end) and 1.5 s (one)
EDITS = dict(text=["a bell", "rain on a roof", "a dog barks"], gt_file=[_clip(8, 220), _clip(4, 330), _clip(2, 440)],
             mask_start=[2.0, 2.0, 0.8], mask_length=[4.0, 4.0, 0.9], boundary=[1.0, 1.0, 0.3], random_seed=[3, 4, 5])


def test_list_equals_scalar_calls_and_pastes(monkeypatch):
    """bf16x3 takes the same GEMM kernels at every token count, so the list must reproduce the three scalar calls bit for bit."""
    from ezaudio_b200.api import edit_plan
    gc.collect()
    ez = _ez(monkeypatch, max_batch=8, precision="bf16x3")
    dec = ez.autoencoder.decoder
    seen = {}
    enc, dect = dec.encode_tiled, dec.decode_tiled

    def spy_enc(*a, **k):
        seen["gt"] = enc(*a, **k)
        return seen["gt"]

    def spy_dec(z, **k):
        seen["pred"] = z.clone()
        return dect(z, **k)
    dec.encode_tiled, dec.decode_tiled = spy_enc, spy_dec
    kw = dict(window_length=2, overlap=0.4, ddim_steps=4, guidance_scale=3.5, guidance_rescale=0.5)
    torch.manual_seed(21)
    sr, batch = ez.editing_long_audio(**EDITS, **kw)
    gt_b, pred_b = seen["gt"], seen["pred"]
    assert len(ez.unet._long_cache) == 1
    torch.manual_seed(21)
    _, again = ez.editing_long_audio(**EDITS, **kw)   # graph replay
    assert all(a.tobytes() == b.tobytes() for a, b in zip(batch, again))
    torch.manual_seed(21)   # the scalar calls draw their bottleneck noise from the global RNG in this order
    for i, got in enumerate(batch):
        one = {k: v[i] for k, v in EDITS.items()}
        _, want = ez.editing_long_audio(**one, **kw)
        assert got.dtype == np.float32 and got.shape == want.shape and np.isfinite(got).all()
        assert got.tobytes() == want.tobytes(), (i, float(np.abs(got - want).max()))
        p = edit_plan(len(one["gt_file"]), sr, 50, HOP, one["boundary"], one["mask_start"], one["mask_length"])
        assert got.shape == (p["n_total"],)
        # kept latent frames are the encoded crop after the paste
        keep = torch.ones(p["frames"], dtype=torch.bool)
        keep[p["m0"]:p["m1"]] = False
        assert torch.equal(pred_b[i, :, :p["frames"]][:, keep.cuda()], gt_b[i, :, :p["frames"]][:, keep.cuda()]), i
        # outside the splice, the prepared clip bit for bit
        ref = post.prepare_wave(torch.from_numpy(one["gt_file"]).cuda().unsqueeze(0), p["n_total"], normalize=True)[0].cpu().numpy()
        lo, hi = p["s0"], p["s0"] + p["n_paste"]
        assert got[:lo].tobytes() == ref[:lo].tobytes() and got[hi:].tobytes() == ref[hi:].tobytes(), i
        assert not np.allclose(got[lo + p["m0"] * HOP:lo + p["m1"] * HOP], ref[lo + p["m0"] * HOP:lo + p["m1"] * HOP], atol=1e-2)
    assert [p for p in (edit_plan(len(f), 24000, 50, HOP, b, s, m)["frames"] for f, b, s, m in
                        zip(EDITS["gt_file"], EDITS["boundary"], EDITS["mask_start"], EDITS["mask_length"]))] == [300, 250, 75]
    assert batch[1].shape == (6 * 24000,)


def test_refusals_leave_no_device_work_and_the_handle_usable(monkeypatch):
    gc.collect()
    ez = _ez(monkeypatch, max_batch=3)   # 6 DiT rows
    one = {k: v[1] for k, v in EDITS.items()}   # 5-s crop: 3 windows x 2 rows = 6
    kw = dict(window_length=2, overlap=0.4, ddim_steps=3)
    gt, gm = _gt([150, 90], seed=3)
    m = ez.unet
    ctx, mask = torch.randn(2, 16, 64), torch.ones(2, 16, dtype=torch.bool)
    torch.cuda.synchronize()
    c0, mem0 = _lib.lib().ezb_launch_count(), torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="max_batch >= 4"):
        ez.editing_long_audio(**{k: v[0] for k, v in EDITS.items()}, **kw)   # 6-s crop: 4 windows x 2 rows
    with pytest.raises(ValueError, match="max_length_s"):
        ez.editing_long_audio(**one, window_length=3, overlap=0.4, ddim_steps=3)
    with pytest.raises(ValueError):
        ez.editing_long_audio(**dict({k: v[:2] for k, v in EDITS.items()}, text=["", "rain"]), **kw)
    for bad in (dict(mask_length=0), dict(mask_start=-1), dict(boundary=-0.5), dict(mask_length=[1, 2])):
        with pytest.raises(ValueError):
            ez.editing_long_audio(**dict(one, **bad), **kw)
    with pytest.raises(NotImplementedError):
        sample_long_latents(m, DDIMScheduler(), ctx, mask, ctx[:1], mask[:1], [150, 90], 100, 20, 3.0, 0.0, 3, 1.0, 1,
                            controlnet=object(), condition=torch.zeros(2, 1, 300), gt=gt, gt_mask=gm)
    with pytest.raises(ValueError, match="gt must be"):   # gt of the wrong length (3 windows x 2 rows fit)
        sample_long_latents(m, DDIMScheduler(), ctx, mask, ctx[:1], mask[:1], [150, 90], 100, 20, 3.0, 0.0, 3, 1.0, 1, gt=gt[:, :, :149],
                            gt_mask=gm[:, :149])
    assert torch.cuda.memory_allocated() == mem0
    torch.cuda.synchronize()
    assert _lib.lib().ezb_launch_count() == c0
    torch.manual_seed(2)
    _, a = ez.editing_long_audio(**one, **kw)
    torch.manual_seed(2)
    _, b = ez.editing_long_audio(**one, **kw)
    assert a.tobytes() == b.tobytes() and np.isfinite(a).all() and a.shape == (6 * 24000,)
