"""Clips of different lengths in one padded batch (per-sample lengths in device memory).

Contract: sample b of a batch padded to L carries lens[b] <= L frames; its frames < lens[b] of the attention output, the DiT output, the
latents and the waveform equal the same request run alone at length lens[b], and nothing in the padded tail (not even NaN) reaches them."""
import functools
import math

import numpy as np
import pytest
import torch

from ezaudio_b200 import synth, weights

pytestmark = pytest.mark.gpu

ATTN6_DEFAULT = 5
LENS = [1, 63, 64, 65, 317, 500]


def _ref(q, k, v):
    s = (q.double() @ k.double().transpose(-1, -2)) / math.sqrt(q.shape[-1])
    o = s.softmax(-1) @ v.double()
    return o.permute(0, 2, 1, 3).reshape(q.shape[0], q.shape[2], -1)


def _tc_layout(q, k, v, dh, row80):
    """[B, H, L, dh] fp32 -> the tensor-core kernel's bf16 q / k [B*H, L, dhp] and V^T [B*H, dvp, ceil8(L)] (padding columns NaN)."""
    B, H, L, _ = q.shape
    dhp = 80 if (row80 and dh == 72) else (dh + 63) // 64 * 64
    dvp, lkp = (dh + 15) // 16 * 16, (L + 7) // 8 * 8
    qb = torch.zeros(B * H, L, dhp, device="cuda", dtype=torch.bfloat16)
    kb = torch.zeros(B * H, L, dhp, device="cuda", dtype=torch.bfloat16)
    vt = torch.zeros(B * H, dvp, lkp, device="cuda", dtype=torch.bfloat16)
    qb[:, :, :dh] = q.reshape(B * H, L, dh)
    kb[:, :, :dh] = k.reshape(B * H, L, dh)
    vt[:, :dh, :L] = v.reshape(B * H, L, dh).transpose(1, 2)
    vt[:, :, L:] = float("nan")
    return qb, kb, vt


def _attention(impl, args, lens, B, H, L, dh):
    from ezaudio_b200 import _lib
    Lib = _lib.lib()
    out = torch.full((B, L, H * dh), 3.0, device="cuda", dtype=torch.bfloat16)
    if lens is None:
        _lib.check(Lib.ezb_test_attention(0, *[_lib.ptr(a) for a in args], None, _lib.ptr(out), B, H, L, L, dh, impl, _lib.stream_ptr()))
    else:
        _lib.check(Lib.ezb_test_attention_lens(0, *[_lib.ptr(a) for a in args], _lib.ptr(lens), _lib.ptr(out), B, H, L, dh, impl, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out


# impl as in ezb_test_attention: 0 fp32 CUDA-core kernel (parity mode); 1 the selected tensor-core variant (4 with attn6 = 0, 4 + RES with
# attn_res); 4 / 6 / 7 forced (generation 8's padded batches are test_attention_wgmma_gpu.py's); +100 the 80-element q / k rows of dh = 72
@pytest.mark.parametrize("dh", [72, 64])
@pytest.mark.parametrize("variant", ["simt", "6", "6r80", "4", "4r80", "4res", "7", "7r80"])
def test_attention_lens_matches_solo_runs(variant, dh):
    from ezaudio_b200 import _lib
    Lib = _lib.lib()
    impl = {"simt": 0, "6": 6, "6r80": 106, "4": 4, "4r80": 104, "4res": 1, "7": 7, "7r80": 107}[variant]
    if variant == "4res":
        _lib.check(Lib.ezb_set_option(b"attn6", 0))
        _lib.check(Lib.ezb_set_option(b"attn_res", 1))
    try:
        B, H, L = len(LENS), 2, 500
        g = torch.Generator(device="cuda").manual_seed(dh)
        q = torch.randn(B, H, L, dh, device="cuda", generator=g) * 1.5
        k = torch.randn(B, H, L, dh, device="cuda", generator=g) * 1.5
        v = torch.randn(B, H, L, dh, device="cuda", generator=g)
        if impl != 0:   # the reference sees the bf16 operands
            q, k, v = q.bfloat16().float(), k.bfloat16().float(), v.bfloat16().float()
        qn, kn, vn = q.clone(), k.clone(), v.clone()
        for b, n in enumerate(LENS):   # NaN in every padded token of q, k and v
            qn[b, :, n:] = float("nan"); kn[b, :, n:] = float("nan"); vn[b, :, n:] = float("nan")
        row80 = impl >= 100
        args = (qn, kn, vn) if impl == 0 else _tc_layout(qn, kn, vn, dh, row80)
        lens = torch.tensor(LENS, dtype=torch.int32, device="cuda")
        out = _attention(impl, args, lens, B, H, L, dh)
        for b, n in enumerate(LENS):
            qs, ks, vs = q[b:b + 1, :, :n].contiguous(), k[b:b + 1, :, :n].contiguous(), v[b:b + 1, :, :n].contiguous()
            solo = _attention(impl, (qs, ks, vs) if impl == 0 else _tc_layout(qs, ks, vs, dh, row80), None, 1, H, n, dh)
            assert torch.equal(out[b, :n], solo[0]), (b, n)                         # bit-identical to the run at Lq = Lk = n
            assert bool((out[b, n:] == 0).all()), (b, n)                            # padded rows are zeros
            err = (out[b:b + 1, :n].double() - _ref(qs, ks, vs)).abs().max().item()
            assert math.isfinite(err) and err < (2e-2 if impl == 0 else 3e-2), (b, n, err)
    finally:
        _lib.check(Lib.ezb_set_option(b"attn_res", 0))
        _lib.check(Lib.ezb_set_option(b"attn6", ATTN6_DEFAULT))


@functools.lru_cache(maxsize=1)
def _xl_state_dict():
    return weights.synthetic_state_dict(weights.dit_param_shapes(synth.model_cfg("xl")), 4)


def _padded_vs_solo(m, x, ctx, mask, t, lens):
    """Padded forward with NaN in every padded input frame, then each sample alone at its length (frames [0, n) of both)."""
    Be, Cc, L = x.shape
    xp = x.clone()
    for b, n in enumerate(lens):
        xp[b, :, n:] = float("nan")
    m.set_context(ctx, mask)
    m.set_timesteps([t])
    out = m.forward_step(xp.cuda().contiguous(), 0, lengths=torch.tensor(lens, dtype=torch.int32, device="cuda"))
    got = [out[b, :, :n].cpu() for b, n in enumerate(lens)]
    solo = []
    for b, n in enumerate(lens):
        o, _ = m(x[b:b + 1, :, :n].cuda().contiguous(), torch.tensor(t), ctx[b:b + 1].cuda(), context_mask=mask[b:b + 1].cuda())
        solo.append(o[0].cpu())
    torch.cuda.synchronize()
    return got, solo


def _same_kernels(precision, Be, L, n):
    """The kernel choices of Dit that depend on the token count M = Be * L (default options): bf16 fp32-output linears run as swap-AB tiles
    when M >= 512, else on 2-CTA cluster tiles (Dit::lin), and gated swap-AB epilogues need clips of >= 32 frames.  bf16x3 takes the same
    kernels at every M."""
    if precision == "bf16x3":
        return True
    return (Be * L >= 512) == (n >= 512) and (L >= 32) == (n >= 32)


TOL = {"bf16x3": (1e-3, 2e-4), "bf16": (6e-2, 1.2e-2)}


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("dh", [72, 64])
def test_dit_forward_lens_tiny(dh, precision):
    from ezaudio_b200.dit import MaskDiT
    from oracle import ezaudio_oracle as O
    cfg = synth.tiny_model(dh)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    lens, L, Lc, t = [96, 70, 33, 20], 96, 12, 479
    Be = len(lens)
    x = synth.synth_latents(Be, L)
    ctx, mask = synth.synth_context(Be, Lc, cfg["context_dim"])
    m = MaskDiT(precision=precision, max_batch=Be, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    got, solo = _padded_vs_solo(m, x, ctx, mask, t, lens)
    for b, n in enumerate(lens):
        assert torch.isfinite(got[b]).all(), (b, n)
        if _same_kernels(precision, Be, L, 1 * n):
            assert torch.equal(got[b], solo[b]), (b, n, float((got[b] - solo[b]).abs().max()))
        else:
            assert float((got[b] - solo[b]).abs().max()) < TOL["bf16"][0], (b, n)
        with torch.no_grad():
            want, _ = O.maskdit_forward(sd, cfg, x[b:b + 1, :, :n], torch.tensor(t), ctx[b:b + 1], mask[b:b + 1])
        err = (got[b] - want[0]).abs()
        assert float(err.max()) < TOL[precision][0] and float(err.mean()) < TOL[precision][1], (b, n, float(err.max()), float(err.mean()))


@pytest.mark.parametrize("swap_ab", [1, 0])
def test_dit_forward_lens_xl(swap_ab):
    """XL in bf16 at L = 500.  With the default options the padded batch (M = 2000) runs its fp32-output linears as swap-AB tiles and each
    solo forward (M < 512) on 2-CTA cluster tiles (Dit::lin), so they are compared at the bf16 floor; a handle built with swap_ab = 0 takes
    the cluster tiles at every M and must match bit for bit.  The fp32 oracle (CPU) checks the shortest clip."""
    from ezaudio_b200 import _lib
    from ezaudio_b200.dit import MaskDiT
    from oracle import ezaudio_oracle as O
    cfg = synth.model_cfg("xl")
    sd = _xl_state_dict()
    lens, L, Lc, t = [500, 350, 275, 137], 500, 100, 479
    Be = len(lens)
    x = synth.synth_latents(Be, L)
    ctx, mask = synth.synth_context(Be, Lc, cfg["context_dim"])
    Lib = _lib.lib()
    _lib.check(Lib.ezb_set_option(b"swap_ab", swap_ab))
    try:
        m = MaskDiT(precision="bf16", max_batch=Be, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    finally:
        _lib.check(Lib.ezb_set_option(b"swap_ab", 1))
    got, solo = _padded_vs_solo(m, x, ctx, mask, t, lens)
    for b, n in enumerate(lens):
        assert torch.isfinite(got[b]).all(), (b, n)
        if swap_ab == 0:
            assert torch.equal(got[b], solo[b]), (b, n, float((got[b] - solo[b]).abs().max()))
        else:
            err = (got[b] - solo[b]).abs()
            assert float(err.max()) < TOL["bf16"][0] and float(err.mean()) < TOL["bf16"][1], (b, n)
    b, n = 3, lens[3]
    with torch.no_grad():
        want, _ = O.maskdit_forward(sd, cfg, x[b:b + 1, :, :n], torch.tensor(t), ctx[b:b + 1], mask[b:b + 1])
    err = (got[b] - want[0]).abs()
    assert float(err.max()) < TOL["bf16"][0] and float(err.mean()) < TOL["bf16"][1], (float(err.max()), float(err.mean()))


def test_cfg_ddim_step_lens_matches_solo_calls():
    from ezaudio_b200.inference import _ddim_step
    B, Cc, L, lens = 3, 128, 100, [100, 37, 1]
    g = torch.Generator(device="cuda").manual_seed(5)
    mo = torch.randn(2 * B, Cc, L, device="cuda", generator=g)
    lat = torch.randn(B, Cc, L, device="cuda", generator=g)
    nz = torch.randn(B, Cc, L, device="cuda", generator=g)
    coef = (0.8, 0.6, 0.9, 0.3, 0.25)   # sigma != 0 (eta > 0)
    mo_p, lat_p, nz_p = mo.clone(), lat.clone(), nz.clone()
    for b, n in enumerate(lens):
        mo_p[b, :, n:] = float("nan"); mo_p[B + b, :, n:] = float("nan"); nz_p[b, :, n:] = float("nan"); lat_p[b, :, n:] = 7.0
    _ddim_step(mo_p, lat_p, nz_p, B, Cc, L, 5.0, 0.75, coef, torch.tensor(lens, dtype=torch.int32, device="cuda"))
    for b, n in enumerate(lens):
        ls = lat[b:b + 1, :, :n].contiguous()
        _ddim_step(torch.cat([mo[b:b + 1, :, :n], mo[B + b:B + b + 1, :, :n]]).contiguous(), ls, nz[b:b + 1, :, :n].contiguous(), 1, Cc, n, 5.0, 0.75, coef)
        torch.cuda.synchronize()
        assert torch.equal(lat_p[b, :, :n], ls[0]), (b, n)
        assert bool((lat_p[b, :, n:] == 7.0).all()), (b, n)   # padded latents untouched


def _loop_setup():
    from ezaudio_b200.dit import MaskDiT
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    B, L, Lc = 3, 40, 12
    ctx, mask = synth.synth_context(B, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    m = MaskDiT(precision="bf16", max_batch=2 * B, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    return m, ctx, mask, uctx, umask, L


def test_sample_latents_lengths_match_solo_runs_and_replay_one_graph():
    from ezaudio_b200.inference import sample_latents
    from ezaudio_b200.scheduler import DDIMScheduler
    m, ctx, mask, uctx, umask, L = _loop_setup()
    seeds = [11, 12, 13]
    kw = dict(audio_frames=L, guidance_scale=5.0, guidance_rescale=0.75, ddim_steps=3, eta=1.0, random_seed=seeds)

    def solo(b, n):
        return sample_latents(m, DDIMScheduler(), ctx[b:b + 1], mask[b:b + 1], uctx, umask, **dict(kw, audio_frames=n, random_seed=[seeds[b]]),
                              use_graphs=False)[0]

    mix1, mix2 = [40, 33, 24], [25, 40, 31]
    a = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, lengths=mix1, **kw)
    cache = m._loop_cache
    n_entries, (entry,) = len(cache), [v for k, v in cache.items()]
    graph, launches = entry["graph"], entry["launches"]
    b2 = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, lengths=mix2, **kw)
    assert len(cache) == n_entries and entry["graph"] is graph and entry["launches"] == launches   # replayed, not recaptured
    e = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, lengths=mix2, use_graphs=False, **kw)
    assert torch.equal(b2, e)
    for lat, mix in ((a, mix1), (b2, mix2)):
        for b, n in enumerate(mix):
            assert torch.equal(lat[b, :, :n], solo(b, n)), (mix, b, n)
            assert bool((lat[b, :, n:] == 0).all())


def test_generate_audio_per_prompt_lengths(monkeypatch):
    from ezaudio_b200 import api, config
    from tests.test_api_gpu import _tiny_params
    tiny = _tiny_params()
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    ez = api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16), max_batch=2,
                     max_length_s=2)
    prompts, lengths, seeds = ["a dog barks", "rain on a roof"], [1, 1.5], [7, 8]
    sr, wavs = ez.generate_audio(prompts, length=lengths, ddim_steps=3, random_seed=seeds, pad_length=2)
    assert sr == 24000 and isinstance(wavs, list) and len(wavs) == 2
    for p, n, s, w in zip(prompts, lengths, seeds, wavs):
        assert w.dtype == np.float32 and w.shape == (int(24000 * n),) and np.isfinite(w).all()
        _, want = ez.generate_audio(p, length=n, ddim_steps=3, random_seed=s)
        assert np.array_equal(w, want), (p, n)


def test_lengths_rejected_before_device_work():
    from ezaudio_b200 import _lib
    from ezaudio_b200.inference import sample_latents
    from ezaudio_b200.scheduler import DDIMScheduler
    m, ctx, mask, uctx, umask, L = _loop_setup()
    torch.cuda.synchronize()
    c0, mem0 = _lib.lib().ezb_launch_count(), torch.cuda.memory_allocated()
    kw = dict(audio_frames=L, guidance_scale=5.0, ddim_steps=2, random_seed=[1, 2, 3])
    gt = torch.zeros(3, 128, L)
    with pytest.raises(NotImplementedError):
        sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, gt=gt, gt_mask=gt.bool(), lengths=[L, L, L], **kw)
    with pytest.raises(NotImplementedError):
        sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, controlnet=object(), condition=gt, lengths=[L, L, L], **kw)
    for bad in ([0, 10, 10], [L + 1, 10, 10], [10, 10], [10, 10, 10, 10]):
        with pytest.raises(ValueError):
            sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, lengths=bad, **kw)
    assert torch.cuda.memory_allocated() == mem0
    with pytest.raises(NotImplementedError):
        m.forward_step(torch.zeros(2, 128, L, device="cuda"), 0, gt=torch.zeros(2, 128, L, device="cuda"),
                       lengths=torch.tensor([L, L], dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    assert _lib.lib().ezb_launch_count() == c0
