"""Edits (inpainting / outpainting) of different crop lengths in one batch: sample_latents with gt, gt_mask and lengths together, and the
list form of EzAudio.editing_audio, against the same edits run one at a time."""
import numpy as np
import pytest
import torch

from ezaudio_b200 import config, synth, weights

pytestmark = pytest.mark.gpu


def test_sample_latents_gt_and_lengths_match_solo_runs():
    """Tiny model in bf16 with every clip >= 32 frames and fewer than 512 tokens per forward, so the padded batch and the solo runs pick the
    same GEMM kernels (the condition tests/test_varlen_gpu.py states) and must agree bit for bit."""
    from ezaudio_b200.dit import MaskDiT
    from ezaudio_b200.inference import sample_latents
    from ezaudio_b200.scheduler import DDIMScheduler
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    B, L, Lc, lens, seeds = 3, 40, 12, [40, 33, 36], [11, 12, 13]
    ctx, mask = synth.synth_context(B, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    m = MaskDiT(precision="bf16", max_batch=2 * B, max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    gt, gm = synth.synth_gt(B, L)
    gm[1, :, :5] = True   # a different mask per clip
    gt_pad, gm_pad = gt.clone(), gm.clone()
    for b, n in enumerate(lens):   # what lies past a clip's end is ignored
        gt_pad[b, :, n:] = float("nan")
        gm_pad[b, :, n:] = False
    kw = dict(guidance_scale=5.0, guidance_rescale=0.75, ddim_steps=3, eta=1.0)
    got = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, gt=gt_pad, gt_mask=gm_pad, audio_frames=L, random_seed=seeds, lengths=lens, padded_gt=True, **kw)
    again = sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, gt=gt_pad, gt_mask=gm_pad, audio_frames=L, random_seed=seeds, lengths=lens, padded_gt=True, **kw)
    assert torch.equal(got, again)   # the captured graph replays to the eager result
    for b, n in enumerate(lens):
        solo = sample_latents(m, DDIMScheduler(), ctx[b:b + 1], mask[b:b + 1], uctx, umask, gt=gt[b:b + 1, :, :n].contiguous(),
                              gt_mask=gm[b:b + 1, :, :n].contiguous(), audio_frames=n, random_seed=[seeds[b]], use_graphs=False, **kw)
        assert torch.equal(got[b, :, :n], solo[0]), (b, n, float((got[b, :, :n] - solo[0]).abs().max()))
        assert bool((got[b, :, n:] == 0).all()), (b, n)
        keep = ~gm[b, 0, :n].cuda()
        assert torch.equal(got[b, :, :n][:, keep], gt[b, :, :n].cuda()[:, keep])   # kept frames are the pasted gt


def _tiny_ez(monkeypatch, precision, max_batch):
    from ezaudio_b200 import api
    tiny = config.load_params("s3_xl")
    tiny["model"] = synth.tiny_model(72)
    tiny["text_encoder"] = dict(tiny["text_encoder"], max_length=16)
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    return api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16), max_batch=max_batch,
                       max_length_s=4, precision=precision)


def _clip(seconds, f, sr=24000):
    t = np.arange(int(seconds * sr)) / sr
    return (0.3 * np.sin(2 * np.pi * f * t) + 0.05 * np.sin(2 * np.pi * 3 * f * t)).astype(np.float32)


# three edits whose crops differ in length (150, 60 and 75 latent frames); the last one outpaints 0.6 s past the end of its 2-s clip
EDITS = dict(text=["a bell", "rain on a roof", "a dog barks"], gt_file=[_clip(4, 220), _clip(3, 330), _clip(2, 440)], mask_start=[1.5, 0.5, 1.6],
             mask_length=[1.0, 0.6, 1.0], boundary=[1, 0.4, 0.5], random_seed=[3, 4, 5])


def test_editing_audio_list_equals_scalar_calls_in_sequence(monkeypatch):
    """bf16x3 takes the same GEMM kernels at every token count, so the batch must reproduce the three scalar calls bit for bit."""
    from ezaudio_b200.api import edit_plan
    ez = _tiny_ez(monkeypatch, "bf16x3", 3)
    torch.manual_seed(21)
    sr, batch = ez.editing_audio(**EDITS, ddim_steps=3)
    assert sr == 24000 and isinstance(batch, list) and len(batch) == 3
    torch.manual_seed(21)   # the scalar calls draw their bottleneck noise from the global RNG in this order
    for i, got in enumerate(batch):
        one = {k: v[i] for k, v in EDITS.items()}
        _, want = ez.editing_audio(**one, ddim_steps=3)
        assert got.dtype == np.float32 and got.shape == want.shape and np.isfinite(got).all()
        assert np.array_equal(got, want), (i, float(np.abs(got - want).max()))
        p = edit_plan(len(one["gt_file"]), sr, 50, 480, one["boundary"], one["mask_start"], one["mask_length"])
        raw = np.zeros(p["n_total"], np.float32)
        raw[:len(one["gt_file"])] = one["gt_file"]
        ref = raw / (np.abs(raw).max() + 1e-9)
        assert got.shape == (p["n_total"],)
        assert np.allclose(got[:p["s0"]], ref[:p["s0"]], atol=1e-6) and np.allclose(got[p["s0"] + p["n_paste"]:], ref[p["s0"] + p["n_paste"]:], atol=1e-6)
        lo, hi = p["s0"] + p["m0"] * 480, p["s0"] + min(p["m1"] * 480, p["n_paste"])
        assert not np.allclose(got[lo:hi], ref[lo:hi], atol=1e-2)   # the masked span is regenerated
    assert batch[2].shape == (int(2.6 * sr),)


def test_second_batch_at_the_same_pad_length_replays_the_graph(monkeypatch):
    ez = _tiny_ez(monkeypatch, "bf16", 3)
    sr, a = ez.editing_audio(**EDITS, ddim_steps=3, pad_length=3.5)
    cache = ez.unet._loop_cache
    (entry,) = cache.values()
    graph, launches = entry["graph"], entry["launches"]
    assert graph is not None
    other = dict(EDITS, mask_start=[1.0, 0.8, 0.2], mask_length=[0.5, 1.2, 0.7], boundary=[0.5, 0.5, 0.3], gt_file=EDITS["gt_file"][::-1])
    _, b = ez.editing_audio(**other, ddim_steps=3, pad_length=3.5)
    assert len(cache) == 1 and entry["graph"] is graph and entry["launches"] == launches   # replayed, not recaptured
    assert [w.shape for w in b] == [(2 * sr,), (3 * sr,), (4 * sr,)] and all(np.isfinite(w).all() for w in a + b)


def test_list_form_is_rejected_before_device_work(monkeypatch):
    from ezaudio_b200 import _lib
    ez = _tiny_ez(monkeypatch, "bf16", 2)
    torch.cuda.synchronize()
    c0, mem0 = _lib.lib().ezb_launch_count(), torch.cuda.memory_allocated()
    two = {k: v[:2] for k, v in EDITS.items()}
    for bad in (EDITS,                                         # three edits, max_batch 2
                dict(two, mask_start=[1.5]),                   # list of the wrong length
                dict(two, gt_file=[_clip(8, 220), _clip(3, 330)], mask_start=[1, 0.5], mask_length=[5, 0.6], boundary=[2, 0.4]),   # 9-s crop, max_length_s 4
                dict(two, text=["", "rain"]),                  # guidance cannot differ inside a batch
                dict(two, mask_length=[0, 0.6])):
        with pytest.raises(ValueError):
            ez.editing_audio(**bad, ddim_steps=3)
    with pytest.raises(ValueError):
        ez.editing_audio(**two, ddim_steps=3, pad_length=5)    # above max_length_s
    with pytest.raises(ValueError):
        ez.editing_audio(**two, ddim_steps=3, pad_length=1)    # below the longest crop
    with pytest.raises(ValueError):
        ez.editing_audio("a bell", 1, EDITS["gt_file"][0], 1.5, 1.0, pad_length=3)   # pad_length belongs to the list form
    assert _lib.lib().ezb_launch_count() == c0 and torch.cuda.memory_allocated() == mem0


def test_padded_gt_lengths_rejected_before_device_work():
    """gt with lengths: refused without padded_gt, and with it bad lengths, a gt of another shape and a ControlNet are refused on the host."""
    from ezaudio_b200 import _lib
    from ezaudio_b200.inference import sample_latents
    from ezaudio_b200.scheduler import DDIMScheduler
    from tests.test_varlen_gpu import _loop_setup
    m, ctx, mask, uctx, umask, L = _loop_setup()
    torch.cuda.synchronize()
    c0, mem0 = _lib.lib().ezb_launch_count(), torch.cuda.memory_allocated()
    kw = dict(audio_frames=L, guidance_scale=5.0, ddim_steps=2, random_seed=[1, 2, 3])
    gt = torch.zeros(3, 128, L)
    with pytest.raises(NotImplementedError):
        sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, gt=gt, gt_mask=gt.bool(), lengths=[L, L, L], **kw)
    with pytest.raises(NotImplementedError):
        sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, gt=gt, gt_mask=gt.bool(), controlnet=object(), condition=gt, lengths=[L, L, L],
                       padded_gt=True, **kw)
    for bad in ([0, 10, 10], [L + 1, 10, 10], [10, 10], [10, 10, 10, 10]):
        with pytest.raises(ValueError):
            sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, gt=gt, gt_mask=gt.bool(), lengths=bad, padded_gt=True, **kw)
    with pytest.raises(ValueError):   # gt must be padded like the batch
        sample_latents(m, DDIMScheduler(), ctx, mask, uctx, umask, gt=gt[:, :, :L - 1], gt_mask=gt[:, :, :L - 1].bool(), lengths=[10, 10, 10],
                       padded_gt=True, **kw)
    assert torch.cuda.memory_allocated() == mem0
    torch.cuda.synchronize()
    assert _lib.lib().ezb_launch_count() == c0
