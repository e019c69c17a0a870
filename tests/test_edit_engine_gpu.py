"""Edits in the continuous-batching engine on the GPU: the all-ones inpainting mask against the forward without gt (bit for bit), an edit's
audio independent of its co-tenants, the admission encode against the scalar call's, the fp32 oracle loop with gt, and the waveform
semantics of editing_audio."""
import dataclasses

import numpy as np
import pytest
import torch

from ezaudio_b200 import synth, weights
from ezaudio_b200.api import edit_plan
from ezaudio_b200.frontend import EditRequest, Request
from ezaudio_b200.inference import scale_shift_re
from oracle import ezaudio_oracle as O
from tests.test_engine_gpu import MIX, TARGET, _model, _tiny_ez

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind,precision", [("tiny", "bf16"), ("tiny", "bf16x3"), ("xl", "bf16")])
def test_all_ones_mask_matches_forward_without_gt(kind, precision):
    """The engine's text-to-audio rows: gt with an all-ones mask packs the operand the forward builds without gt, whatever gt holds."""
    Be, L, Lc = 4, (500 if kind == "xl" else 96), (100 if kind == "xl" else 12)
    cfg, m = _model(kind, precision, Be, L, Lc)
    m.set_timesteps([999, 759, 479, 239, 19])
    x = synth.synth_latents(Be, L).cuda()
    ctx, mask = synth.synth_context(Be, Lc, cfg["context_dim"])
    m.set_context(ctx.cuda(), mask.cuda())
    G = synth.synth_latents(Be, L, seed=77).cuda()
    G[1] = float("nan")
    G[3, :, L // 2:] = float("nan")
    ones = torch.ones(Be, L, dtype=torch.uint8, device="cuda")
    tix = torch.tensor([0, 2, 4, 1], dtype=torch.int32, device="cuda")
    lens = torch.tensor([L, L // 2, 1, L - 3], dtype=torch.int32, device="cuda")
    want = m.forward_step(x, 0, t_index=tix, lengths=lens).clone()
    got = m.forward_step(x, 0, t_index=tix, lengths=lens, gt=G, gt_mask_u8=ones)
    torch.cuda.synchronize()
    for b, n in enumerate(lens.tolist()):
        assert torch.equal(got[b, :, :n].view(torch.int32), want[b, :, :n].view(torch.int32)), (b, n)


def _clip(seconds, f, sr=24000):
    t = np.arange(int(seconds * sr)) / sr
    return (0.3 * np.sin(2 * np.pi * f * t) + 0.05 * np.sin(2 * np.pi * 3 * f * t)).astype(np.float32)


# the target's crop is 1.6 s (80 frames); the other edit outpaints 0.3 s past the end of its 1.5-s clip with a 0.9-s (45-frame) crop
EDIT = EditRequest("a bell", 0.5, _clip(3, 220), 1.2, 0.8, guidance_scale=3.5, guidance_rescale=0, ddim_steps=8, eta=1, random_seed=7)
OTHER = EditRequest("rain on a roof", 0.5, _clip(1.5, 330), 1.2, 0.6, guidance_scale=5, guidance_rescale=0.75, ddim_steps=4, eta=0, random_seed=8)


def _submit(eng, r):
    return eng.submit(**dataclasses.asdict(r))


def _plan(r):
    return edit_plan(len(r.gt_file), 24000, 50, 480, r.boundary, r.mask_start, r.mask_length)


def _check_semantics(got, r):
    """What test_edit_batch_gpu checks of editing_audio: the whole clip, the original outside the pasted crop, the mask regenerated."""
    p = _plan(r)
    raw = np.zeros(p["n_total"], np.float32)
    raw[:len(r.gt_file)] = r.gt_file
    ref = raw / (np.abs(raw).max() + 1e-9)
    assert got.dtype == np.float32 and got.shape == (p["n_total"],) and np.isfinite(got).all()
    s, e = p["s0"], p["s0"] + p["n_paste"]
    assert np.allclose(got[:s], ref[:s], atol=1e-6) and np.allclose(got[e:], ref[e:], atol=1e-6)
    lo, hi = s + p["m0"] * 480, s + min(p["m1"] * 480, p["n_paste"])
    assert not np.allclose(got[lo:hi], ref[lo:hi], atol=1e-2)


def test_edit_audio_independent_of_co_tenants_and_one_graph(monkeypatch):
    from ezaudio_b200.engine import ContinuousEngine
    ez = _tiny_ez("bf16", monkeypatch)
    alone = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8))
    torch.manual_seed(123)   # the global RNG state at an edit's admission fixes its bottleneck noise
    (sr, want), = alone.run([EDIT])
    torch.manual_seed(124)
    (_, want_other), = alone.run([OTHER])
    (_, want_t2a), = alone.run([Request(**TARGET)])
    assert sr == 24000
    _check_semantics(want, EDIT)
    _check_semantics(want_other, OTHER)
    assert want_other.shape == (int(1.8 * 24000),)   # outpainting extends the clip to the mask's end

    eng = ContinuousEngine(ez, slots=3, max_length_s=2, ddim_steps=(4, 8))
    torch.manual_seed(124)                # admitted in one step after a text-to-audio request, which draws nothing from the global RNG
    eng.submit(**MIX[0])                  # text-to-audio, 8 steps
    t_other = _submit(eng, OTHER)         # another edit: other steps, guidance, eta, crop length, outpainting
    out = {}
    for _ in range(3):
        out.update({t: w for t, _, w in eng.step()})
    torch.manual_seed(123)
    t_edit = _submit(eng, EDIT)           # joins at step 4, in slot 2
    t_t2a = eng.submit(**TARGET)          # queued: takes the slot OTHER frees after step 4, next to a generation and an edit
    eng.submit(**MIX[2])
    out.update({t: w for t, _, w in eng.step()})
    # scalar calls in between replace the denoiser's context and table and draw from the global RNG; the engine is unaffected
    ez.editing_audio("a cat", 0.3, _clip(2, 550), 0.5, 0.5, ddim_steps=3, random_seed=2)
    ez.generate_audio("a cat", length=1, ddim_steps=3, random_seed=1)
    for t, _, w in eng.stream():
        out[t] = w
    assert len(out) == 5
    assert out[t_edit].tobytes() == want.tobytes()
    assert out[t_other].tobytes() == want_other.tobytes()
    assert out[t_t2a].tobytes() == want_t2a.tobytes()
    assert eng.backend.captures == 1 and alone.backend.captures == 1
    S = eng.slots
    assert bool((eng.backend.gt == 0).all()) and bool((eng.backend.gt_mask == 1).all()) and eng.backend.edits == [None] * S


class _Recorder:
    """Wraps an Autoencoder and keeps what each call returns (encode) or receives (decode)."""

    def __init__(self, ae):
        self.ae, self.encoded, self.decoded = ae, [], []

    def __getattr__(self, name):
        return getattr(self.ae, name)

    def __call__(self, audio=None, embedding=None, lengths=None):
        out = self.ae(audio=audio, embedding=embedding, lengths=lengths)
        if audio is not None:
            self.encoded.append(out.clone())
        else:
            self.decoded.append(embedding.clone())
        return out


def test_admission_encode_equals_the_scalar_calls(monkeypatch):
    from ezaudio_b200.engine import ContinuousEngine
    ez = _tiny_ez("bf16", monkeypatch)
    eng = ContinuousEngine(ez, slots=2, max_length_s=2, ddim_steps=(4, 8))
    rec = _Recorder(ez.autoencoder)
    ez.autoencoder = rec
    p = _plan(EDIT)
    n = p["frames"]
    torch.manual_seed(5)
    ez.editing_audio(EDIT.prompt, EDIT.boundary, EDIT.gt_file, EDIT.mask_start, EDIT.mask_length, ddim_steps=4, random_seed=7)
    (want,) = rec.encoded
    assert tuple(want.shape) == (1, 128, n)
    eng.submit("x", length=1, ddim_steps=4, random_seed=1)   # slot 0: text-to-audio
    torch.manual_seed(5)
    _submit(eng, EDIT)                                       # slot 1
    eng.step()
    be, S = eng.backend, eng.slots
    for row in (1, S + 1):
        assert torch.equal(be.gt[row, :, :n], want[0]) and bool((be.gt[row, :, n:] == 0).all())
        m = be.gt_mask[row].cpu()
        exp = torch.zeros_like(m)
        exp[p["m0"]:p["m1"]] = 1
        exp[n:] = 1
        assert torch.equal(m, exp)
    for row in (0, S):   # the text-to-audio slot keeps zeros and an all-ones mask
        assert bool((be.gt[row] == 0).all()) and bool((be.gt_mask[row] == 1).all())
    list(eng.stream())
    assert bool((be.gt == 0).all()) and bool((be.gt_mask == 1).all())


def test_edit_latents_match_oracle_loop(monkeypatch):
    from ezaudio_b200.engine import ContinuousEngine
    ez = _tiny_ez("bf16x3", monkeypatch)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(ez.params["model"]), 3)
    eng = ContinuousEngine(ez, slots=2, max_length_s=2, ddim_steps=(4, 8))
    be = eng.backend
    rec = _Recorder(ez.autoencoder)
    ez.autoencoder = rec
    kept = {}
    finish = be.finish

    def keep(k, frames):
        if be.edits[k] is not None:
            kept[k] = (be.lat[k, :, :frames].clone(), be.gt[k, :, :frames].clone(), be.gt_mask[k, :frames].bool().clone(), len(rec.decoded))
        return finish(k, frames)

    be.finish = keep
    reqs = [EDIT, Request(**MIX[0]), OTHER, EditRequest("", 0.2, _clip(2, 440), 0.4, 0.5, ddim_steps=4, eta=1, random_seed=9)]
    slot_of = {}
    admit = be.admit

    def rec_admit(k, prompt, seed, frames, edit=None):
        slot_of[seed] = k
        return admit(k, prompt, seed, frames, edit=edit)

    be.admit = rec_admit
    got = {}
    for r in reqs:
        _submit(eng, r)
    while eng.pending():
        for t, _, _ in eng.step():
            r = reqs[t]
            if isinstance(r, EditRequest):
                got[t] = kept[slot_of[r.random_seed]]
    assert sorted(got) == [0, 2, 3]
    enc = ez.encode_text
    uctx, umask = enc([""])
    sc, sh = ez.params["autoencoder"]["scale"], ez.params["autoencoder"]["shift"]
    for t, (lat, gt, regen, i) in got.items():
        r = reqs[t]
        n = lat.shape[-1]
        g = torch.Generator(device="cuda").manual_seed(r.random_seed)
        noise = torch.randn((1, 128, n), generator=g, device="cuda").cpu()
        steps = [torch.empty((1, 128, n), device="cuda").normal_(generator=g).cpu() for _ in range(r.ddim_steps)] if r.eta > 0 else None
        ctx, mask = enc([r.prompt])
        cfg = r.prompt != ""
        gm = regen.view(1, 1, n).expand(1, 128, n).cpu()
        with torch.no_grad():
            ref = O.sample_loop(sd, ez.params["model"], noise, ctx, mask, uctx, umask, gt=gt.view(1, 128, n).cpu(), gt_mask=gm,
                                guidance_scale=r.guidance_scale if cfg else None, guidance_rescale=r.guidance_rescale, ddim_steps=r.ddim_steps,
                                eta=r.eta, step_noise=steps)
        err = float((torch.where(gm, lat.cpu().view(1, 128, n), gt.cpu().view(1, 128, n)) - ref).abs().max())
        assert err < 5e-3, (t, err)
        # the decoded latent: the rescaled prediction on the regenerated frames, the crop's latent exactly on the kept ones
        emb = rec.decoded[i][0].cpu()
        assert torch.equal(emb[:, ~regen.cpu()], gt.cpu()[:, ~regen.cpu()])
        assert torch.equal(emb[:, regen.cpu()], scale_shift_re(lat, sc, sh).cpu()[:, regen.cpu()])
        assert bool(regen[_plan(r)["m0"]:_plan(r)["m1"]].all()) and not bool(regen.all())


def test_fp8_ezaudio_still_refused(monkeypatch):
    from ezaudio_b200 import api, config
    from ezaudio_b200.engine import ContinuousEngine
    from tests.test_api_gpu import _tiny_params
    tiny = _tiny_params()
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    ez = api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16), max_batch=2,
                     max_length_s=2, precision="fp8")
    with pytest.raises(NotImplementedError):
        ContinuousEngine(ez, slots=2, max_length_s=2, ddim_steps=(4, 8))
