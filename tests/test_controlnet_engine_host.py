"""ControlNet requests in the continuous-batching engine, host side: engine.ContinuousEngine with a stub ControlNet backend (request defaults,
validation before any device work, per-request conditioning scales, admission order) and the per-clip list form of
EzAudio_ControlNet.generate_audio rejecting mismatched lists before device work."""
import dataclasses
import inspect

import numpy as np
import pytest

from ezaudio_b200.engine import ContinuousEngine
from ezaudio_b200.frontend import ControlRequest
from ezaudio_b200.scheduler import DDIMScheduler


class StubControlSlots:
    """Records every call; the 'waveform' of a finished slot is (slot, frames)."""
    control = True
    sr, latent_sr, max_frames, max_timesteps = 24000, 50, 500, 1000

    def __init__(self):
        self.calls = []

    def make_scheduler(self):
        return DDIMScheduler()

    def admit(self, k, prompt, seed, frames, audio=None, surpass_noise=0.0):
        self.calls.append(("admit", k, prompt, seed, frames, audio, surpass_noise))

    def step(self, plan):
        self.calls.append(("step", list(plan)))

    def finish(self, k, frames):
        self.calls.append(("finish", k, frames))
        return ("wav", k, frames)


def _engine(slots=2):
    be = StubControlSlots()
    return ContinuousEngine(None, slots=slots, ddim_steps=(25, 50, 100), backend=be), be


def _clip(n=24000, seed=0):
    return (0.1 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


def test_control_request_defaults_are_generate_audio_defaults():
    from ezaudio_b200.api import EzAudio_ControlNet
    sig = inspect.signature(EzAudio_ControlNet.generate_audio).parameters
    fields = {f.name: f for f in dataclasses.fields(ControlRequest)}
    names = {"text": "prompt", "audio_path": "audio"}
    for p in list(sig.values())[1:]:
        if p.name == "randomize_seed":
            continue
        f = fields[names.get(p.name, p.name)]
        if p.default is inspect.Parameter.empty:
            assert f.default is dataclasses.MISSING, p.name
        else:
            assert f.default == p.default and type(f.default) is type(p.default), p.name
    assert len(fields) == len(sig) - 2   # every argument but self and randomize_seed


@pytest.mark.parametrize("kw", [dict(audio="/nonexistent/clip.wav"), dict(audio=np.zeros((2, 100), np.float32)),
                                dict(audio=np.zeros(0, np.float32)), dict(audio=[0.1, 0.2]), dict(surpass_noise=-0.1),
                                dict(surpass_noise=float("nan")), dict(conditioning_scale=float("inf")), dict(conditioning_scale=float("nan")),
                                dict(conditioning_scale="1"), dict(ddim_steps=30), dict(random_seed=-1), dict(eta=-1),
                                dict(guidance_scale=float("nan"))])
def test_invalid_control_requests_rejected_before_device_work(kw):
    eng, be = _engine()
    args = dict(dict(audio=_clip(), ddim_steps=50, random_seed=1), **kw)
    with pytest.raises(ValueError):
        eng.submit("a siren", **args)
    assert eng.pending() == 0 and eng.step() == [] and be.calls == []


def test_reference_clip_read_at_submit(tmp_path):
    from scipy.io import wavfile
    f = str(tmp_path / "ref.wav")
    wavfile.write(f, 24000, (_clip(36000) * 32767).astype(np.int16))
    eng, be = _engine()
    eng.submit("a siren", audio=f, random_seed=3)
    assert be.calls == []
    eng.step()
    (_, k, prompt, seed, frames, audio, gate), = [c for c in be.calls if c[0] == "admit"]
    assert (k, prompt, seed, frames, gate) == (0, "a siren", 3, 500, 0.0)
    assert audio.dtype == np.float32 and audio.shape == (36000,)


def test_each_slot_step_carries_its_requests_conditioning_scale():
    eng, be = _engine(slots=3)
    reqs = [ControlRequest("a", _clip(seed=1), conditioning_scale=0.5, ddim_steps=25, surpass_noise=0.01, random_seed=1),
            ControlRequest("b", _clip(seed=2), conditioning_scale=1, ddim_steps=50, eta=0, random_seed=2),
            ControlRequest("", _clip(seed=3), conditioning_scale=0, ddim_steps=25, guidance_scale=5, random_seed=3),
            ControlRequest("d", _clip(seed=4), conditioning_scale=1.3, ddim_steps=25, random_seed=4)]
    res = eng.run(reqs)
    assert len(res) == 4
    slot_req, seen, nxt = {}, {i: [] for i in range(4)}, 0
    for c in be.calls:
        if c[0] == "admit":
            r = reqs[nxt]
            assert (c[2], c[3], c[4], c[6]) == (r.prompt, r.random_seed, 500, float(r.surpass_noise))
            assert np.array_equal(c[5], r.audio)
            slot_req[c[1]] = nxt
            nxt += 1
        elif c[0] == "step":
            for k, e in enumerate(c[1]):
                if e is not None:
                    seen[slot_req[k]].append(e)
    for i, r in enumerate(reqs):
        sched = DDIMScheduler()
        sched.set_timesteps(r.ddim_steps)
        ts = [int(t) for t in sched.timesteps]
        got = seen[i]
        assert len(got) == r.ddim_steps and [eng.table[e.t_index] for e in got] == ts
        cfg = bool(r.guidance_scale) and r.prompt != ""
        for e, t in zip(got, ts):
            assert e.conditioning_scale == float(r.conditioning_scale)
            assert e.frames == 500 and e.cfg == cfg and e.guidance_scale == (float(r.guidance_scale) if cfg else 0.0)
            assert e.coef == sched.step_coefficients(t, float(r.eta)) and e.draw_noise == (r.eta > 0)


def test_fifo_admission_and_ticket_order():
    eng, be = _engine(slots=2)
    steps = [25, 50, 25, 100, 25]
    tickets = [eng.submit(f"p{i}", audio=_clip(seed=i), ddim_steps=n, random_seed=i) for i, n in enumerate(steps)]
    assert tickets == [0, 1, 2, 3, 4]
    done = list(eng.stream())
    admits = [(c[1], c[2]) for c in be.calls if c[0] == "admit"]
    assert admits == [(0, "p0"), (1, "p1"), (0, "p2"), (0, "p3"), (1, "p4")]
    assert [t for t, _, _ in done] == [0, 2, 1, 4, 3]
    t = [eng.submit("x", audio=_clip(), ddim_steps=50), eng.submit("y", audio=_clip(), ddim_steps=25)]
    assert t == [5, 6]
    assert [w[1] for _, w in eng.run()] == [0, 1]   # run() returns the queued requests in submission order


@pytest.mark.parametrize("kw", [dict(text=["a", "b"], audio_path=[np.zeros(100, np.float32)]),
                                dict(text="a", audio_path=[np.zeros(100, np.float32)]),
                                dict(text=["a", "b"], audio_path=[np.zeros(100, np.float32)] * 2, surpass_noise=[0.1]),
                                dict(text=["a", "b"], audio_path=[np.zeros(100, np.float32)] * 2, random_seed=[1, 2, 3]),
                                dict(text=["a", "b"], audio_path=[np.zeros(100, np.float32), np.zeros((2, 100), np.float32)])])
def test_per_clip_generate_audio_rejects_mismatched_lists_before_device_work(kw, monkeypatch):
    import torch
    from ezaudio_b200 import api

    def no_device(*a, **k):
        raise AssertionError("device work before validation")

    monkeypatch.setattr(api, "energy_condition", no_device)
    monkeypatch.setattr(api.post, "prepare_wave", no_device)
    monkeypatch.setattr(torch.Tensor, "to", no_device)
    ez = api.EzAudio_ControlNet.__new__(api.EzAudio_ControlNet)   # no weights, no device: only the host-side state the call reads first
    ez.device = "cuda"
    ez.params = {"autoencoder": {"sr": 24000, "latent_sr": 50}, "conditioner": {"condition_type": "energy"}}
    ez._text_embeds = no_device
    with pytest.raises(ValueError):
        ez.generate_audio(**kw)
