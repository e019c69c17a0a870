"""Long ControlNet clips on the host: the latent frame count of a reference clip, the window plan it gives (a clip just over one window
included), and the validation EzAudio_ControlNet.generate_long_audio / sample_long_latents do before any device work."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from ezaudio_b200 import api
from ezaudio_b200.api import long_control_frames
from ezaudio_b200.inference import check_long, sample_long_latents, window_plan


@pytest.mark.parametrize("n,want", [(1, 500), (72000, 500), (239999, 500), (240000, 500), (240001, 501), (240480, 501), (240481, 502),
                                    (1440000, 3000), (720000 + 17, 1501)])
def test_long_control_frames(n, want):
    assert long_control_frames(n, 480, 500) == want
    assert long_control_frames(n, 480, 500) == max(500, int(np.ceil(n / 480)))


def test_plans_of_reference_clips():
    assert window_plan(long_control_frames(240000, 480, 500), 500, 100) == [(0, 500)]   # 10 s: one window, generate_audio's shape
    # just over one window: the last window starts one frame in and overlaps the first by 499 frames, more than `overlap`
    plan = window_plan(long_control_frames(240001, 480, 500), 500, 100)
    assert plan == [(0, 500), (1, 500)] and plan[0][1] - plan[1][0] == 499 > 100
    plan = window_plan(long_control_frames(1440000, 480, 500), 500, 100)   # 60 s in 10 s windows with 2 s overlap: 8 windows
    assert len(plan) == 8 and plan[-1] == (2500, 500) and all(ln == 500 for _, ln in plan)
    check_long([3000], 1, 500, 100, True, 16, 500)                        # x 2 under CFG: 16 rows, max_batch 8
    with pytest.raises(ValueError, match="needs max_batch >= 8"):
        check_long([3000], 1, 500, 100, True, 14, 500)
    # the batch test's clips (4.5 s, 1.5 s, 3 s in 2 s windows, 0.4 s overlap): 3 + 1 + 2 windows, all full-length
    frames = [long_control_frames(int(s * 24000), 480, 100) for s in (4.5, 1.5, 3)]
    assert frames == [225, 100, 150]
    assert [len(window_plan(n, 100, 20)) for n in frames] == [3, 1, 2]


class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device work before validation: {name}")


def _stub(max_batch=4, monkeypatch=None):
    """An EzAudio_ControlNet whose device-facing members fail the test when touched; only the host-side attributes are real."""
    def no_device(*a, **k):
        raise AssertionError("device work before validation")

    monkeypatch.setattr(api, "energy_condition", no_device)
    monkeypatch.setattr(api.post, "prepare_wave", no_device)
    monkeypatch.setattr(api, "sample_long_latents", no_device)
    monkeypatch.setattr(torch.Tensor, "to", no_device)
    ez = object.__new__(api.EzAudio_ControlNet)
    ez.device = "cuda"
    ez.params = {"autoencoder": {"sr": 24000, "latent_sr": 50, "scale": 1.0, "shift": 0.0}, "conditioner": {"condition_type": "energy"}}
    ez.max_length_s = 10.0
    h = SimpleNamespace(_h=SimpleNamespace(desc=SimpleNamespace(max_batch=2 * max_batch, max_len=500)))
    ez.unet, ez.controlnet = h, h
    ez.autoencoder = _NoDevice()
    ez.noise_scheduler = _NoDevice()
    ez._text_embeds = no_device
    return ez


def _wave(seconds):
    return np.zeros(int(seconds * 24000), np.float32)


@pytest.mark.parametrize("kw", [
    dict(text=["a", "b"], audio_path=[_wave(3)]),                                      # one clip per prompt
    dict(text=["a", "b"], audio_path=[_wave(3)] * 3),
    dict(text="a", audio_path=[_wave(3)]),                                             # a string prompt with a list of clips
    dict(text=["a", "b"], audio_path=[_wave(3)] * 2, surpass_noise=[0.1]),             # one gate per prompt
    dict(text=["a", "b"], audio_path=[_wave(3)] * 2, random_seed=[1, 2, 3]),           # one seed per prompt
    dict(text="a", audio_path=_wave(30), window_length=12),                            # window past the handle's 10 s
    dict(text="a", audio_path=_wave(30), overlap=0),                                   # overlap below one frame
    dict(text="a", audio_path=_wave(30), overlap=0.01),                                # overlap rounds to 0 frames
    dict(text="a", audio_path=_wave(30), overlap=6),                                   # overlap past half the window
    dict(text=["a", ""], audio_path=[_wave(3)] * 2),                                   # empty and non-empty prompts mixed
    dict(text="a", audio_path=np.zeros((2, 24000), np.float32)),                       # not mono
    dict(text="a", audio_path=np.zeros(0, np.float32)),                                # empty clip
    dict(text="a", audio_path=_wave(60)),                                              # 8 windows x 2 rows > 2 * max_batch (4)
    dict(text=["a", "b"], audio_path=[_wave(30), _wave(30)]),                          # 2 x 4 windows x 2 = 16 rows > 8
])
def test_generate_long_audio_validates_before_device_work(kw, monkeypatch):
    with pytest.raises(ValueError):
        _stub(monkeypatch=monkeypatch).generate_long_audio(**kw)


def test_generate_long_audio_row_capacity_message(monkeypatch):
    with pytest.raises(ValueError, match="needs max_batch >= 8"):
        _stub(max_batch=4, monkeypatch=monkeypatch).generate_long_audio("a", _wave(60))
    with pytest.raises(ValueError, match="needs max_batch >= 3"):   # an empty prompt runs without guidance: 6 windows, one row each
        _stub(max_batch=2, monkeypatch=monkeypatch).generate_long_audio("", _wave(50))


def _loop_stub(max_batch=8, max_len=500):
    h = SimpleNamespace(_h=SimpleNamespace(desc=SimpleNamespace(max_batch=2 * max_batch, max_len=max_len), dev_index=0))
    return h, SimpleNamespace(_h=SimpleNamespace(desc=SimpleNamespace(max_batch=2 * max_batch, max_len=max_len)))


@pytest.mark.parametrize("case", ["no_condition", "no_controlnet", "shape", "short_clip", "rows"])
def test_sample_long_latents_refuses_before_device_work(case):
    unet, cn = _loop_stub()
    text, mask = torch.zeros(2, 4, 8), torch.ones(2, 4, dtype=torch.bool)
    lens = [700, 520]
    cond = torch.zeros(2, 1, 1400)
    kw = dict(controlnet=cn, condition=cond)
    if case == "no_condition":
        kw = dict(controlnet=cn)
    elif case == "no_controlnet":
        kw = dict(condition=cond)
    elif case == "shape":
        kw["condition"] = torch.zeros(2, 1, 1040)
    elif case == "short_clip":
        lens = [700, 499]
    else:
        unet, cn = _loop_stub(max_batch=2)   # 2 + 2 windows x 2 = 8 rows > 4
        kw["controlnet"] = cn
    with pytest.raises(ValueError):
        sample_long_latents(unet, None, text, mask, text, mask, lens, 500, 100, 3.5, 0.0, 5, 1.0, 1, **kw)
