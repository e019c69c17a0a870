"""Windowed denoising of long clips on the host: the window plan and its crossfade weights against an independent fp64 restatement, the
validation generate_long_audio / sample_long_latents do before any device work, and the VAE decoder's receptive field (decode_tiled's
halo) against its hand derivation."""
import math
from types import SimpleNamespace

import numpy as np
import pytest

from ezaudio_b200 import synth
from ezaudio_b200.api import EzAudio
from ezaudio_b200.inference import check_long, long_plan, window_plan, window_weights
from ezaudio_b200.vae import decoder_receptive_field

CASES = [(n, lw, o) for lw, o in ((500, 100), (500, 1), (500, 250), (64, 16), (40, 20), (7, 3), (2, 1), (10, 4))
         for n in sorted({1, 2, lw - 1, lw, lw + 1, lw + 2, 2 * lw - o, 2 * lw - o + 1, 3 * lw, 3000, 1499, 12 * lw + 5})]


def _plan64(n, lw, o):
    """The plan restated: starts 0, H, 2H, ... while a window of lw ends before n, then one window ending at n."""
    if n <= lw:
        return [(0, n)]
    h = lw - o
    out = []
    s = 0
    while s + lw < n:
        out.append((s, lw))
        s += h
    return out + [(n - lw, lw)]


def _weights64(k, count, length, lw, o):
    j = np.arange(length, dtype=np.float64)
    w = np.ones(length)
    if k > 0:
        w = np.minimum(w, (j + 1) / (o + 1))
    if k < count - 1:
        w = np.minimum(w, (lw - j) / (o + 1))
    return w


@pytest.mark.parametrize("n,lw,o", CASES)
def test_window_plan_covers_the_clip(n, lw, o):
    plan = window_plan(n, lw, o)
    assert plan == _plan64(n, lw, o)
    starts = [s for s, _ in plan]
    assert starts[0] == 0 and starts == sorted(starts)
    assert plan[-1][0] + plan[-1][1] == n                    # the last window ends at the clip's end
    assert all(ln == min(n, lw) for _, ln in plan)
    if n > lw:
        assert len(plan) == math.ceil((n - lw) / (lw - o)) + 1
        assert all(b - a == lw - o for a, b in zip(starts[:-2], starts[1:-1]))
    total, cover = np.zeros(n), np.zeros(n, dtype=int)
    for k, (s, ln) in enumerate(plan):
        w = window_weights(k, len(plan), ln, lw, o)
        assert w.dtype == np.float32 and (w > 0).all() and (w <= 1).all()
        np.testing.assert_allclose(w, _weights64(k, len(plan), ln, lw, o), rtol=2 ** -23, atol=0)
        total[s:s + ln] += w
        cover[s:s + ln] += 1
    assert (cover >= 1).all() and cover.max() <= 3
    assert (total >= 1 - 1e-6).all()                         # every frame has a total weight of at least one


def test_window_plan_examples():
    assert window_plan(3000, 500, 100) == [(k * 400, 500) for k in range(7)] + [(2500, 500)]   # 60 s in 10 s windows, 2 s overlap
    assert window_plan(1500, 500, 100) == [(0, 500), (400, 500), (800, 500), (1000, 500)]
    assert window_plan(500, 500, 100) == [(0, 500)] and window_plan(501, 500, 100) == [(0, 500), (1, 500)]
    assert window_plan(17, 500, 100) == [(0, 17)]
    assert np.array_equal(window_weights(0, 1, 17, 500, 100), np.ones(17, np.float32))   # one window: weight exactly 1


def test_long_plan_lays_the_windows_out_clip_by_clip():
    table, windows = long_plan([1500, 300, 900], 500, 100)
    assert table == [(0, 4, 1500), (4, 1, 300), (5, 2, 900)]
    assert windows[:5] == [(0, 0, 500), (0, 400, 500), (0, 800, 500), (0, 1000, 500), (1, 0, 300)]
    assert [w[0] for w in windows] == [0, 0, 0, 0, 1, 2, 2]
    assert windows[5:] == [(2, s, 500) for s, _ in window_plan(900, 500, 100)]


@pytest.mark.parametrize("o", [0, -1, 251, 500])
def test_window_plan_rejects_bad_overlap(o):
    with pytest.raises(ValueError):
        window_plan(1000, 500, o)


def test_check_long_row_capacity_names_max_batch():
    lens, table, windows = check_long([3000], 1, 500, 100, True, 16, 500)   # 8 windows x 2 = 16 rows: max_batch 8
    assert len(windows) == 8
    with pytest.raises(ValueError, match="max_batch >= 8"):
        check_long([3000], 1, 500, 100, True, 14, 500)
    check_long([3000], 1, 500, 100, False, 8, 500)   # no guidance: one row per window
    with pytest.raises(ValueError, match="max_batch >= 5"):
        check_long([3000, 200, 100], 3, 500, 100, False, 8, 500)
    for bad in ([0], [1.5], [10, 20]):
        with pytest.raises(ValueError):
            check_long(bad, 1, 500, 100, True, 16, 500)
    with pytest.raises(ValueError):
        check_long([1000], 1, 600, 100, True, 16, 500)   # a window past the DiT's max_len


class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device work before validation: {name}")


def _stub_ez(max_batch=4, max_length_s=10.0):
    """An EzAudio whose every device-facing member fails the test when touched; only the host-side attributes are real."""
    ez = object.__new__(EzAudio)
    ez.params = {"autoencoder": {"latent_sr": 50, "sr": 24000, "scale": 1.0, "shift": 0.0}}
    ez.max_length_s = max_length_s
    ez.unet = SimpleNamespace(_h=SimpleNamespace(desc=SimpleNamespace(max_batch=2 * max_batch, max_len=int(max_length_s * 50))))
    ez.autoencoder = _NoDevice()
    ez.noise_scheduler = _NoDevice()

    def enc(prompts):
        raise AssertionError("text encoder called before validation")
    ez.encode_text = enc
    return ez


@pytest.mark.parametrize("kw", [
    dict(text="rain", length=60, window_length=12),                               # window past max_length_s
    dict(text="rain", length=60, overlap=0),                                      # overlap below one frame
    dict(text="rain", length=60, overlap=0.01),                                   # overlap rounds to 0 frames
    dict(text="rain", length=60, overlap=6),                                      # overlap past half the window
    dict(text="rain", length=0),                                                  # empty clip
    dict(text="rain", length=-3),
    dict(text=["rain", "wind"], length=[30, 0.001]),                              # under one frame
    dict(text=["rain", "wind"], length=[30, 20, 10]),                             # one length per prompt
    dict(text=["rain", ""], length=30),                                           # empty and non-empty prompts mixed
    dict(text="rain", length=60),                                                 # 8 windows x 2 rows > 2 * max_batch (4)
    dict(text=["rain", "wind"], length=[30, 30], window_length=10, overlap=2),    # 2 x 4 windows x 2 = 16 rows > 8
    dict(text="rain", length=31, window_length=2, overlap=1),                    # many short windows
])
def test_generate_long_audio_validates_before_device_work(kw):
    with pytest.raises(ValueError):
        _stub_ez().generate_long_audio(**kw)


def test_generate_long_audio_row_capacity_message():
    with pytest.raises(ValueError, match="needs max_batch >= 8"):
        _stub_ez(max_batch=4).generate_long_audio("rain", length=60)


def test_decoder_receptive_field_hand_derived():
    # Perturb latent frame 0 and follow the reach (in samples of each stage's rate):
    #   input conv k 7:                            [-3, 3]
    #   stride 10: convT [i*10 - 5, i*10 + 14] -> [-35, 44];    residual units (k 7, dil 1 + 3 + 9) +-39 -> [-74, 83]
    #   stride 6:  [-74*6 - 3, 83*6 + 8]       -> [-447, 506];  +-39 -> [-486, 545]
    #   stride 4:  [-486*4 - 2, 545*4 + 5]     -> [-1946, 2185]; +-39 -> [-1985, 2224]
    #   stride 2:  [-1985*2 - 1, 2224*2 + 2]   -> [-3971, 4450]; +-39 -> [-4010, 4489]
    #   output conv k 7:                           [-4013, 4492] samples; frame 0 owns samples [0, 480)
    # left: ceil(4013 / 480) = 9 frames; right: ceil((4492 - 479) / 480) = 9 frames.
    assert decoder_receptive_field(synth.VAE_DECODER) == 9
    assert decoder_receptive_field(synth.tiny_vae(16)) == 9       # the tiny config only narrows the channels
    # one stage of stride 2: [-3, 3] -> [-7, 8] -> [-46, 47] -> [-49, 50] samples of a 2-sample frame: 25 frames either side
    assert decoder_receptive_field(dict(synth.VAE_DECODER, strides=[2])) == 25
