"""Long edits on the host: the VAE encoder's receptive field (encode_tiled's halo) against the reach measured through the oracle's encoder
in fp64, the chunk layout tiled encodes and decodes share, the crop arithmetic of continuation and long-crop edits with their window
counts, and the validation editing_long_audio does before any device work."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from ezaudio_b200 import synth, weights
from ezaudio_b200.api import EzAudio, edit_plan
from ezaudio_b200.inference import check_long, window_plan
from ezaudio_b200.vae import decoder_receptive_field, encoder_receptive_field, tile_chunks
from oracle import ezaudio_oracle as O

HOP = 480


# ---------------------------------------------------------------- receptive field
def test_encoder_receptive_field_hand_derived():
    # The samples latent frame 0 reads, walked back from the latent end (strided conv: output o reads o*s - ceil(s/2) .. + 2s - 1):
    #   final conv k 3:                                  [-1, 1] frames
    #   stride 10 (pad 5): [-10 - 5, 10 - 5 + 19]    -> [-15, 24];       residual units (k 7, dil 1 + 3 + 9) +-39 -> [-54, 63]
    #   stride 6 (pad 3):  [-54*6 - 3, 63*6 - 3 + 11] -> [-327, 386];    +-39 -> [-366, 425]
    #   stride 4 (pad 2):  [-366*4 - 2, 425*4 - 2 + 7] -> [-1466, 1705]; +-39 -> [-1505, 1744]
    #   stride 2 (pad 1):  [-1505*2 - 1, 1744*2 - 1 + 3] -> [-3011, 3490]; +-39 -> [-3050, 3529]
    #   input conv k 7:                                  [-3053, 3532] samples; frame 0 owns samples [0, 480)
    # left: ceil(3053 / 480) = 7 frames; right: ceil((3532 - 479) / 480) = 7 frames.
    assert encoder_receptive_field(synth.VAE_ENCODER) == 7
    assert encoder_receptive_field(synth.tiny_vae_encoder(16)) == 7   # the tiny config only narrows the channels
    # one stage of stride 2: [-1, 1] -> [-3, 4] -> [-42, 43] -> [-45, 46] samples of a 2-sample frame: 23 frames either side
    assert encoder_receptive_field(dict(synth.VAE_ENCODER, strides=[2])) == 23


def test_encoder_receptive_field_matches_the_oracle_reach():
    """Perturb one sample (the first and last of a frame mid-clip, and the clip's first and last) through the oracle's encoder in fp64 and
    read which latent frames of the mean change: exactly the frames f whose read span [f * hop - 3053, f * hop + 3532] (derived above)
    holds the sample, clipped to the clip; the widest reach in frames is the derived field."""
    cfg = synth.tiny_vae_encoder(16)
    h = encoder_receptive_field(cfg)
    sd = {k: v.double() for k, v in weights.synthetic_state_dict(weights.vae_encoder_param_shapes(cfg), 6).items()}
    n = 24
    audio = torch.randn(1, 1, n * HOP, generator=torch.Generator().manual_seed(5), dtype=torch.float64) * 0.3
    with torch.no_grad():
        base = O.vae_encode(sd, audio, strides=tuple(cfg["strides"]))
        reach = 0
        for i in (0, HOP - 1, 11 * HOP, 11 * HOP + HOP - 1, n * HOP - HOP, n * HOP - 1):
            a = audio.clone()
            a[0, 0, i] += 0.5
            d = (O.vae_encode(sd, a, strides=tuple(cfg["strides"])) - base)[0].abs().amax(0)
            changed = torch.nonzero(d > 0).flatten().tolist()
            want = list(range(max(0, -(-(i - 3532) // HOP)), min(n - 1, (i + 3053) // HOP) + 1))
            assert changed == want, (i, changed, want)
            q = i // HOP
            reach = max(reach, q - changed[0], changed[-1] - q)
    assert reach == h


# ---------------------------------------------------------------- the shared chunk layout
def _decode_chunks_as_before(host, M, h):
    """decode_tiled's chunk list as the decoder wrote it inline before tile_chunks existed."""
    core = M - 2 * h
    chunks = []
    for b, n in enumerate(host):
        for c0 in range(0, n, core if n > M else n):
            c1 = min(n, c0 + core) if n > M else n
            chunks.append((b, max(0, c0 - h), min(n, c1 + h), c0, c1))
    return chunks


@pytest.mark.parametrize("lens,M,h", [([150], 40, 9), ([150, 61, 23], 40, 9), ([1], 40, 9), ([40, 41, 22, 23], 40, 9),
                                      ([3000, 1750, 500, 499, 501], 500, 7), ([1750], 100, 7), ([87, 86, 300], 100, 7), ([5], 3, 1)])
def test_tile_chunks_cover_every_clip(lens, M, h):
    chunks = tile_chunks(lens, M, h)
    if M == 40 and h == 9:   # the cases of the tiled decode's GPU test: unchanged
        assert chunks == _decode_chunks_as_before(lens, M, h)
    for b, n in enumerate(lens):
        mine = [c for c in chunks if c[0] == b]
        cover = np.zeros(n, dtype=int)
        for _, s, e, c0, c1 in mine:
            assert 0 <= s <= c0 < c1 <= e <= n             # the halo never crosses the clip's ends
            assert e - s <= M                              # every chunk fits the workspace
            if c0 > 0:
                assert c0 - s == min(h, c0)                # an inner edge carries the halo, up to the clip's end
            if c1 < n:
                assert e - c1 == min(h, n - c1)
            cover[c0:c1] += 1
        assert (cover == 1).all(), b                       # the cores tile the clip exactly
        assert [c[3] for c in mine] == sorted(c[3] for c in mine)
        if n <= M:
            assert mine == [(b, 0, n, 0, n)]
    assert [c[0] for c in chunks] == sorted(c[0] for c in chunks)


def test_tile_chunks_examples_and_refusal():
    assert tile_chunks([150], 40, 9) == [(0, 0, 31, 0, 22), (0, 13, 53, 22, 44), (0, 35, 75, 44, 66), (0, 57, 97, 66, 88),
                                         (0, 79, 119, 88, 110), (0, 101, 141, 110, 132), (0, 123, 150, 132, 150)]
    assert tile_chunks([1750], 500, 7)[:2] == [(0, 0, 493, 0, 486), (0, 479, 979, 486, 972)]
    with pytest.raises(ValueError):
        tile_chunks([100], 18, 9)   # no core left inside the halos
    assert decoder_receptive_field(synth.VAE_DECODER) == 9 and encoder_receptive_field(synth.VAE_ENCODER) == 7


# ---------------------------------------------------------------- crop arithmetic
def test_continuation_plan():
    """A 10-s clip continued by 30 s with 5 s of context: a 35-s crop of 1750 frames, 5 windows, 10 rows under guidance."""
    p = edit_plan(10 * 24000, 24000, 50, HOP, 5, 10, 30)
    assert p == dict(n_total=40 * 24000, s0=5 * 24000, s1=40 * 24000, frames=1750, m0=250, m1=1750, n_paste=35 * 24000)
    assert window_plan(p["frames"], 500, 100) == [(0, 500), (400, 500), (800, 500), (1200, 500), (1250, 500)]
    with pytest.raises(ValueError, match="needs max_batch >= 5"):
        check_long([p["frames"]], 1, 500, 100, True, 8, 500)
    _, _, windows = check_long([p["frames"]], 1, 500, 100, True, 10, 500)
    assert len(windows) == 5
    # by 20 s and by 50 s (the measured cases): 25-s and 55-s crops
    p20, p50 = edit_plan(10 * 24000, 24000, 50, HOP, 5, 10, 20), edit_plan(10 * 24000, 24000, 50, HOP, 5, 10, 50)
    assert (p20["frames"], p20["m0"], p20["m1"], p20["n_total"]) == (1250, 250, 1250, 30 * 24000)
    assert (p50["frames"], p50["m0"], p50["m1"], p50["n_total"]) == (2750, 250, 2750, 60 * 24000)
    assert len(window_plan(1250, 500, 100)) == 3 and len(window_plan(2750, 500, 100)) == 7
    check_long([2750], 1, 500, 100, True, 16, 500)   # max_batch=8 holds the 55-s crop


def test_long_crop_inside_a_take():
    """Regenerating 20 s in the middle of a 2-minute take with 5 s of context: a 30-s crop, the clip's length unchanged."""
    p = edit_plan(120 * 24000, 24000, 50, HOP, 5, 50, 20)
    assert p == dict(n_total=120 * 24000, s0=45 * 24000, s1=75 * 24000, frames=1500, m0=250, m1=1250, n_paste=30 * 24000)
    assert len(window_plan(1500, 500, 100)) == 4
    with pytest.raises(ValueError, match="needs max_batch >= 4"):
        check_long([1500], 1, 500, 100, True, 6, 500)
    with pytest.raises(ValueError, match="needs max_batch >= 2"):   # no guidance: one row per window
        check_long([1500], 1, 500, 100, False, 2, 500)
    # a crop that does not end on a whole hop: the last frame is zero-padded, n_paste stops at the crop
    q = edit_plan(100003, 24000, 50, HOP, 0.5, 1.0, 3.0)
    assert q["frames"] == -(-(q["s1"] - q["s0"]) // HOP) and q["n_paste"] == q["s1"] - q["s0"] <= q["frames"] * HOP


# ---------------------------------------------------------------- validation before device work
class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device work before validation: {name}")


class _HopOnly(_NoDevice):
    hop = HOP


def _stub_ez(max_batch=4, max_length_s=10.0):
    """An EzAudio whose every device-facing member fails the test when touched; only the host-side attributes are real."""
    ez = object.__new__(EzAudio)
    ez.params = {"autoencoder": {"latent_sr": 50, "sr": 24000, "scale": 1.0, "shift": 0.0}}
    ez.max_length_s = max_length_s
    ez.device = "cuda"
    ez.unet = SimpleNamespace(_h=SimpleNamespace(desc=SimpleNamespace(max_batch=2 * max_batch, max_len=int(max_length_s * 50))))
    ez.autoencoder = SimpleNamespace(decoder=_HopOnly())
    ez.noise_scheduler = _NoDevice()

    def enc(prompts):
        raise AssertionError("text encoder called before validation")
    ez.encode_text = enc
    return ez


_TEN = np.zeros(10 * 24000, np.float32)
_ARGS = dict(text="thunder", boundary=5, gt_file=_TEN, mask_start=10, mask_length=30)


@pytest.mark.parametrize("kw", [
    dict(_ARGS),                                                                          # 5 windows x 2 rows > 2 * max_batch (4)
    dict(_ARGS, window_length=12),                                                        # window past max_length_s
    dict(_ARGS, overlap=0),                                                               # overlap below one frame
    dict(_ARGS, overlap=6),                                                               # overlap past half the window
    dict(_ARGS, mask_length=0),
    dict(_ARGS, mask_start=-1),
    dict(_ARGS, boundary=-1),
    dict(_ARGS, gt_file=np.zeros(0, np.float32)),                                         # empty clip
    dict(_ARGS, gt_file=np.zeros((2, 100), np.float32)),                                  # not mono
    dict(_ARGS, text=["thunder", ""], mask_length=2),                                     # empty and non-empty prompts mixed
    dict(_ARGS, text=["thunder", "rain"], mask_length=[2, 3, 4]),                         # one value per prompt
    dict(_ARGS, text=["thunder", "rain"], mask_length=2, random_seed=[1, 2, 3]),
    dict(_ARGS, text=[], mask_length=2),
])
def test_editing_long_audio_validates_before_device_work(kw):
    with pytest.raises(ValueError):
        _stub_ez().editing_long_audio(**kw)


def test_editing_long_audio_row_capacity_message():
    with pytest.raises(ValueError, match="needs max_batch >= 5"):
        _stub_ez(max_batch=4).editing_long_audio(**_ARGS)
    with pytest.raises(ValueError, match="needs max_batch >= 8"):   # two edits: 5 + 3 windows
        _stub_ez(max_batch=4).editing_long_audio(["thunder", "rain"], 5, _TEN, 10, [30, 15])
