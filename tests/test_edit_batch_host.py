"""Batched editing, host side: the per-edit index arithmetic against the scalar path's formulas, broadcasting of the list form, length
validation with gt, and the C-ABI of the length-aware VAE."""
import ctypes
import os
import re

import pytest
import torch

from ezaudio_b200.api import _per_clip, edit_plan
from ezaudio_b200.inference import check_lengths


def _scalar_path(n_samples, sr, latent_sr, hop, boundary, mask_start, mask_length):
    """The arithmetic of EzAudio.editing_audio's scalar path, statement by statement, on plain numbers."""
    mask_end = mask_start + mask_length
    audio_length = n_samples / sr
    mask_start = min(mask_start, audio_length)
    n_total = n_samples
    if mask_end > audio_length:
        n_total += round((mask_end - audio_length) * sr)
        audio_length = n_total / sr
    boundary = min((mask_end - mask_start) / 2, boundary)
    start_idx = max(mask_start - boundary, 0)
    end_idx = min(mask_end + boundary, audio_length)
    mask_start -= start_idx
    mask_end -= start_idx
    s0, s1 = round(start_idx * sr), round(end_idx * sr)
    crop = s1 - s0
    L = (crop + (-crop) % hop) // hop                       # OobleckDecoder.encode pads the crop to whole latent frames
    mask = torch.zeros(L)
    mask[round(mask_start * latent_sr):round(mask_end * latent_sr)] = 1
    n = min(round((end_idx - start_idx) * sr), hop * L, n_total - s0)
    return n_total, s0, s1, L, mask, n


@pytest.mark.parametrize("n_samples,boundary,mask_start,mask_length", [
    (4 * 24000, 1, 1.5, 1.0),          # interior edit
    (3 * 24000, 0.4, 0.5, 0.6),        # boundary capped at half the mask
    (2 * 24000, 0.5, 1.6, 1.0),        # outpainting past the clip's end
    (2 * 24000 + 123, 2, 0.0, 0.37),   # crop clipped at the clip's start, ragged sample counts
    (24000, 0.25, 3.0, 0.5),           # mask wholly past the end
    (5 * 24000 + 7, 0.33, 4.9, 0.21),
])
def test_edit_plan_equals_the_scalar_path(n_samples, boundary, mask_start, mask_length):
    sr, latent_sr, hop = 24000, 50, 480
    p = edit_plan(n_samples, sr, latent_sr, hop, boundary, mask_start, mask_length)
    n_total, s0, s1, L, mask, n = _scalar_path(n_samples, sr, latent_sr, hop, boundary, mask_start, mask_length)
    assert (p["n_total"], p["s0"], p["s1"], p["frames"], p["n_paste"]) == (n_total, s0, s1, L, n)
    want = torch.zeros(L)
    want[p["m0"]:p["m1"]] = 1
    assert torch.equal(want, mask) and 0 <= p["m0"] <= p["m1"] <= L
    assert s0 + n <= n_total and n <= hop * L


def test_per_clip_broadcasts_scalars_and_checks_lists():
    num = (int, float)
    assert _per_clip("boundary", 1, 3, num) == [1, 1, 1]
    assert _per_clip("mask_start", [0.5, 1, 2], 3, num) == [0.5, 1, 2]
    assert _per_clip("gt_file", "a.wav", 2, (str,)) == ["a.wav", "a.wav"]
    for bad in ([1, 2], [1, 2, 3, 4], []):
        with pytest.raises(ValueError):
            _per_clip("mask_length", bad, 3, num)


def test_check_lengths_accepts_padded_gt_and_still_refuses_a_controlnet():
    gt = torch.zeros(3, 8, 10)
    assert check_lengths([5, 1, 10], 3, 10, gt=gt, padded_gt=True) == [5, 1, 10]
    with pytest.raises(NotImplementedError):   # without the caller's word that gt is padded like the batch
        check_lengths([5, 1, 10], 3, 10, gt=gt)
    for bad, B in (([0, 5, 5], 3), ([11, 5, 5], 3), ([5, 5], 3), ([2.5, 5, 5], 3)):
        with pytest.raises(ValueError):
            check_lengths(bad, B, 10, gt=gt, padded_gt=True)
    with pytest.raises(ValueError):   # gt is the padded batch
        check_lengths([5, 1, 9], 3, 10, gt=torch.zeros(3, 8, 9), padded_gt=True)
    with pytest.raises(NotImplementedError):
        check_lengths([5], 1, 10, gt=torch.zeros(1, 8, 10), controlnet=object(), padded_gt=True)


def test_library_exports_the_vae_lengths_abi():
    from ezaudio_b200 import _lib, build
    build.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "ezb200.h")).read()
    for name in ("ezb_vae_decode_lens", "ezb_vae_encode_lens"):
        assert hasattr(L, name) and name in _lib.EXPORTS and re.search(rf"\bint {name}\(", header), name
    assert _lib.lib().ezb_version() == 2
