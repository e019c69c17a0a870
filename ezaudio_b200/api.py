"""Public API -- same classes, method signatures, defaults and return types as the reference
(api/ezaudio.py:31-207 `EzAudio`, api/controlnet.py:31-161 `EzAudio_ControlNet`), hosted on the CUDA library.

Extensions (all optional, keyword-only): `text` may be a list of prompts (batched; returns a list of waveforms; for `editing_audio`
the clip, mask, boundary and seed arguments then list one value per prompt and the edits, whatever their crop lengths, run as one batch);
`text_encoder=` injects a callable `(list[str]) -> (emb (B,Lc,ctx) , mask (B,Lc))` standing in for flan-T5 (the image has no
network, so T5 weights cannot be fetched -- BASELINE configs use cached embeddings); `ckpt_path="synthetic:<seed>"` builds
the deterministic random checkpoint of `weights.synthetic_state_dict` instead of reading a file.
"""
from __future__ import annotations

import os
import random
from typing import Callable, List, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib, config, post, weights
from ._lib import EzbError
from .dit import DiTControlNet, MaskDiT
from .inference import (check_long, check_loop, check_timeline, inference, make_generators, sample_long_latents, sample_loop_latents,
                        sample_timeline_latents, scale_shift_re)
from .scheduler import DDIMScheduler, start_index
from .vae import Autoencoder, OobleckDecoder

MAX_SEED = np.iinfo(np.int32).max


class SyntheticTextEncoder:
    """Cached-T5 stand-in (SURVEY 8d): deterministic N(0,1) embeddings keyed by the prompt string; "" -> only the first
    (EOS) token is valid, like the tokenizer's output for the empty negative prompt."""

    def __init__(self, ctx_dim: int, max_length: int = 100):
        self.ctx_dim, self.max_length = ctx_dim, max_length

    def __call__(self, prompts: Sequence[str]):
        embs, masks = [], []
        for p in prompts:
            seed = int.from_bytes(p.encode()[:8].ljust(8, b"\0"), "little") % (2 ** 31) + 7 * len(p)
            g = torch.Generator().manual_seed(seed)
            embs.append(torch.randn(1, self.max_length, self.ctx_dim, generator=g))
            n = 1 if p == "" else min(self.max_length, 2 + len(p.split()) + len(p) // 6)
            m = torch.zeros(1, self.max_length, dtype=torch.bool)
            m[0, :n] = True
            masks.append(m)
        return torch.cat(embs, 0), torch.cat(masks, 0)


def _load_audio(path: str, sr: int) -> np.ndarray:
    """librosa.load(path, sr=sr) stand-in (mono float32, resampled), api/ezaudio.py:146.  librosa / soundfile / torchcodec are
    not in this image: WAV is read with scipy, resampling is polyphase (scipy.signal.resample_poly)."""
    from math import gcd

    from scipy.io import wavfile
    from scipy.signal import resample_poly
    fs, data = wavfile.read(path)
    if data.dtype.kind == "i":
        data = data.astype(np.float32) / float(np.iinfo(data.dtype).max + 1)
    elif data.dtype.kind == "u":
        data = (data.astype(np.float32) - 128.0) / 128.0
    data = data.astype(np.float32)
    if data.ndim == 2:
        data = data.mean(axis=1)
    if fs != sr:
        g = gcd(int(fs), int(sr))
        data = resample_poly(data, sr // g, fs // g).astype(np.float32)
    return data


class HashTokenizer:
    """Offline stand-in for T5Tokenizer (no sentencepiece vocabulary on disk, no network): words -> stable ids in [2, vocab), EOS = 1,
    pad = 0; same call signature / outputs as the tokenizer call at src/inference.py:39-41."""

    def __init__(self, vocab_size: int = 32128):
        self.vocab_size = vocab_size

    def __call__(self, text, max_length=100, padding="max_length", truncation=True, return_tensors="pt"):
        from types import SimpleNamespace
        import zlib
        text = [text] if isinstance(text, str) else list(text)
        ids = torch.zeros(len(text), max_length, dtype=torch.long)
        mask = torch.zeros(len(text), max_length, dtype=torch.long)
        for i, t in enumerate(text):
            toks = [2 + zlib.crc32(w.encode()) % (self.vocab_size - 2) for w in t.lower().split()][: max_length - 1] + [1]
            ids[i, : len(toks)] = torch.tensor(toks)
            mask[i, : len(toks)] = 1
        return SimpleNamespace(input_ids=ids, attention_mask=mask)


class NativeTextEncoder:
    """prompts -> (embeddings, mask) with a tokenizer and the native T5 encoder (ezaudio_b200.t5), i.e. src/inference.py:38-50."""

    def __init__(self, tokenizer, encoder, max_length: int = 100, device="cuda"):
        self.tokenizer, self.encoder, self.max_length, self.device = tokenizer, encoder, max_length, device

    def __call__(self, prompts: Sequence[str]):
        tb = self.tokenizer(list(prompts), max_length=self.max_length, padding="max_length", truncation=True, return_tensors="pt")
        ids, mask = tb.input_ids.to(self.device), tb.attention_mask.to(self.device).bool()
        return self.encoder(input_ids=ids, attention_mask=mask).last_hidden_state, mask


def save_wav(path: str, audio, sr: int = 24000) -> None:
    """soundfile.write(path, audio, sr) stand-in for the step after the path (t2a_demo.py:13,20, controlnet_demo.py:15): float32 mono WAV
    written with scipy (soundfile is not in this image).  Accepts the (sr, ndarray) tuple the API methods return as `audio`."""
    from scipy.io import wavfile
    if isinstance(audio, tuple):
        sr, audio = audio
    a = np.asarray(audio, dtype=np.float32).reshape(-1)
    if not np.isfinite(a).all():
        raise ValueError("save_wav: non-finite samples")
    wavfile.write(path, int(sr), a)


def _load_t5(name: str, device, precision: str = "bf16", max_length: int = 100):
    """api/ezaudio.py:78-79.  transformers is used for the tokenizer and for reading the checkpoint (CPU, I/O only); the encoder that runs
    is the native one.  Returns (None, None) when the checkpoint is not on disk (there is no network here)."""
    try:
        from transformers import T5EncoderModel as HFT5
        from transformers import T5Tokenizer
        tok = T5Tokenizer.from_pretrained(name, local_files_only=True)
        hf = HFT5.from_pretrained(name, local_files_only=True)
    except Exception:
        return None, None
    from .t5 import T5EncoderModel
    c = hf.config
    cfg = dict(vocab_size=c.vocab_size, d_model=c.d_model, d_kv=c.d_kv, num_heads=c.num_heads, d_ff=c.d_ff, num_layers=c.num_layers,
               relative_attention_num_buckets=c.relative_attention_num_buckets,
               relative_attention_max_distance=getattr(c, "relative_attention_max_distance", 128), layer_norm_epsilon=c.layer_norm_epsilon,
               feed_forward_proj=c.feed_forward_proj)
    enc = T5EncoderModel(cfg, precision=precision, max_batch=8, max_len=max_length, device=device).load_state_dict(hf.state_dict())
    return tok, enc


def _state_dict(path, shapes, key):
    if isinstance(path, str) and path.startswith("synthetic"):
        seed = int(path.split(":")[1]) if ":" in path else 0
        return weights.synthetic_state_dict(shapes, seed)
    if path is None or not os.path.exists(path):
        raise FileNotFoundError(f"checkpoint {path!r} not found (no network here: pass a local file or 'synthetic:<seed>')")
    sd = torch.load(path, map_location="cpu")
    return sd[key] if key in sd else sd


class _Base:
    def _text_embeds(self, prompts: List[str], neg: List[str]):
        if self.encode_text is None:
            raise RuntimeError("no text encoder available (flan-T5 weights are not on disk and there is no network); pass "
                               "text_encoder=<callable> to the constructor, e.g. ezaudio_b200.api.SyntheticTextEncoder")
        e, m = self.encode_text(prompts)
        ue, um = self.encode_text(neg)
        return e, m, ue, um

    def _make_text_encoder(self, text_encoder, params, device):
        self.tokenizer = self.text_encoder = None
        if text_encoder is not None:
            return text_encoder
        ml = params["text_encoder"]["max_length"]
        tok, enc = _load_t5(params["text_encoder"]["model"], device, max_length=ml)
        if tok is None:
            return None
        self.tokenizer, self.text_encoder = tok, enc
        return NativeTextEncoder(tok, enc, ml, device)


def edit_plan(n_samples: int, sr: int, latent_sr: int, hop: int, boundary, mask_start, mask_length) -> dict:
    """The index arithmetic of one edit (api/ezaudio.py:140-203), on the host: a clip of n_samples samples, the mask [mask_start,
    mask_start + mask_length) seconds regenerated with `boundary` seconds of context on either side.
    n_total: samples of the output clip (the input zero-padded to the mask's end when outpainting); [s0, s1): samples of the crop that is
    encoded; frames: its latent frames (whole hops, the last one zero-padded); [m0, m1): latent frames regenerated; n_paste: samples of the
    decoded crop pasted back at s0."""
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
    frames = -(-(s1 - s0) // hop)
    m0, m1 = min(round(mask_start * latent_sr), frames), min(round(mask_end * latent_sr), frames)
    n_paste = min(round((end_idx - start_idx) * sr), frames * hop, n_total - s0)
    return dict(n_total=n_total, s0=s0, s1=s1, frames=frames, m0=m0, m1=m1, n_paste=n_paste)


def _per_clip(name: str, value, n: int, scalar_types) -> list:
    """One value per clip: a scalar is repeated, a list must hold n."""
    if isinstance(value, scalar_types):
        return [value] * n
    value = list(value)
    if len(value) != n:
        raise ValueError(f"{name} lists one value per prompt: got {len(value)} for {n} prompts")
    return value


def _vae_precision(precision: str) -> str:
    """The VAE (and T5) have no FP8 mode: precision="fp8" builds them in "bf16"."""
    return "bf16" if precision == "fp8" else precision


class EzAudio(_Base):
    """api/ezaudio.py:31.

    precision: "bf16" (default, throughput), "bf16x3" (fp32-grade parity) or "fp8": the DiT's self-attention QKV and GEGLU up-projections
    run on H100 FP8 tensor cores (e4m3 operands with per-row scales, fp32 accumulation), everything else as in "bf16"; the VAE and the
    text encoder run in "bf16".  See DESIGN.md section 3 for its accuracy."""

    def __init__(self, model_name, ckpt_path=None, vae_path=None, device="cuda", *, text_encoder: Optional[Callable] = None,
                 precision: str = "bf16", max_batch: int = 4, max_length_s: float = 10.0, config_path=None, vae_config_path=None):
        self.device = device
        self.params = config.load_params(model_name, config_path)
        p = self.params
        latent_sr = p["autoencoder"]["latent_sr"]
        max_len = int(round(max_length_s * latent_sr))
        self.max_length_s = float(max_length_s)   # longest clip (seconds) the workspace holds; the batching front-end caps padding at it
        self.noise_scheduler = DDIMScheduler(**p["diff"])
        self.unet = MaskDiT(precision=precision, max_batch=2 * max_batch, max_len=max_len, max_ctx_len=p["text_encoder"]["max_length"],
                            max_timesteps=1000, device=device, **p["model"])
        self.unet.load_state_dict(_state_dict(ckpt_path, weights.dit_param_shapes(p["model"]), "model"))
        dcfg, ecfg = config.load_vae_decoder_config(vae_config_path), config.load_vae_encoder_config(vae_config_path)
        dec = OobleckDecoder(precision=_vae_precision(precision), max_batch=max_batch, max_latent_len=max_len, device=device, encoder_cfg=ecfg,
                             **dcfg)
        vshapes = dict(weights.vae_decoder_param_shapes(dcfg))
        vshapes.update(weights.vae_encoder_param_shapes(ecfg))
        vsd = _state_dict(vae_path, vshapes, "state_dict")
        vsd = {(k[len("autoencoder."):] if k.startswith("autoencoder.") else k): v for k, v in vsd.items()}  # stable_vae/__init__.py:25-31
        dec.load_state_dict(vsd)
        self.autoencoder = Autoencoder(dec)
        self.encode_text = self._make_text_encoder(text_encoder, p, device)

    def generate_audio(self, text, length=10, guidance_scale=5, guidance_rescale=0.75, ddim_steps=100, eta=1, random_seed=None,
                       randomize_seed=False, *, pad_length=None):
        """api/ezaudio.py:101-130.  Returns (sr, float32 waveform); a list of prompts returns (sr, [waveforms]).
        With a list of prompts, `length` may list one length (seconds) per prompt: the prompts run as one batch padded to `pad_length`
        seconds (default: the longest; at most max_length_s), and waveform b has hop * frames(length[b]) samples, equal to that prompt's
        solo call with the same seed (pass one seed per prompt in `random_seed` to make the batch reproduce solo calls)."""
        batched = not isinstance(text, str)
        prompts = list(text) if batched else [text]
        latent_sr = self.params["autoencoder"]["latent_sr"]
        if isinstance(length, (list, tuple)):
            return self._generate_varlen(prompts, batched, length, pad_length, guidance_scale, guidance_rescale, ddim_steps, eta, random_seed,
                                         randomize_seed)
        if pad_length is not None:
            raise ValueError("pad_length applies to a list of per-prompt lengths")
        length = length * latent_sr
        if all(t == "" for t in prompts):
            guidance_scale = None
            print("empyt input")
        if randomize_seed:
            random_seed = random.randint(0, MAX_SEED)
        embeds = self._text_embeds(prompts, [""])
        pred = inference(self.autoencoder, self.unet, None, None, None, None, self.params, self.noise_scheduler, prompts, None,
                         int(length), guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, self.device, text_embeds=embeds)
        pred = pred.cpu().numpy()
        sr = self.params["autoencoder"]["sr"]
        if batched:
            return sr, [pred[i, 0] for i in range(pred.shape[0])]
        return sr, pred.squeeze(0).squeeze(0)

    def _generate_varlen(self, prompts, batched, length, pad_length, guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, randomize_seed):
        latent_sr = self.params["autoencoder"]["latent_sr"]
        if len(length) != len(prompts):
            raise ValueError(f"length lists one value per prompt: got {len(length)} for {len(prompts)} prompts")
        frames = [int(v * latent_sr) for v in length]
        max_frames = int(round(self.max_length_s * latent_sr))
        L = max(frames) if pad_length is None else int(pad_length * latent_sr)
        if pad_length is not None and pad_length > self.max_length_s:
            raise ValueError(f"pad_length {pad_length} s exceeds max_length_s {self.max_length_s} s")
        if L > max_frames or any(f < 1 or f > L for f in frames):
            raise ValueError(f"lengths {list(length)} s must be positive and fit the padded length ({L} frames, at most {max_frames})")
        if all(t == "" for t in prompts):
            guidance_scale = None
            print("empyt input")
        if randomize_seed:
            random_seed = random.randint(0, MAX_SEED)
        embeds = self._text_embeds(prompts, [""])
        wavs = inference(self.autoencoder, self.unet, None, None, None, None, self.params, self.noise_scheduler, prompts, None, L, guidance_scale,
                         guidance_rescale, ddim_steps, eta, random_seed, self.device, text_embeds=embeds, lengths=frames)
        sr = self.params["autoencoder"]["sr"]
        out = [w[0].cpu().numpy() for w in wavs]
        return (sr, out) if batched else (sr, out[0])

    def editing_audio(self, text, boundary, gt_file, mask_start, mask_length, guidance_scale=3.5, guidance_rescale=0, ddim_steps=100,
                      eta=1, random_seed=None, randomize_seed=False, *, pad_length=None):
        """api/ezaudio.py:132-207 (crop -> VAE encode -> masked sampling -> paste -> decode -> splice).
        With a list of prompts, `gt_file` (paths or waveforms), `mask_start`, `mask_length`, `boundary` and `random_seed` list one value per
        prompt (a scalar applies to all) and the call returns (sr, [waveforms]).  The edits run as one batch -- one VAE encode, one sampling
        loop, one decode -- padded to the longest crop, or to `pad_length` seconds (at most max_length_s) so that batches of different crops
        reuse one captured graph.  Each waveform equals the scalar call of that edit with its seed, the calls made in list order (they
        draw the bottleneck noise from the global RNG in that order)."""
        if isinstance(text, (list, tuple)):
            return self._editing_batch(list(text), boundary, gt_file, mask_start, mask_length, guidance_scale, guidance_rescale, ddim_steps, eta,
                                       random_seed, randomize_seed, pad_length)
        if pad_length is not None:
            raise ValueError("pad_length applies to a list of edits")
        sr = self.params["autoencoder"]["sr"]
        if text == "":
            guidance_scale = None
            print("empyt input")
        mask_end = mask_start + mask_length
        gt_raw = _load_audio(gt_file, sr) if isinstance(gt_file, str) else np.asarray(gt_file, dtype=np.float32)
        audio_length = len(gt_raw) / sr
        mask_start = min(mask_start, audio_length)
        n_total = len(gt_raw)
        if mask_end > audio_length:  # outpainting: zero padding up to the end of the mask
            n_total += round((mask_end - audio_length) * sr)
            audio_length = n_total / sr
        # the clip goes to the device ONCE: peak-normalise + pad there (ezb_wave_prepare = api/ezaudio.py:147,152-154 on the device)
        output_audio = post.prepare_wave(torch.from_numpy(gt_raw).to(self.device).unsqueeze(0), n_total, normalize=True)[0]
        boundary = min((mask_end - mask_start) / 2, boundary)
        start_idx = max(mask_start - boundary, 0)
        end_idx = min(mask_end + boundary, audio_length)
        mask_start -= start_idx
        mask_end -= start_idx
        s0, s1 = round(start_idx * sr), round(end_idx * sr)
        gt_t = output_audio[s0:s1].clone().view(1, 1, -1)
        gt_latent = self.autoencoder(audio=gt_t)  # OobleckEncoder + stochastic VAE bottleneck (global RNG, bottleneck.py:69)
        B, D, L = gt_latent.shape
        gt_mask = torch.zeros(B, D, L, device=self.device)
        latent_sr = self.params["autoencoder"]["latent_sr"]
        gt_mask[:, :, round(mask_start * latent_sr):round(mask_end * latent_sr)] = 1
        gt_mask = gt_mask.bool()
        if randomize_seed:
            random_seed = random.randint(0, MAX_SEED)
        embeds = self._text_embeds([text], [""])
        pred = inference(self.autoencoder, self.unet, gt_latent, gt_mask, None, None, self.params, self.noise_scheduler, [text], None, L,
                         guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, self.device, text_embeds=embeds)
        # trim + paste on the device (ezb_wave_splice = api/ezaudio.py:198-203), one download of the finished clip
        n = min(round((end_idx - start_idx) * sr), pred.shape[-1], n_total - s0)
        post.splice_wave(output_audio, pred[0, 0], s0, n)
        return sr, output_audio.cpu().numpy()

    def _editing_batch(self, prompts, boundary, gt_file, mask_start, mask_length, guidance_scale, guidance_rescale, ddim_steps, eta, random_seed,
                       randomize_seed, pad_length):
        sr, latent_sr = self.params["autoencoder"]["sr"], self.params["autoencoder"]["latent_sr"]
        dec = self.autoencoder.decoder
        B, hop = len(prompts), dec.hop
        # ---- everything is checked on the host before any device work
        if B < 1 or B > dec.max_batch:
            raise ValueError(f"{B} edits in one call: 1..{dec.max_batch} (max_batch) fit the workspace")
        num = (int, float, np.integer, np.floating)
        files = _per_clip("gt_file", gt_file, B, (str, np.ndarray))
        starts, lengths_s = _per_clip("mask_start", mask_start, B, num), _per_clip("mask_length", mask_length, B, num)
        bounds = _per_clip("boundary", boundary, B, num)
        if randomize_seed:
            seeds = [random.randint(0, MAX_SEED) for _ in range(B)]
        elif random_seed is None:
            seeds = None
        else:
            seeds = [int(v) for v in _per_clip("random_seed", random_seed, B, num)]
        empty = [t == "" for t in prompts]
        if any(empty) and not all(empty):
            raise ValueError("empty prompts run without guidance: they cannot share a batch with non-empty ones")
        if all(empty):
            guidance_scale = None
            print("empyt input")
        if any(v < 0 for v in starts) or any(v <= 0 for v in lengths_s) or any(v < 0 for v in bounds):
            raise ValueError("mask_start and boundary must be >= 0 and mask_length > 0 for every edit")
        raws = [_load_audio(f, sr) if isinstance(f, str) else np.asarray(f, dtype=np.float32) for f in files]
        if any(r.ndim != 1 or len(r) < 1 for r in raws):
            raise ValueError("every gt_file must be a non-empty mono waveform")
        plans = [edit_plan(len(r), sr, latent_sr, hop, bd, ms, ml) for r, bd, ms, ml in zip(raws, bounds, starts, lengths_s)]
        frames = [p["frames"] for p in plans]
        max_frames = int(round(self.max_length_s * latent_sr))
        if pad_length is not None and pad_length > self.max_length_s:
            raise ValueError(f"pad_length {pad_length} s exceeds max_length_s {self.max_length_s} s")
        L = max(frames) if pad_length is None else int(pad_length * latent_sr)
        if min(frames) < 1 or max(frames) > L or L > max_frames:
            raise ValueError(f"crops of {frames} latent frames must be non-empty and fit the padded length ({L} frames, at most {max_frames}: "
                             f"max_length_s {self.max_length_s} s)")
        # ---- per clip: normalise + pad on the device, crop into the padded batch
        outs, crops = [], torch.zeros(B, 1, L * hop, device=self.device)
        for b, (r, p) in enumerate(zip(raws, plans)):
            o = post.prepare_wave(torch.from_numpy(r).to(self.device).unsqueeze(0), p["n_total"], normalize=True)[0]
            crops[b, 0, :p["s1"] - p["s0"]] = o[p["s0"]:p["s1"]]
            outs.append(o)
        gt_latent = self.autoencoder(audio=crops, lengths=frames)   # clip b's bottleneck noise: (1, C, frames[b]) from the global RNG, in order
        gt_mask = torch.zeros(B, gt_latent.shape[1], L, device=self.device)
        for b, p in enumerate(plans):
            gt_mask[b, :, p["m0"]:p["m1"]] = 1
            gt_mask[b, :, frames[b]:] = 1
        embeds = self._text_embeds(prompts, [""])
        wavs = inference(self.autoencoder, self.unet, gt_latent, gt_mask.bool(), None, None, self.params, self.noise_scheduler, prompts, None, L,
                         guidance_scale, guidance_rescale, ddim_steps, eta, seeds, self.device, text_embeds=embeds, lengths=frames, padded_gt=True)
        for o, w, p in zip(outs, wavs, plans):
            post.splice_wave(o, w[0], p["s0"], p["n_paste"])
        return sr, [o.cpu().numpy() for o in outs]

    def generate_long_audio(self, text, length, window_length=10, overlap=2, guidance_scale=5, guidance_rescale=0.75, ddim_steps=100, eta=1,
                            random_seed=None, randomize_seed=False):
        """Text-to-audio past the denoiser's trained length (`inference.sample_long_latents`): at every step the clip's latent is cut into
        windows of `window_length` seconds overlapping by `overlap` seconds, all windows are denoised as one batch and their predictions
        are crossfaded back into one; the long latent is then decoded in tiles (`OobleckDecoder.decode_tiled`).  No DiT call sees more than
        one window, and no workspace grows with `length`.  `text` is a prompt or a list of prompts, `length` (seconds) one value or one per
        prompt; seeds as in generate_audio (an int gives prompt b seed + b, a list one seed per prompt).  Returns (sr, waveform) or
        (sr, [waveforms]) with hop * int(length * latent_sr) samples each.  A clip no longer than the window equals generate_audio's
        with the same seed and frame count, bit for bit.  The windows (x 2 with guidance) must fit the DiT's 2 * max_batch rows."""
        batched = not isinstance(text, str)
        prompts = list(text) if batched else [text]
        B = len(prompts)
        latent_sr = self.params["autoencoder"]["latent_sr"]
        # ---- everything is checked on the host before any device work
        num = (int, float, np.integer, np.floating)
        frames = [int(v * latent_sr) for v in _per_clip("length", length, B, num)]
        if B < 1 or any(f < 1 for f in frames):
            raise ValueError(f"every length must be positive (at least one latent frame), got {length}")
        if window_length > self.max_length_s:
            raise ValueError(f"window_length {window_length} s exceeds max_length_s {self.max_length_s} s")
        window, hop_over = int(window_length * latent_sr), int(overlap * latent_sr)
        empty = [t == "" for t in prompts]
        if any(empty) and not all(empty):
            raise ValueError("empty prompts run without guidance: they cannot share a batch with non-empty ones")
        if all(empty):
            guidance_scale = None
            print("empyt input")
        check_long(frames, B, window, hop_over, bool(guidance_scale), int(self.unet._h.desc.max_batch), int(self.unet._h.desc.max_len))
        if randomize_seed:
            random_seed = random.randint(0, MAX_SEED)
        text_emb, mask, uemb, umask = self._text_embeds(prompts, [""])
        lat = sample_long_latents(self.unet, self.noise_scheduler, text_emb, mask, uemb, umask, frames, window, hop_over, guidance_scale,
                                  guidance_rescale, ddim_steps, eta, random_seed)
        p = self.params["autoencoder"]
        wav = self.autoencoder.decoder.decode_tiled(scale_shift_re(lat, p["scale"], p["shift"]), lengths=frames)
        hop = self.autoencoder.decoder.hop
        out = [wav[b, 0, :hop * n].cpu().numpy() for b, n in enumerate(frames)]
        return (p["sr"], out) if batched else (p["sr"], out[0])

    def generate_loop_audio(self, text, length, window_length=10, overlap=2, guidance_scale=5, guidance_rescale=0.75, ddim_steps=100, eta=1,
                            random_seed=None, randomize_seed=False):
        """Seamless loops: audio whose last sample runs on into its first, for ambience and effect beds played on repeat.  The latent is
        denoised as a circle (`inference.sample_loop_latents`): windows of `window_length` seconds overlapping by at least `overlap` seconds
        wrap around the loop's end, and all of them move by a golden-ratio stride at every step, so the seam is denoised in context like
        any other frame.  The loop is then decoded with halos that wrap around (`OobleckDecoder.decode_loop`).  Prompts, lengths (seconds,
        one value or one per prompt) and seeds are as in generate_long_audio.  Returns (sr, waveform) or (sr, [waveforms]) with
        hop * int(length * latent_sr) samples each.  The windows (x 2 with guidance) must fit the DiT's 2 * max_batch rows."""
        batched = not isinstance(text, str)
        prompts = list(text) if batched else [text]
        B = len(prompts)
        latent_sr = self.params["autoencoder"]["latent_sr"]
        # ---- everything is checked on the host before any device work
        num = (int, float, np.integer, np.floating)
        frames = [int(v * latent_sr) for v in _per_clip("length", length, B, num)]
        if B < 1 or any(f < 2 for f in frames):
            raise ValueError(f"every loop must be at least two latent frames ({2 / latent_sr} s) long, got {length}")
        if window_length > self.max_length_s:
            raise ValueError(f"window_length {window_length} s exceeds max_length_s {self.max_length_s} s")
        window, hop_over = int(window_length * latent_sr), int(overlap * latent_sr)
        empty = [t == "" for t in prompts]
        if any(empty) and not all(empty):
            raise ValueError("empty prompts run without guidance: they cannot share a batch with non-empty ones")
        if all(empty):
            guidance_scale = None
            print("empyt input")
        check_loop(frames, B, window, hop_over, bool(guidance_scale), int(self.unet._h.desc.max_batch), int(self.unet._h.desc.max_len))
        if randomize_seed:
            random_seed = random.randint(0, MAX_SEED)
        text_emb, mask, uemb, umask = self._text_embeds(prompts, [""])
        lat = sample_loop_latents(self.unet, self.noise_scheduler, text_emb, mask, uemb, umask, frames, window, hop_over, guidance_scale,
                                  guidance_rescale, ddim_steps, eta, random_seed)
        p = self.params["autoencoder"]
        wav = self.autoencoder.decoder.decode_loop(scale_shift_re(lat, p["scale"], p["shift"]), lengths=frames)
        hop = self.autoencoder.decoder.hop
        out = [wav[b, 0, :hop * n].cpu().numpy() for b, n in enumerate(frames)]
        return (p["sr"], out) if batched else (p["sr"], out[0])

    def generate_timeline_audio(self, timeline, length=None, window_length=10, overlap=2, transition=1, guidance_scale=5, guidance_rescale=0.75,
                                ddim_steps=100, eta=1, random_seed=None, randomize_seed=False):
        """Long clips whose prompt changes over time: soundtracks, ambience beds that evolve, sound design for video.  `timeline` is one
        clip's list of (prompt, start_s, end_s) segments, or a list of such lists for a batch; segments may overlap, and together they must
        cover the clip.  `length` (seconds, one value or one per clip) defaults to the clip's largest end_s.  The clip is denoised in
        windows as in generate_long_audio (`inference.sample_timeline_latents`): each window carries one conditioned row per segment within
        `transition` seconds of it, those rows share one unconditional row, and each row's prediction is weighted by its segment's weight,
        1 inside the segment and tapering over `transition` seconds on either side (two abutting segments crossfade over 2 * transition
        seconds; 0 switches hard).  Seeds as in generate_long_audio.  Returns (sr, waveform) or (sr, [waveforms]) with
        hop * int(length * latent_sr) samples each.  The conditioned rows plus one unconditional row per window must fit the DiT's
        2 * max_batch rows.  A one-segment timeline equals generate_long_audio with that prompt, bit for bit."""
        batched = len(timeline) > 0 and not (isinstance(timeline[0], (tuple, list)) and len(timeline[0]) > 0 and isinstance(timeline[0][0], str))
        clips = [list(c) for c in timeline] if batched else [list(timeline)]
        B = len(clips)
        latent_sr = self.params["autoencoder"]["latent_sr"]
        # ---- everything is checked on the host before any device work
        num = (int, float, np.integer, np.floating)
        if B < 1 or any(not c for c in clips):
            raise ValueError("a timeline lists at least one (prompt, start_s, end_s) segment")
        for c in clips:
            for seg in c:
                if len(seg) != 3 or not isinstance(seg[0], str) or not isinstance(seg[1], num) or not isinstance(seg[2], num):
                    raise ValueError(f"a timeline segment is (prompt, start_s, end_s), got {seg!r}")
        if length is None:
            length = [max(e for _, _, e in c) for c in clips]
        frames = [int(v * latent_sr) for v in _per_clip("length", length, B, num)]
        if any(f < 1 for f in frames):
            raise ValueError(f"every length must be positive (at least one latent frame), got {length}")
        if window_length > self.max_length_s:
            raise ValueError(f"window_length {window_length} s exceeds max_length_s {self.max_length_s} s")
        if transition < 0:
            raise ValueError(f"transition must be >= 0 seconds, got {transition}")
        window, hop_over, T = int(window_length * latent_sr), int(overlap * latent_sr), int(transition * latent_sr)
        segs = [[(round(s * latent_sr), min(round(e * latent_sr), n)) for _, s, e in c] for c, n in zip(clips, frames)]
        if all(p == "" for c in clips for p, _, _ in c):
            guidance_scale = None
        check_timeline(segs, frames, B, window, hop_over, T, bool(guidance_scale), int(self.unet._h.desc.max_batch), int(self.unet._h.desc.max_len))
        if randomize_seed:
            random_seed = random.randint(0, MAX_SEED)
        prompts = list(dict.fromkeys(p for c in clips for p, _, _ in c))   # each distinct prompt is encoded once
        index = {p: i for i, p in enumerate(prompts)}
        text_emb, mask, uemb, umask = self._text_embeds(prompts, [""])
        segments = [[(index[p], s, e) for (p, _, _), (s, e) in zip(c, sg)] for c, sg in zip(clips, segs)]
        lat = sample_timeline_latents(self.unet, self.noise_scheduler, text_emb, mask, uemb, umask, segments, frames, window, hop_over, T,
                                      guidance_scale, guidance_rescale, ddim_steps, eta, random_seed)
        p = self.params["autoencoder"]
        wav = self.autoencoder.decoder.decode_tiled(scale_shift_re(lat, p["scale"], p["shift"]), lengths=frames)
        hop = self.autoencoder.decoder.hop
        out = [wav[b, 0, :hop * n].cpu().numpy() for b, n in enumerate(frames)]
        return (p["sr"], out) if batched else (p["sr"], out[0])

    def editing_long_audio(self, text, boundary, gt_file, mask_start, mask_length, window_length=10, overlap=2, guidance_scale=3.5,
                           guidance_rescale=0, ddim_steps=100, eta=1, random_seed=None, randomize_seed=False):
        """editing_audio for crops of any length: inpainting, and continuation past the clip's end (outpainting), over more than the
        denoiser's window.  The arguments and the crop arithmetic are editing_audio's (edit_plan): the mask [mask_start, mask_start +
        mask_length) seconds is regenerated with `boundary` seconds of context on either side, and a mask past the clip's end extends it.
        The crop is encoded in tiles (OobleckDecoder.encode_tiled), denoised in windows of `window_length` seconds overlapping by `overlap`
        seconds with its gt and mask (inference.sample_long_latents), pasted (pred[~mask] = gt[~mask]), decoded in tiles and spliced back.
        Only the window has to fit max_length_s; the crop may be any length.  Returns (sr, the whole edited clip), as editing_audio does.
        A crop that fits one window gives editing_audio's result with the same seed, bit for bit.

        Continuation of a 10-s clip by 30 s with 5 s of context (a 35-s crop: 5 windows, 10 DiT rows with guidance, so
        EzAudio(..., max_batch=5)):

            ez.editing_long_audio("rain turns into a thunderstorm", boundary=5, gt_file="rain_10s.wav", mask_start=10, mask_length=30)

        With a list of prompts, `gt_file`, `mask_start`, `mask_length`, `boundary` and `random_seed` list one value per prompt (a scalar
        applies to all; an int seed gives every edit that seed) and the call returns (sr, [clips]): one tiled encode, one windowed loop and
        one tiled decode.  Each clip equals the scalar call of that edit with its seed, the calls made in list order (the VAE bottleneck
        noise comes from the global RNG in clip order).  Empty prompts run without guidance and cannot share a call with non-empty ones.
        The windows of all edits (x 2 with guidance) must fit the DiT's 2 * max_batch rows."""
        batched = isinstance(text, (list, tuple))
        prompts = list(text) if batched else [text]
        sr, latent_sr = self.params["autoencoder"]["sr"], self.params["autoencoder"]["latent_sr"]
        dec = self.autoencoder.decoder
        B, hop = len(prompts), dec.hop
        # ---- everything is checked on the host before any device work
        if B < 1:
            raise ValueError("no prompt given")
        num = (int, float, np.integer, np.floating)
        scalar = (str, np.ndarray) if batched else (str, np.ndarray, list, tuple)
        files = _per_clip("gt_file", gt_file, B, scalar)
        starts, lengths_s = _per_clip("mask_start", mask_start, B, num), _per_clip("mask_length", mask_length, B, num)
        bounds = _per_clip("boundary", boundary, B, num)
        if randomize_seed:
            seeds = [random.randint(0, MAX_SEED) for _ in range(B)]
        elif random_seed is None:
            seeds = None
        else:
            seeds = [int(v) for v in _per_clip("random_seed", random_seed, B, num)]
        empty = [t == "" for t in prompts]
        if any(empty) and not all(empty):
            raise ValueError("empty prompts run without guidance: they cannot share a batch with non-empty ones")
        if all(empty):
            guidance_scale = None
            print("empyt input")
        if any(v < 0 for v in starts) or any(v <= 0 for v in lengths_s) or any(v < 0 for v in bounds):
            raise ValueError("mask_start and boundary must be >= 0 and mask_length > 0 for every edit")
        if window_length > self.max_length_s:
            raise ValueError(f"window_length {window_length} s exceeds max_length_s {self.max_length_s} s")
        window, hop_over = int(window_length * latent_sr), int(overlap * latent_sr)
        raws = [_load_audio(f, sr) if isinstance(f, str) else np.asarray(f, dtype=np.float32) for f in files]
        if any(r.ndim != 1 or len(r) < 1 for r in raws):
            raise ValueError("every gt_file must be a non-empty mono waveform")
        plans = [edit_plan(len(r), sr, latent_sr, hop, bd, ms, ml) for r, bd, ms, ml in zip(raws, bounds, starts, lengths_s)]
        frames = [p["frames"] for p in plans]
        check_long(frames, B, window, hop_over, bool(guidance_scale), int(self.unet._h.desc.max_batch), int(self.unet._h.desc.max_len))
        # ---- per clip: normalise + pad on the device, crop into the padded batch; one tiled encode (bottleneck noise: global RNG, clip order)
        N = max(frames)
        outs, crops = [], torch.zeros(B, 1, N * hop, device=self.device)
        for b, (r, p) in enumerate(zip(raws, plans)):
            o = post.prepare_wave(torch.from_numpy(r).to(self.device).unsqueeze(0), p["n_total"], normalize=True)[0]
            crops[b, 0, :p["s1"] - p["s0"]] = o[p["s0"]:p["s1"]]
            outs.append(o)
        gt_latent = dec.encode_tiled(crops, lengths=frames)
        gt_mask = torch.ones(B, N, dtype=torch.bool)
        for b, p in enumerate(plans):
            gt_mask[b, :p["m0"]] = False
            gt_mask[b, p["m1"]:frames[b]] = False
        gt_mask = gt_mask.to(self.device)
        text_emb, mask, uemb, umask = self._text_embeds(prompts, [""])
        lat = sample_long_latents(self.unet, self.noise_scheduler, text_emb, mask, uemb, umask, frames, window, hop_over, guidance_scale,
                                  guidance_rescale, ddim_steps, eta, seeds, gt=gt_latent, gt_mask=gt_mask)
        a = self.params["autoencoder"]
        pred = torch.where(gt_mask[:, None, :], scale_shift_re(lat, a["scale"], a["shift"]), gt_latent)   # src/inference.py:104-105
        wav = dec.decode_tiled(pred, lengths=frames)
        for b, (o, p) in enumerate(zip(outs, plans)):
            post.splice_wave(o, wav[b, 0], p["s0"], p["n_paste"])
        res = [o.cpu().numpy() for o in outs]
        return (sr, res) if batched else (sr, res[0])

    def variation_audio(self, text, init_audio, strength=0.8, guidance_scale=5, guidance_rescale=0.75, ddim_steps=100, eta=1, random_seed=None,
                        randomize_seed=False, *, pad_length=None):
        """Audio-to-audio variation (SDEdit; diffusers' img2img, Stable Audio's init_audio): `init_audio` (a WAV path or a float32 mono
        waveform at the model's rate) is peak-normalised, zero-padded to a whole hop, VAE-encoded and noised to the schedule index
        `scheduler.start_index(ddim_steps, strength)`; the last int(ddim_steps * strength) steps then denoise it with `text`.  strength 1
        starts from pure noise (with DDIM the result is then generate_audio's, bit for bit, for the same prompt, seed and frame count);
        smaller strengths keep more of the clip.  Returns (sr, float32 waveform) of the clip's length in samples.
        Prompt b's generator (random_seed as in generate_audio) draws its start noise (1, C, frames) first, then the noise of the steps it
        runs; the VAE bottleneck noise comes from the global RNG in clip order, as in editing_audio.
        With a list of prompts, `init_audio`, `strength` and `random_seed` list one value per prompt (a scalar applies to all) and the call
        returns (sr, [waveforms]): one VAE encode, one sampling loop and one decode, the batch padded to the longest clip or to `pad_length`
        seconds (at most max_length_s).  Each waveform equals the scalar call with its seed, the calls made in list order."""
        if isinstance(text, (list, tuple)):
            return self._variation(list(text), True, init_audio, strength, guidance_scale, guidance_rescale, ddim_steps, eta, random_seed,
                                   randomize_seed, pad_length)
        if pad_length is not None:
            raise ValueError("pad_length applies to a list of variations")
        return self._variation([text], False, [init_audio], [strength], guidance_scale, guidance_rescale, ddim_steps, eta, random_seed,
                               randomize_seed, None)

    def _variation(self, prompts, batched, init_audio, strength, guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, randomize_seed,
                   pad_length):
        sr, latent_sr = self.params["autoencoder"]["sr"], self.params["autoencoder"]["latent_sr"]
        dec = self.autoencoder.decoder
        B, hop = len(prompts), dec.hop
        # ---- everything is checked on the host before any device work
        if B < 1 or B > dec.max_batch:
            raise ValueError(f"{B} variations in one call: 1..{dec.max_batch} (max_batch) fit the workspace")
        num = (int, float, np.integer, np.floating)
        files = _per_clip("init_audio", init_audio, B, (str, np.ndarray))
        strengths = _per_clip("strength", strength, B, num)
        if randomize_seed:
            seeds = [random.randint(0, MAX_SEED) for _ in range(B)]
        elif random_seed is None or isinstance(random_seed, num):
            seeds = random_seed   # an int: prompt b draws from Generator(seed + b), as in generate_audio
        else:
            seeds = [int(v) for v in _per_clip("random_seed", random_seed, B, num)]
        empty = [t == "" for t in prompts]
        if any(empty) and not all(empty):
            raise ValueError("empty prompts run without guidance: they cannot share a batch with non-empty ones")
        if all(empty):
            guidance_scale = None
            print("empyt input")
        starts = [start_index(ddim_steps, v) for v in strengths]
        raws = [_load_audio(f, sr) if isinstance(f, str) else np.asarray(f, dtype=np.float32) for f in files]
        if any(r.ndim != 1 or len(r) < 1 or not np.isfinite(r).all() for r in raws):
            raise ValueError("every init_audio must be a non-empty, finite mono waveform")
        frames = [-(-len(r) // hop) for r in raws]
        max_frames = int(round(self.max_length_s * latent_sr))
        if pad_length is not None and pad_length > self.max_length_s:
            raise ValueError(f"pad_length {pad_length} s exceeds max_length_s {self.max_length_s} s")
        L = max(frames) if pad_length is None else int(pad_length * latent_sr)
        if max(frames) > L or L > max_frames:
            raise ValueError(f"clips of {frames} latent frames must fit the padded length ({L} frames, at most {max_frames}: "
                             f"max_length_s {self.max_length_s} s)")
        sched = self.noise_scheduler
        sched.set_timesteps(ddim_steps)
        ab = [sched.add_noise_coefficients(int(sched.timesteps[k])) for k in starts]
        # ---- per clip: normalise + pad on the device into the padded batch; then the start noise, one fused encode + add_noise
        clips = torch.zeros(B, 1, L * hop, device=self.device)
        for b, r in enumerate(raws):
            clips[b, 0, :frames[b] * hop] = post.prepare_wave(torch.from_numpy(r).to(self.device).unsqueeze(0), frames[b] * hop, normalize=True)[0]
        gens = make_generators(seeds, B, self.device)
        C = self.unet.cfg["out_chans"]
        eps = torch.zeros(B, C, L, device=self.device)
        for b, g in enumerate(gens):   # generate_audio's initial draw, at the clip's own shape
            eps[b, :, :frames[b]] = torch.randn((1, C, frames[b]), generator=g, device=self.device)[0]
        lengths = frames if batched else None
        p = self.params["autoencoder"]
        x_t = dec.encode_noised(clips, ab, eps, p["scale"], p["shift"], lengths=lengths)   # bottleneck noise: global RNG, clip order
        embeds = self._text_embeds(prompts, [""])
        pred = inference(self.autoencoder, self.unet, None, None, None, None, self.params, sched, prompts, None, L, guidance_scale,
                         guidance_rescale, ddim_steps, eta, None, self.device, text_embeds=embeds, lengths=lengths, start_index=starts,
                         init_latents=x_t, generators=gens)
        if not batched:
            return sr, pred[0, 0, :len(raws[0])].cpu().numpy()
        return sr, [w[0, :len(r)].cpu().numpy() for w, r in zip(pred, raws)]


def energy_condition(audio: torch.Tensor, hop_size=240, window_size=1920, padding="reflect", min_db=-60, norm=True, quantize_levels=None,
                     **unused):
    """EnergyExtractor + Conditioner (src/models/conditions/energy.py:19-56, condition_wrapper.py:26-42): (B,T) -> (B,1,T/hop).
    One CUDA kernel (ezb_energy_condition); no torch fallback."""
    if padding != "reflect":
        raise NotImplementedError("energy conditioner: only padding='reflect' (the shipped config)")
    if not audio.is_cuda:
        raise EzbError("energy_condition needs a CUDA tensor")
    a = audio.detach().to(torch.float32).contiguous()
    B, T = a.shape
    out = torch.empty(B, 1, T // hop_size, dtype=torch.float32, device=a.device)
    _lib.check(_lib.lib().ezb_energy_condition(a.device.index or 0, a.data_ptr(), out.data_ptr(), B, T, int(hop_size), int(window_size), float(min_db),
                                               int(bool(norm)), int(quantize_levels or 0), torch.cuda.current_stream(a.device).cuda_stream))
    return out


class EzAudio_ControlNet(_Base):
    """api/controlnet.py:31.  precision as for EzAudio ("fp8" applies to the DiT and the ControlNet).  It has no audio-to-audio variation
    call: a variation starts from its own clip, a ControlNet call from the reference clip's energy; use EzAudio.variation_audio."""

    def __init__(self, model_name, ckpt_path=None, controlnet_path=None, vae_path=None, device="cuda", *,
                 text_encoder: Optional[Callable] = None, precision: str = "bf16", max_batch: int = 4, config_path=None,
                 vae_config_path=None, params: Optional[dict] = None):
        self.device = device
        self.params = params if params is not None else config.load_params(model_name, config_path, config.BUILTIN_CONTROLNET)
        p = self.params
        max_len = 10 * p["autoencoder"]["latent_sr"]  # the reference ControlNet API is hard-wired to 10 s (api/controlnet.py:131-138)
        self.max_length_s = 10.0
        self.noise_scheduler = DDIMScheduler(**p["diff"])
        kw = dict(precision=precision, max_batch=2 * max_batch, max_len=max_len, max_ctx_len=p["text_encoder"]["max_length"], max_timesteps=1000,
                  device=device)
        self.unet = MaskDiT(**kw, **p["model"])
        sd = _state_dict(ckpt_path, weights.dit_param_shapes(p["model"]), "model")
        self.unet.load_state_dict(sd)
        self.controlnet = DiTControlNet(**kw, **p["model"], **p["controlnet"])
        csd = _state_dict(controlnet_path, weights.controlnet_param_shapes(p["model"], p["controlnet"]), "model")
        self.controlnet.load_state_dict(csd, mask_embed=sd["mask_embed"])
        dcfg = config.load_vae_decoder_config(vae_config_path)
        dec = OobleckDecoder(precision=_vae_precision(precision), max_batch=max_batch, max_latent_len=max_len, device=device, **dcfg)
        vsd = _state_dict(vae_path, weights.vae_decoder_param_shapes(dcfg), "state_dict")
        vsd = {(k[len("autoencoder."):] if k.startswith("autoencoder.") else k): v for k, v in vsd.items()}
        dec.load_state_dict(vsd)
        self.autoencoder = Autoencoder(dec)
        if p["conditioner"]["condition_type"] != "energy":
            raise NotImplementedError("only the shipped energy conditioner")
        self.encode_text = self._make_text_encoder(text_encoder, p, device)

    def generate_audio(self, text, audio_path, surpass_noise=0, guidance_scale=3.5, guidance_rescale=0, ddim_steps=50, eta=1,
                       conditioning_scale=1, random_seed=None, randomize_seed=False):
        """api/controlnet.py:113-161.  `audio_path` may also be a float32 numpy waveform at the model sample rate.
        With a list of prompts, `audio_path` may list one reference clip per prompt (and `surpass_noise` one gate per prompt, or one for
        all): each clip is prepared on its own, the batch runs once and waveform b is trimmed to clip b's length.  Pass one seed per prompt
        in `random_seed` to make the batch reproduce the scalar calls."""
        if isinstance(audio_path, (list, tuple)):
            return self._generate_per_clip(text, list(audio_path), surpass_noise, guidance_scale, guidance_rescale, ddim_steps, eta,
                                           conditioning_scale, random_seed, randomize_seed)
        sr = self.params["autoencoder"]["sr"]
        gt = _load_audio(audio_path, sr) if isinstance(audio_path, str) else np.asarray(audio_path, dtype=np.float32)
        original_length = len(gt)
        num_samples = int(10 * sr)
        audio_frames = round(num_samples / sr * self.params["autoencoder"]["latent_sr"])
        # normalise, noise-gate and pad / crop to 10 s on the device (ezb_wave_prepare = api/controlnet.py:119-136)
        gt_audio = post.prepare_wave(torch.from_numpy(gt).to(self.device).unsqueeze(0), num_samples, normalize=True, gate=float(surpass_noise or 0))
        # the reference encodes gt_audio only to read its latent SHAPE (api/controlnet.py:141-142): (1, 128, audio_frames)
        cond_kw = {k: v for k, v in self.params["conditioner"].items() if k != "condition_type"}
        condition = energy_condition(gt_audio, **cond_kw)
        if randomize_seed:
            random_seed = random.randint(0, MAX_SEED)
        batched = not isinstance(text, str)
        prompts = list(text) if batched else [text]
        condition = condition.expand(len(prompts), -1, -1)
        embeds = self._text_embeds(prompts, [""])
        pred = inference(self.autoencoder, self.unet, None, None, None, None, self.params, self.noise_scheduler, prompts, None, audio_frames,
                         guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, self.device, text_embeds=embeds,
                         controlnet=self.controlnet, condition=condition, conditioning_scale=conditioning_scale)
        pred = pred.cpu().numpy()
        if batched:
            return sr, [pred[i, 0][:original_length] for i in range(pred.shape[0])]
        return sr, pred.squeeze(0).squeeze(0)[:original_length]

    def _generate_per_clip(self, text, audio_paths, surpass_noise, guidance_scale, guidance_rescale, ddim_steps, eta, conditioning_scale,
                           random_seed, randomize_seed):
        sr = self.params["autoencoder"]["sr"]
        # ---- everything is checked on the host before any device work
        if isinstance(text, str):
            raise ValueError("a list of reference clips takes a list of prompts (one clip per prompt)")
        prompts = list(text)
        B = len(prompts)
        if len(audio_paths) != B:
            raise ValueError(f"audio_path lists one clip per prompt: got {len(audio_paths)} for {B} prompts")
        num = (int, float, np.integer, np.floating)
        gates = [float(g or 0) for g in _per_clip("surpass_noise", surpass_noise, B, num)]
        if isinstance(random_seed, (list, tuple)) and len(random_seed) != B:
            raise ValueError(f"random_seed lists one seed per prompt: got {len(random_seed)} for {B} prompts")
        raws = [_load_audio(a, sr) if isinstance(a, str) else np.asarray(a, dtype=np.float32) for a in audio_paths]
        if any(r.ndim != 1 or len(r) < 1 for r in raws):
            raise ValueError("every reference clip must be a non-empty mono waveform")
        num_samples = int(10 * sr)
        audio_frames = round(num_samples / sr * self.params["autoencoder"]["latent_sr"])
        cond_kw = {k: v for k, v in self.params["conditioner"].items() if k != "condition_type"}
        # ---- per clip: normalise, noise-gate, pad / crop to 10 s and the energy condition, as the scalar call does; stacked (B, 1, 2L)
        condition = torch.cat([energy_condition(post.prepare_wave(torch.from_numpy(r).to(self.device).unsqueeze(0), num_samples, normalize=True,
                                                                  gate=g), **cond_kw) for r, g in zip(raws, gates)], 0)
        if randomize_seed:
            random_seed = random.randint(0, MAX_SEED)
        embeds = self._text_embeds(prompts, [""])
        pred = inference(self.autoencoder, self.unet, None, None, None, None, self.params, self.noise_scheduler, prompts, None, audio_frames,
                         guidance_scale, guidance_rescale, ddim_steps, eta, random_seed, self.device, text_embeds=embeds,
                         controlnet=self.controlnet, condition=condition, conditioning_scale=conditioning_scale)
        pred = pred.cpu().numpy()
        return sr, [pred[b, 0][:len(r)] for b, r in enumerate(raws)]

    def generate_long_audio(self, text, audio_path, window_length=10, overlap=2, surpass_noise=0, guidance_scale=3.5, guidance_rescale=0,
                            ddim_steps=50, eta=1, conditioning_scale=1, random_seed=None, randomize_seed=False):
        """generate_audio for reference clips of any length: the output is as long as the clip (generate_audio cuts it to 10 s).
        The clip's latent is denoised in windows of `window_length` seconds overlapping by `overlap` seconds, as in
        EzAudio.generate_long_audio (inference.sample_long_latents), and decoded in tiles.  Clip b of n_b samples gets
        long_control_frames(n_b, hop, window) latent frames: a clip shorter than the window is padded to it, as generate_audio pads to 10 s.
        The condition is the energy contour of the whole prepared clip (one peak normalisation and one noise gate per clip, then
        energy_condition over all of it), so overlapping windows see the same condition values on the frames they share; each window's
        slice of it goes through the ControlNet's stem once per call.
        `audio_path`: a path or a float32 waveform, or a list of one per prompt; `surpass_noise` and `random_seed` one value or one per
        prompt, as in generate_audio; `conditioning_scale` one value for the call.  Returns (sr, waveform) or, for a list of prompts,
        (sr, [waveforms]), waveform b trimmed to n_b samples.  An empty prompt runs without guidance (as in EzAudio.generate_long_audio) and
        cannot share a call with non-empty ones.  With window_length=10, a clip of at most 10 s is one window and the result equals
        generate_audio with the same arguments and seed, bit for bit (for an empty prompt: generate_audio with guidance_scale=0).  The
        windows (x 2 with guidance) must fit the 2 * max_batch rows of the DiT and the ControlNet: a 60 s clip in 10 s windows with 2 s
        overlap is 8 windows, which needs max_batch=8 with guidance."""
        batched = not isinstance(text, str)
        prompts = list(text) if batched else [text]
        B = len(prompts)
        p = self.params["autoencoder"]
        sr, latent_sr = p["sr"], p["latent_sr"]
        # ---- everything is checked on the host before any device work
        if isinstance(audio_path, (list, tuple)):
            if not batched:
                raise ValueError("a list of reference clips takes a list of prompts (one clip per prompt)")
            clips = list(audio_path)
            if len(clips) != B:
                raise ValueError(f"audio_path lists one clip per prompt: got {len(clips)} for {B} prompts")
        else:
            clips = [audio_path] * B
        num = (int, float, np.integer, np.floating)
        gates = [float(g or 0) for g in _per_clip("surpass_noise", surpass_noise, B, num)]
        if isinstance(random_seed, (list, tuple)) and len(random_seed) != B:
            raise ValueError(f"random_seed lists one seed per prompt: got {len(random_seed)} for {B} prompts")
        if B < 1:
            raise ValueError("no prompt given")
        if window_length > self.max_length_s:
            raise ValueError(f"window_length {window_length} s exceeds the ControlNet's {self.max_length_s} s")
        window, hop_over = int(window_length * latent_sr), int(overlap * latent_sr)
        empty = [t == "" for t in prompts]
        if any(empty) and not all(empty):
            raise ValueError("empty prompts run without guidance: they cannot share a batch with non-empty ones")
        if all(empty):
            guidance_scale = None
        raws = [_load_audio(a, sr) if isinstance(a, str) else np.asarray(a, dtype=np.float32) for a in clips]
        if any(r.ndim != 1 or len(r) < 1 for r in raws):
            raise ValueError("every reference clip must be a non-empty mono waveform")
        hop = int(round(sr / latent_sr))
        frames = [long_control_frames(len(r), hop, window) for r in raws]
        rows = min(int(self.unet._h.desc.max_batch), int(self.controlnet._h.desc.max_batch))
        check_long(frames, B, window, hop_over, bool(guidance_scale), rows, int(self.unet._h.desc.max_len))
        if randomize_seed:
            random_seed = random.randint(0, MAX_SEED)
        cond_kw = {k: v for k, v in self.params["conditioner"].items() if k != "condition_type"}
        condition = torch.zeros(B, 1, 2 * max(frames), device=self.device)   # clip b's frames past 2 * frames[b] are never read
        for b, (r, g, n) in enumerate(zip(raws, gates, frames)):
            wave = post.prepare_wave(torch.from_numpy(r).to(self.device).unsqueeze(0), n * hop, normalize=True, gate=g)
            condition[b:b + 1, :, :2 * n] = energy_condition(wave, **cond_kw)
        text_emb, mask, uemb, umask = self._text_embeds(prompts, [""])
        lat = sample_long_latents(self.unet, self.noise_scheduler, text_emb, mask, uemb, umask, frames, window, hop_over, guidance_scale,
                                  guidance_rescale, ddim_steps, eta, random_seed, controlnet=self.controlnet, condition=condition,
                                  conditioning_scale=conditioning_scale)
        wav = self.autoencoder.decoder.decode_tiled(scale_shift_re(lat, p["scale"], p["shift"]), lengths=frames)
        out = [wav[b, 0, :len(r)].cpu().numpy() for b, r in enumerate(raws)]
        return (sr, out) if batched else (sr, out[0])


def long_control_frames(n_samples: int, hop: int, window: int) -> int:
    """Latent frames of EzAudio_ControlNet.generate_long_audio for a reference clip of n_samples samples: enough whole hops to hold the
    clip, and at least one window (a shorter clip is zero-padded to it, as generate_audio pads to 10 s)."""
    return max(int(window), -(-int(n_samples) // int(hop)))
