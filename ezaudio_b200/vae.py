"""VAE side of the hot path: `Autoencoder(embedding=z)` (src/modules/autoencoder_wrapper.py:74-77) ->
OobleckDecoder (src/modules/stable_vae/models/autoencoders.py:149-190), backed by libezb200.so."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from . import _lib, weights
from .dit import PRECISIONS, _as_f32c


def decoder_receptive_field(cfg) -> int:
    """Latent frames on either side of a latent frame that can change the decoder's samples of that frame (the halo decode_tiled gives
    each chunk): the interval a perturbed frame reaches, propagated through the input conv (k 7), every stage's transposed conv (k 2s,
    stride s, padding s / 2) and its three residual units (k 7 at dilations 1, 3, 9; the 1x1 convs reach nothing), and the output conv
    (k 7), in decoder order (the config's strides reversed), then rounded up to whole frames of hop samples."""
    lo, hi = -3, 3                                        # input conv, in latent frames
    for s in reversed(list(cfg["strides"])):
        lo, hi = lo * s - s // 2, hi * s - s // 2 + 2 * s - 1   # outputs input frame i reaches: i*s - s/2 .. i*s - s/2 + 2s - 1
        lo, hi = lo - 3 * (1 + 3 + 9), hi + 3 * (1 + 3 + 9)
    lo, hi = lo - 3, hi + 3                               # output conv
    hop = 1
    for s in cfg["strides"]:
        hop *= s
    return max(-(lo // hop), -(-(hi - (hop - 1)) // hop))


def encoder_receptive_field(cfg) -> int:
    """Latent frames on either side of a latent frame whose samples can change that frame (the halo encode_tiled gives each chunk): the
    samples latent frame 0 reads, propagated back through the encoder in encoder order -- the input conv (k 7, pad 3); per stage, three
    residual units (k 7 at dilations 1, 3, 9; the 1x1 convs reach nothing), then the strided conv (k 2s, stride s, pad ceil(s/2)), which
    reads inputs o*s - ceil(s/2) .. o*s - ceil(s/2) + 2s - 1 for output o; and the final conv (k 3, pad 1) at the latent rate -- then rounded
    up to whole frames of hop samples.  Walked from the latent end: [-1, 1] -> per stage (last first) -> [lo, hi] samples."""
    lo, hi = -1, 1                                        # final conv, in latent frames
    for s in reversed(list(cfg["strides"])):
        p = -(-s // 2)
        lo, hi = lo * s - p, hi * s - p + 2 * s - 1       # the strided conv's inputs
        lo, hi = lo - 3 * (1 + 3 + 9), hi + 3 * (1 + 3 + 9)
    lo, hi = lo - 3, hi + 3                               # input conv
    hop = 1
    for s in cfg["strides"]:
        hop *= s
    return max(-(lo // hop), -(-(hi - (hop - 1)) // hop))


def tile_chunks(lengths, max_len: int, halo: int):
    """The chunks decode_tiled and encode_tiled cut a batch of clips into, in latent frames: [(clip, first frame, end frame, core start,
    core end)].  A clip of at most max_len frames is one chunk [0, n); a longer one is cut into cores of max_len - 2 * halo frames, each
    chunk reaching `halo` frames past its core on either side, clipped to the clip's ends."""
    core = max_len - 2 * halo
    if core < 1:
        raise ValueError(f"max_latent_len {max_len} leaves no core inside a halo of {halo} frames on each side")
    chunks = []
    for b, n in enumerate(lengths):
        for c0 in range(0, n, core if n > max_len else n):
            c1 = min(n, c0 + core) if n > max_len else n
            chunks.append((b, max(0, c0 - halo), min(n, c1 + halo), c0, c1))
    return chunks


def loop_chunks(lengths, max_len: int, halo: int):
    """The chunks decode_loop cuts a batch of seamless loops into: [(loop, core start, core end, frames)].  A loop of n frames is cut into
    cores of at most max_len - 2 * halo frames (one core [0, n) when it fits); each chunk is its core with `halo` frames on either side,
    the frame indices taken mod n, so the halos wrap around the loop's ends (more than once when n < halo)."""
    core = max_len - 2 * halo
    if core < 1:
        raise ValueError(f"max_latent_len {max_len} leaves no core inside a halo of {halo} frames on each side")
    chunks = []
    for b, n in enumerate(lengths):
        for c0 in range(0, n, core):
            c1 = min(n, c0 + core)
            chunks.append((b, c0, c1, [f % n for f in range(c0 - halo, c1 + halo)]))
    return chunks


class OobleckDecoder:
    """OobleckDecoder (and, when `encoder_cfg` is given, OobleckEncoder + VAE bottleneck) on one ezb_vae handle."""

    def __init__(self, precision="bf16", max_batch=4, max_latent_len=512, device="cuda", encoder_cfg=None, **dec_cfg):
        self.shapes = weights.vae_decoder_param_shapes(dec_cfg)
        odd = [s for s in dec_cfg["strides"] if s < 2 or s % 2]
        if odd:  # ConvTranspose1d(k = 2s, stride s, padding ceil(s/2)) yields T*s - 1 frames for odd s, the library T*s
            raise NotImplementedError(f"VAE decoder strides {list(dec_cfg['strides'])}: only even strides >= 2 are implemented")
        self.encoder_cfg = dict(encoder_cfg) if encoder_cfg else None
        if self.encoder_cfg is not None:
            weights.vae_encoder_param_shapes(self.encoder_cfg)  # validates the switches
            if (self.encoder_cfg["channels"], list(self.encoder_cfg["c_mults"]), list(self.encoder_cfg["strides"])) != \
                    (dec_cfg["channels"], list(dec_cfg["c_mults"]), list(dec_cfg["strides"])):
                raise NotImplementedError("encoder and decoder must mirror each other (ckpts/vae/config.json)")
        self.cfg = dict(dec_cfg)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.EzbError("ezaudio_b200 runs on CUDA devices only (no CPU path)")
        self.dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        n = len(dec_cfg["c_mults"])
        d = _lib.VaeDesc(latent_dim=dec_cfg["latent_dim"], channels=dec_cfg["channels"], out_channels=dec_cfg["out_channels"], n_stages=n,
                         max_batch=max_batch, max_latent_len=max_latent_len, precision=PRECISIONS[precision],
                         with_encoder=1 if encoder_cfg else 0, in_channels=encoder_cfg["in_channels"] if encoder_cfg else 0,
                         enc_latent_dim=encoder_cfg["latent_dim"] if encoder_cfg else 0)
        for i in range(n):
            d.c_mults[i] = dec_cfg["c_mults"][i]
            d.strides[i] = dec_cfg["strides"][i]
        self.hop = 1
        for s in dec_cfg["strides"]:
            self.hop *= s
        self.max_batch = max_batch
        self.max_latent_len = max_latent_len
        self.h = C.c_void_p()
        with torch.cuda.device(self.dev_index):
            _lib.check(_lib.lib().ezb_vae_create(C.byref(self.h), C.byref(d), self.dev_index))

    def __del__(self):
        try:
            if getattr(self, "h", None) and self.h.value:
                _lib.lib().ezb_vae_destroy(self.h)
                self.h = C.c_void_p()
        except Exception:
            pass

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """Accepts the reference VAE state-dict after its 'autoencoder.' prefix strip (stable_vae/__init__.py:25-31);
        only `decoder.*` entries are consumed."""
        L = _lib.lib()
        with torch.cuda.device(self.dev_index):
            st = _lib.stream_ptr()
            for k, v in sd.items():
                if not (k.startswith("decoder.") or (self.encoder_cfg is not None and k.startswith("encoder."))):
                    continue
                t = _as_f32c(v).to(self.device)
                shape = (C.c_int64 * t.dim())(*t.shape)
                _lib.check(L.ezb_vae_load_weight(self.h, k.encode(), _lib.ptr(t), shape, t.dim(), st))
            torch.cuda.current_stream().synchronize()
            _lib.check(L.ezb_vae_finalize_weights(self.h, st))
        return self

    def _lens(self, lengths, B: int, L: int):
        """lengths (list of ints, or a cuda int32 tensor read on the device when the kernels run) -> (device int32 [B], host list or None).
        A list is validated here, before any device work; a tensor's values are the caller's to validate (the kernels clamp to 1..L)."""
        if isinstance(lengths, torch.Tensor):
            if lengths.dtype != torch.int32 or not lengths.is_cuda or tuple(lengths.shape) != (B,) or not lengths.is_contiguous():
                raise ValueError(f"lengths must be a contiguous cuda int32 tensor of shape ({B},)")
            return lengths, None
        host = [int(v) for v in lengths]
        if len(host) != B or any(v != w for v, w in zip(host, lengths)) or any(v < 1 or v > L for v in host):
            raise ValueError(f"lengths lists one whole frame count in 1..{L} per clip ({B} clips), got {list(lengths)}")
        return torch.tensor(host, dtype=torch.int32).to(self.device), host

    def __call__(self, z: torch.Tensor, lengths=None) -> torch.Tensor:
        """z (B,latent,L) -> (B,1,hop*L).  `lengths` (latent frames per clip, a list or a cuda int32 tensor): z is a padded batch; clip b's
        hop * lengths[b] samples equal the decode of z[b:b+1, :, :lengths[b]] alone, bit for bit, whatever the padded frames hold, and the
        samples past them are zeros."""
        z = _as_f32c(z).to(self.device)
        B, Cz, L = z.shape
        lens = None if lengths is None else self._lens(lengths, B, L)[0]
        wav = torch.empty(B, 1, L * self.hop, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.dev_index):
            for b0 in range(0, B, self.max_batch):
                nb = min(self.max_batch, B - b0)
                zs, ws = _lib.ptr(z[b0:b0 + nb]), C.c_void_p(wav[b0:b0 + nb].data_ptr())
                if lens is None:
                    _lib.check(_lib.lib().ezb_vae_decode(self.h, zs, ws, nb, L, _lib.stream_ptr()))
                else:
                    _lib.check(_lib.lib().ezb_vae_decode_lens(self.h, zs, ws, nb, L, _lib.ptr(lens[b0:b0 + nb]), _lib.stream_ptr()))
        return wav

    forward = __call__

    def decode_tiled(self, z: torch.Tensor, lengths=None) -> torch.Tensor:
        """z (B,latent,L) -> (B,1,hop*L) for L longer than the workspace's max_latent_len, on this handle: each clip is cut into chunks
        of at most max_latent_len frames whose inner edges carry a halo of decoder_receptive_field frames, up to max_batch chunks go to one
        length-aware decode, and each chunk's core is pasted into the output.  Every core sample depends only on latent frames inside its
        chunk, so the result equals a one-shot decode (on a workspace that holds L) bit for bit.  `lengths` (a list of latent frames per
        clip, or None): z is a padded batch, as in __call__; samples past hop * lengths[b] are zeros."""
        z = _as_f32c(z).to(self.device)
        B, Cz, L = z.shape
        host = [L] * B if lengths is None else self._lens(lengths, B, L)[1]
        if host is None:
            raise ValueError("decode_tiled takes the lengths as a list")
        chunks = tile_chunks(host, self.max_latent_len, decoder_receptive_field(self.cfg))
        wav = torch.zeros(B, 1, L * self.hop, device=self.device, dtype=torch.float32)
        hop = self.hop
        for g0 in range(0, len(chunks), self.max_batch):
            group = chunks[g0:g0 + self.max_batch]
            Lc = max(e - s for _, s, e, _, _ in group)
            zs = torch.zeros(len(group), Cz, Lc, device=self.device, dtype=torch.float32)
            for k, (b, s, e, _, _) in enumerate(group):
                zs[k, :, :e - s] = z[b, :, s:e]
            ws = self(zs, lengths=[e - s for _, s, e, _, _ in group])
            for k, (b, s, _, c0, c1) in enumerate(group):
                wav[b, :, c0 * hop:c1 * hop] = ws[k, :, (c0 - s) * hop:(c1 - s) * hop]
        return wav

    def decode_loop(self, z: torch.Tensor, lengths=None) -> torch.Tensor:
        """Seamless decode of loops: z (B,latent,L), loop b being its first lengths[b] frames (all L for None), followed by its frame 0
        after its last -> (B,1,hop*L), samples past hop * lengths[b] zero.  decode_tiled on a circle: each loop is cut into cores of at most
        max_latent_len - 2h frames (h = decoder_receptive_field) carrying h halo frames on either side taken mod lengths[b] (loop_chunks),
        the chunks are gathered by one index, up to max_batch go to one length-aware decode, and their cores are pasted.  Every core sample
        depends only on frames inside its chunk, so loop b's samples equal the middle period of a one-shot decode of the loop repeated,
        bit for bit: sample hop * lengths[b] - 1 runs on into sample 0."""
        z = _as_f32c(z).to(self.device)
        B, Cz, L = z.shape
        host = [L] * B if lengths is None else self._lens(lengths, B, L)[1]
        if host is None:
            raise ValueError("decode_loop takes the lengths as a list")
        h = decoder_receptive_field(self.cfg)
        chunks = loop_chunks(host, self.max_latent_len, h)
        wav = torch.zeros(B, 1, L * self.hop, device=self.device, dtype=torch.float32)
        hop = self.hop
        zf = z.transpose(0, 1).reshape(Cz, B * L)
        for g0 in range(0, len(chunks), self.max_batch):
            group = chunks[g0:g0 + self.max_batch]
            Lc = max(len(fr) for *_, fr in group)
            idx = torch.tensor([[b * L + f for f in fr] + [b * L] * (Lc - len(fr)) for b, _, _, fr in group], dtype=torch.int64)
            zs = zf[:, idx.to(self.device)].transpose(0, 1).contiguous()   # (chunks, latent, Lc); past a chunk's length never read
            ws = self(zs, lengths=[len(fr) for *_, fr in group])
            for k, (b, c0, c1, _) in enumerate(group):
                wav[b, :, c0 * hop:c1 * hop] = ws[k, :, h * hop:(h + c1 - c0) * hop]
        return wav

    def encode(self, audio: torch.Tensor, noise=None, lengths=None) -> torch.Tensor:
        """audio (B,1,T) -> latents (B,latent,T/hop): encoder + z = mean + (softplus(scale)+1e-4) * noise
        (`noise=None` draws torch.randn from the global RNG like the reference's vae_sample; pass False for the mean).
        `lengths` (latent frames per clip, a list or a cuda int32 tensor): audio is a padded batch, clip b being its first hop * lengths[b]
        samples; frames < lengths[b] of the result equal the encode of that clip alone, bit for bit, and the frames past them are zeros.
        With `noise=None` the bottleneck noise of clip b is drawn as (1, latent, lengths[b]) from the global RNG, in clip order -- the draws
        consecutive solo calls make -- which needs the lengths on the host (a list)."""
        a, T, L, lens, nz = self._encode_inputs(audio, noise, lengths)
        z = torch.empty(a.shape[0], self.cfg["latent_dim"], L, device=self.device, dtype=torch.float32)

        def launch(args, lb, b0, nb):
            if lb is None:
                return _lib.lib().ezb_vae_encode(*args, _lib.stream_ptr())
            return _lib.lib().ezb_vae_encode_lens(*args, lb, _lib.stream_ptr())
        self._run_encode(a, T, nz, z, lens, launch)
        return z

    def encode_tiled(self, audio: torch.Tensor, noise=None, lengths=None) -> torch.Tensor:
        """encode for clips longer than the workspace's max_latent_len, on this handle: audio (B,1,T) is zero-padded to a whole hop, each
        clip is cut into chunks of at most max_latent_len frames (tile_chunks) whose inner edges carry a halo of encoder_receptive_field
        frames, up to max_batch chunks go to one length-aware encode, and each chunk's core frames are pasted into the result.  Every core
        frame depends only on samples inside its chunk, so the result equals a one-shot encode (on a workspace that holds the whole length)
        bit for bit.  `lengths` (a list of latent frames per clip, or None for all of them): audio is a padded batch, as in encode; frames
        past lengths[b] are zeros.  With `noise=None` the bottleneck noise of clip b is drawn from the global RNG as (1, latent, lengths[b]),
        in clip order -- the draws of encode(lengths=list), and of consecutive solo encodes -- and each chunk reads its slice; a given
        noise (B, latent, L) is sliced the same way; `noise=False` gives the mean."""
        if self.encoder_cfg is None:
            raise _lib.EzbError("this handle was created without encoder_cfg")
        a = _as_f32c(audio).to(self.device)
        B, ch, T = a.shape
        if ch != 1:
            raise ValueError("mono audio (B,1,T) expected")
        hop, Cz = self.hop, self.cfg["latent_dim"]
        L = -(-T // hop)
        host = [L] * B if lengths is None else self._lens(lengths, B, L)[1]
        if host is None:
            raise ValueError("encode_tiled takes the lengths as a list")
        if noise is not None and noise is not False and tuple(noise.shape) != (B, Cz, L):
            raise ValueError(f"noise must be ({B}, {Cz}, {L}), got {tuple(noise.shape)}")
        chunks = tile_chunks(host, self.max_latent_len, encoder_receptive_field(self.encoder_cfg))
        if T % hop:   # strided convs floor the length; zero-pad to a whole latent frame, as encode does
            a = torch.nn.functional.pad(a, (0, L * hop - T))
        if noise is None:
            noise = torch.zeros(B, Cz, L, device=self.device, dtype=torch.float32)
            for b, n in enumerate(host):
                noise[b, :, :n] = torch.randn(1, Cz, n, device=self.device, dtype=torch.float32)[0]
        elif noise is not False:
            noise = _as_f32c(noise).to(self.device)
        z = torch.zeros(B, Cz, L, device=self.device, dtype=torch.float32)
        for g0 in range(0, len(chunks), self.max_batch):
            group = chunks[g0:g0 + self.max_batch]
            Lc = max(e - s for _, s, e, _, _ in group)
            xs = torch.zeros(len(group), 1, Lc * hop, device=self.device, dtype=torch.float32)
            ns = False if noise is False else torch.zeros(len(group), Cz, Lc, device=self.device, dtype=torch.float32)
            for k, (b, s, e, _, _) in enumerate(group):
                xs[k, :, :(e - s) * hop] = a[b, :, s * hop:e * hop]
                if ns is not False:
                    ns[k, :, :e - s] = noise[b, :, s:e]
            zs = self.encode(xs, noise=ns, lengths=[e - s for _, s, e, _, _ in group])
            for k, (b, s, _, c0, c1) in enumerate(group):
                z[b, :, c0:c1] = zs[k, :, c0 - s:c1 - s]
        return z

    def encode_noised(self, audio: torch.Tensor, ab, eps: torch.Tensor, scale: float, shift: float, noise=None, lengths=None) -> torch.Tensor:
        """The start latent of an audio-to-audio variation in one pass (ezb_vae_encode_noised): with z = encode(audio, noise, lengths),
        x_t = a_b * ((z + shift) * scale) + s_b * eps_b -- scale_shift, then diffusers' add_noise with clip b's (a_b, s_b) = ab[b]
        (`DDIMScheduler.add_noise_coefficients`).  ab: (B, 2) fp32 (a cuda tensor is read when the kernel runs), eps (B, latent, L).
        noise and lengths as in `encode`; with lengths, frames past a clip's end come out as zeros and eps is not read there."""
        B, L = audio.shape[0], -(-audio.shape[-1] // self.hop)   # checked before _encode_inputs draws the bottleneck noise
        abt = torch.as_tensor(ab, dtype=torch.float32)
        if tuple(abt.shape) != (B, 2) or tuple(eps.shape) != (B, self.cfg["latent_dim"], L):
            raise ValueError(f"ab must be ({B}, 2) and eps ({B}, {self.cfg['latent_dim']}, {L}), got {tuple(abt.shape)} and {tuple(eps.shape)}")
        a, T, L, lens, nz = self._encode_inputs(audio, noise, lengths)
        abt = abt.to(self.device).contiguous()
        e = _as_f32c(eps).to(self.device)
        x_t = torch.empty(B, self.cfg["latent_dim"], L, device=self.device, dtype=torch.float32)
        sc, sh = float(scale), float(shift)

        def launch(args, lb, b0, nb):
            h, au, vn, out, n, t = args
            return _lib.lib().ezb_vae_encode_noised(h, au, vn, C.c_void_p(e[b0:b0 + nb].data_ptr()), C.c_void_p(abt[b0:b0 + nb].data_ptr()), sc, sh,
                                                    out, n, t, lb, _lib.stream_ptr())
        self._run_encode(a, T, nz, x_t, lens, launch)
        return x_t

    def _encode_inputs(self, audio, noise, lengths):
        """encode's argument handling: (audio zero-padded to a whole hop, T, L, device lens or None, bottleneck noise or None)."""
        if self.encoder_cfg is None:
            raise _lib.EzbError("this handle was created without encoder_cfg")
        a = _as_f32c(audio).to(self.device)
        B, ch, T = a.shape
        if ch != 1:
            raise ValueError("mono audio (B,1,T) expected")
        pad = (-T) % self.hop
        if pad:  # strided convs floor the length; zero-pad to a whole latent frame (the reference silently truncates)
            a = torch.nn.functional.pad(a, (0, pad))
            T += pad
        L = T // self.hop
        Cz = self.cfg["latent_dim"]
        lens = host = None
        if lengths is not None:
            lens, host = self._lens(lengths, B, L)
        if noise is None and lens is not None:
            if host is None:
                raise ValueError("encode(lengths=<tensor>) cannot size the per-clip noise draws: pass the lengths as a list, or the noise")
            noise = torch.zeros(B, Cz, L, device=self.device, dtype=torch.float32)
            for b, n in enumerate(host):
                noise[b, :, :n] = torch.randn(1, Cz, n, device=self.device, dtype=torch.float32)[0]
        elif noise is None:
            noise = torch.randn(B, Cz, L, device=self.device, dtype=torch.float32)
        nz = None if noise is False else _as_f32c(noise).to(self.device)
        return a, T, L, lens, nz

    def _run_encode(self, a, T, nz, out, lens, launch):
        """Calls launch((handle, audio, noise, out, nb, T), lens or None, b0, nb) on each run of at most max_batch clips."""
        B = a.shape[0]
        with torch.cuda.device(self.dev_index):
            for b0 in range(0, B, self.max_batch):
                nb = min(self.max_batch, B - b0)
                args = (self.h, _lib.ptr(a[b0:b0 + nb]), None if nz is None else C.c_void_p(nz[b0:b0 + nb].data_ptr()),
                        C.c_void_p(out[b0:b0 + nb].data_ptr()), nb, T)
                lb = None if lens is None else _lib.ptr(lens[b0:b0 + nb])
                _lib.check(launch(args, lb, b0, nb))


class Autoencoder:
    """Call contract of src/modules/autoencoder_wrapper.py:7-83 for model_type 'stable_vae', quantization_first=True:
    exactly one of audio / embedding.  Decode is the hot path; encode = VAE encoder + bottleneck sampling (SURVEY 8f row 1)."""

    def __init__(self, decoder: OobleckDecoder):
        self.decoder = decoder

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def __call__(self, audio=None, embedding=None, lengths=None):
        """`lengths`: latent frames per clip of a padded batch (OobleckDecoder.__call__ / .encode)."""
        if embedding is not None:
            return self.decoder(embedding, lengths=lengths)
        if audio is not None:
            return self.decoder.encode(audio, lengths=lengths)
        raise ValueError("Either audio or embedding must be provided.")

    forward = __call__
