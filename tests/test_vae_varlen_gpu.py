"""Length-aware Oobleck encode / decode: a padded batch with per-clip lengths in device memory.

Contract: clip b of a batch padded to L latent frames carries lens[b] <= L of them; its hop * lens[b] samples (decode) or lens[b] latent
frames (encode) are the bits the same clip computes alone at its own length, nothing in the padded tail (not even NaN) reaches them, and
everything past the clip's end comes out as zeros."""
import functools

import pytest
import torch

from ezaudio_b200 import synth, weights

pytestmark = pytest.mark.gpu

CONFIGS = {"tiny": (synth.tiny_vae_encoder(16), synth.tiny_vae(16), 150), "full": (synth.VAE_ENCODER, synth.VAE_DECODER, 140)}
REL = {"bf16x3": 1e-3, "bf16": 6e-2}   # of max|ref|, as tests/test_vae_gpu.py


@functools.lru_cache(maxsize=None)
def _state_dict(name):
    ecfg, dcfg, _ = CONFIGS[name]
    sd = dict(weights.synthetic_state_dict(weights.vae_decoder_param_shapes(dcfg), 6))
    sd.update(weights.synthetic_state_dict(weights.vae_encoder_param_shapes(ecfg), 8))
    return sd


def _codec(name, precision, B=4):
    from ezaudio_b200.vae import OobleckDecoder
    ecfg, dcfg, L = CONFIGS[name]
    return OobleckDecoder(precision=precision, max_batch=B, max_latent_len=L, encoder_cfg=ecfg, **dcfg).load_state_dict(_state_dict(name)), L


def _lens(L):
    return [L, 1, 37, L - 1]   # the padded length itself, one frame, an interior length, one frame short (L > 128: two M tiles at the top)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("name", ["tiny", "full"])
def test_decode_lens_matches_solo_decodes(name, precision):
    from oracle import ezaudio_oracle as O
    dec, L = _codec(name, precision)
    lens, hop, Cz = _lens(L), dec.hop, dec.cfg["latent_dim"]
    z = synth.synth_latents(4, L, Cz, seed=31).cuda()
    outs = []
    for fill in (float("nan"), 1e30):   # whatever the padded frames hold
        zp = z.clone()
        for b, n in enumerate(lens):
            zp[b, :, n:] = fill
        outs.append(dec(zp, lengths=lens))
    torch.cuda.synchronize()
    wav = outs[0]
    assert wav.shape == (4, 1, hop * L) and torch.equal(outs[0], outs[1])
    sd = {k: v.double() for k, v in _state_dict(name).items()}
    for b, n in enumerate(lens):
        solo = dec(z[b:b + 1, :, :n].contiguous())
        assert torch.equal(wav[b, :, :hop * n], solo[0]), (b, n)          # bit-identical to the clip decoded alone at its length
        assert bool((wav[b, :, hop * n:] == 0).all()), (b, n)              # zeros past the clip's end
        if n <= 37:                                                        # fp64 oracle on the short clips (CPU)
            ref = O.vae_decode(sd, z[b:b + 1, :, :n].cpu().double(), strides=tuple(dec.cfg["strides"]))
            err = float((wav[b:b + 1, :, :hop * n].cpu().double() - ref).abs().max())
            assert err < REL[precision] * float(ref.abs().max()) + 1e-5, (b, n, err)
    assert torch.equal(dec(z, lengths=[L] * 4), dec(z))                    # full lengths: the kernels without lengths, bit for bit


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("name", ["tiny", "full"])
def test_encode_lens_matches_solo_encodes(name, precision):
    from oracle import ezaudio_oracle as O
    enc, L = _codec(name, precision)
    lens, hop, Cz = _lens(L), enc.hop, enc.cfg["latent_dim"]
    audio = 0.3 * torch.randn(4, 1, hop * L, generator=torch.Generator().manual_seed(41)).cuda()
    noise = torch.randn(4, Cz, L, generator=torch.Generator().manual_seed(5)).cuda()
    ap, npad = audio.clone(), noise.clone()
    for b, n in enumerate(lens):
        ap[b, :, hop * n:] = float("nan")
        npad[b, :, n:] = float("nan")
    mean = enc.encode(ap, noise=False, lengths=lens)
    z = enc.encode(ap, noise=npad, lengths=torch.tensor(lens, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    assert mean.shape == (4, Cz, L)
    sd = {k: v.double() for k, v in _state_dict(name).items()}
    for b, n in enumerate(lens):
        a1, n1 = audio[b:b + 1, :, :hop * n].contiguous(), noise[b:b + 1, :, :n].contiguous()
        assert torch.equal(mean[b, :, :n], enc.encode(a1, noise=False)[0]), (b, n)
        assert torch.equal(z[b, :, :n], enc.encode(a1, noise=n1)[0]), (b, n)
        assert bool((mean[b, :, n:] == 0).all()) and bool((z[b, :, n:] == 0).all()), (b, n)
        if n <= 37:
            ref = O.vae_encode(sd, a1.cpu().double(), noise=n1.cpu().double(), strides=tuple(enc.cfg["strides"]))
            scale = float(O.vae_encode(sd, a1.cpu().double(), strides=tuple(enc.cfg["strides"])).abs().max())
            assert float((z[b:b + 1, :, :n].cpu().double() - ref).abs().max()) < 4 * REL[precision] * scale + 1e-5, (b, n)
    assert torch.equal(enc.encode(audio, noise=noise, lengths=[L] * 4), enc.encode(audio, noise=noise))


def test_encode_draws_the_noise_of_consecutive_solo_calls():
    enc, L = _codec("tiny", "bf16")
    lens, hop = [40, 7, L], enc.hop
    audio = 0.3 * torch.randn(3, 1, hop * L, generator=torch.Generator().manual_seed(2)).cuda()
    torch.manual_seed(11)
    z = enc.encode(audio, lengths=lens)
    torch.manual_seed(11)
    for b, n in enumerate(lens):
        assert torch.equal(z[b, :, :n], enc.encode(audio[b:b + 1, :, :hop * n].contiguous())[0]), (b, n)
    with pytest.raises(ValueError):   # a device tensor cannot size the host-side draws
        enc.encode(audio, lengths=torch.tensor(lens, dtype=torch.int32, device="cuda"))


def test_one_captured_graph_follows_new_lengths():
    dec, L = _codec("tiny", "bf16")
    z = synth.synth_latents(4, L, dec.cfg["latent_dim"], seed=3).cuda()
    audio = 0.3 * torch.randn(4, 1, dec.hop * L, generator=torch.Generator().manual_seed(4)).cuda()
    la, lb = _lens(L), [5, L, L - 3, 130]
    lens = torch.tensor(la, dtype=torch.int32, device="cuda")
    want = {}
    for key, v in (("a", la), ("b", lb)):
        want[key] = (dec(z, lengths=v), dec.encode(audio, noise=False, lengths=v))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        dec(z, lengths=lens); dec.encode(audio, noise=False, lengths=lens)   # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        wav, lat = dec(z, lengths=lens), dec.encode(audio, noise=False, lengths=lens)
    for key, v in (("a", la), ("b", lb), ("a", la)):
        lens.copy_(torch.tensor(v, dtype=torch.int32))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(wav, want[key][0]) and torch.equal(lat, want[key][1]), key


def test_lengths_are_validated_on_the_host():
    from ezaudio_b200 import _lib
    dec, L = _codec("tiny", "bf16")
    z = torch.zeros(4, dec.cfg["latent_dim"], L, device="cuda")
    torch.cuda.synchronize()
    c0 = _lib.lib().ezb_launch_count()
    for bad in ([L, 1, 37], [0, 1, 2, 3], [L + 1, 1, 2, 3], [1.5, 1, 2, 3], torch.tensor([1, 2, 3, 4]), torch.ones(3, dtype=torch.int32, device="cuda")):
        with pytest.raises(ValueError):
            dec(z, lengths=bad)
        with pytest.raises(ValueError):
            dec.encode(torch.zeros(4, 1, dec.hop * L, device="cuda"), noise=False, lengths=bad)
    assert _lib.lib().ezb_launch_count() == c0
