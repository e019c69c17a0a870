"""CPU oracle for the EzAudio hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference`
legs may import this file.  The product path (`ezaudio_b200/`) never imports it and has no
CPU fallback.

What it is: a plain-PyTorch fp32 (or fp64) *functional* restatement of the reference's
algorithm for the path SURVEY.md section 8(a) names, operating directly on the reference's
state-dict wire format (SURVEY Appendix D) -- no nn.Module, no einops, no caching, every
step-invariant quantity recomputed exactly as the reference does.  Each function cites the
reference file:line it follows (paths relative to the reference root).

Pinning: the reference has NO tests or golden vectors of its own (SURVEY section 4), so the
oracle is pinned against outputs of the reference itself: `oracle/gen_golden.py` imports the
reference modules in the build container, loads the same deterministic state-dict, and
writes `tests/golden/*.npz`; `tests/test_oracle_golden.py` checks this file against them
(and, when the reference tree is present, against the live reference modules).
The DDIM scheduler (`diffusers`, third-party, un-pinned, absent -- requirements.txt:2) is
restated from its published algorithm; for that piece parity is UNPINNED (closed-form
invariants only), see DESIGN.md.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]


# --------------------------------------------------------------------------- primitives
def layer_norm(x, w, b, eps=1e-5):
    """nn.LayerNorm over the last dim (blocks.py:68,83,85,91,100; attention.py:63-65)."""
    return F.layer_norm(x, (x.shape[-1],), w, b, eps)


def film_modulate(x, shift, scale):
    """src/models/utils/modules.py:15-16."""
    return x * (1 + scale) + shift


def timestep_embedding(t, dim=256, max_period=10000):
    """src/models/utils/modules.py:19-39: [cos | sin] of t * exp(-ln(1e4) i / half)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def linear(x, sd: SD, key: str):
    return F.linear(x, sd[key + ".weight"], sd.get(key + ".bias"))


def rotate_half(x):
    """src/models/utils/rotary.py:6-8."""
    x1, x2 = x.chunk(2, dim=-1)
    return torch.cat((-x2, x1), dim=-1)


def rope(q, k, inv_freq):
    """src/models/utils/rotary.py:48-91 ('shared' mode, positions 0..L-1, fp32 tables)."""
    L = q.shape[-2]
    t = torch.arange(L, dtype=torch.float32)
    freqs = torch.einsum("i,j->ij", t, inv_freq.float())
    emb = torch.cat((freqs, freqs), dim=-1)
    cos, sin = emb.cos()[None, None], emb.sin()[None, None]
    qf, kf = q.float(), k.float()
    return ((qf * cos) + rotate_half(qf) * sin).to(q.dtype), ((kf * cos) + rotate_half(kf) * sin).to(k.dtype)


def attention(x, sd: SD, p: str, H: int, context=None, context_mask=None, use_rope=False):
    """src/models/utils/attention.py:122-150 (Attention.forward), qk_norm='layernorm',
    SDPA math restated: softmax(q k^T / sqrt(dh) masked with -inf on ~key_mask) v; a query whose keys are all masked gets zeros, as
    F.scaled_dot_product_attention with a boolean mask returns them."""
    B, L, C = x.shape
    ctx = x if context is None else context
    q = F.linear(x, sd[p + ".to_q.weight"])
    k = F.linear(ctx, sd[p + ".to_k.weight"])
    v = F.linear(ctx, sd[p + ".to_v.weight"])
    dh = C // H
    split = lambda z: z.reshape(z.shape[0], z.shape[1], H, dh).permute(0, 2, 1, 3)
    q, k, v = split(q), split(k), split(v)
    q = layer_norm(q, sd[p + ".norm_q.weight"], sd[p + ".norm_q.bias"])
    k = layer_norm(k, sd[p + ".norm_k.weight"], sd[p + ".norm_k.bias"])
    if use_rope:
        q, k = rope(q, k, sd[p + ".rotary.inv_freq"])
    s = (q @ k.transpose(-2, -1)) * (dh ** -0.5)
    if context_mask is not None:  # attention.py:30-37,131-135: bool (B,1,L,Lc), True = keep
        s = s.masked_fill(~context_mask[:, None, None, :], float("-inf"))
    a = s.softmax(dim=-1)
    if context_mask is not None:
        a = a.masked_fill(~context_mask.any(-1)[:, None, None, None], 0.0)
    o = (a @ v).permute(0, 2, 1, 3).reshape(B, L, C)
    return linear(o, sd, p + ".proj")


def feed_forward(x, sd: SD, p: str):
    """GEGLU FeedForward: modules.py:263-277 (proj, chunk -> hidden, gate; hidden*gelu_erf(gate))
    then modules.py:366 Linear(inner -> D)."""
    u = linear(x, sd, p + ".net.0.proj")
    h, g = u.chunk(2, dim=-1)
    return linear(h * F.gelu(g), sd, p + ".net.2")


def adaln(sd: SD, p: str, time_token, time_ada, alpha_over_r: float):
    """src/models/blocks.py:39-45 ('ada_sola_bias')."""
    B = time_ada.shape[0]
    lora = F.linear(F.linear(time_token, sd[p + ".lora_a.weight"]), sd[p + ".lora_b.weight"]) * alpha_over_r
    return (time_ada + lora).reshape(B, 6, -1) + sd[p + ".scale_shift_table"][None]


def dit_block(x, sd: SD, p: str, cfg, time_token, time_ada, skip, context, context_mask):
    """src/models/blocks.py:120-160 (DiTBlock._forward)."""
    H = cfg["num_heads"]
    if skip is not None:  # :124-128
        cat = torch.cat([x, skip], dim=-1)
        cat = layer_norm(cat, sd[p + ".skip_norm.weight"], sd[p + ".skip_norm.bias"])
        x = linear(cat, sd, p + ".skip_linear")
    ada = adaln(sd, p + ".adaln", time_token, time_ada, cfg["ada_sola_alpha"] / cfg["ada_sola_rank"])
    sh_a, sc_a, g_a, sh_m, sc_m, g_m = ada.chunk(6, dim=1)  # :132-133
    xn = film_modulate(layer_norm(x, sd[p + ".norm1.weight"], sd[p + ".norm1.bias"]), sh_a, sc_a)
    x = x + (1 - g_a) * attention(xn, sd, p + ".attn", H, use_rope=True)  # :137-141
    xn = layer_norm(x, sd[p + ".norm2.weight"], sd[p + ".norm2.bias"])
    cn = layer_norm(context, sd[p + ".norm_context.weight"], sd[p + ".norm_context.bias"])
    x = x + attention(xn, sd, p + ".cross_attn", H, context=cn, context_mask=context_mask)  # :147-151
    xn = film_modulate(layer_norm(x, sd[p + ".norm3.weight"], sd[p + ".norm3.bias"]), sh_m, sc_m)
    x = x + (1 - g_m) * feed_forward(xn, sd, p + ".mlp")  # :155-156
    return x


def _time_path(sd: SD, p: str, timesteps, B, final=True):
    """udit.py:286-287,305-316: TimestepEmbedder -> SiLU -> time_ada(_final)."""
    if timesteps.dim() == 0:
        timesteps = timesteps.expand(B).long()
    te = timestep_embedding(timesteps).to(sd[p + "time_embed.mlp.0.weight"].dtype)
    tok = linear(F.silu(linear(te, sd, p + "time_embed.mlp.0")), sd, p + "time_embed.mlp.2")
    tok = F.silu(tok)
    ada_f = linear(tok, sd, p + "time_ada_final") if final else None
    ada = linear(tok, sd, p + "time_ada")
    return tok, ada, ada_f


def _embed(sd: SD, p: str, x, context):
    """udit.py:289-296: PatchEmbed Conv1d k=1 (modules.py:100-111) + context_embed MLP."""
    h = F.conv1d(x, sd[p + "patch_embed.proj.weight"], sd[p + "patch_embed.proj.bias"]).transpose(1, 2)
    c = linear(F.silu(linear(context, sd, p + "context_embed.0")), sd, p + "context_embed.2")
    return h, c


def udit_forward(sd: SD, cfg, x, timesteps, context, context_mask=None,
                 controlnet_skips: Optional[List[torch.Tensor]] = None, prefix="model."):
    """src/models/udit.py:281-362 for the shipped configuration (1d, ada_sola_bias, cross,
    rope shared, qk layernorm, geglu, skip+skip_norm, use_conv, pe none)."""
    p = prefix
    n_half = cfg["depth"] // 2
    B = x.shape[0]
    h, ctx = _embed(sd, p, x, context)
    tok, ada, ada_f = _time_path(sd, p, timesteps, B)
    skips = []
    for i in range(n_half):
        h = dit_block(h, sd, f"{p}in_blocks.{i}", cfg, tok, ada, None, ctx, context_mask)
        skips.append(h)
    h = dit_block(h, sd, f"{p}mid_block", cfg, tok, ada, None, ctx, context_mask)
    cskips = list(controlnet_skips) if controlnet_skips else None
    for i in range(n_half):
        skip = skips.pop()
        if cskips:
            skip = skip + cskips.pop()  # udit.py:345-348
        h = dit_block(h, sd, f"{p}out_blocks.{i}", cfg, tok, ada, skip, ctx, context_mask)
    # FinalBlock: blocks.py:199-211 ; unpatchify modules.py:80-84 (patch 1 -> transpose)
    shift, scale = ada_f.reshape(B, 2, -1).chunk(2, dim=1)
    h = film_modulate(layer_norm(h, sd[p + "final_block.norm.weight"], sd[p + "final_block.norm.bias"]), shift, scale)
    h = linear(h, sd, p + "final_block.linear").transpose(1, 2)
    return F.conv1d(h, sd[p + "final_block.final_layer.weight"], sd[p + "final_block.final_layer.bias"], padding=1)


def maskdit_concat(sd: SD, x, gt=None, mae_mask_infer=None):
    """src/models/conditioners.py:156-176 inference branches: returns (x257, mae_mask).
    NOTE (quirk, SURVEY 3.7): the reference overwrites `gt` in place; the oracle clones."""
    mae_mask = torch.ones_like(x)
    me = sd["mask_embed"].view(1, -1, 1)
    if gt is not None:
        mask = mae_mask_infer.expand_as(gt)
        gt = torch.where(mask, me.expand_as(gt), gt)  # conditioners.py:150-153
        mae_mask = mask.type_as(gt)
    else:
        gt = me.expand_as(x)
    return torch.cat([x, gt, mae_mask[:, 0:1, :]], dim=1), mae_mask


def maskdit_forward(sd: SD, cfg, x, timesteps, context, context_mask=None, gt=None,
                    mae_mask_infer=None, forward_model=True):
    """src/models/conditioners.py:156-183 (MaskDiT.forward)."""
    x257, mae_mask = maskdit_concat(sd, x, gt, mae_mask_infer)
    if forward_model:
        x257 = udit_forward(sd, cfg, x257, timesteps, context, context_mask)
    return x257, mae_mask


def controlnet_embed(sd: SD, p: str, condition):
    """src/models/controlnet.py:65-84 eval path: conv_in, cat an all-zero mask channel,
    [conv3+SiLU, conv3 stride2+SiLU] per block, conv_out, -> (B, L, D)."""
    e = F.conv1d(condition, sd[p + "conv_in.weight"], sd[p + "conv_in.bias"])
    e = torch.cat([e, torch.zeros_like(e[:, 0:1, :])], dim=1)  # cond_mask_infer = zeros
    i = 0
    while f"{p}blocks.{i}.0.weight" in sd:
        e = F.silu(F.conv1d(e, sd[f"{p}blocks.{i}.0.weight"], sd[f"{p}blocks.{i}.0.bias"], padding=1))
        e = F.silu(F.conv1d(e, sd[f"{p}blocks.{i}.2.weight"], sd[f"{p}blocks.{i}.2.bias"], padding=1, stride=2))
        i += 1
    e = F.conv1d(e, sd[p + "conv_out.weight"], sd[p + "conv_out.bias"])
    return e.transpose(1, 2).contiguous()


def controlnet_forward(sd: SD, cfg, x, timesteps, context, context_mask=None, condition=None,
                       conditioning_scale=1.0):
    """src/models/controlnet.py:252-315 (DiTControlNet.forward) -> list of depth/2 (B,L,D)."""
    B = x.shape[0]
    h, ctx = _embed(sd, "", x, context)
    h = h + controlnet_embed(sd, "controlnet_pre.", condition)
    tok, ada, _ = _time_path(sd, "", timesteps, B, final=False)
    skips = []
    for i in range(cfg["depth"] // 2):
        h = dit_block(h, sd, f"in_blocks.{i}", cfg, tok, ada, None, ctx, context_mask)
        skips.append(h)
    return [linear(s, sd, f"controlnet_zero_blocks.{i}") * conditioning_scale for i, s in enumerate(skips)]


# --------------------------------------------------------------------------- VAE decoder
def wn_weight(sd: SD, p: str):
    """torch.nn.utils.weight_norm (old style, dim=0): w = g * v / ||v|| with the norm over all
    dims except 0 (stable_vae/models/nn/layers.py:9-14).  For ConvTranspose1d dim 0 is C_in."""
    v, g = sd[p + ".weight_v"], sd[p + ".weight_g"]
    return g * v / v.flatten(1).norm(dim=1).view(-1, 1, 1)


def snake_beta(x, sd: SD, p: str):
    """stable_vae/models/blocks.py:317-318,350-359 (alpha_logscale=True)."""
    a = torch.exp(sd[p + ".alpha"]).view(1, -1, 1)
    b = torch.exp(sd[p + ".beta"]).view(1, -1, 1)
    return x + (1.0 / (b + 1e-9)) * torch.sin(x * a).pow(2)


def vae_res_unit(x, sd: SD, p: str, dilation: int):
    """stable_vae/models/autoencoders.py:38-61."""
    y = snake_beta(x, sd, p + ".layers.0")
    y = F.conv1d(y, wn_weight(sd, p + ".layers.1"), sd[p + ".layers.1.bias"], dilation=dilation, padding=3 * dilation)
    y = snake_beta(y, sd, p + ".layers.2")
    y = F.conv1d(y, wn_weight(sd, p + ".layers.3"), sd[p + ".layers.3.bias"])
    return y + x


def vae_decode(sd: SD, z, strides=(2, 4, 6, 10), prefix="decoder."):
    """OobleckDecoder.forward: stable_vae/models/autoencoders.py:149-190 with
    ckpts/vae/config.json:18-28 (snake, final_tanh false). z (B,128,L) -> (B,1,480 L)."""
    p = prefix + "layers."
    x = F.conv1d(z, wn_weight(sd, p + "0"), sd[p + "0.bias"], padding=3)
    for j, s in enumerate(reversed(strides)):  # decoder blocks use strides[i-1] for i = depth-1..1
        q = f"{p}{j + 1}.layers."
        x = snake_beta(x, sd, q + "0")
        x = F.conv_transpose1d(x, wn_weight(sd, q + "1"), sd[q + "1.bias"], stride=s, padding=math.ceil(s / 2))
        for u, d in enumerate((1, 3, 9)):
            x = vae_res_unit(x, sd, f"{q}{u + 2}", d)
    n = len(strides) + 1
    x = snake_beta(x, sd, f"{p}{n}")
    return F.conv1d(x, wn_weight(sd, f"{p}{n + 1}"), None, padding=3)


def vae_encode(sd: SD, audio, noise=None, strides=(2, 4, 6, 10), prefix="encoder."):
    """OobleckEncoder.forward (stable_vae/models/autoencoders.py:115-146; EncoderBlock :63-80) followed by
    VAEBottleneck.encode = vae_sample (stable_vae/models/bottleneck.py:66-70,77-87): audio (B,1,T) -> (B,128,T/480).
    `noise` replaces torch.randn_like(mean) (None -> returns the mean, for deterministic checks)."""
    p = prefix + "layers."
    x = F.conv1d(audio, wn_weight(sd, p + "0"), sd[p + "0.bias"], padding=3)
    for j, s in enumerate(strides):
        q = f"{p}{j + 1}.layers."
        for u, d in enumerate((1, 3, 9)):
            x = vae_res_unit(x, sd, f"{q}{u}", d)
        x = snake_beta(x, sd, q + "3")
        x = F.conv1d(x, wn_weight(sd, q + "4"), sd[q + "4.bias"], stride=s, padding=math.ceil(s / 2))
    n = len(strides) + 1
    x = snake_beta(x, sd, f"{p}{n}")
    x = F.conv1d(x, wn_weight(sd, f"{p}{n + 1}"), sd[f"{p}{n + 1}.bias"], padding=1)
    mean, scale = x.chunk(2, dim=1)
    if noise is None:
        return mean
    return noise * (F.softplus(scale) + 1e-4) + mean


def energy_extract(audio, hop_size=240, window_size=1920, min_db=-60.0, norm=True, quantize_levels=None):
    """EnergyExtractor.forward (src/models/conditions/energy.py:19-56), reflect padding: audio (B,T) -> (B, T//hop, 1)."""
    B, T = audio.shape
    n_frames = T // hop_size
    pad = (window_size - hop_size) // 2
    sq = F.pad(audio[:, None, :], (pad, pad), mode="reflect")[:, 0].double() ** 2
    csum = torch.cat([sq.new_zeros(B, 1), sq.cumsum(-1)], dim=-1)
    start = torch.arange(n_frames) * hop_size
    energy = ((csum[:, start + window_size] - csum[:, start]) / window_size).float()
    gain_db = 10 * torch.log10(torch.clamp(energy, min=10 ** (min_db / 10)))
    if norm:
        gain_db = (gain_db - min_db) / (gain_db.max(dim=-1, keepdim=True)[0] - min_db + 1e-8)
    if quantize_levels is not None:
        gain_db = torch.round(gain_db * (quantize_levels - 1)) / (quantize_levels - 1)
    return gain_db.unsqueeze(-1)


# --------------------------------------------------------------------------- T5 text encoder (the step before the path, SURVEY 8(f) row 3)
def t5_relative_position_bucket(relative_position, num_buckets=32, max_distance=128):
    """transformers T5Attention._relative_position_bucket, bidirectional branch (third-party dependency of the reference: `transformers`,
    un-pinned in requirements.txt; 5.5.0 is installed here and generated the goldens).  Same float32 arithmetic, operation by operation."""
    num_buckets //= 2
    ret = (relative_position > 0).to(torch.long) * num_buckets
    rp = torch.abs(relative_position)
    max_exact = num_buckets // 2
    is_small = rp < max_exact
    large = max_exact + (torch.log(rp.float() / max_exact) / math.log(max_distance / max_exact) * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return ret + torch.where(is_small, rp, large)


def t5_rms_norm(x, w, eps):
    """T5LayerNorm: no mean subtraction, no bias, variance in fp32."""
    return w * (x * torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + eps))


def t5_encode(sd: SD, cfg, input_ids, attention_mask):
    """T5EncoderModel(input_ids=, attention_mask=).last_hidden_state as the reference calls it (src/inference.py:38-50; model loaded at
    api/ezaudio.py:78-79): gated-GELU (gelu_new) T5 v1.1 / flan-T5 encoder, unscaled attention, relative position bias of block 0 shared by
    every block, additive key mask.  (B, L) int64 ids, (B, L) 0/1 mask -> (B, L, d_model)."""
    H, dk, eps = cfg["num_heads"], cfg["d_kv"], cfg.get("layer_norm_epsilon", 1e-6)
    B, L = input_ids.shape
    x = sd["shared.weight"][input_ids]
    pos = torch.arange(L)
    bucket = t5_relative_position_bucket(pos[None, :] - pos[:, None], cfg["relative_attention_num_buckets"],
                                         cfg.get("relative_attention_max_distance", 128))   # [query, key]
    bias = sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"][bucket].permute(2, 0, 1)[None]  # (1, H, L, L)
    bias = bias + (1.0 - attention_mask[:, None, None, :].to(x.dtype)) * torch.finfo(x.dtype).min
    for i in range(cfg["num_layers"]):
        a = f"encoder.block.{i}.layer.0."
        h = t5_rms_norm(x, sd[a + "layer_norm.weight"], eps)
        q, k, v = (F.linear(h, sd[a + f"SelfAttention.{n}.weight"]).view(B, L, H, dk).transpose(1, 2) for n in ("q", "k", "v"))
        w = torch.softmax((q @ k.transpose(-1, -2) + bias).float(), dim=-1).to(x.dtype)
        o = (w @ v).transpose(1, 2).reshape(B, L, H * dk)
        x = x + F.linear(o, sd[a + "SelfAttention.o.weight"])
        f = f"encoder.block.{i}.layer.1."
        h = t5_rms_norm(x, sd[f + "layer_norm.weight"], eps)
        g = F.linear(h, sd[f + "DenseReluDense.wi_0.weight"])
        g = 0.5 * g * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (g + 0.044715 * g.pow(3))))   # NewGELUActivation
        x = x + F.linear(g * F.linear(h, sd[f + "DenseReluDense.wi_1.weight"]), sd[f + "DenseReluDense.wo.weight"])
    return t5_rms_norm(x, sd["encoder.final_layer_norm.weight"], eps)


# --------------------------------------------------------------------------- sampling loop
class DDIM:
    """Restatement of diffusers.DDIMScheduler for ckpts/ezaudio-xl.yml:52-60 (scaled_linear,
    rescale_betas_zero_snr, trailing, v_prediction, clip_sample False, set_alpha_to_one True).
    Call sites: api/ezaudio.py:92-97, src/inference.py:64,71,98-100.  PARITY UNPINNED
    (third-party, source absent): checked by closed-form invariants in tests only."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
        self.T = num_train_timesteps
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, self.T, dtype=torch.float32) ** 2
        abar_sqrt = torch.cumprod(1.0 - betas, dim=0).sqrt()
        s0, sT = abar_sqrt[0].clone(), abar_sqrt[-1].clone()
        abar_sqrt = (abar_sqrt - sT) * (s0 / (s0 - sT))
        abar = abar_sqrt ** 2
        alphas = torch.cat([abar[0:1], abar[1:] / abar[:-1]])
        # diffusers stores betas' = 1 - alphas, then alphas_cumprod = cumprod(1 - betas')
        self.alphas_cumprod = torch.cumprod(1.0 - (1.0 - alphas), dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0)

    def set_timesteps(self, n):
        import numpy as np
        self.n = n
        ts = np.round(np.arange(self.T, 0, -self.T / n)).astype(np.int64) - 1
        self.timesteps = torch.from_numpy(ts)
        return self.timesteps

    def coeffs(self, t: int, eta: float):
        """Scalars of one step: x_prev = c_x0*x0 + c_eps*eps + sigma*z."""
        tp = t - self.T // self.n
        a = self.alphas_cumprod[t]
        ap = self.alphas_cumprod[tp] if tp >= 0 else self.final_alpha_cumprod
        b = 1 - a
        var = ((1 - ap) / b) * (1 - a / ap)
        sigma = eta * var ** 0.5
        return a, ap, b, sigma

    def step(self, v, t: int, x, eta=0.0, noise=None):
        a, ap, b, sigma = self.coeffs(int(t), eta)
        x0 = (a ** 0.5) * x - (b ** 0.5) * v
        eps = (a ** 0.5) * v + (b ** 0.5) * x
        prev = ap ** 0.5 * x0 + (1 - ap - sigma ** 2) ** 0.5 * eps
        if eta > 0:
            prev = prev + sigma * noise
        return prev


def rescale_noise_cfg(cfg_out, text_out, guidance_rescale):
    """src/inference.py:12-23 (unbiased std over dims 1..)."""
    dims = list(range(1, text_out.ndim))
    std_t = text_out.std(dim=dims, keepdim=True)
    std_c = cfg_out.std(dim=dims, keepdim=True)
    return guidance_rescale * (cfg_out * (std_t / std_c)) + (1 - guidance_rescale) * cfg_out


def cfg_combine(out_text, out_uncond, guidance_scale, guidance_rescale):
    """src/inference.py:88-93."""
    pred = out_uncond + guidance_scale * (out_text - out_uncond)
    if guidance_rescale > 0.0:
        pred = rescale_noise_cfg(pred, out_text, guidance_rescale)
    return pred


@torch.no_grad()
def sample_loop(sd: SD, cfg, noise, text, text_mask, uncond_text=None, uncond_mask=None,
                gt=None, gt_mask=None, guidance_scale=None, guidance_rescale=0.0,
                ddim_steps=50, eta=0.0, step_noise=None, controlnet=None):
    """src/inference.py:58-105 with cached text embeddings and injected RNG draws
    (`noise` = initial latent, `step_noise[i]` = eta-noise of step i).  Batched over prompts
    (the reference is B=1; SURVEY 0.8).  `controlnet` = (sd_cn, cfg_cn, condition, scale)
    follows src/inference_controlnet.py:74-122.  Returns the final latent (before VAE)."""
    sched = DDIM()
    latents = noise
    for i, t in enumerate(sched.set_timesteps(ddim_steps)):
        if guidance_scale:
            lc = torch.cat([latents, latents], 0)
            tc = torch.cat([text, uncond_text], 0)
            mc = torch.cat([text_mask, uncond_mask], 0)
            gc = torch.cat([gt, gt], 0) if gt is not None else None
            gmc = torch.cat([gt_mask, gt_mask], 0) if gt is not None else None
        else:
            lc, tc, mc, gc, gmc = latents, text, text_mask, gt, gt_mask
        if controlnet is None:
            out, _ = maskdit_forward(sd, cfg, lc, t, tc, mc, gc, gmc)
        else:
            sd_cn, cfg_cn, cond, scale = controlnet
            x257, _ = maskdit_forward(sd, cfg, lc, t, tc, mc, gc, gmc, forward_model=False)
            cc = torch.cat([cond, cond], 0) if guidance_scale else cond
            sk = controlnet_forward(sd_cn, cfg_cn, x257, t, tc, mc, cc, scale)
            out = udit_forward(sd, cfg, x257, t, tc, mc, controlnet_skips=sk)
        if guidance_scale:
            o_t, o_u = out.chunk(2, 0)
            out = cfg_combine(o_t, o_u, guidance_scale, guidance_rescale)
        latents = sched.step(out, int(t), latents, eta, None if step_noise is None else step_noise[i])
    if gt is not None:  # inference.py:104-105
        latents = torch.where(gt_mask, latents, gt)
    return latents
