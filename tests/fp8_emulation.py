"""CPU emulation of the library's FP8 mode (precision "fp8") on top of the oracle (oracle/ezaudio_oracle.py, used unchanged): the operands
of every block's self-attention QKV and GEGLU up-projections -- the norm1 / norm3 outputs and those weights -- pass through fp8_rows,
nothing else changes.  The weights are rounded to bf16 first, as the library quantises its packed bf16 copy."""
import contextlib

import torch

from oracle import ezaudio_oracle as O

FP8_WEIGHTS = (".to_q.weight", ".to_k.weight", ".to_v.weight")


def fp8_rows(x):
    """Every row (last dim) quantised to e4m3 with its own fp32 scale s = amax / 448, q = e4m3(x * (448 / amax)) rounded to nearest even
    and saturated (amax = 0: zeros), then dequantised as q * s in x's dtype."""
    xf = x.float()
    amax = xf.abs().amax(-1, keepdim=True)
    inv = torch.where(amax > 0, 448.0 / amax, torch.zeros_like(amax))
    q = (xf * inv).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    return q.to(x.dtype) * (amax / 448.0).to(x.dtype)


def _w(w):
    return fp8_rows(w.to(torch.bfloat16).to(w.dtype))


@contextlib.contextmanager
def emulate():
    """Inside the block, O.dit_block (and everything built on it) runs the FP8 mode's numerics."""
    attention, feed_forward = O.attention, O.feed_forward

    def attention8(x, sd, p, H, context=None, context_mask=None, use_rope=False):
        if context is not None:   # cross-attention: unchanged
            return attention(x, sd, p, H, context, context_mask, use_rope)
        sd = dict(sd, **{p + k: _w(sd[p + k]) for k in FP8_WEIGHTS})
        return attention(fp8_rows(x), sd, p, H, None, None, use_rope)

    def feed_forward8(x, sd, p):
        k = p + ".net.0.proj.weight"
        return feed_forward(fp8_rows(x), dict(sd, **{k: _w(sd[k])}), p)

    O.attention, O.feed_forward = attention8, feed_forward8
    try:
        yield
    finally:
        O.attention, O.feed_forward = attention, feed_forward


def maskdit_forward(*args, **kw):
    with emulate():
        return O.maskdit_forward(*args, **kw)


def controlnet_forward(*args, **kw):
    with emulate():
        return O.controlnet_forward(*args, **kw)
