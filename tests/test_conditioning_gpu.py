"""The kernels that turn the prompt and the reference audio into DiT inputs, against float64 references of the operation each one computes.

The T5 kernels (csrc/t5.cuh: embedding gather, RMSNorm, head permute, position bias, gated GELU, and attn_simt_kernel in T5 mode: scale 1,
bias [H, L, L], key mask) and the ControlNet stem's four convolutions (conv1d_direct_kernel) run through ezb_test_cond, which launches them
with the grid and shared memory T5::forward and Dit::controlnet_stem use.  The energy condition runs through the public
ezb_energy_condition.  Tests at the end cover the T5 encoder's own bucket table, conditioning_scale 0 and fully masked attention rows.

Each reference is float64 torch computed from exactly the values the kernel read.  Tolerances follow tests/test_step_kernels_gpu.py:
  * a bf16 output: 2^-8 |ref| (one rounding) + the fp32 error of the kernel's arithmetic, propagated;
  * bf16x3 ([hi | lo | hi], kmul 3): hi + lo within 2^-16 |ref| + the same fp32 error, the third block bit-equal to the first;
  * an fp32 output: the roundings its accumulation order implies, stated per kernel.
Outputs are prefilled with a NaN sentinel and the rows past the written region must still hold it afterwards."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from ezaudio_b200 import synth, weights
from tests.test_step_kernels_gpu import _check_bf16

pytestmark = pytest.mark.gpu

SENT16 = 0x7FAB        # a bf16 NaN pattern no kernel produces
SENT32 = 0x7FC0ABCD    # an fp32 NaN pattern no kernel produces
U = 2.0 ** -24         # fp32 unit roundoff
EZB_ERR_ARG, EZB_ERR_SHAPE, EZB_ERR_UNSUPPORTED = -1, -2, -3
K_EMBED, K_RMS, K_HEADS, K_BIAS, K_GELU, K_ATTN, K_CONV = range(7)


# ------------------------------------------------------------------------------------------------------------------------------ plumbing
def _call(**kw):
    from ezaudio_b200 import _lib
    a = _lib.TestCondArgs()
    for k, v in kw.items():
        k = "in_" if k == "in" else k
        if torch.is_tensor(v):
            setattr(a, k, v.data_ptr())
        elif v is not None:
            setattr(a, k, v)
    return _lib.lib().ezb_test_cond(0, C.byref(a), _lib.stream_ptr())


def _run(**kw):
    from ezaudio_b200 import _lib
    _lib.check(_call(**kw))
    torch.cuda.synchronize()


def _sent16(rows, cols):
    return torch.full((rows, cols), SENT16, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _sent32(*shape):
    return torch.full(shape, SENT32, dtype=torch.int32, device="cuda").view(torch.float32)


def _bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _untouched(t):
    return bool((_bits(t) == (SENT32 if t.dtype == torch.float32 else SENT16)).all())


def _check_f32(got, ref, allow, what):
    err = (got.double() - ref).abs()
    i = int((err / (allow + 1e-300)).argmax())
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output"
    assert bool((err <= allow).all()), f"{what}: err {float(err.flatten()[i]):.3e} > {float(allow.flatten()[i]):.3e} at flat index {i}"
    return float(err.max())


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------------------ embedding
@pytest.mark.parametrize("M,D,vocab", [(1, 192, 50), (37, 1024, 300), (300, 2048, 32128)])
def test_t5_embed_gathers_rows_and_clamps_ids(M, D, vocab):
    g = _gen(M + D)
    table = torch.randn(vocab, D, device="cuda", generator=g)
    ids = torch.randint(0, vocab, (M,), device="cuda", generator=g, dtype=torch.int32)
    edge = torch.tensor([-1, -(2 ** 31), vocab, vocab + 7, 2 ** 31 - 1, 0, vocab - 1], dtype=torch.int32, device="cuda")
    ids[:min(M, len(edge))] = edge[:M]
    out = _sent32(M + 2, D)
    _run(kind=K_EMBED, M=M, D=D, vocab=vocab, **{"in": ids}, w=table, out=out)
    want = table[ids.long().clamp(0, vocab - 1)]
    assert torch.equal(_bits(out[:M]), _bits(want))
    assert _untouched(out[M:])


# ------------------------------------------------------------------------------------------------------------------------------ RMSNorm
def _rms_rows(M, D, g):
    """randn rows; every 5th scaled to 1e-4 (mean square 1e-8 << eps: eps sets the scale), every 7th to 1e-30 (squares underflow), every 3rd
    to 1e15 (squares near 1e30)."""
    x = torch.randn(M, D, device="cuda", generator=g)
    r = torch.arange(M, device="cuda")
    x[r % 5 == 1] *= 1e-4
    x[r % 7 == 2] *= 1e-30
    x[r % 3 == 0] *= 1e15
    return x


@pytest.mark.parametrize("D", [192, 1024, 2048])
@pytest.mark.parametrize("M", [1, 13, 100])
@pytest.mark.parametrize("kmul,outs", [(1, "16"), (3, "16"), (1, "32"), (1, "both"), (3, "both")])
def test_t5_rms(M, D, kmul, outs):
    """y = w x rsqrt(mean(x^2) + eps).  fp32 error: a lane sums D/128 float4 groups of squares, the warp tree adds 5 levels, then /D, + eps,
    rsqrtf (2 ulp) and two products: |err| <= (D/128 + 24) 2^-24 |y|."""
    eps = 1e-6
    g = _gen(M * 7 + D + kmul)
    x = _rms_rows(M, D, g)
    w = 1.0 + 0.3 * torch.randn(D, device="cuda", generator=g)
    o16 = _sent16(M + 2, kmul * D) if outs in ("16", "both") else None
    o32 = _sent32(M + 2, D) if outs in ("32", "both") else None
    _run(kind=K_RMS, M=M, D=D, kmul=kmul, eps=eps, **{"in": x}, w=w, out=o16, out32=o32)
    xd = x.double()
    ref = w.double() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
    slack = (D / 128 + 24) * U * ref.abs()
    if o32 is not None:
        _check_f32(o32[:M], ref, slack, "t5_rms out32")
        assert _untouched(o32[M:])
        if outs == "both":   # the bf16 operand is the rounding of the same fp32 values
            assert torch.equal(_bits(o16[:M, :D]), _bits(o32[:M].bfloat16()))
    if o16 is not None:
        _check_bf16(o16[:M], ref, slack, kmul, "t5_rms out16")
        assert _untouched(o16[M:])
    # eps matters: on the 1e-4 rows a kernel without it would be ~10x off
    small = torch.arange(M, device="cuda") % 5 == 1
    if bool(small.any()):
        no_eps = w.double() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True))
        assert float((no_eps[small] - ref[small]).abs().max()) > 100 * float(slack[small].max() + 2.0 ** -8 * ref[small].abs().max())


# ------------------------------------------------------------------------------------------------------------------------------ heads / bias
@pytest.mark.parametrize("B,L,H,dk", [(1, 1, 2, 64), (2, 7, 3, 32), (3, 65, 4, 96), (2, 100, 32, 64)])
def test_t5_heads_permutes_bit_exactly(B, L, H, dk):
    g = _gen(B + L + H + dk)
    qkv = torch.randn(B * L, 3 * H * dk, device="cuda", generator=g)
    n = B * H * L * dk
    q, k, v = _sent32(n + 64), _sent32(n + 64), _sent32(n + 64)
    _run(kind=K_HEADS, B=B, L=L, H=H, dk=dk, **{"in": qkv}, out=q, out32=k, out_v=v)
    want = qkv.view(B, L, 3, H, dk).permute(2, 0, 3, 1, 4).reshape(3, n)
    for i, t in enumerate((q, k, v)):
        assert torch.equal(_bits(t[:n]), _bits(want[i])), "qkv"[i]
        assert _untouched(t[n:])


@pytest.mark.parametrize("L", [1, 7, 64, 65, 100])
def test_t5_bias_looks_up_the_bucket_table(L):
    from ezaudio_b200.t5 import relative_position_buckets
    H, nb = 6, 32
    table = torch.randn(nb, H, device="cuda", generator=_gen(L))
    buckets = relative_position_buckets(L, nb, 128).cuda()
    out = _sent32(H * L * L + 64)
    _run(kind=K_BIAS, L=L, H=H, **{"in": buckets}, w=table, out=out)
    want = table[buckets.long()].permute(2, 0, 1).reshape(-1)
    assert torch.equal(_bits(out[:H * L * L]), _bits(want))
    assert _untouched(out[H * L * L:])


# ------------------------------------------------------------------------------------------------------------------------------ gated GELU
@pytest.mark.parametrize("M,F_", [(1, 64), (37, 200), (130, 1024)])
@pytest.mark.parametrize("kmul", [1, 3])
def test_t5_gated_gelu_tanh_form(M, F_, kmul):
    """gelu_new(g) h = 0.5 g (1 + tanh(sqrt(2/pi) (g + 0.044715 g^3))) h.  fp32 error: the tanh argument carries ~6 roundings (constants
    included), moving t by (1 - t^2) |arg| 6 2^-24; tanhf adds 2 ulp; the products 4 roundings of the result."""
    g_ = _gen(M + F_ + kmul)
    h = torch.randn(M, F_, device="cuda", generator=g_)
    gate = 3.0 * torch.randn(M, F_, device="cuda", generator=g_)
    sweep = torch.linspace(-20.0, 20.0, M * F_, device="cuda").view(M, F_)   # the tail where tanhf saturates, both signs
    gate[::2] = sweep[::2]
    u = torch.cat([h, gate], 1).contiguous()
    out = _sent16(M + 2, kmul * F_)
    _run(kind=K_GELU, M=M, F=F_, kmul=kmul, **{"in": u}, out=out)
    gd, hd = gate.double(), h.double()
    arg = math.sqrt(2.0 / math.pi) * (gd + 0.044715 * gd.pow(3))
    t = torch.tanh(arg)
    ref = 0.5 * gd * (1.0 + t) * hd
    slack = 0.5 * (gd * hd).abs() * ((1 - t * t) * arg.abs() * 6 * U + 4 * U) + 4 * U * ref.abs()
    _check_bf16(out[:M], ref, slack, kmul, "t5_gated_gelu")
    assert _untouched(out[M:])


# ------------------------------------------------------------------------------------------------------------------------------ T5 attention
def _t5_attn_inputs(B, H, L, dk, seed):
    g = _gen(seed)
    q = 0.5 * torch.randn(B, H, L, dk, device="cuda", generator=g)
    k = 0.5 * torch.randn(B, H, L, dk, device="cuda", generator=g)
    v = torch.randn(B, H, L, dk, device="cuda", generator=g)
    bias = 30.0 * (2 * torch.rand(H, L, L, device="cuda", generator=g) - 1)   # up to +-30
    bias[0, :, : min(L, 3)] = 30.0
    bias[-1, :, -1] = -30.0
    mask = torch.ones(B, L, dtype=torch.uint8, device="cuda")
    if B > 1:
        mask[1, max(1, L - L // 3):] = 0                      # padded key tail
    if B > 2:
        mask[2] = (torch.rand(L, device="cuda", generator=g) > 0.3).to(torch.uint8)
        mask[2, 0] = 1
    return q, k, v, bias, mask


def _t5_attn_ref(q, k, v, bias, mask):
    """fp64 softmax(q k^T + bias, masked keys excluded) v -> [B, L, H dk]; a row whose keys are all masked is the mean of V over the L keys
    (transformers adds finfo.min to every masked score)."""
    qd, kd, vd = q.double(), k.double(), v.double()
    s = qd @ kd.transpose(-1, -2) + bias.double()[None]
    keep = mask.bool()[:, None, None, :]
    s = s.masked_fill(~keep, float("-inf"))
    p = s.softmax(-1)
    none = ~keep.any(-1, keepdim=True)
    p = torch.where(none, torch.full_like(p, 1.0 / q.shape[2]), p)
    o = p @ vd
    B, H, L, dk = q.shape
    return o.permute(0, 2, 1, 3).reshape(B, L, H * dk)


def _t5_attn_slack(q, k, v, bias):
    """fp32 error of attn_simt: each score is a dk-long fma chain plus the bias (error (dk + 2) 2^-24 (sum |q_i k_i| + |bias|)), which moves
    each probability by up to twice that relatively; the P V and l sums over L keys and the per-tile rescales add (L + 32) 2^-24 max |v|."""
    B, H, L, dk = q.shape
    qk = q.double().abs() @ k.double().abs().transpose(-1, -2) + bias.double().abs()[None]
    ds = (dk + 2) * U * qk.amax(-1)                                  # [B, H, L]
    vmax = v.double().abs().amax((-1, -2))                           # [B, H]
    s = vmax[:, :, None] * (2 * 2 * ds + (L + 32) * U)               # [B, H, L]
    return s.permute(0, 2, 1)[..., None].expand(B, L, H, dk).reshape(B, L, H * dk)


def _t5_attn_run(q, k, v, bias, mask, kmul):
    B, H, L, dk = q.shape
    out = _sent16(B * L + 2, kmul * H * dk)
    _run(kind=K_ATTN, B=B, H=H, L=L, dk=dk, kmul=kmul, **{"in": q}, k=k, v=v, b=bias, key_mask=mask, out=out)
    assert _untouched(out[B * L:])
    return out[:B * L]


@pytest.mark.parametrize("dk", [32, 64, 96])
@pytest.mark.parametrize("L", [1, 63, 64, 65, 100, 129])
def test_t5_attention(dk, L):
    B, H = 3, 2
    q, k, v, bias, mask = _t5_attn_inputs(B, H, L, dk, dk * 1000 + L)
    ref = _t5_attn_ref(q, k, v, bias, mask).reshape(B * L, H * dk)
    slack = _t5_attn_slack(q, k, v, bias).reshape(B * L, H * dk)
    for kmul in (1, 3):
        got = _t5_attn_run(q, k, v, bias, mask, kmul)
        _check_bf16(got, ref, slack, kmul, f"T5 attention kmul {kmul}")
    # no mask: the same as a mask of ones, bit for bit
    a = _t5_attn_run(q, k, v, bias, None, 1)
    b = _t5_attn_run(q, k, v, bias, torch.ones_like(mask), 1)
    assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("dk,L", [(64, 1), (64, 20), (32, 65), (96, 100), (64, 129)])
def test_t5_attention_fully_masked_row_is_mean_of_v(dk, L):
    """A sample whose keys are all masked (an all-zero attention_mask row) gets the mean of V over the L keys in every query row, as
    transformers' additive finfo.min mask gives; the other samples come out bit-identical to a batch without it."""
    B, H = 3, 2
    q, k, v, bias, mask = _t5_attn_inputs(B, H, L, dk, 77 + L)
    mask[1] = 0
    ref = _t5_attn_ref(q, k, v, bias, mask)
    slack = _t5_attn_slack(q, k, v, bias)
    want_mean = v.double().mean(2)                                   # [B, H, dk]
    assert torch.allclose(ref[1].view(L, H, dk), want_mean[1][None].expand(L, H, dk))
    others = torch.tensor([0, 2], device="cuda")
    for kmul in (1, 3):
        got = _t5_attn_run(q, k, v, bias, mask, kmul).view(B, L, kmul * H * dk)
        _check_bf16(got[1], ref[1], slack[1], kmul, f"fully masked row, kmul {kmul}")
        alone = _t5_attn_run(q[others].contiguous(), k[others].contiguous(), v[others].contiguous(), bias, mask[others].contiguous(), kmul)
        assert torch.equal(_bits(got[others].reshape(2 * L, -1)), _bits(alone))


# ------------------------------------------------------------------------------------------------------------------------------ ControlNet stem
C0, C1 = synth.CONTROLNET["cond_blocks"]


def _stem_case(stage, B, L, D, g):
    """-> (input the kernel reads, weight, bias, fp64 reference) of stem convolution `stage` (oracle controlnet_embed's order)."""
    T = 2 * L
    if stage == 0:
        x = torch.rand(B, 1, T, device="cuda", generator=g)
        w, b = torch.randn(C0, 1, 1, device="cuda", generator=g), torch.randn(C0, device="cuda", generator=g)
        ref = F.conv1d(x.double(), w.double(), b.double())
    elif stage == 1:
        x = torch.randn(B, C0, T, device="cuda", generator=g)    # conv_in's output; the mask channel is appended as zeros
        w, b = 0.2 * torch.randn(C0 + 1, C0 + 1, 3, device="cuda", generator=g), torch.randn(C0 + 1, device="cuda", generator=g)
        xz = torch.cat([x.double(), torch.zeros(B, 1, T, dtype=torch.float64, device="cuda")], 1)
        ref = F.silu(F.conv1d(xz, w.double(), b.double(), padding=1))
    elif stage == 2:
        x = torch.randn(B, C0 + 1, T, device="cuda", generator=g)
        w, b = 0.2 * torch.randn(C1, C0 + 1, 3, device="cuda", generator=g), torch.randn(C1, device="cuda", generator=g)
        ref = F.silu(F.conv1d(x.double(), w.double(), b.double(), padding=1, stride=2))
    else:
        x = torch.randn(B, C1, L, device="cuda", generator=g)
        w, b = 0.2 * torch.randn(D, C1, 1, device="cuda", generator=g), torch.randn(D, device="cuda", generator=g)
        ref = F.conv1d(x.double(), w.double(), b.double()).transpose(1, 2)   # conv_out writes (B, L, D)
    xs = torch.cat([x, torch.zeros_like(x[:, :1])], 1) if stage == 1 else x
    taps = F.conv1d(xs.double().abs(), w.double().abs(), b.double().abs(), padding=w.shape[-1] // 2, stride=2 if stage == 2 else 1)
    mag = taps.transpose(1, 2) if stage == 3 else taps
    return x.contiguous(), w.contiguous(), b, ref.contiguous(), mag.contiguous(), w.shape[1] * w.shape[2]


@pytest.mark.parametrize("stage", [0, 1, 2, 3])
@pytest.mark.parametrize("L", [1, 25, 500])
def test_controlnet_stem_conv(stage, L):
    """Each convolution of Dit::controlnet_stem against F.conv1d in fp64.  fp32 error: an fma chain over Cin * K taps,
    (Cin K + 2) 2^-24 (sum |w x| + |b|), SiLU (expf and a division) 1.2x that plus 6 roundings of the result."""
    B, D = 2, 1152
    x, w, b, ref, mag, n = _stem_case(stage, B, L, D, _gen(stage * 1000 + L))
    out = _sent32(ref.numel() + 64)
    _run(kind=K_CONV, stage=stage, B=B, L=L, c0=C0, c1=C1, D=D, **{"in": x}, w=w, b=b, out=out)
    allow = 1.2 * (n + 2) * U * mag + 6 * U * ref.abs()
    _check_f32(out[:ref.numel()].view_as(ref), ref, allow, f"stem conv {stage}")
    assert _untouched(out[ref.numel():])


def test_cond_hook_refuses_bad_arguments():
    x = torch.zeros(64, device="cuda")
    assert _call(kind=7, **{"in": x}, out=x) == EZB_ERR_ARG
    assert _call(kind=K_RMS, M=4, D=6, kmul=1, eps=1e-6, **{"in": x}, w=x, out=x) == EZB_ERR_SHAPE
    assert _call(kind=K_RMS, M=4, D=8, kmul=2, eps=1e-6, **{"in": x}, w=x, out=x) == EZB_ERR_ARG
    assert _call(kind=K_ATTN, B=1, H=1, L=4, dk=30, kmul=1, **{"in": x}, k=x, v=x, b=x, out=x) == EZB_ERR_UNSUPPORTED
    assert _call(kind=K_ATTN, B=1, H=1, L=4, dk=100, kmul=1, **{"in": x}, k=x, v=x, b=x, out=x) == EZB_ERR_UNSUPPORTED
    assert _call(kind=K_ATTN, B=1, H=1, L=4, dk=32, kmul=1, **{"in": x}, k=x, v=x, out=x) == EZB_ERR_ARG
    assert _call(kind=K_HEADS, B=1, H=1, L=4, dk=8, **{"in": x}, out=x) == EZB_ERR_ARG
    assert _call(kind=K_CONV, stage=4, B=1, L=4, c0=4, c1=4, D=4, **{"in": x}, w=x, b=x, out=x) == EZB_ERR_ARG
    assert _call(kind=K_EMBED, M=2, D=8, vocab=4, **{"in": x[1:]}, w=x, out=x) == EZB_ERR_ARG   # misaligned float4 rows


# ------------------------------------------------------------------------------------------------------------------------------ energy
def _energy_ref(audio, hop, win, min_db=-60.0, norm=True, q=None):
    """EnergyExtractor.forward (src/models/conditions/energy.py:19-56) restated in fp64: (B, T) -> (B, T // hop)."""
    a = audio.double()
    n, pad = a.shape[-1] // hop, (win - hop) // 2
    p = F.pad(a[:, None], (pad, pad), mode="reflect")[:, 0]
    e = p.unfold(-1, win, hop)[:, :n].pow(2).mean(-1)
    gdb = 10 * torch.log10(torch.clamp(e, min=10 ** (min_db / 10)))
    if norm:
        gdb = (gdb - min_db) / (gdb.max(-1, keepdim=True)[0] - min_db + 1e-8)
    if q:
        gdb = torch.round(gdb * (q - 1)) / (q - 1)
    return gdb


def _energy(audio, hop, win, min_db=-60.0, norm=True, q=0):
    from ezaudio_b200 import _lib
    B, T = audio.shape
    out = _sent32(B, T // hop + 8)
    rc = _lib.lib().ezb_energy_condition(0, _lib.ptr(audio), _lib.ptr(out), B, T, hop, win, float(min_db), int(norm), int(q), _lib.stream_ptr())
    torch.cuda.synchronize()
    if rc != 0:
        return rc
    n = T // hop
    flat = out.view(-1)
    assert _untouched(flat[B * n:])
    return flat[:B * n].view(B, n)


def _energy_tol(audio, hop, win, norm, min_db=-60.0):
    """Allowed error: in dB, the fp32 sum of win squares (win / 32 lane adds + 5 tree levels), log10f (2 ulp) and the product; normalised,
    twice that over the clip's range max - min_db (the frame and the maximum both move), plus 4 roundings."""
    g = _energy_ref(audio, hop, win, min_db, norm=False)
    db = (10 / math.log(10)) * (win / 32 + 10) * U + 4 * U * (g.abs() + 1)
    if not norm:
        return db
    rng = g.max(-1, keepdim=True)[0] - min_db + 1e-8
    return 2 * db.max(-1, keepdim=True)[0] / rng + 4 * U


def _clips(B, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    env = torch.exp(3 * torch.sin(torch.linspace(0, 13, T, device="cuda")))[None]
    return (0.1 * torch.randn(B, T, device="cuda", generator=g) * env).contiguous()


@pytest.mark.parametrize("T,hop,win", [(24000, 240, 1920), (24000 + 137, 240, 1920), (1000, 240, 1920), (841, 240, 1920), (50, 8, 16),
                                       (3, 1, 3), (7, 2, 6)])
@pytest.mark.parametrize("norm,q", [(True, 0), (False, 0), (True, 16)])
def test_energy_condition(T, hop, win, norm, q):
    """T a multiple of hop or not; T just above the reflect padding ((1920 - 240) / 2 = 840 < 841); one-sample hops."""
    audio = _clips(3, T, T + hop)
    got = _energy(audio, hop, win, norm=norm, q=q)
    ref = _energy_ref(audio, hop, win, norm=norm, q=q)
    if not q:
        _check_f32(got, ref, _energy_tol(audio, hop, win, norm), f"energy norm={norm}")
    else:   # quantised: k / (q - 1) rounded to fp32, except where the unquantised value sits within the error of a rounding boundary
        raw = _energy_ref(audio, hop, win, norm=True) * (q - 1)
        near = (raw - raw.floor() - 0.5).abs() < 1e-4
        assert bool((got == ref.float())[~near].all()) and bool(((got.double() - ref).abs() <= 1.0 / (q - 1) + 1e-6).all())


def test_energy_condition_silence_constant_and_batch_independence():
    T, hop, win = 4800, 240, 1920
    clips = torch.stack([torch.zeros(T, device="cuda"), torch.full((T,), 0.25, device="cuda"), _clips(1, T, 3)[0] * 1e-3,
                         _clips(1, T, 4)[0] * 100.0]).contiguous()         # silence, a constant, levels 1e-4 and 10
    for norm in (True, False):
        got = _energy(clips, hop, win, norm=norm)
        ref = _energy_ref(clips, hop, win, norm=norm)
        assert bool(torch.isfinite(got).all())
        _check_f32(got, ref, _energy_tol(clips, hop, win, norm), f"energy norm={norm}")
        # silence hits the floor: min_db, or 0 once normalised (0 / 1e-8)
        assert bool((got[0] == (0.0 if norm else -60.0)).all())
        for b in range(clips.shape[0]):
            assert torch.equal(_bits(got[b:b + 1]), _bits(_energy(clips[b:b + 1].contiguous(), hop, win, norm=norm))), b


def test_energy_condition_refuses_what_it_cannot_compute():
    a = torch.zeros(2, 60000 * 4, device="cuda")
    assert _energy(a[:, :100].contiguous(), 240, 1920) == EZB_ERR_SHAPE        # T < hop
    assert _energy(a[:, :840].contiguous(), 240, 1920) == EZB_ERR_SHAPE        # reflect padding 840 needs more than 840 samples
    full = _energy(a[:, :51200 * 4].contiguous(), 4, 4)                        # 51200 frames fill the shared-memory table exactly
    assert torch.is_tensor(full) and bool((full == 0).all())
    assert _energy(a[:, :51201 * 4].contiguous(), 4, 4) == EZB_ERR_SHAPE       # one frame more is refused
    # an odd window - hop: the reference would pad (win - hop - 1) / 2 and return (T - 1) // hop frames; the library refuses
    assert _energy(a[:, :2400].contiguous(), 240, 1921) == EZB_ERR_UNSUPPORTED
    assert _energy(a[:, :2400].contiguous(), 2, 5) == EZB_ERR_UNSUPPORTED


# ------------------------------------------------------------------------------------------------------------------------------ T5 encoder
@pytest.mark.parametrize("L", [1, 2, 15, 16, 17, 33, 64, 100, 128])
def test_t5_library_bucket_table_equals_the_callers(L):
    """ezb_t5_forward with buckets = NULL builds the table on the host with float32 logf; at distances 16, 32 and 64 the exact bucket value
    is an integer, so the truncation (int)t must land where torch's float32 ops land.  The output is bit-equal to a run on the caller's
    table (128 = max_len, distances up to 127)."""
    from ezaudio_b200 import _lib
    from ezaudio_b200.t5 import T5EncoderModel, relative_position_buckets
    cfg = synth.tiny_t5()
    m = T5EncoderModel(cfg, precision="bf16x3", max_batch=2, max_len=128).load_state_dict(weights.synthetic_state_dict(weights.t5_param_shapes(cfg), 12))
    ids, mask = synth.synth_tokens(2, L, cfg["vocab_size"])
    i32, m8 = ids.cuda().to(torch.int32).contiguous(), mask.cuda().to(torch.uint8).contiguous()
    table = relative_position_buckets(L).cuda()
    outs = []
    for buckets in (table, None):
        o = _sent32(2, L, cfg["d_model"])
        _lib.check(_lib.lib().ezb_t5_forward(m.h, _lib.ptr(i32), _lib.ptr(m8), _lib.ptr(buckets), _lib.ptr(o), 2, L, _lib.stream_ptr()))
        torch.cuda.synchronize()
        outs.append(o)
    assert bool(torch.isfinite(outs[0]).all())
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))


@pytest.mark.parametrize("precision,tol", [("bf16x3", 1e-3), ("bf16", 6e-2)])
def test_t5_encoder_with_an_all_zero_mask_row_matches_oracle(precision, tol):
    """Cached uncond embeddings can carry an all-zero attention mask row; transformers (and the oracle) then attend uniformly over the L
    keys.  Tolerances as tests/test_t5_gpu.py."""
    from ezaudio_b200.t5 import T5EncoderModel
    from oracle import ezaudio_oracle as O
    cfg = synth.tiny_t5()
    sd = weights.synthetic_state_dict(weights.t5_param_shapes(cfg), 12)
    ids, mask = synth.synth_tokens(3, 20, cfg["vocab_size"])
    mask[1] = 0
    m = T5EncoderModel(cfg, precision=precision, max_batch=3, max_len=20).load_state_dict(sd)
    out = m(input_ids=ids.cuda(), attention_mask=mask.cuda()).last_hidden_state
    with torch.no_grad():
        ref = O.t5_encode(sd, cfg, ids, mask)
    assert bool(torch.isfinite(out).all())
    err = (out.cpu() - ref).abs()
    assert float(err.max()) < tol, float(err.max())


# ------------------------------------------------------------------------------------------------------------------------------ DiT attention
def _attn_operands(impl, q, k, v):
    """impl 0 reads fp32 [B, H, L, dh]; the tensor-core generations bf16 q / k rows of dhp and V^T [B*H, dvp, Lk padded to 8]."""
    if impl == 0:
        return q.contiguous(), k.contiguous(), v.contiguous()
    B, H, Lq, dh = q.shape
    Lk = k.shape[2]
    dhp, dvp, lkp = (80 if impl >= 100 and dh == 72 else (dh + 63) // 64 * 64), (dh + 15) // 16 * 16, (Lk + 7) // 8 * 8
    qb = torch.zeros(B * H, Lq, dhp, device="cuda", dtype=torch.bfloat16)
    kb = torch.zeros(B * H, Lk, dhp, device="cuda", dtype=torch.bfloat16)
    vt = torch.zeros(B * H, dvp, lkp, device="cuda", dtype=torch.bfloat16)
    qb[:, :, :dh] = q.reshape(B * H, Lq, dh)
    kb[:, :, :dh] = k.reshape(B * H, Lk, dh)
    vt[:, :dh, :Lk] = v.reshape(B * H, Lk, dh).transpose(1, 2)
    vt[:, :, Lk:] = 7.0
    return qb, kb, vt


def _attention(impl, q, k, v, mask):
    from ezaudio_b200 import _lib
    B, H, Lq, dh = q.shape
    ops = _attn_operands(impl, q, k, v)
    out = _sent16(B * Lq, H * dh)
    _lib.check(_lib.lib().ezb_test_attention(0, _lib.ptr(ops[0]), _lib.ptr(ops[1]), _lib.ptr(ops[2]), _lib.ptr(mask), _lib.ptr(out), B, H, Lq,
                                             k.shape[2], dh, impl, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out.view(B, Lq, H * dh)


@pytest.mark.parametrize("impl", [0, 4, 6, 7, 8, 104, 106, 108])
@pytest.mark.parametrize("Lq,Lk,dh", [(40, 12, 72), (130, 100, 64), (500, 385, 72)])
def test_attention_fully_masked_row_is_zero(impl, Lq, Lk, dh):
    """A sample whose keys are all masked comes out as zeros from every attention kernel (SDPA with a boolean mask returns zeros there);
    the partly masked samples come out bit-identical to a batch without it."""
    B, H = 3, 2
    g = _gen(impl + Lq + dh)
    q = 1.5 * torch.randn(B, H, Lq, dh, device="cuda", generator=g)
    k = 1.5 * torch.randn(B, H, Lk, dh, device="cuda", generator=g)
    v = torch.randn(B, H, Lk, dh, device="cuda", generator=g)
    mask = torch.zeros(B, Lk, dtype=torch.uint8, device="cuda")
    mask[0, :8] = 1
    mask[2] = (torch.rand(Lk, device="cuda", generator=g) > 0.5).to(torch.uint8)
    mask[2, -1] = 1
    got = _attention(impl, q, k, v, mask)
    assert bool((got[1].float() == 0).all()), f"fully masked sample: {got[1].float().abs().max()}"
    keep = torch.tensor([0, 2], device="cuda")
    alone = _attention(impl, q[keep], k[keep], v[keep], mask[keep].contiguous())
    assert torch.equal(_bits(got[keep]), _bits(alone))


def test_oracle_attention_gives_zeros_for_a_fully_masked_row():
    from oracle import ezaudio_oracle as O
    D, H = 16, 2
    g = torch.Generator().manual_seed(0)
    sd = {f"a.{n}.weight": torch.randn(D, D, generator=g) for n in ("to_q", "to_k", "to_v", "proj")}
    sd.update({"a.proj.bias": torch.zeros(D), "a.norm_q.weight": torch.ones(D // H), "a.norm_q.bias": torch.zeros(D // H),
               "a.norm_k.weight": torch.ones(D // H), "a.norm_k.bias": torch.zeros(D // H)})
    x, ctx = torch.randn(2, 5, D, generator=g), torch.randn(2, 3, D, generator=g)
    cm = torch.tensor([[True, False, True], [False, False, False]])
    out = O.attention(x, sd, "a", H, context=ctx, context_mask=cm)
    assert torch.equal(out[1], F.linear(torch.zeros(5, D), sd["a.proj.weight"], sd["a.proj.bias"]))
    assert bool(torch.isfinite(out).all())


# ------------------------------------------------------------------------------------------------------------------------------ conditioning_scale 0
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_controlnet_scale_zero_gives_zero_skips(precision):
    """conditioning_scale 0 multiplies the skips by 0 (controlnet.py:311-313): ezb_controlnet_forward writes zeros, as the device-scale path
    does, and a later non-zero scale is unaffected."""
    from tests.test_controlnet_engine_gpu import _cond, _controlnet, _host_index_forward, _tdev_forward
    Be, L, Lc = 4, 96, 12
    cfg, net = _controlnet("tiny", precision, Be, L, Lc)
    x = synth.synth_latents(Be, L).cuda()
    cond = _cond(Be, L, 9)
    net.set_condition(cond)
    before = _host_index_forward(net, x, [0, 2, 4, 1], cond, 0.5)
    outs = [_sent32(Be, L, cfg["embed_dim"]) for _ in range(net.half)]
    got = [o.clone() for o in net.forward_step(x, 2, cond, 0.0, outs=outs)]
    tdev = _tdev_forward(net, x, [2] * Be, [0.0] * Be)
    torch.cuda.synchronize()
    for gz, tz in zip(got, tdev):
        assert bool((gz == 0).all()) and torch.equal(gz, tz)
    after = _host_index_forward(net, x, [0, 2, 4, 1], cond, 0.5)
    torch.cuda.synchronize()
    for b, a in zip(before, after):
        assert bool((a != 0).any()) and torch.equal(_bits(a), _bits(b))


def test_generate_audio_conditioning_scale_zero_matches_oracle_loop(monkeypatch):
    """EzAudio_ControlNet.generate_audio(conditioning_scale=0) on the tiny models: the latents match the fp32 oracle loop at scale 0 (and
    differ from it at scale 1 by far more than the tolerance)."""
    from ezaudio_b200 import inference, post
    from ezaudio_b200.api import energy_condition
    from oracle import ezaudio_oracle as O
    from tests.test_controlnet_engine_gpu import _clip, _tiny_cn
    ez = _tiny_cn("bf16x3", max_batch=1)
    cfg = ez.params["model"]
    seen = {}
    real = inference.sample_latents

    def spy(*a, **kw):
        seen["lat"] = real(*a, **kw)
        return seen["lat"]

    monkeypatch.setattr(inference, "sample_latents", spy)
    clip, seed = _clip(2, 31), 11
    ez.generate_audio("a siren", clip, guidance_scale=3.5, ddim_steps=3, eta=0, conditioning_scale=0, random_seed=seed)
    got = seen["lat"].cpu()
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 5)
    sd_cn = weights.synthetic_state_dict(weights.controlnet_param_shapes(cfg, synth.CONTROLNET), 6)
    noise = torch.randn((1, 128, 500), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda").cpu()
    ckw = {k: v for k, v in ez.params["conditioner"].items() if k != "condition_type"}
    cond = energy_condition(post.prepare_wave(torch.from_numpy(clip).cuda().unsqueeze(0), 240000, normalize=True, gate=0.0), **ckw).cpu()
    ctx, mask = ez.encode_text(["a siren"])
    uctx, umask = ez.encode_text([""])
    refs = {}
    with torch.no_grad():
        for s in (0.0, 1.0):
            refs[s] = O.sample_loop(sd, cfg, noise, ctx.cpu(), mask.cpu(), uctx.cpu(), umask.cpu(), guidance_scale=3.5, guidance_rescale=0,
                                    ddim_steps=3, eta=0.0, controlnet=(sd_cn, cfg, cond, s))
    err = float((got - refs[0.0]).abs().max())
    assert err < 5e-3, err
    assert float((refs[1.0] - refs[0.0]).abs().max()) > 20 * 5e-3
