"""FP8 mode (precision "fp8", include/ezb200.h): its kernels through ezb_test_fp8 against fp64 references of the dequantised operands, and
whole forwards against the oracle's FP8 emulation (tests/fp8_emulation.py) and the reference goldens.

Kernel bounds.  The GEMM references are fp64 products of exactly the e4m3 values and scales the kernels read (the hook returns the packed
weight), through the same epilogue math, so what remains is the fp32 / tensor-core accumulation and the bf16 rounding of the output:
    |got - ref| <= 2^-8 |ref| + FP8_ACC    per element (mean: 0.75 * 2^-8 mean |ref| + FP8_ACC).
FP8_ACC bounds the accumulation error of e4m3 wgmma over K = 1024 / 1152 on O(1) projections, read off the printed "excess over one bf16
rounding" on an H100 (700 W): largest 8.1e-3 after the per-head LayerNorm (|w| / std(u) <= 2 scales it: bound 2 FP8_ACC) and 3.0e-2 after
GEGLU, whose product h * gelu(g) of two projections of |.| <~ 5 scales it up to 8x (bound 8 FP8_ACC).  DESIGN.md section 3 compares it with
the operand quantisation error.
Model bounds.  Against the reference goldens: FP8_TOL of tests/test_fp8_host.py (the emulation's own distance from them, with margin).
Against the FP8 emulation: TOL_EMU, measured max 0.127 / mean 0.019 (dit_tiny72), 0.121 / 0.018 (dit_XL), with 1.5x margin.  The bf16 mode's
6e-2 / 1.2e-2 cannot hold here: the bf16 operands of the other layers move each norm1 / norm3 output by ~2^-8, which sends a few percent of
the elements to the neighbouring e4m3 value (a 2^-4 step) and the two runs drift apart by a fraction of the FP8 noise itself."""
import ctypes as C
import math

import pytest
import torch

from ezaudio_b200 import synth, weights
from tests import helpers
from tests.test_fp8_host import FP8_TOL
from tests.test_heads_gpu import ROPE_MUFU, _dvp, _lpad, _reference

pytestmark = pytest.mark.gpu

FP8_ACC = 8e-3
TOL_EMU = (0.2, 0.03)


def _e4m3(q):
    return q.view(torch.float8_e4m3fn).double()


def _call(a):
    from ezaudio_b200 import _lib
    _lib.check(_lib.lib().ezb_test_fp8(0, C.byref(a), _lib.stream_ptr()))
    torch.cuda.synchronize()


def _ln_quant(x, w, b, shift, scale):
    from ezaudio_b200 import _lib
    M, D = x.shape
    q = torch.empty(M, D, dtype=torch.uint8, device="cuda")
    s = torch.empty(M, device="cuda")
    a = _lib.TestFp8Args(kind=0, M=M, D=D, x=x.data_ptr(), weight=w.data_ptr(), bias=b.data_ptr(),
                         shift=None if shift is None else shift.data_ptr(), scale=None if scale is None else scale.data_ptr(), q=q.data_ptr(),
                         s=s.data_ptr())
    _call(a)
    return q, s


def _operand(M, D, seed):
    """A LayerNorm-like e4m3 operand with row scales, made by the kernel under test in kind 0."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 1
    w, b = 1 + 0.3 * torch.randn(D, device="cuda", generator=g), 0.3 * torch.randn(D, device="cuda", generator=g)
    return _ln_quant(x, w, b, None, None)


@pytest.mark.parametrize("D,modulate", [(1152, True), (1024, False), (144, True)])
def test_layernorm_quantise(D, modulate):
    M = 333
    g = torch.Generator(device="cuda").manual_seed(D)
    x = torch.randn(M, D, device="cuda", generator=g) * 2 + 0.5
    w, b = 1 + 0.3 * torch.randn(D, device="cuda", generator=g), 0.3 * torch.randn(D, device="cuda", generator=g)
    shift, scale = (0.5 * torch.randn(D, device="cuda", generator=g), 0.5 * torch.randn(D, device="cuda", generator=g)) if modulate else (None, None)
    q, s = _ln_quant(x, w, b, shift, scale)
    xd = x.double()
    y = (xd - xd.mean(-1, keepdim=True)) / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-5) * w.double() + b.double()
    if modulate:
        y = y * (1 + scale.double()) + shift.double()
    s_ref = y.abs().amax(-1) / 448
    assert float(((s.double() - s_ref).abs() / s_ref).max()) < 1e-5          # fp32 round-off of the LayerNorm and the division
    deq = _e4m3(q) * s.double()[:, None]
    u = (y / s_ref[:, None]).abs()                                            # position on the e4m3 grid
    step = torch.exp2(torch.clamp(torch.floor(torch.log2(u.clamp_min(1e-30))), min=-6) - 3) * s_ref[:, None]
    err = (deq - y).abs()
    print(f"[fp8 ln] D {D}: max error / e4m3 step {float((err / step).max()):.3f}")
    assert bool((err <= step).all())


def _geglu_ref(A, W, bp, inner):
    u = A @ W.T + bp                                   # packed columns: per 256-wide tile 128 hidden then 128 gate
    u = u.reshape(u.shape[0], -1, 2, 128)
    h, gt = u[:, :, 0], u[:, :, 1]
    return (h * 0.5 * gt * (1 + torch.special.erf(gt / math.sqrt(2)))).reshape(u.shape[0], inner)


@pytest.mark.parametrize("D,inner", [(1152, 4608), (1024, 4096)])
@pytest.mark.parametrize("M", [128, 4000, 333])
def test_geglu_fp8(D, inner, M):
    from ezaudio_b200 import _lib
    q, s = _operand(M, D, M + D)
    g = torch.Generator(device="cuda").manual_seed(7)
    W = torch.randn(2 * inner, D, device="cuda", generator=g) / math.sqrt(D)
    b = 0.1 * torch.randn(2 * inner, device="cuda", generator=g)
    out = torch.empty(M, inner, dtype=torch.bfloat16, device="cuda")
    wq = torch.empty(2 * inner, D, dtype=torch.uint8, device="cuda")
    ws = torch.empty(2 * inner, device="cuda")
    a = _lib.TestFp8Args(kind=1, M=M, D=D, q=q.data_ptr(), s=s.data_ptr(), inner=inner, w=W.data_ptr(), b=b.data_ptr(), out=out.data_ptr(),
                         w_q=wq.data_ptr(), w_s=ws.data_ptr())
    _call(a)
    # packing: output row (m // 128) * 256 + g * 128 + m % 128 holds reference row g * inner + m (g = 0 hidden, 1 gate)
    idx = torch.arange(2 * inner, device="cuda")
    src = (idx % 256 >= 128).long() * inner + (idx // 256) * 128 + idx % 128
    Wd = _e4m3(wq) * ws.double()[:, None]
    ws_ref = W[src].bfloat16().double().abs().amax(-1) / 448
    assert float(((ws.double() - ws_ref).abs() / ws_ref).max()) < 1e-6
    ref = _geglu_ref(_e4m3(q) * s.double()[:, None], Wd, b[src].double(), inner)
    err = (out.double() - ref).abs()
    excess = err - 2.0 ** -8 * ref.abs()
    print(f"[fp8 geglu] M {M} D {D}: max-abs {float(err.max()):.3e}, largest excess over one bf16 rounding {float(excess.max()):.3e}")
    assert bool((excess <= 8 * FP8_ACC).all())
    assert float(err.mean()) <= 0.75 * 2.0 ** -8 * float(ref.abs().mean()) + FP8_ACC


@pytest.mark.parametrize("dh,H", [(72, 16), (64, 16)])
@pytest.mark.parametrize("B,L", [(1, 128), (8, 500), (3, 111)])
def test_qkv_heads_fp8(dh, H, B, L):
    from ezaudio_b200 import _lib
    D, M = H * dh, B * L
    q, s = _operand(M, D, M + dh)
    g = torch.Generator(device="cuda").manual_seed(11)
    W = torch.randn(3 * D, D, device="cuda", generator=g) / math.sqrt(D)
    nq = torch.stack([1 + 0.3 * torch.randn(dh, device="cuda", generator=g), 0.3 * torch.randn(dh, device="cuda", generator=g)]).contiguous()
    nk = torch.stack([1 + 0.3 * torch.randn(dh, device="cuda", generator=g), 0.3 * torch.randn(dh, device="cuda", generator=g)]).contiguous()
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dh, 2, device="cuda", dtype=torch.float32) / dh))
    ld_qk, dvp, Lpad, bn = (80 if dh == 72 else 64), _dvp(dh), _lpad(L), (224 if dh == 72 else 192)
    outs = {0: torch.zeros(B * H, L, ld_qk, dtype=torch.bfloat16, device="cuda"), 1: torch.zeros(B * H, L, ld_qk, dtype=torch.bfloat16, device="cuda"),
            2: torch.zeros(B * H, dvp, Lpad, dtype=torch.bfloat16, device="cuda")}
    wq = torch.empty(H * bn, D, dtype=torch.uint8, device="cuda")
    ws = torch.empty(H * bn, device="cuda")
    a = _lib.TestFp8Args(kind=2, M=M, D=D, q=q.data_ptr(), s=s.data_ptr(), w=W.data_ptr(), B=B, L=L, H=H, dh=dh, norm_q=nq.data_ptr(),
                         norm_k=nk.data_ptr(), inv_freq=inv_freq.data_ptr(), rope=ROPE_MUFU, q_out=outs[0].data_ptr(), k_out=outs[1].data_ptr(),
                         vt_out=outs[2].data_ptr(), ld_qk=ld_qk, dvp=dvp, Lpad=Lpad, w_q=wq.data_ptr(), w_s=ws.data_ptr())
    _call(a)
    # unpack: global head gh of [q | k | v] sits at rows (gh // 3) * bn + (gh % 3) * dh of the packed weight
    gh = torch.arange(3 * H, device="cuda")
    rows = ((gh // 3) * bn + (gh % 3) * dh)[:, None] + torch.arange(dh, device="cuda")[None]
    Wd = (_e4m3(wq) * ws.double()[:, None])[rows.reshape(-1)]
    u = (_e4m3(q) * s.double()[:, None]) @ Wd.T
    refs = _reference(u, B=B, L=L, H=H, dh=dh, kinds=(0, 1, 2), nq=nq, nk=nk, inv_freq=inv_freq, rope=ROPE_MUFU)
    for kd in (0, 1, 2):
        ref, extra = refs[kd]
        got = outs[kd][:, :dh, :L].double() if kd == 2 else outs[kd][:, :, :dh].double()
        err = (got - ref).abs()
        excess = err - 2.0 ** -8 * ref.abs()
        print(f"[fp8 heads] dh {dh} M {M} kind {kd}: max-abs {float(err.max()):.3e}, largest excess over one bf16 rounding {float((excess - extra).max()):.3e}")
        assert bool((excess <= 2 * FP8_ACC + extra).all()), kd          # per-head LayerNorm: |w| / std(u) <= 2 scales the accumulation error
        assert float(err.mean()) <= 0.75 * 2.0 ** -8 * float(ref.abs().mean()) + 2 * FP8_ACC + float(extra.mean() if extra.dim() else 0.0)


def _dit_fp8(name):
    from ezaudio_b200.dit import MaskDiT
    from tests import fp8_emulation as E
    cfg, sd, inp, g = helpers.dit_case_inputs(name)
    B, _, L = inp["x"].shape
    m = MaskDiT(precision="fp8", max_batch=B, max_len=L, max_ctx_len=inp["ctx"].shape[1], max_timesteps=8, **cfg).load_state_dict(sd)
    out, _ = m(inp["x"].cuda(), inp["t"], inp["ctx"].cuda(), context_mask=inp["mask"].cuda())
    out = out.cpu()
    with torch.no_grad():
        emu, _ = E.maskdit_forward(sd, cfg, inp["x"], inp["t"], inp["ctx"], inp["mask"])
    return out, emu, g


@pytest.mark.parametrize("name", ["dit_tiny72", "dit_tiny64", "dit_XL"])
def test_maskdit_fp8(name):
    out, emu, g = _dit_fp8(name)
    assert torch.isfinite(out).all()
    e = (out - emu).abs()
    r = (helpers.golden_view(g, out) - torch.from_numpy(g["out"])).abs()
    print(f"[fp8] {name}: vs FP8 emulation max {float(e.max()):.3e} mean {float(e.mean()):.3e}; vs reference golden max {float(r.max()):.3e} "
          f"mean {float(r.mean()):.3e}")
    assert float(e.max()) < TOL_EMU[0] and float(e.mean()) < TOL_EMU[1]
    assert float(r.max()) < FP8_TOL[0] and float(r.mean()) < FP8_TOL[1]


def test_controlnet_fp8():
    from ezaudio_b200.dit import DiTControlNet
    from oracle import ezaudio_oracle as O
    from tests import fp8_emulation as E
    cfg, cn, L, Lc = synth.tiny_model(72), synth.CONTROLNET, 40, 12
    g = helpers.load_golden("controlnet_tiny72")
    stride = int(g["skip_stride"]) if "skip_stride" in g.files else 1
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 5)
    sd_cn = weights.synthetic_state_dict(weights.controlnet_param_shapes(cfg, cn), 6)
    x = synth.synth_latents(2, L)
    ctx, mask = synth.synth_context(2, Lc, cfg["context_dim"])
    cond = torch.rand(2, 1, 2 * L, generator=torch.Generator().manual_seed(9))
    t = torch.tensor(499)
    with torch.no_grad():
        x257, _ = O.maskdit_forward(sd, cfg, x, t, ctx, mask, forward_model=False)
        emu = E.controlnet_forward(sd_cn, cfg, x257, t, ctx, mask, cond, 0.8)
    kw = dict(precision="fp8", max_batch=2, max_len=L, max_ctx_len=Lc, max_timesteps=8)
    net = DiTControlNet(**kw, **cfg, **cn).load_state_dict(sd_cn, mask_embed=sd["mask_embed"])
    skips = [s.cpu() for s in net(x257.cuda(), t, ctx.cuda(), context_mask=mask.cuda(), condition=cond.cuda(), conditioning_scale=0.8)]
    for i, key in ((0, "skip0"), (len(skips) - 1, "skip_last")):
        e = (skips[i] - emu[i]).abs()
        r = (skips[i][:, ::stride] - torch.from_numpy(g[key])).abs()
        print(f"[fp8] controlnet {key}: vs emulation max {float(e.max()):.3e} mean {float(e.mean()):.3e}; vs golden max {float(r.max()):.3e}")
        assert torch.isfinite(skips[i]).all()
        assert float(e.max()) < TOL_EMU[0] and float(e.mean()) < TOL_EMU[1]
        assert float(r.max()) < FP8_TOL[0] and float(r.mean()) < FP8_TOL[1]


@pytest.mark.parametrize("dh", [72, 64])
def test_fp8_padded_batch_matches_solo_runs(dh):
    """NaN in every padded input frame stays in its own rows: per-row scales keep it out of the valid rows' operands."""
    from ezaudio_b200.dit import MaskDiT
    from tests.test_varlen_gpu import _padded_vs_solo, _same_kernels
    cfg = synth.tiny_model(dh)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    lens, L, Lc, t = [96, 70, 33, 20], 96, 12, 479
    x = synth.synth_latents(len(lens), L)
    ctx, mask = synth.synth_context(len(lens), Lc, cfg["context_dim"])
    m = MaskDiT(precision="fp8", max_batch=len(lens), max_len=L, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    got, solo = _padded_vs_solo(m, x, ctx, mask, t, lens)
    for b, n in enumerate(lens):
        assert torch.isfinite(got[b]).all(), (b, n)
        if _same_kernels("bf16", len(lens), L, n):
            assert torch.equal(got[b], solo[b]), (b, n, float((got[b] - solo[b]).abs().max()))
        else:
            assert float((got[b] - solo[b]).abs().max()) < TOL_EMU[0], (b, n)


def test_ezaudio_fp8_end_to_end(monkeypatch):
    from ezaudio_b200 import api, config
    from tests.test_api_gpu import _tiny_params
    tiny = _tiny_params()
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    seen = []
    real = api.OobleckDecoder
    monkeypatch.setattr(api, "OobleckDecoder", lambda **kw: seen.append(kw["precision"]) or real(**kw))
    ez = api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16), max_batch=2,
                     max_length_s=2, precision="fp8")
    assert seen == ["bf16"] and ez.unet.precision == "fp8"
    sr, wav = ez.generate_audio("a dog barks", length=1, ddim_steps=4, random_seed=7)
    assert sr == 24000 and wav.shape == (24000,) and bool(torch.isfinite(torch.from_numpy(wav)).all())
