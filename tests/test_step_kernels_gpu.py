"""The bandwidth kernels of a DiT step (csrc/elementwise.cuh) against float64 references of the operation each one computes.

The LayerNorm family, qk_prep, patch_pack, final_conv, small_linear and timestep_embed run through ezb_test_step, which launches them with the
grid and shared memory the model uses (csrc/dit.cuh ln_launch and friends; for the LayerNorm, "auto" is the model's own kernel selection).
cfg_ddim runs through the public ezb_cfg_ddim_step.  Two tests at the end drive the model itself through schedules longer than the
timestep-upload chunk (240 entries) and than the precombined LayerNorm tables (128 entries).

Each reference is float64 torch computed from exactly the values the kernel read (the same fp32 inputs; the bf16 values where the kernel
reads bf16).  Tolerances:
  * a bf16 output: 2^-8 |ref| (one rounding to nearest) + the fp32 error of the kernel's arithmetic, propagated;
  * bf16x3 ([hi | lo | hi], kmul 3): hi + lo within 2^-16 |ref| + the same fp32 error, the third block bit-equal to the first;
  * an fp32 output: a few fp32 roundings of the accumulated magnitude (stated per kernel below).
The fp32 error of a LayerNorm is dominated by the mean: a lane sums 4 NCH values, the warp tree adds 5 levels, so |mu_err| <= 48 * 2^-24 *
max |x| and the normalised value moves by that times rstd.  Rows with mean 100 and std 1e-2 make this visible (a one-pass E[x^2] - E[x]^2
variance loses every digit there); rows with mean 0 and std 1e-2 make the 1e-5 in rstd = (var + 1e-5)^-1/2 a 4 % effect.
Outputs are prefilled with a bf16 NaN sentinel or fp32 NaN, and every region a kernel must not write (rows >= M, frames >= lens[b], V^T columns
>= L, pitch padding, the padded frames of cfg_ddim's latents) must still hold it afterwards."""
import contextlib
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tests import helpers

pytestmark = pytest.mark.gpu

SENT = 0x7FAB   # a bf16 NaN pattern no kernel produces
EZB_ERR_ARG, EZB_ERR_SHAPE, EZB_ERR_UNSUPPORTED = -1, -2, -3
K_LN, K_QK, K_PATCH, K_FCONV, K_SLIN, K_TEMB = range(6)
AUTO, GENERIC, REG1, REG8, GC, CAT = range(6)
VARIANT_NAMES = {AUTO: "auto", GENERIC: "generic", REG1: "reg1", REG8: "reg8", GC: "gc", CAT: "cat"}
LN_SLACK = 48 * 2.0 ** -24   # LayerNorm mean error per unit of max |x| (lane chain of <= 36 adds + 5 tree levels, with margin)


# ------------------------------------------------------------------------------------------------------------------------------ plumbing
def _args(**kw):
    from ezaudio_b200 import _lib
    a = _lib.TestStepArgs()
    for k, v in kw.items():
        if k in ("kinds", "col_off"):
            for i, e in enumerate(v):
                getattr(a, k)[i] = e
        elif k in ("f32_out", "bf_out"):
            for i, e in enumerate(v):
                getattr(a, k)[i] = None if e is None else e.data_ptr()
        elif torch.is_tensor(v):
            setattr(a, k, v.data_ptr())
        elif v is not None:
            setattr(a, k, v)
    return a


def _call(**kw):
    from ezaudio_b200 import _lib
    return _lib.lib().ezb_test_step(0, C.byref(_args(**kw)), _lib.stream_ptr())


def _run(**kw):
    from ezaudio_b200 import _lib
    _lib.check(_call(**kw))
    torch.cuda.synchronize()


def _sentinel(n):
    return torch.full((n,), SENT, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _is_sent(t):
    return bool((_bits(t) == SENT).all())


def _split(x, kmul):
    """fp32 [..., K] -> the bf16 operand the kernels store: hi, or [hi | lo | hi]."""
    hi = x.bfloat16()
    if kmul == 1:
        return hi
    return torch.cat([hi, (x - hi.float()).bfloat16(), hi], -1)


def _check_bf16(got, ref, slack, kmul, what):
    """got bf16 [M, kmul*D] vs float64 ref [M, D] with the fp32 allowance `slack`; returns (max |err|, max err / allowance)."""
    D = ref.shape[-1]
    hi = got[:, :D].double()
    if kmul == 1:
        val, rnd = hi, 2.0 ** -8
    else:
        assert torch.equal(_bits(got[:, 2 * D:]), _bits(got[:, :D])), f"{what}: third block != hi"
        val, rnd = hi + got[:, D:2 * D].double(), 2.0 ** -16
    err = (val - ref).abs()
    allow = rnd * ref.abs() + (1 + 2.0 ** -7) * slack + 1e-30
    q = err / allow
    i = int(q.argmax())
    assert bool((err <= allow).all()), f"{what}: err {float(err.flatten()[i]):.3e} > {float(allow.flatten()[i]):.3e} at {divmod(i, D)}"
    assert float(err.mean()) <= 0.5 * float(allow.mean()), f"{what}: mean err {float(err.mean()):.3e} vs allowance {float(allow.mean()):.3e}"
    return float(err.max()), float(q.max())


OPTION_DEFAULTS = {"ln_variant": 2, "ln_tail": 0, "ln_fold": 0}


@contextlib.contextmanager
def _options(**kw):
    from ezaudio_b200 import _lib
    L = _lib.lib()
    for k, v in kw.items():
        _lib.check(L.ezb_set_option(k.encode(), int(v)))
    try:
        yield
    finally:
        for k in kw:
            _lib.check(L.ezb_set_option(k.encode(), OPTION_DEFAULTS[k]))


def _ln_counts():
    from ezaudio_b200 import _lib
    return {v: int(_lib.lib().ezb_ln_launch_count(v)) for v in (GENERIC, REG1, REG8, GC, CAT)}


# ------------------------------------------------------------------------------------------------------------------------------ LayerNorm
def _ln_rows(M, D, g):
    """randn rows, every 7th shifted to mean 100 / std 1e-2, every 11th scaled to std 1e-2."""
    x = torch.randn(M, D, device="cuda", generator=g)
    r = torch.arange(M, device="cuda")
    big, small = r % 7 == 3, r % 11 == 5
    x[big] = 100.0 + 1e-2 * x[big]
    x[small] = 1e-2 * x[small]
    return x


def _ln_params(D, g):
    return 1.0 + 0.2 * torch.randn(D, device="cuda", generator=g), 0.2 * torch.randn(D, device="cuda", generator=g)


def _mod_table(M, D, mode, g):
    """-> (table, shift view, scale view, mod_bstride, rows_per_batch): shift / scale live in one [batches, 3 D] table as in the model's
    [t][block][6 D] modulation rows (stride > D)."""
    if mode is None:
        return None, None, None, 0, 1
    rpb = 1 if mode == "shared" else mode
    nb = 1 if mode == "shared" else (M + rpb - 1) // rpb
    tab = 0.3 * torch.randn(nb, 3 * D, device="cuda", generator=g)
    return tab, tab[:, :D], tab[:, D:2 * D], (0 if mode == "shared" else 3 * D), rpb


def _ln_ref(x, x2=None, x3=None, w=None, b=None, tab=None, mbs=0, rpb=1, G=None, Cc=None):
    """float64 LayerNorm (+ modulate) of the fp32 values the kernel reads -> (ref, fp32 allowance)."""
    xs = x if x2 is None else torch.cat([x, x2 if x3 is None else x2 + x3], 1)   # x2 + x3: the kernel's fp32 add
    xs = xs.double()
    M, D = xs.shape
    if w is None and G is None:
        return xs, torch.zeros_like(xs)
    mu = xs.mean(1, keepdim=True)
    rstd = (((xs - mu) ** 2).mean(1, keepdim=True) + 1e-5).rsqrt()
    xh = (xs - mu) * rstd
    if G is not None:
        gain, y = G.double().expand(M, D), xh * G.double() + Cc.double()
        mag = (xh * gain).abs() + Cc.double().abs()
    else:
        w, b = w.double(), b.double()
        y, gain = xh * w + b, w.expand(M, D)
        mag = (xh * w).abs() + b.abs()
        if tab is not None:
            flat = tab.double().flatten()
            idx = (torch.arange(M, device="cuda") // rpb * mbs)[:, None] + torch.arange(D, device="cuda")[None]
            sh, sc = flat[idx], flat[idx + D]
            y, gain, mag = y * (1 + sc) + sh, gain * (1 + sc), mag * (1 + sc).abs() + sh.abs()
    slack = 2.0 ** -18 * mag + gain.abs() * rstd * LN_SLACK * xs.abs().amax(1, keepdim=True)
    return y, slack


def _ln_call(M, D1, kmul, variant, x, x2=None, x3=None, D2=0, w=None, b=None, sh=None, sc=None, mbs=0, rpb=1, G=None, Cc=None):
    W = kmul * (D1 + D2)
    out = _sentinel((M + 2) * W)
    _run(kind=K_LN, variant=variant, M=M, D1=D1, D2=D2, kmul=kmul, x=x, x2=x2, x3=x3, w=w, b=b, shift=sh, scale=sc, mod_bstride=mbs,
         rows_per_batch=rpb, G=G, Cc=Cc, out=out)
    assert _is_sent(out[M * W:]), "rows >= M written"
    return out[:M * W].view(M, W)


def _gc_tables(w, b, sh, sc):
    """G = w (1 + scale), C = b (1 + scale) + shift in fp32 (fold_gc_kernel)."""
    return (w * (1 + sc[0])).contiguous(), (b * (1 + sc[0]) + sh[0]).contiguous()


LN_M_MOD = [(1, None), (3, "shared"), (5, 25), (127, 25), (4000, 500), (8001, "shared"), (20000, 500)]


@pytest.mark.parametrize("D", [1152, 1024])
@pytest.mark.parametrize("variant", [REG1, REG8, GENERIC, GC], ids=lambda v: VARIANT_NAMES[v])
@pytest.mark.parametrize("M,mode", LN_M_MOD)
def test_layernorm_forced_variant(D, variant, M, mode):
    """Every kernel Dit::ln can select for one D-wide source, at the model's widths, over row counts that leave a partial last CTA (reg:
    4 rows per CTA; generic: 8) and that make ln_gc's warps (grid capped at 4 CTAs per SM) walk several rows with a partial last round."""
    g = torch.Generator(device="cuda").manual_seed(M + D + variant)
    x = _ln_rows(M, D, g)
    w, b = _ln_params(D, g)
    if variant == GC:   # precombined affine: one modulation row for the whole batch
        tab, sh, sc, _, _ = _mod_table(M, D, "shared", g)
        G, Cc = _gc_tables(w, b, sh, sc)
        got = _ln_call(M, D, 1, GC, x, G=G, Cc=Cc)
        ref, slack = _ln_ref(x, G=G, Cc=Cc)
    else:
        tab, sh, sc, mbs, rpb = _mod_table(M, D, mode, g)
        got = _ln_call(M, D, 1, variant, x, w=w, b=b, sh=sh, sc=sc, mbs=mbs, rpb=rpb)
        ref, slack = _ln_ref(x, w=w, b=b, tab=tab, mbs=mbs, rpb=rpb)
    e, q = _check_bf16(got, ref, slack, 1, f"LayerNorm {VARIANT_NAMES[variant]} D{D} M{M}")
    print(f"[step] LayerNorm {VARIANT_NAMES[variant]} D{D} M{M} mod {mode}: max err {e:.3e}, {q:.2f} of the allowance")


@pytest.mark.parametrize("D", [1152, 1024])
def test_layernorm_gc_within_one_ulp_of_reg1(D):
    """The precombined affine (fmaf(xhat, G, C)) and the plain one (((xhat w + b)(1 + scale) + shift) round differently in fp32 only: the bf16
    outputs may differ by one bf16 ulp of the larger value, plus the fp32 difference where the terms cancel."""
    M = 4000
    g = torch.Generator(device="cuda").manual_seed(D)
    x = _ln_rows(M, D, g)
    w, b = _ln_params(D, g)
    tab, sh, sc, mbs, rpb = _mod_table(M, D, "shared", g)
    G, Cc = _gc_tables(w, b, sh, sc)
    a = _ln_call(M, D, 1, REG1, x, w=w, b=b, sh=sh, sc=sc, mbs=0, rpb=1).double()
    c = _ln_call(M, D, 1, GC, x, G=G, Cc=Cc).double()
    _, slack = _ln_ref(x, w=w, b=b, tab=tab, mbs=0, rpb=1)
    big = torch.maximum(a.abs(), c.abs())
    ulp = torch.where(big > 0, torch.exp2(torch.floor(torch.log2(big.clamp_min(1e-38))) - 7), torch.zeros_like(big))
    d = (a - c).abs()
    assert bool((d <= ulp + 2 * slack).all()), float((d - ulp - 2 * slack).max())
    print(f"[step] LayerNorm gc vs reg1 D{D}: {int((d > ulp).sum())} of {d.numel()} elements beyond one ulp (cancellation), "
          f"{int((d > 0).sum())} differ")


@pytest.mark.parametrize("D", [1152, 1024])
def test_layernorm_auto_follows_ln_variant(D):
    """'auto' is Dit::ln's own selection: for each option value it must give the bits of the kernel that option names."""
    M = 1000
    g = torch.Generator(device="cuda").manual_seed(7 * D)
    x, x2, x3 = _ln_rows(M, D, g), torch.randn(M, D, device="cuda", generator=g), torch.randn(M, D, device="cuda", generator=g)
    w, b = _ln_params(D, g)
    w2, b2 = _ln_params(2 * D, g)
    tab, sh, sc, _, _ = _mod_table(M, D, "shared", g)
    G, Cc = _gc_tables(w, b, sh, sc)
    single = dict(x=x, w=w, b=b, sh=sh, sc=sc, mbs=0, rpb=1, G=G, Cc=Cc)   # a modulated norm whose tables exist: what norm1 / norm3 pass
    cat = dict(x=x, x2=x2, x3=x3, D2=D, w=w2, b=b2)                         # skip_norm
    for opt, want_single, want_cat in ((0, REG1, GENERIC), (1, REG8, GENERIC), (2, GC, CAT)):
        with _options(ln_variant=opt):
            for kw, want, kmul in ((single, want_single, 1), (cat, want_cat, 1), (cat, GENERIC, 3)):
                got = _ln_call(M, D, kmul, AUTO, **kw)
                forced = _ln_call(M, D, kmul, want, **kw)
                assert torch.equal(_bits(got), _bits(forced)), (opt, VARIANT_NAMES[want], kmul)


@pytest.mark.parametrize("D,kmul,M", [(128, 1, 127), (128, 3, 4000), (144, 1, 4000), (144, 3, 127)])
def test_layernorm_generic_tiny_widths(D, kmul, M):
    """The tiny models' widths (128, 144: a lane takes 1 or 2 float4 per pass) with per-clip modulation, in bf16 and bf16x3."""
    g = torch.Generator(device="cuda").manual_seed(D * kmul + M)
    x = _ln_rows(M, D, g)
    w, b = _ln_params(D, g)
    tab, sh, sc, mbs, rpb = _mod_table(M, D, 25, g)
    got = _ln_call(M, D, kmul, AUTO, x, w=w, b=b, sh=sh, sc=sc, mbs=mbs, rpb=rpb)
    ref, slack = _ln_ref(x, w=w, b=b, tab=tab, mbs=mbs, rpb=rpb)
    e, q = _check_bf16(got, ref, slack, kmul, f"LayerNorm generic D{D} kmul {kmul}")
    print(f"[step] LayerNorm generic D{D} kmul {kmul} M{M}: max err {e:.3e}, {q:.2f} of the allowance")


@pytest.mark.parametrize("D,kmul,M", [(2048, 1, 5), (2048, 3, 4000), (1024, 1, 4000), (1024, 3, 3)])
def test_layernorm_cast_only_is_exact(D, kmul, M):
    """w = b = NULL (the context cast, the ControlNet zero-linear input): bf16 round-to-nearest of x, bit for bit, and lo = bf16(x - hi)."""
    x = 10.0 * torch.randn(M, D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(D + M))
    got = _ln_call(M, D, kmul, AUTO, x)
    assert torch.equal(_bits(got), _bits(_split(x, kmul)))


@pytest.mark.parametrize("D", [1152, 1024])
@pytest.mark.parametrize("with_x3", [False, True])
@pytest.mark.parametrize("variant,kmul,M", [(CAT, 1, 4000), (GENERIC, 1, 127), (GENERIC, 3, 4000)], ids=["cat", "generic", "generic-x3"])
def test_layernorm_skip_concat(D, with_x3, variant, kmul, M):
    """skip_norm over [x | skip (+ ControlNet skip)]: 2 D features from two (three) sources."""
    g = torch.Generator(device="cuda").manual_seed(D + M + with_x3)
    x, x2 = _ln_rows(M, D, g), torch.randn(M, D, device="cuda", generator=g)
    x3 = 0.5 * torch.randn(M, D, device="cuda", generator=g) if with_x3 else None
    w, b = _ln_params(2 * D, g)
    got = _ln_call(M, D, kmul, variant, x, x2=x2, x3=x3, D2=D, w=w, b=b)
    ref, slack = _ln_ref(x, x2, x3, w=w, b=b)
    e, q = _check_bf16(got, ref, slack, kmul, f"skip LayerNorm {VARIANT_NAMES[variant]} D{D}")
    print(f"[step] skip LayerNorm {VARIANT_NAMES[variant]} D{D} x3 {with_x3} kmul {kmul} M{M}: max err {e:.3e}, {q:.2f} of the allowance")


# ------------------------------------------------------------------------------------------------------------------------------ qk_prep
def _qk_ref(xin, off, kind, B, L, H, dh, norm, inv_freq):
    """float64 per-head LayerNorm + rotate-half RoPE (positions 0..L-1) of the values the kernel read -> ([B, H, L, dh] ref, fp32 allowance)."""
    v = xin[:, off:off + H * dh].double().view(B, L, H, dh)
    if kind == 2:
        return v.permute(0, 2, 1, 3), torch.zeros_like(v).permute(0, 2, 1, 3)
    mu = v.mean(-1, keepdim=True)
    xh = (v - mu) * (((v - mu) ** 2).mean(-1, keepdim=True) + 1e-5).rsqrt()
    y = xh * norm[0].double() + norm[1].double()
    slack = 2.0 ** -16 * ((xh * norm[0].double()).abs() + norm[1].double().abs())
    if inv_freq is not None:
        half = dh // 2
        th = torch.arange(L, device="cuda", dtype=torch.float64)[:, None] * inv_freq.double()[None]   # the same fp32 inv_freq
        th = torch.cat([th, th], -1)[None, :, None, :]
        rot = torch.cat([-y[..., half:], y[..., :half]], -1)
        slack = (slack + 2.0 ** -16 * (y.abs() + rot.abs())) + (y.abs() + rot.abs()) * 2.0 ** -23 * th   # (float) l * inv_freq, sincosf
        y = y * torch.cos(th) + rot * torch.sin(th)
    return y.permute(0, 2, 1, 3), slack.permute(0, 2, 1, 3)


QK_CASES = [  # (B, L, H, dh, sections (kinds), rope, input bf16, outputs): the parity-mode self-attention, the fast path's own
    (2, 1500, 16, 72, (0, 1, 2), True, False, "f32"),           # qk_prep (no fused heads), the cross-Q and cross-K/V layouts
    (3, 7, 2, 64, (0, 1, 2), True, True, "bf16"),
    (1, 1500, 16, 72, (0, 1, 2), True, True, "bf16"),
    (2, 500, 16, 64, (0, 1, 2), True, False, "both"),
    (3, 33, 16, 72, (0,), False, False, "both"),
    (2, 100, 2, 72, (1, 2), False, True, "bf16"),
]


@pytest.mark.parametrize("B,L,H,dh,kinds,rope,in_bf16,outs", QK_CASES)
def test_qk_prep(B, L, H, dh, kinds, rope, in_bf16, outs):
    g = torch.Generator(device="cuda").manual_seed(B * L + H + dh)
    D, nsec = H * dh, len(kinds)
    ld_in = nsec * D + 8
    xin = torch.randn(B * L, ld_in, device="cuda", generator=g) + 0.5
    if in_bf16:
        xin = xin.bfloat16()
    norms = {0: torch.stack(_ln_params(dh, g)).contiguous(), 1: torch.stack(_ln_params(dh, g)).contiguous()}
    inv_freq = (1.0 / 10000 ** (torch.arange(0, dh, 2, dtype=torch.float32) / dh)).cuda() if rope else None
    ld_qk, dv_pad = (80 if dh == 72 else 64), (dh + 15) // 16 * 16
    Lpad = (L + 7) // 8 * 8 + 8   # 8 more columns than the model's pitch: V^T columns >= L must stay untouched
    f32o, bfo = [None] * 3, [None] * 3
    for s, kd in enumerate(kinds):
        if outs in ("f32", "both"):
            f32o[s] = torch.full((B * H * L * dh + 64,), float("nan"), device="cuda")
        if outs in ("bf16", "both"):
            bfo[s] = _sentinel((B * H * dv_pad * Lpad if kd == 2 else B * H * L * ld_qk) + 64)
    off = [s * D for s in range(nsec)]
    _run(kind=K_QK, B=B, L=L, H=H, dh=dh, nsec=nsec, kinds=kinds, col_off=off, ld_in=ld_in, in_bf16=int(in_bf16), x=xin,
         norm_q=norms[0] if 0 in kinds else None, norm_k=norms[1] if 1 in kinds else None, inv_freq=inv_freq, f32_out=f32o, bf_out=bfo,
         ld_qk=ld_qk, Lpad=Lpad, dv_pad=dv_pad, out=f32o[0] if f32o[0] is not None else bfo[0])
    worst = 0.0
    for s, kd in enumerate(kinds):
        ref, slack = _qk_ref(xin.float(), off[s], kd, B, L, H, dh, norms.get(kd), inv_freq)
        if f32o[s] is not None:
            got = f32o[s][:B * H * L * dh].view(B, H, L, dh).double()
            assert bool(torch.isnan(f32o[s][B * H * L * dh:]).all()), "fp32 output: written past its end"
            if kd == 2:
                assert torch.equal(got, ref), "v section must be copied exactly"
            else:
                err = (got - ref).abs()
                assert bool((err <= slack).all()), f"section {s}: fp32 err {float(err.max()):.3e} > {float(slack.flatten()[int((err - slack).argmax())]):.3e}"
                worst = max(worst, float((err / slack).max()))
        if bfo[s] is not None:
            o = bfo[s]
            if kd == 2:   # V^T [B, H, dv_pad, Lpad]: values, zero pad rows, untouched columns >= L
                vt = o[:B * H * dv_pad * Lpad].view(B, H, dv_pad, Lpad)
                assert torch.equal(_bits(vt[:, :, :dh, :L]), _bits(ref.to(torch.float32).bfloat16().transpose(-1, -2)))
                assert bool((_bits(vt[:, :, dh:, :L]) == 0).all()), "V^T pad rows dh..dv_pad must be zeros"
                assert _is_sent(vt[..., L:]), "V^T columns >= L written"
            else:         # q / k [B, H, L, ld_qk]: dims >= dh untouched (the model clears them once)
                qk = o[:B * H * L * ld_qk].view(B, H, L, ld_qk)
                e, q = _check_bf16(qk[..., :dh].reshape(-1, dh), ref.reshape(-1, dh), slack.reshape(-1, dh), 1, f"qk_prep section {s}")
                worst = max(worst, q)
                assert _is_sent(qk[..., dh:]), "q / k pitch padding written"
            assert _is_sent(o[-64:]), "bf16 output: written past its end"
    print(f"[step] qk_prep B{B} L{L} H{H} dh{dh} kinds {kinds} rope {rope} in {'bf16' if in_bf16 else 'fp32'} out {outs}: "
          f"{worst:.2f} of the allowance")


# ------------------------------------------------------------------------------------------------------------------------------ patch_pack
@pytest.mark.parametrize("B,L,Cc,gt_mode,kmul", [(1, 1, 128, "none", 1), (3, 31, 128, "mask", 3), (16, 33, 128, "nomask", 1), (2, 500, 16, "mask", 1),
                                                  (4, 1500, 128, "none", 3), (16, 500, 128, "mask", 3), (2, 33, 16, "nomask", 3)])
def test_patch_pack_bit_exact(B, L, Cc, gt_mode, kmul):
    """A[b L + l] = [x[b, :, l] | gt[b, :, l] or mask_embed (no gt, or gt_mask[b, l]) | mask channel | zeros up to Kp], rounded to bf16 (hi |
    lo | hi in bf16x3): equal bit for bit to torch's rounding, rows >= B L untouched."""
    g = torch.Generator(device="cuda").manual_seed(B * L + Cc)
    Kp = (2 * Cc + 1 + 7) // 8 * 8
    x = torch.randn(B, Cc, L, device="cuda", generator=g)
    me = torch.randn(Cc, device="cuda", generator=g)
    gt = torch.randn(B, Cc, L, device="cuda", generator=g) if gt_mode != "none" else None
    gm = (torch.rand(B, L, device="cuda", generator=g) < 0.4).to(torch.uint8) if gt_mode == "mask" else None
    out = _sentinel((B * L + 2) * kmul * Kp)
    _run(kind=K_PATCH, B=B, L=L, C=Cc, Kp=Kp, kmul=kmul, x=x, gt=gt, gt_mask=gm, mask_embed=me, out=out)
    X = x.permute(0, 2, 1)
    if gt is None:
        Gc, m = me.expand(B, L, Cc), torch.ones(B, L, device="cuda")
    else:
        masked = gm.bool() if gm is not None else torch.zeros(B, L, dtype=torch.bool, device="cuda")
        Gc, m = torch.where(masked[..., None], me.expand(B, L, Cc), gt.permute(0, 2, 1)), masked.float()
    A = torch.cat([X, Gc, m[..., None], torch.zeros(B, L, Kp - 2 * Cc - 1, device="cuda")], -1).reshape(B * L, Kp)
    want = torch.cat([_split(A, 1), (A - _split(A, 1).float()).bfloat16(), _split(A, 1)], -1) if kmul == 3 else _split(A, 1)
    assert torch.equal(_bits(out[:B * L * kmul * Kp].view(B * L, kmul * Kp)), _bits(want))
    assert _is_sent(out[B * L * kmul * Kp:]), "rows >= B L written"


# ------------------------------------------------------------------------------------------------------------------------------ final_conv
FC_CASES = [(1, 1, None), (2, 2, [1, 2]), (3, 31, None), (2, 32, [32, 1]), (4, 33, [33, 17, 1, 33]),
            (16, 500, [500, 1, 250, 499, 37, 500, 7, 33, 32, 31, 100, 2, 480, 481, 64, 300]), (2, 1500, [1500, 1013])]


@pytest.mark.parametrize("B,L,lens", FC_CASES, ids=[f"B{b}-L{l}-{'nolens' if n is None else 'lens'}" for b, l, n in FC_CASES])
def test_final_conv(B, L, lens):
    """Conv1d(C, C, k=3, padding=1) over each clip's own frames (a clip of lens[b] frames sees zeros past its end); frames >= lens[b] keep
    their sentinel.  fp32 accumulation: a chain of 96 fmaf per input-channel group plus the four-group sum, |err| <= 2^-17 S with
    S = conv(|y|, |W|) + |bias| (worst case 100 roundings of 2^-24)."""
    Cc = 128
    g = torch.Generator(device="cuda").manual_seed(B * L)
    y = torch.randn(B * L, Cc, device="cuda", generator=g)
    W = 0.1 * torch.randn(Cc, Cc, 3, device="cuda", generator=g)
    bias = 0.1 * torch.randn(Cc, device="cuda", generator=g)
    wp = W.permute(2, 1, 0).contiguous()   # [tap][in][out], as Dit::init packs it
    ln = None if lens is None else torch.tensor(lens, dtype=torch.int32, device="cuda")
    out = torch.full((B + 1, Cc, L), float("nan"), device="cuda")
    _run(kind=K_FCONV, B=B, L=L, C=Cc, x=y, w=wp, b=bias, lens=ln, out=out)
    assert bool(torch.isnan(out[B]).all()), "written past the batch"
    worst = (0.0, 0.0)
    for b in range(B):
        n = L if lens is None else min(max(lens[b], 1), L)
        yb = y[b * L:b * L + n].double().T[None]
        ref = F.conv1d(yb, W.double(), bias.double(), padding=1)[0]
        S = F.conv1d(yb.abs(), W.double().abs(), bias.double().abs(), padding=1)[0]
        err = (out[b, :, :n].double() - ref).abs()
        allow = 2.0 ** -17 * S
        assert bool((err <= allow).all()), f"clip {b}: err {float(err.max()):.3e}"
        assert bool(torch.isnan(out[b, :, n:]).all()), f"clip {b}: frames >= {n} written"
        worst = max(worst, (float(err.max()), float((err / allow).max())), key=lambda t: t[1])
    print(f"[step] final_conv B{B} L{L} lens {lens if lens is None or len(lens) < 5 else 'mixed'}: max err {worst[0]:.3e}, {worst[1]:.2f} of the allowance")


# ------------------------------------------------------------------------------------------------------------------------------ small_linear
SL_CASES = [  # (K, R, N, act, add, out_scale): the time path's shapes (lora_b: K = 6 r, add = time_ada, scale = alpha / r) and the pass edges
    (6 * 36, 50, 6 * 1152, 0, True, 1.0), (6 * 4, 128, 6 * 144, 0, True, 1.0), (256, 128, 1152, 1, False, 1.0), (1152, 1, 6 * 1152, 0, False, 1.0),
    (1280, 50, 1024, 1, False, 1.0), (1281, 50, 1152, 0, True, 0.5), (2048, 128, 1024, 1, False, 1.0), (2560, 1, 300, 1, True, 0.25)]


@pytest.mark.parametrize("K,R,N,act,with_add,scale", SL_CASES)
def test_small_linear(K, R, N, act, with_add, scale):
    """out = act(scale (x W^T) + bias) + add, accumulated in passes of 1280 columns (K = 1280: one pass; 1281: a second pass of one column).
    Error: per lane a chain of <= 40 fmaf per pass, 5 tree levels, one add per pass: |err| <= (K / 32 + 48) 2^-24 S, S = |x| |W|^T, plus
    2^-21 of the activation's magnitude."""
    g = torch.Generator(device="cuda").manual_seed(K + R + N)
    ld_in, ld_out, ld_add = K + 3, N + 5, N + 2
    x = torch.randn(R, ld_in, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    bias = 0.5 * torch.randn(N, device="cuda", generator=g)
    add = torch.randn(R, ld_add, device="cuda", generator=g) if with_add else None
    out = torch.full((R + 1, ld_out), float("nan"), device="cuda")
    _run(kind=K_SLIN, R=R, N=N, K=K, act=act, out_scale=scale, x=x, ld_in=ld_in, w=W, b=bias, add=add, ld_add=ld_add if with_add else 0,
         out=out, ld_out=ld_out)
    xd, Wd = x[:, :K].double(), W.double()
    pre = scale * (xd @ Wd.T) + bias.double()
    ref = pre * torch.sigmoid(pre) if act == 1 else pre
    slack = 1.1 * (K / 32 + 48) * 2.0 ** -24 * (abs(scale) * (xd.abs() @ Wd.abs().T) + bias.double().abs()) + 2.0 ** -21 * ref.abs()
    if with_add:
        ref = ref + add[:, :N].double()
        slack = slack + 2.0 ** -24 * ref.abs()
    err = (out[:R, :N].double() - ref).abs()
    assert bool((err <= slack).all()), f"err {float(err.max()):.3e} > {float(slack.flatten()[int((err - slack).argmax())]):.3e}"
    assert bool(torch.isnan(out[:R, N:]).all()) and bool(torch.isnan(out[R]).all()), "written outside [R, N]"
    print(f"[step] small_linear K{K} R{R} N{N} act {act}: max err {float(err.max()):.3e}, {float((err / slack).max()):.2f} of the allowance")


# ------------------------------------------------------------------------------------------------------------------------------ timestep_embed
def test_timestep_embed():
    """[cos(t f_i) | sin(t f_i)], f_i = exp(-ln(1e4) i / 128): against torch's own fp32 formula (modules.py:19-39, restated in
    oracle.ezaudio_oracle.timestep_embedding) within a few ulp of the argument, and against float64 within the fp32 rounding of f and t f."""
    from oracle import ezaudio_oracle as O
    ts = [0, 1, 20, 499, 979, 999]
    t = torch.tensor(ts, dtype=torch.float32, device="cuda")
    out = torch.full((len(ts) + 1, 256), float("nan"), device="cuda")
    _run(kind=K_TEMB, M=len(ts), x=t, out=out)
    assert bool(torch.isnan(out[len(ts)]).all())
    got = out[:len(ts)].double().cpu()
    arg = torch.tensor(ts, dtype=torch.float64)[:, None] * torch.exp(-torch.log(torch.tensor(1e4, dtype=torch.float64)) * torch.arange(128) / 128)[None]
    arg2 = torch.cat([arg, arg], -1)
    e32 = (got - O.timestep_embedding(torch.tensor(ts)).double()).abs()
    assert bool((e32 <= 2.0 ** -21 * arg2 + 2.0 ** -21).all()), float(e32.max())
    e64 = (got - torch.cat([torch.cos(arg), torch.sin(arg)], -1)).abs()
    assert bool((e64 <= 2.0 ** -21 * arg2 + 2.0 ** -21).all()), float(e64.max())
    print(f"[step] timestep_embed: max err vs torch fp32 {float(e32.max()):.3e}, vs float64 {float(e64.max()):.3e} (t up to 999)")


# ------------------------------------------------------------------------------------------------------------------------------ cfg_ddim
def _cfg_ddim_ref(t, u, x, z, n, gs, gr, c):
    """float64 rescale_noise_cfg (unbiased std per sample, src/inference.py:12-23) + DDIM v-prediction update of one sample's first n frames
    -> (prev, fp32 allowance).  Only the ratio std(text) / std(cfg) enters the update, so the (n - 1) of the unbiased std cancels: no
    output can tell it from a biased std.  A divisor that differs between the two stds (n - 1 on one, n on the other) does show, most at
    small n (C = 3, L = 1: sqrt(2 / 3))."""
    t, x = t.double(), x.double()
    if u is None:
        v, V = t, t.abs()
    else:
        u = u.double()
        v = u + gs * (t - u)
        V = u.abs() + abs(gs) * (t.abs() + u.abs())
        if gr > 0:
            ratio = float(t.std() / v.std())
            v = gr * (v * ratio) + (1 - gr) * v
            V = V * (1 + ratio)
    c0, c1, c2, c3, c4 = (float(e) for e in c)
    prev = c2 * (c0 * x - c1 * v) + c3 * (c0 * v + c1 * x)
    mag = (abs(c0) + abs(c1)) * (abs(c2) + abs(c3)) * (x.abs() + V)
    if z is not None:
        prev = prev + c4 * z.double()
        mag = mag + abs(c4) * z.double().abs()
    return prev, 2.0 ** -20 * mag


CFG_CASES = [  # (B, C, L, guidance, rescale, eta, lens)
    (1, 128, 1, 5.0, 0.75, 0.0, None), (4, 128, 1, 5.0, 0.75, 1.0, None), (4, 128, 500, 5.0, 0.75, 1.0, None),
    (4, 128, 1500, 5.0, 0.75, 1.0, [1500, 1, 777, 1499]), (8, 128, 7, 1.0, 0.75, 0.0, None),
    (16, 128, 500, 0.0, 0.75, 1.0, [500, 1, 250, 499, 37, 500, 7, 33, 32, 31, 100, 2, 480, 481, 64, 300]),
    (16, 128, 1500, 5.0, 0.75, 1.0, None), (2, 3, 1, 5.0, 0.75, 1.0, None), (2, 130, 7, 5.0, 0.75, 0.0, [7, 3]), (1, 3, 7, 5.0, 0.0, 1.0, None)]


@pytest.mark.parametrize("B,Cc,L,gs,gr,eta,lens", CFG_CASES)
def test_cfg_ddim_step(B, Cc, L, gs, gr, eta, lens):
    """The fused CFG + rescale + DDIM update: 8 CTAs per sample, each over a slice of C len / 8 elements rounded up to a multiple of 4 (C = 3
    and 130 leave short or empty last slices).  Frames >= lens[b] of the latents keep their (NaN) values; a second call on the same inputs
    gives the same bits."""
    from ezaudio_b200 import _lib
    from ezaudio_b200.scheduler import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(50)
    coef = s.step_coefficients(479, eta)
    g = torch.Generator(device="cuda").manual_seed(B * Cc * L)
    text = torch.randn(B, Cc, L, device="cuda", generator=g) + 0.3
    unc = 0.8 * text + 0.3 * torch.randn(B, Cc, L, device="cuda", generator=g)
    model_out = torch.cat([text, unc]) if gs != 0 else text.clone()
    noise = torch.randn(B, Cc, L, device="cuda", generator=g) if eta > 0 else None
    lat0 = torch.full((B + 1, Cc, L), float("nan"), device="cuda")
    lat0[:B] = torch.randn(B, Cc, L, device="cuda", generator=g)
    n = [L] * B if lens is None else [min(max(v, 1), L) for v in lens]
    for b in range(B):   # what a clip must not read: NaN in every padded frame of every input
        lat0[b, :, n[b]:] = float("nan")
        model_out[b, :, n[b]:] = float("nan")
        if gs != 0:
            model_out[B + b, :, n[b]:] = float("nan")
        if noise is not None:
            noise[b, :, n[b]:] = float("nan")
    ln = None if lens is None else torch.tensor(lens, dtype=torch.int32, device="cuda")
    runs = []
    for _ in range(2):
        lat = lat0.clone()
        _lib.check(_lib.lib().ezb_cfg_ddim_step(0, _lib.ptr(model_out), _lib.ptr(lat), _lib.ptr(noise), B, Cc, L, gs, gr, (C.c_float * 5)(*coef),
                                                _lib.stream_ptr(), _lib.ptr(ln)))
        torch.cuda.synchronize()
        runs.append(lat)
    assert torch.equal(_bits(runs[0]), _bits(runs[1])), "second call differs"
    lat = runs[0]
    assert bool(torch.isnan(lat[B]).all()), "written past the batch"
    c32 = [float(torch.tensor(v, dtype=torch.float32)) for v in coef]   # the kernel's fp32 coefficients
    worst = (0.0, 0.0)
    for b in range(B):
        sl = (b, slice(None), slice(0, n[b]))
        ref, allow = _cfg_ddim_ref(text[sl], unc[sl] if gs != 0 else None, lat0[sl], None if noise is None else noise[sl], n[b], gs, gr, c32)
        err = (lat[sl].double() - ref).abs()
        assert bool((err <= allow).all()), f"sample {b}: err {float(err.max()):.3e} > {float(allow.flatten()[int((err - allow).argmax())]):.3e}"
        assert bool(torch.isnan(lat[b, :, n[b]:]).all()), f"sample {b}: padded frames written"
        worst = max(worst, (float(err.max()), float((err / allow).max())), key=lambda t: t[1])
    print(f"[step] cfg_ddim B{B} C{Cc} L{L} gs {gs} gr {gr} eta {eta}: max err {worst[0]:.3e}, {worst[1]:.2f} of the allowance")


# ------------------------------------------------------------------------------------------------------------------------------ argument checks
def test_step_hook_rejects_bad_arguments():
    """Refused before any device work (the buffers are large enough that a launch could not leave them)."""
    buf, obuf = torch.zeros(1 << 22, device="cuda"), torch.zeros(1 << 22, device="cuda")
    good = dict(kind=K_LN, variant=AUTO, M=4, D1=1152, kmul=1, x=buf, w=buf, b=buf, out=obuf)
    assert _call(**good) == 0
    torch.cuda.synchronize()
    for kw, rc in [(dict(kind=6), EZB_ERR_ARG), (dict(kind=-1), EZB_ERR_ARG), (dict(variant=6), EZB_ERR_ARG),
                   (dict(variant=REG1, D1=512), EZB_ERR_UNSUPPORTED), (dict(variant=REG8, D1=1152 + 128), EZB_ERR_UNSUPPORTED),
                   (dict(variant=GC), EZB_ERR_UNSUPPORTED), (dict(variant=GC, D1=768, G=buf, Cc=buf), EZB_ERR_ARG),
                   (dict(variant=REG1, kmul=3), EZB_ERR_UNSUPPORTED), (dict(variant=REG8, kmul=3), EZB_ERR_UNSUPPORTED),
                   (dict(variant=CAT), EZB_ERR_UNSUPPORTED), (dict(variant=CAT, x2=buf, D2=1024), EZB_ERR_UNSUPPORTED),
                   (dict(kmul=2), EZB_ERR_ARG), (dict(D1=1150), EZB_ERR_SHAPE), (dict(M=0), EZB_ERR_SHAPE), (dict(x=None), EZB_ERR_ARG),
                   (dict(out=None), EZB_ERR_ARG), (dict(b=None), EZB_ERR_ARG), (dict(scale=buf), EZB_ERR_ARG), (dict(x3=buf), EZB_ERR_ARG),
                   (dict(x2=buf), EZB_ERR_ARG),
                   # alignment: G / Cc are not read by the register kernel and one row at rows_per_batch 1 reads shift / scale at offset 0, so
                   # these calls would stay inside aligned accesses even if the check were missing
                   (dict(variant=REG1, G=buf[1:], Cc=buf), EZB_ERR_ARG), (dict(variant=REG1, G=buf, Cc=buf[2:]), EZB_ERR_ARG),
                   (dict(M=1, shift=buf, scale=buf[4:], mod_bstride=2, rows_per_batch=1), EZB_ERR_ARG)]:
        assert _call(**{**good, **kw}) == rc, kw
    qk = dict(kind=K_QK, B=2, L=8, H=2, dh=72, nsec=1, kinds=(0,), col_off=(0,), ld_in=144, x=buf, norm_q=buf, f32_out=(buf,), out=buf)
    assert _call(**{**qk, "norm_q": None}) == EZB_ERR_ARG
    assert _call(**{**qk, "dh": 98}) == EZB_ERR_SHAPE
    assert _call(**{**qk, "ld_in": 100}) == EZB_ERR_SHAPE
    assert _call(**{**qk, "f32_out": (None,)}) == EZB_ERR_ARG
    assert _call(**{**qk, "kinds": (2,), "f32_out": (None,), "bf_out": (buf,), "Lpad": 4, "dv_pad": 80}) == EZB_ERR_SHAPE
    assert _call(kind=K_PATCH, B=1, L=8, C=128, Kp=256, kmul=1, x=buf, mask_embed=buf, out=buf) == EZB_ERR_SHAPE   # Kp < 2C + 1
    assert _call(kind=K_PATCH, B=1, L=8, C=128, Kp=264, kmul=1, x=buf, out=buf) == EZB_ERR_ARG
    assert _call(kind=K_PATCH, B=1, L=8, C=128, Kp=264, kmul=1, x=buf, mask_embed=buf, gt_mask=buf, out=buf) == EZB_ERR_ARG
    assert _call(kind=K_FCONV, B=1, L=8, C=128, x=buf, b=buf, out=buf) == EZB_ERR_ARG
    assert _call(kind=K_FCONV, B=1, L=8, C=130, x=buf, w=buf, b=buf, out=buf) == EZB_ERR_SHAPE
    assert _call(kind=K_SLIN, R=1, N=8, K=16, ld_in=8, ld_out=8, x=buf, w=buf, out=buf) == EZB_ERR_SHAPE
    assert _call(kind=K_SLIN, R=1, N=8, K=16, ld_in=16, ld_out=8, act=2, x=buf, w=buf, out=buf) == EZB_ERR_ARG
    assert _call(kind=K_TEMB, M=0, x=buf, out=buf) == EZB_ERR_SHAPE
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------------ long schedules
TOL = {"bf16x3": (1e-3, 2e-4), "bf16": (6e-2, 1.2e-2)}


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_schedule_past_one_timestep_chunk(precision):
    """A 250-entry schedule uploads its timesteps in two 240-entry chunks.  The golden's timestep at indices 3, 130 and 245 (second chunk)
    must give the same bits at all three, and each must hold the tolerance against the fp32 reference's output at that timestep."""
    from ezaudio_b200.dit import MaskDiT
    cfg, sd, inp, g = helpers.dit_case_inputs("dit_tiny72")
    B, _, L = inp["x"].shape
    t0 = int(g["t"])
    ts = [4 * i for i in range(250)]
    assert t0 not in ts
    for i in (3, 130, 245):
        ts[i] = t0
    m = MaskDiT(precision=precision, max_batch=B, max_len=L, max_ctx_len=inp["ctx"].shape[1], max_timesteps=300, **cfg).load_state_dict(sd)
    m.set_context(inp["ctx"].cuda(), inp["mask"].cuda())
    m.set_timesteps(ts)
    x = inp["x"].cuda().contiguous()
    outs = [m.forward_step(x, i).clone() for i in (3, 130, 245)]
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    ref = torch.from_numpy(g["out"])
    err = (helpers.golden_view(g, outs[2].cpu()) - ref).abs()
    print(f"[step] 250-entry schedule [{precision}], index 245: max-abs {float(err.max()):.3e} mean-abs {float(err.mean()):.3e}")
    assert float(err.max()) < TOL[precision][0] and float(err.mean()) < TOL[precision][1]


def test_xl_schedule_past_the_layernorm_tables():
    """With more than 128 timesteps the precombined LayerNorm tables are not built and every modulated LayerNorm of EzAudio-XL runs
    ln_mod_cast_reg_kernel instead of ln_gc_kernel.  The golden's timestep at index 150 of a 200-entry schedule holds the bf16 tolerance
    against the golden and against the same forward on a 1-entry schedule (ln_gc_kernel).  The per-kernel launch counts show the dispatch:
    norm1 and norm3 of every block and the final norm (the modulated ones) on the register kernel for the long schedule and on ln_gc_kernel
    for the short one; norm2 (no modulation: G = weight) on ln_gc_kernel in both.  Stand-alone LayerNorms only: no GEMM tail, no fold."""
    from ezaudio_b200.dit import MaskDiT
    cfg, sd, inp, g = helpers.dit_case_inputs("dit_XL")
    B, _, L = inp["x"].shape
    t0 = int(g["t"])
    ts = [5 * i for i in range(200)]
    assert t0 not in ts
    ts[150] = t0
    nblk = cfg["depth"] + 1
    with _options(ln_variant=2, ln_tail=0, ln_fold=0):
        m = MaskDiT(precision="bf16", max_batch=B, max_len=L, max_ctx_len=inp["ctx"].shape[1], max_timesteps=200, **cfg).load_state_dict(sd)
        m.set_context(inp["ctx"].cuda(), inp["mask"].cuda())
        x = inp["x"].cuda().contiguous()
        m.set_timesteps(ts)
        c0 = _ln_counts()
        long = m.forward_step(x, 150).clone()
        c1 = _ln_counts()
        m.set_timesteps([t0])
        c2 = _ln_counts()
        short = m.forward_step(x, 0).clone()
        c3 = _ln_counts()
        torch.cuda.synchronize()
    d_long = {v: c1[v] - c0[v] for v in c0}
    d_short = {v: c3[v] - c2[v] for v in c2}
    print(f"[step] XL LayerNorm launches per forward, 200-entry schedule {d_long}, 1-entry schedule {d_short}")
    assert d_long[REG1] == 2 * nblk + 1 and d_long[GC] == nblk, d_long
    assert d_short[REG1] == 0 and d_short[GC] == 3 * nblk + 1, d_short
    ref = torch.from_numpy(g["out"])
    for name, out in (("200-entry", long), ("1-entry", short)):
        err = (helpers.golden_view(g, out.cpu()) - ref).abs()
        print(f"[step] XL {name} schedule [bf16]: max-abs {float(err.max()):.3e} mean-abs {float(err.mean()):.3e}")
        assert float(err.max()) < TOL["bf16"][0] and float(err.mean()) < TOL["bf16"][1]
    d = (long - short).abs()
    print(f"[step] XL 200-entry vs 1-entry schedule: max-abs {float(d.max()):.3e} mean-abs {float(d.mean()):.3e}")
    assert float(d.max()) < TOL["bf16"][0] and float(d.mean()) < TOL["bf16"][1]
