"""Oobleck VAE layers (csrc/vae.cuh), launched through ezb_test_vae exactly as Vae::decode / Vae::encode launch them, against fp64 references.

GEMM convs (Conv1d, ConvTranspose1d, strided Conv1d) get two references:

* Exact operands.  The packed bf16 weights the hook returns are unpacked into an fp64 kernel over all kmul*cin input channels and run with
  F.conv1d / F.conv_transpose1d on the same bf16 A.  In bf16x3 A is [hi | lo | hi] and W [hi | hi | lo] per tap, so the kernel multiplies
  exactly these operands; every product is exact in fp32 and only the fp32 accumulation is left.  Per element
      |raw - ref| <= EPS * S,   S = conv(|A'|, |W'|) + |bias| + |resid|.
  The wgmma accumulator is rounded once per 16-term step (at most 2^-23 relative, truncation), n = K / 16 steps for K = kmul * cin * taps
  <= 21 504 terms (n <= 1344).  With incoherent term signs the partial sums P_j grow like sqrt(j) and the rounding errors keep the sign of
  P_j, so the error is about 2^-23 sum_j |P_j| ~ 2^-23 * 0.2 sqrt(n) S <= 2^-20 S at n = 1344.  The epilogue's bias and residual adds are
  two more fp32 roundings (2^-23 S).  EPS = 2^-17 keeps a margin of about 8.  The mean error per tensor must stay under EPS / 4 * mean S,
  which a systematic offset such as a missing bias, or another phase's bias, does not.
* Impulses.  A is zero except for +-1 at rows 0, 1, T-2, T-1 and a few interior rows of every clip, each in one random channel (any of the
  hi / lo / hi blocks).  Every output then sums at most a handful of exact products and the bias, so the bound is EPS_IMPULSE = 2^-19 (a few
  fp32 roundings).  A dense input cannot see one dropped tap among thousands of terms; here a dropped, shifted or misplaced tap (tap order,
  dilation, the conv-transpose phase r and k = r + pad - delta*s, the strided conv's r / dq split for negative offsets, the zero halo at a
  clip edge) changes an output by a whole term.

The packing itself is checked against the fp64 weight-normed weight w = g v / ||v|| (norm over every dim but 0; dim 0 is C_in for the
conv-transpose): hi within one bf16 ulp (2^-7 |w|), the second hi block equal to the first, hi + lo within 2^-16 |w|; pad columns and the
conv-transpose's out-of-range taps are zero.

The fused SnakeBeta output is checked against ref + sin(a ref)^2 / (exp(beta) + 1e-9), a = exp(alpha), on the fp64 raw reference:
  bf16:   2^-8 |want| (one rounding) + EPS S |d snake / dv| + (|theta| 2^-22 + 2^-20) 2 |sin| / b   (__sinf, as in test_heads_gpu.py);
  bf16x3: 2^-16 |want| (hi + lo) + EPS S |d snake / dv| + (|theta| 2^-22 + 2^-22) 2 |sin| / b   (exact sinf),
  both + 2^-22 (|v| + sin^2 / b) for the fp32 arithmetic.  The third bf16x3 block must equal the first.

Layout: outputs are prefilled with NaN (fp32) or a bf16 NaN sentinel, and hold one spare clip past the end.  The first B clips must be
fully written and the spare clip untouched.  Clip b of a B = 3 call equals the B = 1 call on that clip, bit for bit, and with NaN in all
of clip 1's inputs, clips 0 and 2 are unchanged.

Shapes: every conv Vae::decode and Vae::encode run, at the shipped widths and at tiny_vae(16) (N = 32 < the 128-wide N-tile), in both
precisions.  The latent-rate layers (conv_in, the first conv-transpose, the last strided conv, e_out) run at T in {1, 2, 9, 127, 128,
129, 500}; the others at the rates of L = 1 and 3, which puts T = 10 under the dilation-9 halo of 27 rows.  The encoder's residual units
run at the same (channels, T) pairs as the decoder's, so the decoder's cases cover them.

The non-GEMM kernels (wave out, encoder stem, bottleneck sample, latent pack) and the whole decoder at short lengths follow below."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from ezaudio_b200 import synth, weights

gpu = pytest.mark.gpu

SENT = 0x7FAB   # a bf16 NaN pattern no kernel produces
CONV, CONVT, STRIDED, WAVE, STEM, SAMPLE, LATENT = range(7)
EPS = 2.0 ** -17
EPS_IMPULSE = 2.0 ** -19
T_LATENT = (1, 2, 9, 127, 128, 129, 500)


def _p(t):
    return None if t is None else t.data_ptr()


def _call(kind, precision, B, T, *, cin=0, cout=0, taps=0, dil=1, stride=0, w=None, x=None, resid=None, noise=None, raw=None, act=None,
          out=None, w_packed=None, stream=None):
    from ezaudio_b200 import _lib
    a = _lib.TestVaeArgs(kind=kind, precision=precision, B=B, T=T, cin=cin, cout=cout, taps=taps, dil=dil, stride=stride)
    w = w or {}
    a.weight_v, a.weight_g, a.bias, a.alpha, a.beta = (_p(w.get(k)) for k in ("v", "g", "bias", "alpha", "beta"))
    a.x, a.resid, a.noise, a.raw, a.act, a.out, a.w_packed = map(_p, (x, resid, noise, raw, act, out, w_packed))
    return _lib.lib().ezb_test_vae(0, C.byref(a), _lib.stream_ptr() if stream is None else stream)


def _run(*args, **kw):
    from ezaudio_b200 import _lib
    _lib.check(_call(*args, **kw))
    torch.cuda.synchronize()


def _sentinel(*shape):
    return torch.full(shape, SENT, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _split(x, kmul):
    """fp32 [..., C] -> the bf16 operand the library stores: hi, or [hi | lo | hi]."""
    hi = x.bfloat16()
    if kmul == 1:
        return hi.contiguous()
    return torch.cat([hi, (x - hi.float()).bfloat16(), hi], -1).contiguous()


def _wn64(w):
    v = w["v"].double()
    return w["g"].double().view(-1, *([1] * (v.dim() - 1))) * v / v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))


def _snake_weights(C, g):
    return dict(alpha=0.5 * torch.randn(C, device="cuda", generator=g), beta=0.5 * torch.randn(C, device="cuda", generator=g))


def _conv_weights(kind, cin, cout, K, s, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    shape = (cin, cout, 2 * s) if kind == CONVT else (cout, cin, 2 * s if kind == STRIDED else K)
    w = dict(v=torch.randn(*shape, device="cuda", generator=g), g=0.5 + torch.rand(shape[0], 1, 1, device="cuda", generator=g),
             bias=0.3 * torch.randn(cout, device="cuda", generator=g))
    w.update(_snake_weights(cout, g))
    return w


def _snake_check(got_act, ref, bound, w, kmul, cout):
    """Fused SnakeBeta output vs fp64 snake of the fp64 raw reference; returns max error / allowance."""
    a, binv = torch.exp(w["alpha"].double()), 1.0 / (torch.exp(w["beta"].double()) + 1e-9)
    th = a * ref
    sn = torch.sin(th)
    want = ref + binv * sn * sn
    prop = bound * (1 + binv * a * torch.sin(2 * th).abs()) + 2.0 ** -22 * (ref.abs() + binv * sn * sn)
    hi = got_act[..., :cout].double()
    if kmul == 1:
        got, rnd, mean_rnd = hi, 2.0 ** -8 * want.abs(), 0.75 * 2.0 ** -8
        prop = prop + (th.abs() * 2.0 ** -22 + 2.0 ** -20) * 2 * sn.abs() * binv
    else:
        assert torch.equal(_bits(got_act[..., 2 * cout:]), _bits(got_act[..., :cout])), "bf16x3: third block != hi"
        got, rnd, mean_rnd = hi + got_act[..., cout:2 * cout].double(), 2.0 ** -16 * want.abs(), 0.75 * 2.0 ** -16
        prop = prop + (th.abs() * 2.0 ** -22 + 2.0 ** -22) * 2 * sn.abs() * binv
    err = (got - want).abs()
    prop = (1 + 2.0 ** -7) * prop   # the rounding acts on the kernel's value, want + (up to) prop
    allow = rnd + prop
    i = int((err - allow).argmax())
    assert bool((err <= allow).all()), f"act: err {float(err.flatten()[i]):.3e} > {float(allow.flatten()[i]):.3e} at {i}"
    assert float(err.mean()) <= mean_rnd * float(want.abs().mean()) + float(prop.mean())
    return float((err / allow).max())


def _unpack(kind, wp, cin, cout, s, kmul):
    """Packed weights -> fp64 kernel over all kmul*cin input channels: [cout, kmul*cin, taps] (conv) or [kmul*cin, cout, 2s] (conv-T)."""
    width = kmul * cin
    if kind != CONVT:
        return wp[:, :, :width].double().permute(0, 2, 1)
    P, p = wp.double().view(s, cout, 3, -1)[..., :width], s // 2
    W = torch.empty(width, cout, 2 * s, dtype=torch.float64, device="cuda")
    for k in range(2 * s):
        r = (k - p) % s
        W[:, :, k] = P[r, :, (r + p - k) // s + 1, :].t()
    return W


def _check_packing(kind, wp, w, cin, cout, s, kmul):
    w64 = _wn64(w)
    assert bool((wp[:, :, kmul * cin:].float() == 0).all()), "pad columns not zero"
    if kind == CONVT:
        P, p = wp.view(s, cout, 3, -1), s // 2
        blocks, targets = [], []
        for r in range(s):
            for tap in range(3):
                k = r + p - (tap - 1) * s
                if 0 <= k < 2 * s:
                    blocks.append(P[r, :, tap])
                    targets.append(w64[:, :, k].t())
                else:
                    assert bool((P[r, :, tap].float() == 0).all()), f"conv-transpose phase {r} tap {tap} (k = {k}) not zero"
        blk, tgt = torch.stack(blocks), torch.stack(targets)
    else:
        blk, tgt = wp, w64.permute(0, 2, 1)
    hi = blk[..., :cin]
    assert bool(((hi.double() - tgt).abs() <= 2.0 ** -7 * tgt.abs()).all()), "hi not within one bf16 ulp of g v / |v|"
    if kmul == 3:
        assert torch.equal(_bits(blk[..., cin:2 * cin]), _bits(hi))
        assert bool(((hi.double() + blk[..., 2 * cin:3 * cin].double() - tgt).abs() <= 2.0 ** -16 * tgt.abs()).all()), "hi + lo"


def _conv_ref(kind, Ad, W, bias, *, K, dil, s):
    if kind == CONVT:
        return F.conv_transpose1d(Ad, W, bias, stride=s, padding=s // 2)
    if kind == STRIDED:
        return F.conv1d(Ad, W, bias, stride=s, padding=(s + 1) // 2)
    return F.conv1d(Ad, W, bias, padding=dil * (K - 1) // 2, dilation=dil)


def _conv_run(kind, prec, B, T, cin, cout, K, dil, s, w, A, resid, mode):
    kmul = 3 if prec else 1
    T_out = T * s if kind == CONVT else T
    raw = _nan(B + 1, T_out, cout) if mode in ("raw", "raw_act", "inplace") else None
    if mode == "inplace":
        raw[:B] = resid
    act = _sentinel(B + 1, T_out, kmul * cout) if mode != "raw" else None
    N, taps = (s * cout, 3) if kind == CONVT else (cout, 2 * s if kind == STRIDED else K)
    wp = torch.empty(N, taps, (kmul * cin + 63) // 64 * 64, dtype=torch.bfloat16, device="cuda")
    _run(kind, prec, B, T, cin=cin, cout=cout, taps=K, dil=dil, stride=s, w=w, x=A, raw=raw, act=act, w_packed=wp,
         resid=raw if mode == "inplace" else (resid if mode == "resid_act" else None))
    return raw, act, wp


def _impulses(B, T_in, width, g):
    A = torch.zeros(B, T_in, width, device="cuda")
    rows = sorted({r for r in (0, 1, T_in - 2, T_in - 1, T_in // 3, T_in // 2 + 1, 2 * T_in // 3 + 2) if 0 <= r < T_in})
    for b in range(B):
        ch = torch.randint(width, (len(rows),), device="cuda", generator=g)
        sign = torch.randint(2, (len(rows),), device="cuda", generator=g).float() * 2 - 1
        A[b, rows, ch] = sign
    return A.bfloat16()


def _check_conv(tag, kind, prec, B, T, cin, cout, K, dil, s, w, A, resid, mode, eps, outs):
    raw, act, wp = outs
    kmul = 3 if prec else 1
    W = _unpack(kind, wp, cin, cout, s, kmul)
    Ad = A.double().transpose(1, 2)
    ref = _conv_ref(kind, Ad, W, w["bias"].double(), K=K, dil=dil, s=s).transpose(1, 2)
    S = _conv_ref(kind, Ad.abs(), W.abs(), w["bias"].double().abs(), K=K, dil=dil, s=s).transpose(1, 2)
    assert ref.shape[1] == (T * s if kind == CONVT else T)
    if mode in ("inplace", "resid_act"):
        ref, S = ref + resid.double(), S + resid.double().abs()
    bound = eps * S
    r_raw = r_act = float("nan")
    if raw is not None:
        assert bool(torch.isnan(raw[B]).all()), "raw: spare clip written"
        err = (raw[:B].double() - ref).abs()
        i = int((err - bound).argmax())
        assert bool((err <= bound).all()), f"{tag} raw: err {float(err.flatten()[i]):.3e} > {float(bound.flatten()[i]):.3e} at {i}"
        assert float(err.mean()) <= 0.25 * float(bound.mean()), f"{tag} raw: mean error {float(err.mean()):.3e}"
        r_raw = float((err / bound).max())
    if act is not None:
        assert bool((_bits(act[B]) == SENT).all()), "act: spare clip written"
        assert bool((_bits(act[:B]) != SENT).all()), "act: not fully written"
        r_act = _snake_check(act[:B], ref, bound, w, kmul, cout)
    return r_raw, r_act


def _layer_cases():
    cases, seen = [], set()

    def add(tag, kind, cin, cout, K, dil, s, T, mode):
        key = (kind, cin, cout, K, dil, s, T, mode)
        if key not in seen:
            seen.add(key)
            cases.append(pytest.param(kind, cin, cout, K, dil, s, T, mode, id=tag))

    for cname, dcfg in (("full", synth.VAE_DECODER), ("tiny", synth.tiny_vae(16))):
        ch, n, lat = dcfg["channels"], len(dcfg["strides"]), dcfg["latent_dim"]
        mults = [1] + list(dcfg["c_mults"])
        dec_in, dec_out = [mults[i] * ch for i in range(n, 0, -1)], [mults[i - 1] * ch for i in range(n, 0, -1)]
        dec_s, enc_s = list(dcfg["strides"])[::-1], list(dcfg["strides"])
        enc_in, enc_out = [mults[i] * ch for i in range(n)], [mults[i + 1] * ch for i in range(n)]
        hop = math.prod(enc_s)
        for T in T_LATENT:
            add(f"{cname}-conv_in-T{T}", CONV, lat, dec_in[0], 7, 1, 0, T, "act")
            add(f"{cname}-up1-s{dec_s[0]}-T{T}", CONVT, dec_in[0], dec_out[0], 3, 1, dec_s[0], T, "raw_act")
            add(f"{cname}-down{n}-s{enc_s[-1]}-T{T}", STRIDED, enc_in[-1], enc_out[-1], 0, 1, enc_s[-1], T, "act")
            add(f"{cname}-e_out-T{T}", CONV, enc_out[-1], 2 * lat, 3, 1, 0, T, "raw")
        for L in (1, 3):
            T = L
            for j in range(n):
                if j:
                    add(f"{cname}-up{j + 1}-s{dec_s[j]}-T{T}", CONVT, dec_in[j], dec_out[j], 3, 1, dec_s[j], T, "raw_act")
                T *= dec_s[j]
                c = dec_out[j]
                for d in (1, 3, 9):
                    add(f"{cname}-res7-C{c}-d{d}-T{T}", CONV, c, c, 7, d, 0, T, "act")
                add(f"{cname}-res1-inplace-C{c}-T{T}", CONV, c, c, 1, 1, 0, T, "inplace")
                add(f"{cname}-res1-last-C{c}-T{T}", CONV, c, c, 1, 1, 0, T, "resid_act")
            T = L * hop
            for j in range(n - 1):
                T //= enc_s[j]
                add(f"{cname}-down{j + 1}-s{enc_s[j]}-T{T}", STRIDED, enc_in[j], enc_out[j], 0, 1, enc_s[j], T, "raw_act")
    for s in (3, 5):   # the encoder's strided conv is also right for odd strides (floor((T s + 1) / s) = T output rows)
        add(f"odd-down-s{s}-T129", STRIDED, 64, 64, 0, 1, s, 129, "raw_act")
    return cases


@gpu
@pytest.mark.parametrize("prec", [0, 1], ids=["bf16", "bf16x3"])
@pytest.mark.parametrize("kind,cin,cout,K,dil,s,T,mode", _layer_cases())
def test_vae_conv_layer(kind, cin, cout, K, dil, s, T, mode, prec):
    """One conv of the decoder / encoder: packing, dense and impulse inputs against the exact-operand fp64 reference, layout, and clip
    independence (B = 3 equals three B = 1 calls bit for bit; NaN in clip 1 leaves clips 0 and 2 unchanged)."""
    B, kmul = 3, 3 if prec else 1
    T_in, T_out = (T * s if kind == STRIDED else T), (T * s if kind == CONVT else T)
    seed = hash((kind, cin, cout, K, dil, s, T, mode)) % 100_000
    w = _conv_weights(kind, cin, cout, K, s, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    A = _split(torch.randn(B, T_in, cin, device="cuda", generator=g), kmul)
    resid = 0.5 * torch.randn(B, T_out, cout, device="cuda", generator=g) if mode in ("inplace", "resid_act") else None
    run = lambda A_, r_, b=B: _conv_run(kind, prec, b, T, cin, cout, K, dil, s, w, A_, r_, mode)
    outs = run(A, resid)
    _check_packing(kind, outs[2], w, cin, cout, s, kmul)
    r_raw, r_act = _check_conv("dense", kind, prec, B, T, cin, cout, K, dil, s, w, A, resid, mode, EPS, outs)
    Ai = _impulses(B, T_in, kmul * cin, g)
    i_raw, i_act = _check_conv("impulse", kind, prec, B, T, cin, cout, K, dil, s, w, Ai, resid, mode, EPS_IMPULSE, run(Ai, resid))
    print(f"[vae-layer] err / bound: dense raw {r_raw:.3f} act {r_act:.3f}; impulse raw {i_raw:.3f} act {i_act:.3f}")
    got = [o for o in outs[:2] if o is not None]
    for b in range(B):
        solo = run(A[b:b + 1], None if resid is None else resid[b:b + 1], 1)
        for o, o1 in zip(got, [o for o in solo[:2] if o is not None]):
            assert torch.equal(_bits(o[b]), _bits(o1[0])), f"clip {b} of B = 3 differs from its B = 1 call"
    An = A.clone()
    An[1] = float("nan")
    rn = None if resid is None else resid.clone()
    if rn is not None:
        rn[1] = float("nan")
    for o, on in zip(got, [o for o in run(An, rn)[:2] if o is not None]):
        for b in (0, 2):
            assert torch.equal(_bits(o[b]), _bits(on[b])), f"NaN in clip 1 changed clip {b}"


@gpu
@pytest.mark.parametrize("prec", [0, 1], ids=["bf16", "bf16x3"])
@pytest.mark.parametrize("kind,cin,cout,K,dil,s,T,mode", [
    pytest.param(CONV, 128, 128, 7, 9, 0, 30000, "act", id="res7-d9-T30000"),
    pytest.param(CONV, 128, 128, 1, 1, 0, 30000, "inplace", id="res1-inplace-T30000"),
    pytest.param(CONVT, 128, 128, 3, 1, 2, 15000, "raw_act", id="up-s2-T15000"),
    pytest.param(STRIDED, 128, 128, 0, 1, 2, 15000, "raw_act", id="down-s2-T15000")])
def test_vae_conv_layer_large(kind, cin, cout, K, dil, s, T, mode, prec):
    """Clips of a 62.5-s waveform's rate, B = 2: hundreds of tiles per launch, so the persistent CTAs wrap many times."""
    B, kmul = 2, 3 if prec else 1
    T_in, T_out = (T * s if kind == STRIDED else T), (T * s if kind == CONVT else T)
    w = _conv_weights(kind, cin, cout, K, s, 77)
    g = torch.Generator(device="cuda").manual_seed(78)
    A = _split(torch.randn(B, T_in, cin, device="cuda", generator=g), kmul)
    resid = 0.5 * torch.randn(B, T_out, cout, device="cuda", generator=g) if mode == "inplace" else None
    outs = _conv_run(kind, prec, B, T, cin, cout, K, dil, s, w, A, resid, mode)
    _check_packing(kind, outs[2], w, cin, cout, s, kmul)
    r = _check_conv("dense", kind, prec, B, T, cin, cout, K, dil, s, w, A, resid, mode, EPS, outs)
    Ai = _impulses(B, T_in, kmul * cin, g)
    ri = _check_conv("impulse", kind, prec, B, T, cin, cout, K, dil, s, w, Ai, resid, mode, EPS_IMPULSE,
                     _conv_run(kind, prec, B, T, cin, cout, K, dil, s, w, Ai, resid, mode))
    print(f"[vae-layer] err / bound: dense raw {r[0]:.3f} act {r[1]:.3f}; impulse raw {ri[0]:.3f} act {ri[1]:.3f}")


# ---------------------------------------------------------------------------------------------------------------------------------------
# wave out: Conv1d(C -> 1, k 7, pad 3) of the last snake's output.  Each output is a chain of 28 fmaf per lane (7 taps x 4 channels) and
# a 5-level shuffle tree: at most 33 fp32 roundings of partial sums bounded by S = conv(|x|, |w|), so |err| <= 33 * 2^-24 S < 2^-18 S.
EPS_WAVE = 2.0 ** -18


@gpu
@pytest.mark.parametrize("prec", [0, 1], ids=["bf16", "bf16x3"])
@pytest.mark.parametrize("C", [16, 128])
@pytest.mark.parametrize("T", [1, 31, 33, 200, 480, 960, 4800, 240000])
def test_wave_out(T, C, prec):
    kmul = 3 if prec else 1
    B = 2 if T > 100_000 else 3
    g = torch.Generator(device="cuda").manual_seed(T * 7 + C)
    w = dict(v=torch.randn(1, C, 7, device="cuda", generator=g), g=torch.rand(1, 1, 1, device="cuda", generator=g) + 0.5)
    x = torch.randn(B, T, C, device="cuda", generator=g)
    act = _split(x, kmul)
    out, wf = _nan(B + 1, T), torch.empty(7, C, device="cuda")
    _run(WAVE, prec, B, T, cin=C, w=w, x=act, out=out, w_packed=wf)
    w64 = _wn64(w)[0]                               # [C, 7]
    assert bool(((wf.double().t() - w64).abs() <= 2.0 ** -18 * w64.abs()).all()), "folded wave-out weights"
    xd = act[..., :C].double() + (act[..., C:2 * C].double() if kmul == 3 else 0)
    k = wf.double().t().unsqueeze(0)               # [1, C, 7]
    ref = F.conv1d(xd.transpose(1, 2), k, padding=3)[:, 0]
    S = F.conv1d(xd.abs().transpose(1, 2), k.abs(), padding=3)[:, 0]
    assert bool(torch.isnan(out[B]).all()), "spare clip written"
    err = (out[:B].double() - ref).abs()
    assert bool((err <= EPS_WAVE * S).all()), float((err / S).max())
    print(f"[vae-wave-out] err / bound {float((err / (EPS_WAVE * S)).max()):.3f}")
    if B == 3:
        one = _nan(2, T)
        _run(WAVE, prec, 1, T, cin=C, w=w, x=act[1:2].contiguous(), out=one)
        assert torch.equal(_bits(one[0]), _bits(out[1])), "clip 1 of B = 3 differs from its B = 1 call"


# encoder stem: Conv1d(1 -> C, k 7, pad 3) of the waveform, a chain of 7 fmaf from the bias: |err| <= 8 * 2^-24 S.
EPS_STEM = 2.0 ** -20


@gpu
@pytest.mark.parametrize("prec", [0, 1], ids=["bf16", "bf16x3"])
@pytest.mark.parametrize("C", [16, 128])
@pytest.mark.parametrize("T", [1, 31, 480, 240000])
def test_encoder_stem(T, C, prec):
    kmul = 3 if prec else 1
    B = 2 if T > 100_000 else 3
    g = torch.Generator(device="cuda").manual_seed(T + C)
    w = dict(v=torch.randn(C, 1, 7, device="cuda", generator=g), g=torch.rand(C, 1, 1, device="cuda", generator=g) + 0.5,
             bias=0.3 * torch.randn(C, device="cuda", generator=g))
    w.update(_snake_weights(C, g))
    audio = 0.3 * torch.randn(B, T, device="cuda", generator=g)
    raw, act, wf = _nan(B + 1, T, C), _sentinel(B + 1, T, kmul * C), torch.empty(7, C, device="cuda")
    _run(STEM, prec, B, T, cout=C, w=w, x=audio, raw=raw, act=act, w_packed=wf)
    w64 = _wn64(w)[:, 0]                             # [C, 7]
    assert bool(((wf.double().t() - w64).abs() <= 2.0 ** -20 * w64.abs()).all()), "folded stem weights"
    k = wf.double().t().unsqueeze(1)                 # [C, 1, 7]
    ref = F.conv1d(audio.double().unsqueeze(1), k, w["bias"].double(), padding=3).transpose(1, 2)
    S = F.conv1d(audio.double().abs().unsqueeze(1), k.abs(), w["bias"].double().abs(), padding=3).transpose(1, 2)
    bound = EPS_STEM * S
    err = (raw[:B].double() - ref).abs()
    assert bool((err <= bound).all()), float((err / S).max())
    assert bool(torch.isnan(raw[B]).all()) and bool((_bits(act[B]) == SENT).all()), "spare clip written"
    # the stem's snake takes the exact sinf in both precisions: the bf16x3 allowance, plus one bf16 rounding in bf16 mode
    r_act = _snake_check(act[:B], ref, bound, w, kmul, C) if prec else _snake_check_exact_bf16(act[:B], ref, bound, w, C)
    print(f"[vae-stem] err / bound: raw {float((err / bound).max()):.3f} act {r_act:.3f}")


def _snake_check_exact_bf16(got, ref, bound, w, C):
    a, binv = torch.exp(w["alpha"].double()), 1.0 / (torch.exp(w["beta"].double()) + 1e-9)
    th = a * ref
    sn = torch.sin(th)
    want = ref + binv * sn * sn
    allow = 2.0 ** -8 * want.abs() + bound * (1 + binv * a * torch.sin(2 * th).abs()) + 2.0 ** -22 * (ref.abs() + binv * sn * sn) + \
        (th.abs() * 2.0 ** -22 + 2.0 ** -22) * 2 * sn.abs() * binv
    err = (got.double() - want).abs()
    assert bool((err <= allow).all()), float((err / allow).max())
    return float((err / allow).max())


# bottleneck sample: z = noise (softplus(scale) + 1e-4) + mean, softplus(x) = x above 20.  log1pf(expf(x)) is within ~4 fp32 ulps
# (its condition number in exp(x) is <= 1), then three roundings: |err| <= 2^-20 (|noise| (sp + 1e-4) + |mean|).
@gpu
@pytest.mark.parametrize("noise", [True, False], ids=["noise", "mean"])
@pytest.mark.parametrize("L", [1, 7, 500])
def test_vae_sample(L, noise):
    B, Cz = 3, 128
    g = torch.Generator(device="cuda").manual_seed(L)
    n = B * L * Cz
    scale = torch.cat([torch.linspace(-30, 30, n // 2, device="cuda"), 20 + torch.linspace(-1e-3, 1e-3, n - n // 2, device="cuda")])
    scale = scale[torch.randperm(n, device="cuda", generator=g)]
    scale[:3] = torch.tensor([20.0, 20.0 + 2.0 ** -19, 20.0 - 2.0 ** -19])   # 20 and its fp32 neighbours
    enc = torch.cat([torch.randn(B * L, Cz, device="cuda", generator=g), scale.view(B * L, Cz)], 1).contiguous()
    nz = torch.randn(B, Cz, L, device="cuda", generator=g) if noise else None
    z = _nan(B + 1, Cz, L)
    _run(SAMPLE, 0, B, L, cout=Cz, x=enc, noise=nz, out=z)
    mean = enc[:, :Cz].view(B, L, Cz).transpose(1, 2)
    assert bool(torch.isnan(z[B]).all())
    if not noise:
        assert torch.equal(_bits(z[:B]), _bits(mean.contiguous()))
        return
    sp = F.softplus(enc[:, Cz:].double(), threshold=20).view(B, L, Cz).transpose(1, 2)
    want = nz.double() * (sp + 1e-4) + mean.double()
    allow = 2.0 ** -20 * (nz.double().abs() * (sp + 1e-4) + mean.double().abs())
    err = (z[:B].double() - want).abs()
    assert bool((err <= allow).all()), float((err / allow).max())
    print(f"[vae-sample] err / bound {float((err / allow).max()):.3f}")


@gpu
@pytest.mark.parametrize("prec", [0, 1], ids=["bf16", "bf16x3"])
@pytest.mark.parametrize("L", [1, 31, 33, 500])
def test_latent_pack(L, prec):
    """z (B, C, L) -> channels-last bf16 [hi | lo | hi], bit for bit against torch's round-to-nearest-even."""
    B, C, kmul = 3, 128, 3 if prec else 1
    z = torch.randn(B, C, L, device="cuda", generator=torch.Generator(device="cuda").manual_seed(L))
    act = _sentinel(B + 1, L, kmul * C)
    _run(LATENT, prec, B, L, cin=C, x=z, act=act)
    assert torch.equal(_bits(act[:B]), _bits(_split(z.transpose(1, 2), kmul)))
    assert bool((_bits(act[B]) == SENT).all())


# ---------------------------------------------------------------------------------------------------------------------------------------
def _vae_sd(dcfg, ecfg=None):
    sd = dict(weights.synthetic_state_dict(weights.vae_decoder_param_shapes(dcfg), 6))
    if ecfg:
        sd.update(weights.synthetic_state_dict(weights.vae_encoder_param_shapes(ecfg), 8))
    return sd


@gpu
@pytest.mark.parametrize("L", [1, 2, 3, 37])
@pytest.mark.parametrize("name,dcfg", [("tiny", synth.tiny_vae(16)), ("full", synth.VAE_DECODER)])
def test_decoder_short_clips_match_oracle(name, dcfg, L):
    """Whole bf16x3 decoder at lengths the goldens skip, down to L = 1 (early layers shorter than their halo), against the fp32 oracle on
    the host, with the bound of test_vae_gpu.py."""
    from ezaudio_b200.vae import OobleckDecoder
    from oracle import ezaudio_oracle as O
    sd = _vae_sd(dcfg)
    dec = OobleckDecoder(precision="bf16x3", max_batch=1, max_latent_len=L, **dcfg).load_state_dict(sd)
    z = synth.synth_latents(1, L, dcfg["latent_dim"], seed=31)
    wav = dec(z.cuda()).cpu()
    ref = O.vae_decode(sd, z, strides=tuple(dcfg["strides"]))
    assert wav.shape == ref.shape == (1, 1, 480 * L)
    err, scale = float((wav - ref).abs().max()), float(ref.abs().max())
    print(f"[vae-short] {name} L {L}: max-abs {err:.3e} (|ref|max {scale:.3e})")
    assert err < 1e-3 * scale + 1e-5


@gpu
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("name,dcfg,ecfg", [("tiny", synth.tiny_vae(16), synth.tiny_vae_encoder(16)),
                                            ("full", synth.VAE_DECODER, synth.VAE_ENCODER)])
def test_batch_equals_solo(name, dcfg, ecfg, precision):
    """Decoding (and encoding) a batch of three clips gives each clip's solo result bit for bit: the varlen API's per-length groups rely
    on a clip's waveform not depending on its neighbours."""
    from ezaudio_b200.vae import OobleckDecoder
    B, L = 3, 7
    codec = OobleckDecoder(precision=precision, max_batch=B, max_latent_len=L, encoder_cfg=ecfg, **dcfg).load_state_dict(_vae_sd(dcfg, ecfg))
    z = synth.synth_latents(B, L, dcfg["latent_dim"], seed=5).cuda()
    wav = codec(z)
    audio = 0.3 * torch.randn(B, 1, 480 * L, generator=torch.Generator().manual_seed(9)).cuda()
    mean = codec.encode(audio, noise=False)
    torch.cuda.synchronize()
    for b in range(B):
        assert torch.equal(_bits(codec(z[b:b + 1])[0]), _bits(wav[b])), f"decode: clip {b}"
        assert torch.equal(_bits(codec.encode(audio[b:b + 1], noise=False)[0]), _bits(mean[b])), f"encode: clip {b}"


# ---------------------------------------------------------------------------------------------------------------------------------------
ODD = dict(synth.VAE_DECODER, strides=[2, 3, 6, 10])


def test_decoder_rejects_odd_strides():
    """ConvTranspose1d(k = 2s, stride s, padding ceil(s/2)) yields T s - 1 frames for odd s; the decoder refuses such a config before it
    touches a device."""
    from ezaudio_b200.vae import OobleckDecoder
    for strides in ([2, 3, 6, 10], [1, 4, 6, 10]):
        with pytest.raises(NotImplementedError, match="even strides"):
            OobleckDecoder(precision="bf16", **dict(synth.VAE_DECODER, strides=strides))


@gpu
def test_library_rejects_odd_decoder_stride():
    from ezaudio_b200 import _lib
    d = _lib.VaeDesc(latent_dim=128, channels=128, out_channels=1, n_stages=4, max_batch=1, max_latent_len=8, precision=0)
    for i, (m, s) in enumerate(zip(ODD["c_mults"], ODD["strides"])):
        d.c_mults[i], d.strides[i] = m, s
    h = C.c_void_p()
    assert _lib.lib().ezb_vae_create(C.byref(h), C.byref(d), 0) == -3   # EZB_ERR_UNSUPPORTED
    assert not h.value
    assert "stride 3" in _lib.lib().ezb_last_error().decode()


def test_test_hook_rejects_bad_arguments_before_device_work():
    """ezb_test_vae refuses impossible shapes, odd conv-transpose strides and an activated output without a snake before any device work
    (the pointers below are never dereferenced)."""
    from ezaudio_b200 import _lib

    class Fake:
        def __init__(self, p):
            self.p = p

        def data_ptr(self):
            return self.p

    f = Fake(256)
    w = dict(v=f, g=f, bias=f, alpha=f, beta=f)
    ok = dict(cin=64, cout=64, taps=7, dil=1, w=w, x=f, raw=f, act=f)
    bad = [(CONV, dict(ok, cin=12), -2), (CONV, dict(ok, cout=20), -2), (CONV, dict(ok, taps=4), -2),
           (CONVT, dict(ok, stride=3), -3), (CONVT, dict(ok, stride=0), -3), (STRIDED, dict(ok, stride=1), -2),
           (CONV, dict(ok, w=dict(w, alpha=None)), -1), (CONV, dict(ok, raw=None, act=None), -1),
           (WAVE, dict(cin=18, w=w, x=f, out=f), -2), (STEM, dict(cout=16, w=w, x=f, raw=f), -1), (LATENT, dict(cin=16, x=f), -1)]
    st = C.c_void_p()
    for kind, kw, rc in bad:
        assert _call(kind, 0, 1, 8, stream=st, **kw) == rc, (kind, kw)
    assert _call(CONV, 0, 1, 0, stream=st, **ok) == -2       # T < 1
    assert _call(CONV, 0, 0, 8, stream=st, **ok) == -2       # B < 1
    assert _call(7, 0, 1, 8, stream=st, **ok) == -1          # no such kind
    assert _call(CONV, 2, 1, 8, stream=st, **ok) == -1       # no such precision
