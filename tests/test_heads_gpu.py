"""Fused Q/K/V-heads epilogue (csrc/gemm.cuh EpiHeads, launched through host.cuh heads_gemm exactly as Dit::lin_heads launches it) against an
fp64 reference of the same operation on the same bf16 A and bf16-rounded W:

    u = A W^T  ->  per head LayerNorm(dh), eps 1e-5, with the affine of the section's kind  ->  rotate-half RoPE at the position within the
    clip  ->  q / k rows [b*H + h, l, :dh] (pitch ld_qk), V^T [b*H + h, d, l] (pitch Lpad).

The RoPE angle is l * inv_freq rounded to fp32, as the model's fp32 frequency table holds it; its cos / sin are taken in fp64.

Per element:  |got - ref| <= 2^-8 |ref| + EPS_ABS  (+ the MUFU term below).
  2^-8 |ref| is the bf16 rounding of the output (half an ulp of 8 significant bits).  EPS_ABS covers the fp32 arithmetic before the rounding,
  on values of O(1) (u ~ N(0, 1), LayerNorm outputs |w z + b| <~ 6):
  - GEMM: K <= 1152 bf16 products, exact in fp32, accumulated in fp32: ~sqrt(K) 2^-24 |u| <~ 1e-5, scaled by rstd |w| <~ 2: 2e-5;
  - LayerNorm(dh): fp32 sums of dh <= 72 values, rsqrtf (2 ulp): ~1e-6 relative, 6e-6;
  - table RoPE: sincosf of the same fp32 angle (<= 2 ulp) and two fp32 products per element: ~1e-6;
  - fold: rstd * (acc - mu u) + v in fp32 on O(1..5) terms, mu and rstd from fp32 partial sums: ~5e-6.
  Together ~3e-5; EPS_ABS = 1e-4 keeps a 3x margin.
MUFU RoPE (__sincosf, the default): the hardware reduces the argument as theta * (1 / 2 pi) in fp32, so the angle is off by up to
  |theta| 2^-23 (product and constant rounding) + 2^-21.4 (MUFU.SIN / COS absolute error), and the rotated pair (a, b) moves by that angle
  times r = sqrt(a^2 + b^2).  Bound: EPS_ABS + (|theta| 2^-22 + 2^-20) r per element (2x margin); theta reaches 1499 rad here.
Mean per output tensor:  mean |got - ref| <= 0.75 * 2^-8 mean |ref| + EPS_ABS (+ the mean MUFU term).  A bf16 rounding averages about
  2^-9.5 relative, so a systematic bias (a dropped LayerNorm bias, the other kind's affine) fails here even where it hides under the
  per-element bound.

Layout: the outputs are filled with a sentinel first.  q / k pad columns dh..ld_qk and V^T columns L..Lpad come back untouched (attention
relies on the allocator's zeroing of the q / k pads and never reads the V^T pad columns), V^T rows dh..dvp come back zero, and one extra
slab past the last b*H + h is never written."""
import ctypes as C
import math

import pytest
import torch

gpu = pytest.mark.gpu

EPS_ABS = 1e-4
SENT = 0x7FAB   # a bf16 NaN pattern no epilogue produces

# heads_gemm variants (csrc/host.cuh HeadsVariant; 2 is the retired 128-deep-slot id)
PACKED3, PACKED3_PARKED, PAIR, PAIR_PARKED, SINGLE = 0, 1, 3, 4, 5
ROPE_NONE, ROPE_TABLE, ROPE_MUFU = 0, 1, 2


def _dvp(dh):
    return (dh + 15) // 16 * 16


def _lpad(L):
    return (L + 7) // 8 * 8


def _run(A, W, *, B, L, H, dh, kinds, variant, rope=ROPE_NONE, nq=None, nk=None, inv_freq=None, ld_qk=None, fold=None):
    """One launch; returns {kind: output buffer} (bf16, one spare slab past the last b*H + h, filled with the sentinel beforehand)."""
    from ezaudio_b200 import _lib
    D = H * dh
    ld_qk = ld_qk or (80 if dh == 72 else 64)
    dvp, Lpad, BH = _dvp(dh), _lpad(L), B * H
    outs = {}
    for kd in kinds:
        shape = (BH + 1, dvp, Lpad) if kd == 2 else (BH + 1, L, ld_qk)
        outs[kd] = torch.full(shape, SENT, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    a = _lib.TestHeadsArgs()
    a.B, a.L, a.D, a.H, a.dh, a.nsec = B, L, D, H, dh, len(kinds)
    for i, kd in enumerate(kinds):
        a.kinds[i] = kd
    a.norm_q, a.norm_k = (None if nq is None else nq.data_ptr()), (None if nk is None else nk.data_ptr())
    a.inv_freq = None if inv_freq is None else inv_freq.data_ptr()
    a.rope = rope
    a.q, a.k, a.vt = (outs[kd].data_ptr() if kd in outs else None for kd in (0, 1, 2))
    a.ld_qk, a.dvp, a.Lpad, a.variant = ld_qk, dvp, Lpad, variant
    if fold is not None:
        a.fold_st, a.fold_slots, a.fold_ld_st = fold["st"].data_ptr(), fold["st"].shape[0], fold["st"].shape[1]
        a.fold_u, a.fold_v = fold["u"].data_ptr(), fold["v"].data_ptr()
    _lib.check(_lib.lib().ezb_test_heads(0, _lib.ptr(A), _lib.ptr(W), C.byref(a), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return outs


def _inputs(seed, M, D, nsec, dh):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, D, device="cuda", generator=g).bfloat16()
    W = torch.randn(nsec * D, D, device="cuda", generator=g) / math.sqrt(D)
    # q and k affines differ everywhere, so either one applied to the other kind shows
    nq = torch.stack([1 + 0.3 * torch.randn(dh, device="cuda", generator=g), 0.3 * torch.randn(dh, device="cuda", generator=g)]).contiguous()
    nk = torch.stack([1 + 0.3 * torch.randn(dh, device="cuda", generator=g), 0.3 * torch.randn(dh, device="cuda", generator=g)]).contiguous()
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dh, 2, device="cuda", dtype=torch.float32) / dh))
    return A, W, nq, nk, inv_freq


def _reference(u, *, B, L, H, dh, kinds, nq, nk, inv_freq, rope):
    """u: fp64 [B*L, nsec*D] projection.  Returns {kind: (ref, extra)}, ref shaped like the valid part of the output, extra = the MUFU
    allowance per element (0 elsewhere)."""
    D = H * dh
    out = {}
    for s, kd in enumerate(kinds):
        x = u[:, s * D:(s + 1) * D].reshape(B, L, H, dh)
        if kd == 2:
            out[kd] = (x.permute(0, 2, 3, 1).reshape(B * H, dh, L), torch.zeros((), dtype=torch.float64, device=u.device))
            continue
        p = (nq if kd == 0 else nk).double()
        mu = x.mean(-1, keepdim=True)
        y = (x - mu) / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-5) * p[0] + p[1]
        extra = torch.zeros((), dtype=torch.float64, device=u.device)
        if rope != ROPE_NONE:
            theta = (torch.arange(L, device=u.device, dtype=torch.float32)[:, None] * inv_freq[None, :]).double()   # [L, dh/2], fp32 angle
            c, sn = torch.cos(theta)[None, :, None, :], torch.sin(theta)[None, :, None, :]
            a, b = y[..., :dh // 2], y[..., dh // 2:]
            y = torch.cat([a * c - b * sn, b * c + a * sn], -1)
            if rope == ROPE_MUFU:
                ang = (theta.abs() * 2.0 ** -22 + 2.0 ** -20)[None, :, None, :] * torch.sqrt(a * a + b * b)
                extra = torch.cat([ang, ang], -1).permute(0, 2, 1, 3).reshape(B * H, L, dh)
        out[kd] = (y.permute(0, 2, 1, 3).reshape(B * H, L, dh), extra)
    return out


def _check(outs, refs, *, B, L, H, dh, tag):
    """Values against the fp64 reference (per element and mean) and the layout contract.  Prints, per output, the largest excess of the error
    over one bf16 rounding, max(|got - ref| - 2^-8 |ref|): it approaches the fp32 error before the rounding, which the allowance EPS_ABS (+ the
    MUFU term) bounds.  Returns that excess."""
    BH, worst = B * H, float("-inf")
    for kd, buf in outs.items():
        ref, extra = refs[kd]
        bits = buf.view(torch.int16)
        if kd == 2:
            got = buf[:BH, :dh, :L].double()
            assert bool((bits[:BH, dh:, :L] == 0).all()), f"{tag}: V^T pad rows dh..dvp not written as zeros"
            assert bool((bits[:BH, :, L:] == SENT).all()), f"{tag}: V^T pad columns L..Lpad written"
        else:
            got = buf[:BH, :, :dh].double()
            assert bool((bits[:BH, :, dh:] == SENT).all()), f"{tag}: kind {kd} pad columns dh..ld_qk written"
        assert bool((bits[BH:] == SENT).all()), f"{tag}: kind {kd}: a slab past b*H + h written"
        err = (got - ref).abs()
        excess = (err - 2.0 ** -8 * ref.abs()).nan_to_num(nan=float("inf"))
        ok = excess <= EPS_ABS + extra          # NaN (an unwritten sentinel) fails
        i = int(excess.argmax())
        worst = max(worst, float(excess.max()))
        print(f"[heads] {tag} kind {kd}: max-abs err {float(err.max()):.3e}, mean-abs err {float(err.mean()):.3e}; largest excess over one bf16 "
              f"rounding {float(excess.max()):.3e} (allowance there {EPS_ABS + float(extra.flatten()[i] if extra.dim() else 0.0):.3e})")
        assert bool(ok.all()), f"{tag}: kind {kd}: {int((~ok).sum())} elements out of bound, largest excess {float(excess.max()):.3e}"
        mean_bound = 0.75 * 2.0 ** -8 * float(ref.abs().mean()) + EPS_ABS + float(extra.mean() if extra.dim() else 0.0)
        assert float(err.mean()) <= mean_bound, f"{tag}: kind {kd}: mean error {float(err.mean()):.3e} > {mean_bound:.3e}"
    return worst


def _same_bits(a, b):
    return all(torch.equal(a[k].view(torch.int16), b[k].view(torch.int16)) for k in a)


# dh, H, B, L, ld_qk, RoPE.  H = 16: the XL shape (5 1/3 packed tiles per section, tiles straddle q / k / v); H = 2 / 4 at dh = 72: K = 144 /
# 288, i.e. 3 / 5 64-wide k-blocks.  M = 25 / 75 / 200: clips shorter than a 32-row group; M = 320: three 128-row tiles (the cluster kernels'
# empty fourth tile); L = 1500: positions up to 1499.
SELF = [(72, 16, 2, 1500, 80, ROPE_MUFU), (72, 16, 2, 1500, 80, ROPE_TABLE), (72, 16, 1, 25, 128, ROPE_MUFU), (72, 2, 3, 130, 80, ROPE_TABLE),
        (72, 2, 8, 40, 128, ROPE_MUFU), (72, 4, 1, 500, 80, ROPE_TABLE), (72, 4, 3, 25, 80, ROPE_MUFU), (72, 2, 2, 1500, 128, ROPE_MUFU),
        (64, 4, 3, 130, 64, ROPE_TABLE), (64, 16, 2, 1500, 64, ROPE_MUFU), (64, 4, 8, 25, 64, ROPE_MUFU), (64, 16, 1, 40, 64, ROPE_TABLE)]


@gpu
@pytest.mark.parametrize("dh,H,B,L,ld_qk,rope", SELF)
def test_self_attention_qkv_heads(dh, H, B, L, ld_qk, rope):
    """nsec = 3 (q, k, v) with RoPE: every instantiation the model can dispatch for it.  Three heads per tile on the register fragment and on
    the parked tile run the same MMAs in the same k order and the same epilogue arithmetic, so they must agree bit for bit; so must the
    two-heads-per-tile cluster kernels on either schedule and the single-CTA kernel."""
    D, M, kinds = H * dh, B * L, (0, 1, 2)
    A, W, nq, nk, inv_freq = _inputs(dh * 1000 + H * 100 + L + B, M, D, 3, dh)
    kw = dict(B=B, L=L, H=H, dh=dh, kinds=kinds, rope=rope, nq=nq, nk=nk, inv_freq=inv_freq, ld_qk=ld_qk)
    u = A.double() @ W.bfloat16().double().t()
    refs = _reference(u, B=B, L=L, H=H, dh=dh, kinds=kinds, nq=nq, nk=nk, inv_freq=inv_freq, rope=rope)
    packed = _run(A, W, variant=PACKED3, **kw)
    excess = _check(packed, refs, B=B, L=L, H=H, dh=dh, tag=f"qkv dh{dh} H{H} B{B} L{L} ld{ld_qk} rope{rope} packed-3")
    assert _same_bits(packed, _run(A, W, variant=PACKED3_PARKED, **kw)), "packed-3 fragment != parked"
    pair = _run(A, W, variant=PAIR, **kw)
    _check(pair, refs, B=B, L=L, H=H, dh=dh, tag=f"qkv dh{dh} H{H} B{B} L{L} ld{ld_qk} rope{rope} pair-2")
    assert _same_bits(pair, _run(A, W, variant=PAIR_PARKED, **kw)), "pair-2 fragment != parked"
    assert _same_bits(pair, _run(A, W, variant=SINGLE, **kw)), "single-CTA != pair-2"
    if rope == ROPE_MUFU:   # on record: what __sincosf costs against the table at these angles
        trefs = _reference(u, B=B, L=L, H=H, dh=dh, kinds=kinds, nq=nq, nk=nk, inv_freq=inv_freq, rope=ROPE_TABLE)
        table = _check(_run(A, W, variant=PACKED3, **{**kw, "rope": ROPE_TABLE}), trefs, B=B, L=L, H=H, dh=dh, tag=f"qkv dh{dh} H{H} B{B} L{L} table")
        print(f"[heads] qkv dh{dh} H{H} B{B} L{L}: largest excess over one bf16 rounding, MUFU RoPE {excess:.3e} vs table {table:.3e} "
              f"(positions up to {L - 1}; table allowance {EPS_ABS:.0e})")


@gpu
@pytest.mark.parametrize("dh,H,B,Lc", [(72, 16, 8, 1), (72, 16, 8, 12), (72, 16, 8, 100), (72, 2, 5, 12), (64, 4, 3, 12), (64, 16, 8, 100)])
def test_cross_attention_kv_cache_heads(dh, H, B, Lc):
    """nsec = 2, kinds (k, v), no RoPE: the context K / V^T cache.  Several clips share one 32-row group (the staged store loop wraps rows
    across clip boundaries)."""
    D, M, kinds = H * dh, B * Lc, (1, 2)
    A, W, nq, nk, _ = _inputs(dh * 1000 + H * 100 + Lc + B, M, D, 2, dh)
    kw = dict(B=B, L=Lc, H=H, dh=dh, kinds=kinds, nk=nk)
    refs = _reference(A.double() @ W.bfloat16().double().t(), B=B, L=Lc, H=H, dh=dh, kinds=kinds, nq=None, nk=nk, inv_freq=None, rope=ROPE_NONE)
    pair = _run(A, W, variant=PAIR, **kw)
    _check(pair, refs, B=B, L=Lc, H=H, dh=dh, tag=f"ctx-kv dh{dh} H{H} B{B} Lc{Lc}")
    assert _same_bits(pair, _run(A, W, variant=PAIR_PARKED, **kw)), "pair-2 fragment != parked"
    assert _same_bits(pair, _run(A, W, variant=SINGLE, **kw)), "single-CTA != pair-2"


@gpu
@pytest.mark.parametrize("dh,H,B,L", [(72, 16, 2, 1500), (72, 16, 3, 25), (64, 4, 2, 130)])
def test_cross_attention_q_heads(dh, H, B, L):
    """nsec = 1, kind q, no RoPE, no k LayerNorm: the cross-attention query on 2-CTA clusters and on the single-CTA kernel (option
    cq_single)."""
    D, M, kinds = H * dh, B * L, (0,)
    A, W, nq, _, _ = _inputs(dh * 1000 + H * 100 + L + B + 7, M, D, 1, dh)
    kw = dict(B=B, L=L, H=H, dh=dh, kinds=kinds, nq=nq)
    refs = _reference(A.double() @ W.bfloat16().double().t(), B=B, L=L, H=H, dh=dh, kinds=kinds, nq=nq, nk=None, inv_freq=None, rope=ROPE_NONE)
    pair = _run(A, W, variant=PAIR, **kw)
    _check(pair, refs, B=B, L=L, H=H, dh=dh, tag=f"cross-q dh{dh} H{H} B{B} L{L}")
    assert _same_bits(pair, _run(A, W, variant=PAIR_PARKED, **kw)), "pair-2 fragment != parked"
    assert _same_bits(pair, _run(A, W, variant=SINGLE, **kw)), "single-CTA != pair-2"


def _packed_columns(H, dh, nsec, packed):
    """Packed output column of every reference column n = s*D + h*dh + j (pack_weight_kernel's h3 layout), and the packed width."""
    n = torch.arange(nsec * H * dh, device="cuda")
    if not packed:
        return n, nsec * H * dh
    bn = 224 if dh == 72 else 3 * dh
    g, j = n // dh, n % dh          # global head in [q heads | k heads | v heads]
    return (g // 3) * bn + (g % 3) * dh + j, H * bn


def _fold_inputs(seed, M, D, W, H, dh, nsec, packed):
    """x fp32, the LayerNorm affine g, c (incl. a modulation) -> A = bf16(x g), per-row partials of x in 32-feature slots, u = W g, v = W c in
    the packed column order (zeros in the pad columns)."""
    g_ = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, D, device="cuda", generator=g_) * 1.3 + 0.4
    gv = 1 + 0.3 * torch.randn(D, device="cuda", generator=g_)
    cv = 0.3 * torch.randn(D, device="cuda", generator=g_)
    A = (x * gv).bfloat16()
    slots = (D + 31) // 32   # D = 144 (H = 2): the last slot holds 16 features
    xs = torch.nn.functional.pad(x, (0, 32 * slots - D)).view(M, slots, 32)
    st = torch.stack([xs.sum(-1), (xs * xs).sum(-1)], -1).transpose(0, 1).contiguous()   # float2 [slots][M]
    Wb = W.bfloat16().double()
    cols, width = _packed_columns(H, dh, nsec, packed)
    u = torch.zeros(width, device="cuda")
    v = torch.zeros(width, device="cuda")
    u[cols] = (Wb @ gv.double()).float()
    v[cols] = (Wb @ cv.double()).float()
    xd = x.double()
    mu = xd.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-5)
    uref = rstd * (A.double() @ Wb.t() - mu * u[cols].double()) + v[cols].double()
    return A, dict(st=st, u=u, v=v), uref


@gpu
@pytest.mark.parametrize("dh,H,B,L,ld_qk,rope,nsec", [(72, 16, 2, 1500, 80, ROPE_MUFU, 3), (72, 2, 8, 40, 128, ROPE_TABLE, 3),
                                                      (64, 4, 3, 130, 64, ROPE_MUFU, 3), (72, 16, 2, 500, 80, ROPE_NONE, 1),
                                                      (64, 4, 3, 25, 64, ROPE_NONE, 1)])
def test_folded_layernorm_heads(dh, H, B, L, ld_qk, rope, nsec):
    """FOLD instantiations (LayerNorm of the block input folded into the projection): the epilogue's rstd * (A W^T - mu u) + v followed by
    the same per-head LayerNorm, RoPE and layout.  Whether the fold equals the true LayerNorm is test_fold_layers_gpu.py's job."""
    D, M = H * dh, B * L
    kinds = (0, 1, 2) if nsec == 3 else (0,)
    _, W, nq, nk, inv_freq = _inputs(dh * 1000 + H * 100 + L + B + 11, M, D, nsec, dh)
    kw = dict(B=B, L=L, H=H, dh=dh, kinds=kinds, rope=rope, nq=nq, nk=nk if nsec == 3 else None, inv_freq=inv_freq, ld_qk=ld_qk)
    for variant in ((PACKED3, PAIR) if nsec == 3 else (PAIR,)):
        A, fold, uref = _fold_inputs(M + nsec, M, D, W, H, dh, nsec, variant == PACKED3)
        refs = _reference(uref, B=B, L=L, H=H, dh=dh, kinds=kinds, nq=nq, nk=nk, inv_freq=inv_freq, rope=rope)
        out = _run(A, W, variant=variant, fold=fold, **kw)
        _check(out, refs, B=B, L=L, H=H, dh=dh, tag=f"fold nsec{nsec} dh{dh} H{H} B{B} L{L} rope{rope} variant{variant}")


def test_heads_hook_rejects_bad_arguments():
    """Argument validation happens before any device work (this runs without a GPU): the hook refuses shapes its kernels would run out of
    range on instead of launching them."""
    from ezaudio_b200 import _lib
    L_ = _lib.lib()
    buf = (C.c_float * 16)()
    p = C.c_void_p(C.addressof(buf))
    good = dict(B=2, L=40, D=1152, H=16, dh=72, kinds=(0, 1, 2), ld_qk=80, Lpad=40, variant=PACKED3)

    def rc(**over):
        c = {**good, **over}
        a = _lib.TestHeadsArgs()
        a.B, a.L, a.D, a.H, a.dh, a.nsec = c["B"], c["L"], c["D"], c["H"], c["dh"], len(c["kinds"])
        for i, kd in enumerate(c["kinds"]):
            a.kinds[i] = kd
        a.norm_q = a.norm_k = a.inv_freq = a.q = a.k = a.vt = p.value
        a.rope, a.ld_qk, a.dvp, a.Lpad, a.variant = ROPE_TABLE, c["ld_qk"], 80, c["Lpad"], c["variant"]
        return L_.ezb_test_heads(0, p, p, C.byref(a), None)

    EZB_ERR_ARG, EZB_ERR_SHAPE = -1, -2
    assert rc(dh=80, D=1280) == EZB_ERR_SHAPE       # head dimension other than 64 / 72
    assert rc(H=3, D=216) == EZB_ERR_SHAPE          # odd head count
    assert rc(D=1088) == EZB_ERR_SHAPE              # D != H * dh
    assert rc(ld_qk=64) == EZB_ERR_SHAPE            # q / k pitch narrower than a head
    assert rc(Lpad=32) == EZB_ERR_SHAPE             # V^T pitch shorter than the clip
    assert rc(kinds=(0,)) == EZB_ERR_SHAPE          # the packed-3 layout needs all three sections
    assert rc(variant=6) == EZB_ERR_ARG
    mid = C.c_void_p(C.addressof(buf))
    assert L_.ezb_test_mlp(0, p, p, p, p, p, p, p, 6 * 1152, 16, mid, p, 64, 1152, 4608, 0, None) == EZB_ERR_SHAPE   # clips < 32 rows
    assert L_.ezb_test_mlp(0, p, p, p, p, p, p, p, 6 * 1152, 64, mid, p, 64, 1152, 4608, 3, None) == EZB_ERR_ARG
