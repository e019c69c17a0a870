"""Swap-AB GEMM with 288-token tiles against the same GEMM with 256-token tiles (ezb_test_gemm kind 21 forces the width, kind 20 takes the
width the model would).  Each output element gets the same k-ordered chain of k16 wgmma steps at either width, so every output is
bit-identical: bias -> f32, gated residual in place, plain residual in place, and the fold epilogue's outputs (LayerNorm folded in, the
next GEMM's bf16 operands and the per-token partial sums folded out).  Rows past the last token and columns past the last feature of the
padded outputs must stay NaN.  The 288-wide results are also held to an fp64 reference."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

PAD_ROWS, PAD_COLS = 40, 32
SHAPES = [(4000, 1152, 264, 500), (4000, 1152, 1152, 500), (4000, 1152, 2304, 500), (4000, 1152, 4608, 500), (8000, 1152, 1152, 500),
          (777, 1024, 264, 259),     # ragged last tile
          (1000, 1152, 1152, 140),   # clip boundaries at 140 and 280: inside the half chunks next to the 144-token warp boundary of a 288 tile
          (1000, 1152, 1152, 150)]   # clip boundary at 150: in the first chunk of the second warp


def _run(A, W, e, M, N, K, kind, bn):
    from ezaudio_b200 import _lib
    _lib.check(_lib.lib().ezb_test_gemm(0, _lib.ptr(A), A.stride(0), _lib.ptr(W), W.stride(0), M, N, K, bn, kind, C.byref(e), 0, 0, 0, 0, 0, 0,
                                        _lib.stream_ptr()))
    torch.cuda.synchronize()


def _epi(**kw):
    from ezaudio_b200 import _lib
    e = _lib.TestEpilogue()
    for k, v in kw.items():
        setattr(e, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return e


def _nan(rows, cols, dtype=torch.float32):
    return torch.full((rows, cols), float("nan"), device="cuda", dtype=dtype)


def _padded(x):
    out = _nan(x.shape[0] + PAD_ROWS, x.shape[1] + PAD_COLS)
    out[:x.shape[0], :x.shape[1]] = x
    return out


def _pads_nan(t, M, N):
    t = t.float()
    return bool(t[M:].isnan().all()) and bool(t[:, N:].isnan().all())


WIDTHS = [(21, 256), (21, 288), (20, 0)]   # kind 20: the width the model dispatches for this shape


@pytest.mark.parametrize("M,N,K,L", SHAPES)
def test_swap_ab_288_matches_256(M, N, K, L):
    g = torch.Generator(device="cuda").manual_seed(M + N + K + L)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g)
    nb = (M + L - 1) // L
    gate = torch.randn(nb, 6 * N, device="cuda", generator=g) * 0.3
    mm = A.double() @ W.double().t()
    keep = 1 - gate[:, 5 * N:].double().repeat_interleave(L, 0)[:M]
    tol = 3e-3 * max(1.0, math.sqrt(K / 1024))
    ld = N + PAD_COLS
    gate_kw = dict(gate=gate[:, 5 * N:], gate_bstride=6 * N, rows_per_batch=L)

    def variants():
        out = _nan(M + PAD_ROWS, ld)
        yield "bias", [out], _epi(bias=bias, out_f32=out, ld32=ld), mm + bias.double()
        xg = _padded(x)
        yield "gated residual", [xg], _epi(bias=bias, resid=xg, ldr=ld, out_f32=xg, ld32=ld, **gate_kw), x.double() + keep * (mm + bias.double())
        xr = _padded(x)
        yield "residual", [xr], _epi(bias=bias, resid=xr, ldr=ld, out_f32=xr, ld32=ld), x.double() + mm + bias.double()

    results = {}
    for kind, bn in WIDTHS:
        for name, outs, e, ref in variants():
            _run(A, W, e, M, N, K, kind, bn)
            for o in outs:
                assert _pads_nan(o, M, N), (name, kind, bn)
            results.setdefault(name, []).append((bn, outs[0][:M, :N].clone()))
            if bn == 288:
                err = float((outs[0][:M, :N].double() - ref).abs().max())
                assert err < tol, (name, err)
    for name, rs in results.items():
        for bn, r in rs[1:]:
            assert torch.equal(r, rs[0][1]), (name, bn)


@pytest.mark.parametrize("M,N,K,L", [s for s in SHAPES if s[2] in (264, 1152)])
def test_swap_ab_288_matches_256_fold(M, N, K, L):
    """The fold epilogue (EpiLinearTF): LayerNorm statistics folded in from per-token partials, gated residual, and folded out: two bf16
    operands x * g0, x * g1 and one (sum, sum of squares) partial per token and 32-feature slot."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K + L + 1)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g)
    nb = (M + L - 1) // L
    gate = torch.randn(nb, 6 * N, device="cuda", generator=g) * 0.3
    # fold-in: partials of a previous 1152-wide row, slot-major [slots][ld_st]
    Din, slots = 1152, 36
    xp = torch.randn(M, Din, device="cuda", generator=g) * 2 + 0.5
    st_in = torch.zeros(slots, M + 16, 2, device="cuda")
    st_in[:, :M, 0] = xp.view(M, slots, 32).sum(2).t()
    st_in[:, :M, 1] = (xp * xp).view(M, slots, 32).sum(2).t()
    u = torch.randn(N, device="cuda", generator=g) * 0.1
    v = torch.randn(N, device="cuda", generator=g) * 0.1
    g0 = torch.rand(N, device="cuda", generator=g) + 0.5
    g1 = torch.rand(N, device="cuda", generator=g) + 0.5
    ld, ld_st = N + PAD_COLS, M + PAD_ROWS
    res = []
    for kind, bn in WIDTHS:
        xo = _padded(x)
        a0, a1 = _nan(M + PAD_ROWS, ld, torch.bfloat16), _nan(M + PAD_ROWS, ld, torch.bfloat16)
        st = torch.full((N // 32, ld_st, 2), float("nan"), device="cuda")
        e = _epi(bias=bias, resid=xo, ldr=ld, out_f32=xo, ld32=ld, gate=gate[:, 5 * N:], gate_bstride=6 * N, rows_per_batch=L,
                 fin_st=st_in, fin_slots=slots, fin_ld_st=st_in.shape[1], fin_inv_dim=1.0 / Din, fin_u=u, fin_v=v,
                 fout_st=st, fout_ld_st=ld_st, fout_a0=a0, fout_ld0=ld, fout_g0=g0, fout_a1=a1, fout_ld1=ld, fout_g1=g1)
        _run(A, W, e, M, N, K, kind, bn)
        assert _pads_nan(xo, M, N) and _pads_nan(a0, M, N) and _pads_nan(a1, M, N), (kind, bn)
        assert bool(st[:, M:].isnan().all()), (kind, bn)
        res.append((bn, xo[:M, :N].clone(), a0[:M, :N].clone(), a1[:M, :N].clone(), st[:, :M].clone()))
    for bn, *outs in res[1:]:
        for i, (o, o0) in enumerate(zip(outs, res[0][1:])):
            assert torch.equal(o.view(torch.int16) if o.dtype == torch.bfloat16 else o,
                               o0.view(torch.int16) if o0.dtype == torch.bfloat16 else o0), (bn, i)
    _, xo, a0, a1, st = res[1]   # 288 wide
    mean = xp.double().mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(xp.double().var(1, unbiased=False, keepdim=True) + 1e-5)
    keep = 1 - gate[:, 5 * N:].double().repeat_interleave(L, 0)[:M]
    ref = x.double() + keep * (rstd * (A.double() @ W.double().t()) - rstd * mean * u.double() + v.double() + bias.double())
    err = float((xo.double() - ref).abs().max())
    assert err < 3e-3 * max(1.0, math.sqrt(K / 1024)) * float(rstd.max()), err
    assert torch.equal(a0.view(torch.int16), (xo * g0).bfloat16().view(torch.int16))
    assert torch.equal(a1.view(torch.int16), (xo * g1).bfloat16().view(torch.int16))
    part = xo.double().view(M, N // 32, 32)
    assert torch.allclose(st[..., 0].double(), part.sum(2).t(), rtol=1e-5, atol=1e-4)
    assert torch.allclose(st[..., 1].double(), (part * part).sum(2).t(), rtol=1e-5, atol=1e-3)
