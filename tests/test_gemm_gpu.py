"""wgmma GEMM kernels through ezb_test_gemm.  The linear-epilogue tests (bn 64 / 128 / 256, single-CTA and 2-CTA cluster) hold the kernel
to the fp64 bounds of test_linear_gpu.py on exactly the bf16 operands it reads, with outputs framed by a NaN / sentinel border that must
stay untouched.  The GEGLU and conv-addressing tests compare with a PyTorch fp32 reference of the same op (bf16-rounded operands, fp32
math): only summation order differs, |err| <= 2e-3 * sqrt(K/1024) on O(1..30) outputs for fp32 out; bf16 outputs add one bf16 rounding
(rel 2^-8)."""
import ctypes as C
import math

import pytest
import torch

from tests.test_linear_gpu import ACT_SILU, PADC, _check_bf16, _check_f32, _check_layout_bf16, _check_layout_f32, _f32_out, _sentinel

pytestmark = pytest.mark.gpu


def _run(A, W, epi, M, N, K, bn, kind=0, conv=(0, 0, 0, 0, 0, 0)):
    from ezaudio_b200 import _lib
    L = _lib.lib()
    _lib.check(L.ezb_test_gemm(0, _lib.ptr(A), A.stride(-2), _lib.ptr(W), W.stride(0), M, N, K, bn, kind, C.byref(epi), *conv,
                               _lib.stream_ptr()))
    torch.cuda.synchronize()


def _epi(**kw):
    from ezaudio_b200 import _lib
    e = _lib.TestEpilogue()
    for k, v in kw.items():
        setattr(e, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return e


def _mm64(A, W, bias=None):
    """fp64 A W^T (+ bias) and S = |A| |W|^T (+ |bias|) of the bf16 operands."""
    a, w = A.double(), W.double()
    ref, S = a @ w.t(), a.abs() @ w.abs().t()
    if bias is not None:
        ref, S = ref + bias.double(), S + bias.double().abs()
    return ref, S


@pytest.mark.parametrize("M,N,K,bn", [(4000, 1152, 1152, 128), (300, 144, 144, 128), (4000, 1152, 4608, 128), (1000, 3456, 1152, 256),
                                      (257, 128, 1152, 64), (128, 128, 64, 128), (777, 2304, 264, 128)])
def test_gemm_f32_out(M, N, K, bn):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    out = _f32_out(M, N)
    _run(A, W, _epi(out_f32=out, ld32=N + PADC), M, N, K, bn)
    _check_layout_f32(out, M, N, f"bn {bn}")
    ref, S = _mm64(A, W)
    _check_f32(out[:M, :N], ref, S, f"bn {bn} M {M} N {N} K {K}")


def test_gemm_bias_gate_residual():
    M, N, K, L = 1000, 1152, 1152, 250
    g = torch.Generator(device="cuda").manual_seed(1)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g)
    gate = torch.randn(M // L, 6 * N, device="cuda", generator=g) * 0.3
    out = _f32_out(M, N)
    _run(A, W, _epi(bias=bias, resid=x, ldr=N, gate=gate[:, 2 * N:], gate_bstride=6 * N, rows_per_batch=L, out_f32=out, ld32=N + PADC), M, N, K, 128)
    _check_layout_f32(out, M, N, "gated residual")
    ref, S = _mm64(A, W, bias)
    keep = 1 - gate[:, 2 * N:3 * N].double().repeat_interleave(L, 0)
    _check_f32(out[:M, :N], x.double() + keep * ref, keep.abs() * S + x.double().abs(), "gated residual")
    # in-place residual (out aliases resid), no gate
    x2 = _f32_out(M, N, x)
    _run(A, W, _epi(bias=bias, resid=x2, ldr=N + PADC, out_f32=x2, ld32=N + PADC), M, N, K, 128)
    _check_layout_f32(x2, M, N, "residual")
    _check_f32(x2[:M, :N], x.double() + ref, S + x.double().abs(), "residual")


@pytest.mark.parametrize("split", [False, True])
def test_gemm_bf16_silu_and_split(split):
    M, N, K = 800, 1152, 2048
    g = torch.Generator(device="cuda").manual_seed(2)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    width = 3 * N if split else N
    out = _sentinel(M + 1, width + PADC)
    _run(A, W, _epi(bias=bias, out_bf16=out, ld16=width + PADC, split_stride=N if split else 0, act=1), M, N, K, 128)
    _check_layout_bf16(out, M, width, f"split {split}")
    ref, S = _mm64(A, W, bias)
    _check_bf16(out[:M], N, split, ref, S, ACT_SILU, f"split {split}")


@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_geglu(bn):
    M, D, inner = 900, 1152, 4608
    g = torch.Generator(device="cuda").manual_seed(3)
    A = torch.randn(M, D, device="cuda", generator=g).bfloat16()
    W = (torch.randn(2 * inner, D, device="cuda", generator=g) / math.sqrt(D)).bfloat16()  # reference layout: [hidden; gate]
    bias = torch.randn(2 * inner, device="cuda", generator=g) * 0.1
    half = bn // 2
    Wp = torch.stack([W[:inner].view(inner // half, half, D), W[inner:].view(inner // half, half, D)], 1).reshape(2 * inner, D).contiguous()
    bp = torch.stack([bias[:inner].view(-1, half), bias[inner:].view(-1, half)], 1).reshape(-1).contiguous()
    out = torch.zeros(M, inner, device="cuda", dtype=torch.bfloat16)
    _run(A, Wp, _epi(bias=bp, out_bf16=out, ld16=inner), M, 2 * inner, D, bn, kind=1)
    u = A.float() @ W.float().t() + bias
    ref = u[:, :inner] * torch.nn.functional.gelu(u[:, inner:])
    assert (out.float() - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item() / 4)


@pytest.mark.parametrize("Cin,Cout,taps,dil,T,B", [(128, 128, 7, 9, 1000, 2), (256, 128, 7, 1, 300, 1), (32, 64, 7, 3, 200, 2), (1024, 512, 3, 1, 130, 2)])
def test_gemm_conv_addressing(Cin, Cout, taps, dil, T, B):
    """Implicit-GEMM conv over channels-last activations == F.conv1d with zero padding, + snake epilogue."""
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(B, T, Cin, device="cuda", generator=g).bfloat16()
    w = (torch.randn(Cout, Cin, taps, device="cuda", generator=g) / math.sqrt(Cin * taps)).bfloat16()
    bias = torch.randn(Cout, device="cuda", generator=g) * 0.1
    a, binv = torch.rand(Cout, device="cuda", generator=g) + 0.5, torch.rand(Cout, device="cuda", generator=g) + 0.5
    cin_pad = (Cin + 63) // 64 * 64
    Wp = torch.zeros(Cout, taps, cin_pad, device="cuda", dtype=torch.bfloat16)
    Wp[:, :, :Cin] = w.permute(0, 2, 1)
    Wp = Wp.reshape(Cout, taps * cin_pad).contiguous()
    raw = torch.empty(B * T, Cout, device="cuda")
    act = torch.empty(B * T, Cout, device="cuda", dtype=torch.bfloat16)
    center = (taps - 1) // 2
    _run(x, Wp, _epi(bias=bias, out_f32=raw, ld32=Cout, out_bf16=act, ld16=Cout, act=2, act_a=a, act_b=binv), B * T, Cout, Cin, 128 if Cout >= 128 else 64,
         conv=(taps, center, dil, cin_pad, T, B))
    ref = torch.nn.functional.conv1d(x.float().transpose(1, 2), w.float(), bias, dilation=dil, padding=center * dil).transpose(1, 2).reshape(B * T, Cout)
    assert (raw - ref).abs().max().item() < 3e-3
    sref = ref + binv * torch.sin(ref * a) ** 2
    assert (act.float() - sref).abs().max().item() < 3e-2


@pytest.mark.parametrize("M,N,K,bn", [(4000, 1152, 1152, 128), (300, 144, 144, 128), (4000, 1152, 4608, 128), (1000, 3456, 1152, 256), (129, 256, 64, 256),
                                      (777, 2304, 264, 128)])
def test_pair_gemm_f32_out(M, N, K, bn):
    """2-CTA cluster kernel (W tile multicast to both CTAs), same bound as the single-CTA one."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    out = _f32_out(M, N)
    _run(A, W, _epi(out_f32=out, ld32=N + PADC, bias=bias), M, N, K, bn, kind=10)
    _check_layout_f32(out, M, N, f"pair bn {bn}")
    ref, S = _mm64(A, W, bias)
    _check_f32(out[:M, :N], ref, S, f"pair bn {bn} M {M} N {N} K {K}")


def test_pair_gemm_geglu():
    M, D, inner, bn = 900, 1152, 4608, 256
    g = torch.Generator(device="cuda").manual_seed(3)
    A = torch.randn(M, D, device="cuda", generator=g).bfloat16()
    W = (torch.randn(2 * inner, D, device="cuda", generator=g) / math.sqrt(D)).bfloat16()
    bias = torch.randn(2 * inner, device="cuda", generator=g) * 0.1
    half = bn // 2
    Wp = torch.stack([W[:inner].view(inner // half, half, D), W[inner:].view(inner // half, half, D)], 1).reshape(2 * inner, D).contiguous()
    bp = torch.stack([bias[:inner].view(-1, half), bias[inner:].view(-1, half)], 1).reshape(-1).contiguous()
    out = torch.zeros(M, inner, device="cuda", dtype=torch.bfloat16)
    _run(A, Wp, _epi(bias=bp, out_bf16=out, ld16=inner), M, 2 * inner, D, bn, kind=11)
    u = A.float() @ W.float().t() + bias
    ref = u[:, :inner] * torch.nn.functional.gelu(u[:, inner:])
    assert (out.float() - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item() / 4)


def _geglu_ref(A, W, bias, inner):
    """fp64 h * gelu_erf(g), [h; g] = A W^T + bias in the reference row order."""
    u = A.double() @ W.double().t() + bias.double()
    return u[:, :inner] * torch.nn.functional.gelu(u[:, inner:])


@pytest.mark.parametrize("M,L,D,inner", [(64, 32, 1152, 4608), (300, 100, 1152, 512), (1000, 40, 1152, 4608), (4000, 500, 1152, 4608),
                                         (1000, 250, 384, 512)])
def test_mlp_fused_matches_two_launch_and_fp64(M, L, D, inner):
    """The persistent MLP kernel (GEGLU GEMM on 2-CTA clusters, grid barrier, swap-AB output projection with the gated residual) against
    the same two GEMMs as two launches (the same tiles and k order: bit-identical), the two-launch path with the GEGLU on the parked tile
    instead of the register-fragment schedule (also bit-identical) and fp64.  Clips of L rows do not align to the 128-row / 256-token tiles.  The reference takes the kernel's own bf16
    `mid` (checked separately to one bf16 rounding) so that the second GEMM is held to the swap-AB bound 3e-3 sqrt(K / 1024)."""
    from ezaudio_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(M + L + D + inner)
    A = torch.randn(M, D, device="cuda", generator=g).bfloat16()
    W1 = torch.randn(2 * inner, D, device="cuda", generator=g) / math.sqrt(D)      # reference layout [hidden; gate], packed by the hook
    b1 = torch.randn(2 * inner, device="cuda", generator=g) * 0.1
    W2 = (torch.randn(D, inner, device="cuda", generator=g) / math.sqrt(inner)).bfloat16()
    b2 = torch.randn(D, device="cuda", generator=g)
    x = torch.randn(M, D, device="cuda", generator=g)
    nb = (M + L - 1) // L
    gate = torch.randn(nb, 6 * D, device="cuda", generator=g) * 0.3
    bar = torch.zeros(2, dtype=torch.int32, device="cuda")

    def run(variant):
        xo = x.clone()
        mid = torch.full((M, inner), float("nan"), device="cuda", dtype=torch.bfloat16)
        _lib.check(lib.ezb_test_mlp(0, _lib.ptr(A), _lib.ptr(W1), _lib.ptr(b1), _lib.ptr(W2), _lib.ptr(b2), _lib.ptr(xo), _lib.ptr(gate[:, 5 * D:]),
                                    6 * D, L, _lib.ptr(mid), _lib.ptr(bar), M, D, inner, variant, _lib.stream_ptr()))
        torch.cuda.synchronize()
        return xo, mid

    x2, mid2 = run(1)
    xk, midk = run(2)
    assert torch.equal(midk.view(torch.int16), mid2.view(torch.int16)) and torch.equal(xk, x2)
    for i in range(3):   # the barrier resets itself: count back to 0, one generation per launch
        gen = int(bar[1])
        xf, midf = run(0)
        assert int(bar[0]) == 0 and int(bar[1]) == gen + 1, (i, bar.tolist())
        assert torch.equal(midf.view(torch.int16), mid2.view(torch.int16)), i
        assert torch.equal(xf, x2), i
    mid_ref = _geglu_ref(A, W1.bfloat16(), b1, inner)
    err = (mid2.double() - mid_ref).abs()
    assert bool((err <= 2.0 ** -8 * mid_ref.abs() + 2e-4).all()), float(err.max())
    keep = 1 - gate[:, 5 * D:].double().repeat_interleave(L, 0)[:M]
    ref = x.double() + keep * (mid2.double() @ W2.double().t() + b2.double())
    err = float((x2.double() - ref).abs().max())
    print(f"[mlp] M {M} L {L} D {D} inner {inner}: mid max-abs err {float((mid2.double() - mid_ref).abs().max()):.3e}, x max-abs err {err:.3e}")
    assert err < 3e-3 * max(1.0, math.sqrt(inner / 1024)), err


@pytest.mark.parametrize("M,N,K,L", [(4000, 1152, 1152, 500), (1000, 1152, 4608, 250), (300, 144, 144, 100), (777, 1024, 264, 259), (4000, 1152, 2304, 500)])
def test_swap_ab_gemm_gated_residual(M, N, K, L):
    """Swap-AB kernel (features on accumulator rows): bias + gated residual in place, and plain bias -> f32."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g)
    nb = (M + L - 1) // L
    gate = torch.randn(nb, 6 * N, device="cuda", generator=g) * 0.3
    ref_mm = A.float() @ W.float().t() + bias
    tol = 3e-3 * max(1.0, math.sqrt(K / 1024))
    out = torch.full((M, N), float("nan"), device="cuda")
    _run(A, W, _epi(bias=bias, out_f32=out, ld32=N), M, N, K, 256, kind=20)
    assert (out - ref_mm).abs().max().item() < tol
    x2 = x.clone()
    _run(A, W, _epi(bias=bias, resid=x2, ldr=N, gate=gate[:, 5 * N:], gate_bstride=6 * N, rows_per_batch=L, out_f32=x2, ld32=N), M, N, K, 256, kind=20)
    ref = x + (1 - gate[:, 5 * N:].repeat_interleave(L, 0)[:M]) * ref_mm
    assert (x2 - ref).abs().max().item() < tol
    x3 = x.clone()
    _run(A, W, _epi(bias=bias, resid=x3, ldr=N, out_f32=x3, ld32=N), M, N, K, 256, kind=20)
    assert (x3 - (x + ref_mm)).abs().max().item() < tol


@pytest.mark.parametrize("M,N,K,L", [(4000, 1152, 1152, 500), (4000, 1152, 4608, 500), (2000, 1152, 1152, 500), (4000, 1024, 1024, 500)])
def test_swap_ab_multicast_matches_plain(M, N, K, L):
    """wip: clusters of 3 feature tiles share the activation tile (TMA multicast).  Shapes that do not split into whole clusters
    (N = 1024: 8 feature tiles) or do not fit one wave must fall back and still be right."""
    from ezaudio_b200 import _lib
    L_ = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(M + N + K + 1)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g)
    ref = x + A.float() @ W.float().t() + bias
    tol = 3e-3 * max(1.0, math.sqrt(K / 1024))
    _lib.check(L_.ezb_set_option(b"swap_mc", 1))
    try:
        for _ in range(3):   # stage / phase wrap-around across launches
            x2 = x.clone()
            _run(A, W, _epi(bias=bias, resid=x2, ldr=N, out_f32=x2, ld32=N), M, N, K, 256, kind=20)
            torch.cuda.synchronize()
            assert (x2 - ref).abs().max().item() < tol
    finally:
        _lib.check(L_.ezb_set_option(b"swap_mc", 0))
