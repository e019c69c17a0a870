"""The GEGLU GEMM's overlapped schedule (gemm.cuh EpiGegluFrag: epilogue on the wgmma registers, TMA box stores, the producer streaming the next
tile's k-blocks meanwhile) against the parked-tile schedule it replaces, bit for bit, and against fp64."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(A, W, epi, M, N, K, kind):
    from ezaudio_b200 import _lib
    L = _lib.lib()
    _lib.check(L.ezb_test_gemm(0, _lib.ptr(A), A.stride(-2), _lib.ptr(W), W.stride(0), M, N, K, 256, kind, C.byref(epi), 0, 0, 0, 0, 0, 0,
                               _lib.stream_ptr()))
    torch.cuda.synchronize()


def _epi(**kw):
    from ezaudio_b200 import _lib
    e = _lib.TestEpilogue()
    for k, v in kw.items():
        setattr(e, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return e


# Many tiles per CTA with the ring phase wrapping inside and across tiles (M >= 4000), a partial last M tile and the empty padding tile of an
# odd M-tile count (M = 130: 2 tiles; 257 / 300: 3 tiles + 1 padding); K = 64 is one k-block, 1088 / 1216 leave the ring mid-phase at a
# tile's end.
@pytest.mark.parametrize("M,K,inner", [(4000, 1152, 4608), (4000, 64, 1024), (6000, 1216, 4608), (8000, 1088, 1024), (32000, 1152, 4608),
                                       (130, 64, 1024), (130, 1088, 4608), (257, 1152, 4608), (257, 1216, 1024), (900, 64, 1024), (300, 1088, 1024),
                                       (1000, 1216, 1024), (257, 1152, 1024)])
def test_geglu_overlapped_matches_parked(M, K, inner):
    """Kind 11 (what Dit::block dispatches: the overlapped schedule) == kind 12 (the parked-tile schedule, which bf16x3 and outputs without
    16-byte alignment run): the same MMAs in the same k order and the same epilogue arithmetic, so bit-identical.  Outputs sit in a NaN-filled
    buffer with a wider row pitch and extra rows: nothing outside [M, inner) may be written.  Against fp64: one bf16 rounding of the output
    (2^-8 relative) plus 2e-4 for the fp32 accumulation and the fast erf (|err| <= 1.5e-7 + 2 MUFU ulp, on |h gelu(g)| <~ 30)."""
    bn, half = 256, 128
    g = torch.Generator(device="cuda").manual_seed(M + K + inner)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(2 * inner, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(2 * inner, device="cuda", generator=g) * 0.1
    Wp = torch.stack([W[:inner].view(inner // half, half, K), W[inner:].view(inner // half, half, K)], 1).reshape(2 * inner, K).contiguous()
    bp = torch.stack([bias[:inner].view(-1, half), bias[inner:].view(-1, half)], 1).reshape(-1).contiguous()
    ld16 = inner + 64
    outs = {}
    for kind in (11, 12):
        buf = torch.full((M + 64, ld16), float("nan"), device="cuda", dtype=torch.bfloat16)
        _run(A, Wp, _epi(bias=bp, out_bf16=buf, ld16=ld16), M, 2 * inner, K, kind)
        assert bool(buf[M:].isnan().all()) and bool(buf[:M, inner:].isnan().all()), kind
        outs[kind] = buf[:M, :inner]
    assert torch.equal(outs[11].view(torch.int16), outs[12].view(torch.int16))
    u = A.double() @ W.double().t() + bias.double()
    ref = u[:, :inner] * torch.nn.functional.gelu(u[:, inner:])
    del u
    err = (outs[11].double() - ref).abs()
    assert bool((err <= 2.0 ** -8 * ref.abs() + 2e-4).all()), float(err.max())


@pytest.mark.parametrize("pitch_pad,offset", [(4, 0), (64, 4)])
def test_geglu_outputs_without_tma_alignment(pitch_pad, offset):
    """Outputs with only the 8-byte alignment the parked epilogue needs (a row pitch that is not a multiple of 8 elements, or a base 8 bytes
    past a 16-byte boundary) cannot take the TMA stores: the launch still succeeds, on the parked tile, with the same bits."""
    M, K, inner, half = 600, 1152, 1024, 128
    g = torch.Generator(device="cuda").manual_seed(7 + pitch_pad + offset)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(2 * inner, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(2 * inner, device="cuda", generator=g) * 0.1
    Wp = torch.stack([W[:inner].view(inner // half, half, K), W[inner:].view(inner // half, half, K)], 1).reshape(2 * inner, K).contiguous()
    bp = torch.stack([bias[:inner].view(-1, half), bias[inner:].view(-1, half)], 1).reshape(-1).contiguous()
    ld16 = inner + pitch_pad
    outs = {}
    for kind in (11, 12):
        flat = torch.full((offset + (M + 1) * ld16,), float("nan"), device="cuda", dtype=torch.bfloat16)
        out = flat[offset:offset + M * ld16].view(M, ld16)
        _run(A, Wp, _epi(bias=bp, out_bf16=out, ld16=ld16), M, 2 * inner, K, kind)
        assert bool(flat[:offset].isnan().all()) and bool(flat[offset + M * ld16:].isnan().all()) and bool(out[:, inner:].isnan().all()), kind
        outs[kind] = out[:, :inner]
    assert not bool(outs[11].isnan().any())
    assert torch.equal(outs[11].view(torch.int16), outs[12].view(torch.int16))
