"""Attention kernels vs a plain PyTorch fp32 reference of the same op (softmax(q k^T/sqrt(dh) + key mask) v).
impl 0 = fp32 CUDA-core kernel (parity mode): tolerance 2e-2 is the bf16 rounding of the OUTPUT only (values O(1));
impl 1 = tensor-core kernel: q, k, v and P are bf16 operands -> tolerance 3e-2 abs on O(1) outputs."""
import math

import pytest
import torch

ATTN6_DEFAULT = 5   # csrc/attention_mma.cuh opt_attn6(): generation 6 (bits 1 / 2 have no effect on sm_90a)

pytestmark = pytest.mark.gpu


def _ref(q, k, v, mask):
    s = (q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1])
    if mask is not None:
        s = s.masked_fill(~mask[:, None, None, :].bool(), float("-inf"))
    o = s.softmax(-1) @ v
    return o.permute(0, 2, 1, 3).reshape(q.shape[0], q.shape[2], -1)


# 0 = fp32 CUDA-core kernel (parity mode); 1 = the tensor-core kernel the options select (generation 8 of attention_wgmma.cuh for dh 64 / 72
# by default, generation 6 of attention_mma.cuh for other head dims); 4 = generation 4 (128 query rows per CTA); +100 = q / k rows of 80 elements for dh = 72 (160-byte pitch) instead of 128
@pytest.mark.parametrize("impl", [0, 1, 4, 101, 104])
@pytest.mark.parametrize("B,H,Lq,Lk,dh,masked", [(2, 4, 500, 500, 72, False), (2, 3, 256, 256, 64, False), (3, 2, 500, 100, 72, True),
                                                 (2, 2, 40, 12, 72, True), (1, 2, 130, 130, 64, False), (1, 16, 1500, 1500, 72, False),
                                                 (2, 2, 37, 100, 64, True), (8, 16, 500, 500, 72, False), (2, 5, 700, 700, 72, "grow")])
def test_attention(impl, B, H, Lq, Lk, dh, masked):
    from ezaudio_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(Lq * 7 + Lk + dh)
    q = torch.randn(B, H, Lq, dh, device="cuda", generator=g) * 1.5
    k = torch.randn(B, H, Lk, dh, device="cuda", generator=g) * 1.5
    v = torch.randn(B, H, Lk, dh, device="cuda", generator=g)
    if masked == "grow":  # scores grow by orders of magnitude from key block to key block: exercises the in-place O rescale
        k = k * torch.linspace(0.2, 3.0, Lk, device="cuda")[None, None, :, None]
        masked = False
    mask = None
    if masked:
        mask = torch.zeros(B, Lk, dtype=torch.uint8, device="cuda")
        for i in range(B):
            mask[i, : (1 if i == B - 1 else min(Lk, 8 + 5 * i))] = 1
    out = torch.zeros(B, Lq, H * dh, device="cuda", dtype=torch.bfloat16)
    L = _lib.lib()
    if impl == 0:
        args = (q.contiguous(), k.contiguous(), v.contiguous())
        ref = _ref(q, k, v, mask)
    else:
        dhp, dvp, lkp = (dh + 63) // 64 * 64, (dh + 15) // 16 * 16, (Lk + 7) // 8 * 8
        if impl >= 100 and dh == 72:
            dhp = 80
        qb = torch.zeros(B * H, Lq, dhp, device="cuda", dtype=torch.bfloat16)
        kb = torch.zeros(B * H, Lk, dhp, device="cuda", dtype=torch.bfloat16)
        vt = torch.zeros(B * H, dvp, lkp, device="cuda", dtype=torch.bfloat16)
        qb[:, :, :dh] = q.reshape(B * H, Lq, dh)
        kb[:, :, :dh] = k.reshape(B * H, Lk, dh)
        vt[:, :dh, :Lk] = v.reshape(B * H, Lk, dh).transpose(1, 2)
        vt[:, :, Lk:] = 7.0  # beyond the true length: must never be read
        args = (qb, kb, vt)
        ref = _ref(q.bfloat16().float(), k.bfloat16().float(), v.bfloat16().float(), mask)
    _run(L, _lib, args, mask, out, B, H, Lq, Lk, dh, impl)
    torch.cuda.synchronize()
    err = (out.float() - ref).abs().max().item()
    assert math.isfinite(err) and err < (2e-2 if impl == 0 else 3e-2), err


def _run(L, _lib, args, mask, out, B, H, Lq, Lk, dh, impl):
    _lib.check(L.ezb_test_attention(0, _lib.ptr(args[0]), _lib.ptr(args[1]), _lib.ptr(args[2]), _lib.ptr(mask), _lib.ptr(out), B, H, Lq, Lk, dh, impl,
                                    _lib.stream_ptr()))
    torch.cuda.synchronize()


@pytest.mark.parametrize("B,H,Lq,Lk,dh,masked", [(2, 4, 500, 500, 72, False), (3, 2, 500, 100, 72, True), (2, 2, 40, 12, 72, True), (1, 16, 1500, 1500, 72, False),
                                                 (2, 3, 256, 256, 64, False), (8, 16, 500, 500, 72, False), (2, 5, 400, 512, 72, "grow"), (5, 3, 300, 100, 64, True),
                                                 (16, 16, 500, 500, 72, False), (2, 2, 130, 385, 72, True)])
def test_attention_kv_resident(B, H, Lq, Lk, dh, masked):
    """Generation 4 with the K / V^T key blocks of a head resident in shared memory (option attn_res; falls back above 512 keys): odd and even
    numbers of query tiles per head, one to eight key blocks, more heads than SMs (two waves of CTAs), masks, growth."""
    from ezaudio_b200 import _lib
    L = _lib.lib()
    _lib.check(L.ezb_set_option(b"attn6", 0))   # generation-4 kernel (the default is generation 8)
    _lib.check(L.ezb_set_option(b"attn_res", 1))
    try:
        test_attention(1, B, H, Lq, Lk, dh, masked)
        test_attention(101, B, H, Lq, Lk, dh, masked)
    finally:
        _lib.check(L.ezb_set_option(b"attn_res", 0))
        _lib.check(L.ezb_set_option(b"attn6", ATTN6_DEFAULT))


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,Lq,Lk,dh,masked", [(2, 4, 500, 500, 72, False), (3, 2, 500, 100, 72, True), (2, 2, 40, 12, 72, True), (1, 16, 1500, 1500, 72, False),
                                                 (2, 3, 256, 256, 64, False), (8, 16, 500, 500, 72, False), (2, 5, 400, 512, 72, "grow"), (5, 3, 300, 100, 64, True),
                                                 (16, 16, 500, 500, 72, False), (2, 2, 130, 385, 72, True), (1, 1, 100, 300, 72, False), (1, 3, 128, 128, 72, True)])
@pytest.mark.parametrize("res", [0, 1])
def test_attention_mufu_token(B, H, Lq, Lk, dh, masked, res):
    """Generation 4 with the option attn_pp set (it scheduled the softmax groups of the sm_100a kernel and leaves the sm_90a kernel unchanged):
    a single query tile, one to twelve key blocks, with and without resident K / V^T."""
    from ezaudio_b200 import _lib
    L = _lib.lib()
    _lib.check(L.ezb_set_option(b"attn6", 0))   # generation-4 kernel (the default is generation 8)
    _lib.check(L.ezb_set_option(b"attn_pp", 1))
    _lib.check(L.ezb_set_option(b"attn_res", res))
    try:
        test_attention(1, B, H, Lq, Lk, dh, masked)
        test_attention(101, B, H, Lq, Lk, dh, masked)
    finally:
        _lib.check(L.ezb_set_option(b"attn_pp", 0))
        _lib.check(L.ezb_set_option(b"attn_res", 0))
        _lib.check(L.ezb_set_option(b"attn6", ATTN6_DEFAULT))


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,Lq,Lk,dh,masked", [(2, 4, 500, 500, 72, False), (3, 2, 500, 100, 72, True), (2, 2, 40, 12, 72, True), (1, 16, 1500, 1500, 72, False),
                                                 (2, 3, 256, 256, 64, False), (8, 16, 500, 500, 72, False), (2, 5, 400, 512, 72, "grow"), (5, 3, 300, 100, 64, True),
                                                 (16, 16, 500, 500, 72, False), (2, 2, 130, 385, 72, True), (1, 1, 100, 300, 72, False), (1, 3, 128, 128, 72, True)])
@pytest.mark.parametrize("mode", [0, 1, 3, 5, 7])
def test_attention_gen6(B, H, Lq, Lk, dh, masked, mode):
    """Every value of the option attn6 (bit 0: generation 6, 64 query rows per CTA, else generation 4; bits 1 and 2 are accepted and change
    nothing on sm_90a): a single query tile, one to twelve key blocks, key masks, score growth (O rescale), dh = 64 and 72, both q / k row
    pitches."""
    from ezaudio_b200 import _lib
    L = _lib.lib()
    _lib.check(L.ezb_set_option(b"attn6", mode))
    try:
        test_attention(1, B, H, Lq, Lk, dh, masked)
        test_attention(101, B, H, Lq, Lk, dh, masked)
    finally:
        _lib.check(L.ezb_set_option(b"attn6", ATTN6_DEFAULT))


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,Lq,Lk,dh,masked", [(2, 4, 500, 500, 72, False), (3, 2, 500, 100, 72, True), (2, 2, 40, 12, 72, True), (1, 16, 1500, 1500, 72, False),
                                                 (2, 3, 256, 256, 64, False), (8, 16, 500, 500, 72, False), (2, 5, 400, 512, 72, "grow"), (5, 3, 300, 100, 64, True),
                                                 (16, 16, 500, 500, 72, False), (2, 2, 130, 385, 72, True), (1, 1, 100, 300, 72, False), (1, 3, 128, 128, 72, True),
                                                 (3, 5, 200, 65, 72, True), (1, 2, 640, 192, 64, False), (37, 4, 512, 512, 72, False)])
def test_attention_gen7(B, H, Lq, Lk, dh, masked):
    """Generation 7 (128-key blocks): partial last blocks (385, 65, 192 keys), a lone key in the last block, up to 12 blocks, key masks, score
    growth (O rescale), dh = 64 and 72, both q / k row pitches, Lk below one block, many CTAs."""
    test_attention(7, B, H, Lq, Lk, dh, masked)
    test_attention(107, B, H, Lq, Lk, dh, masked)
