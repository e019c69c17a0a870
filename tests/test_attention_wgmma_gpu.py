"""Generation 8 of the tensor-core attention (attention_wgmma.cuh: TMA-fed, warp-specialised wgmma) against a float64 reference on the same
bf16 operands, against generation 6, with NaN in the padding, across batch sizes, and which generation the options select."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

ATTN6_DEFAULT = 5


def _ref(q, k, v, mask):
    s = (q.double() @ k.double().transpose(-1, -2)) / math.sqrt(q.shape[-1])
    if mask is not None:
        s = s.masked_fill(~mask[:, None, None, :].bool(), float("-inf"))
    o = s.softmax(-1) @ v.double()
    return o.permute(0, 2, 1, 3).reshape(q.shape[0], q.shape[2], -1)


def _layout(q, k, v, row80, fill=7.0):
    """[B, H, L, dh] -> bf16 q / k [B*H, L, dhp] and V^T [B*H, dvp, ceil8(Lk)] with `fill` past Lk."""
    B, H, Lq, dh = q.shape
    Lk = k.shape[2]
    dhp = 80 if (row80 and dh == 72) else (dh + 63) // 64 * 64
    dvp, lkp = (dh + 15) // 16 * 16, (Lk + 7) // 8 * 8
    qb = torch.zeros(B * H, Lq, dhp, device="cuda", dtype=torch.bfloat16)
    kb = torch.zeros(B * H, Lk, dhp, device="cuda", dtype=torch.bfloat16)
    vt = torch.zeros(B * H, dvp, lkp, device="cuda", dtype=torch.bfloat16)
    qb[:, :, :dh] = q.reshape(B * H, Lq, dh)
    kb[:, :, :dh] = k.reshape(B * H, Lk, dh)
    vt[:, :dh, :Lk] = v.reshape(B * H, Lk, dh).transpose(1, 2)
    vt[:, :, Lk:] = fill
    return qb, kb, vt


def _run(impl, args, mask, B, H, Lq, Lk, dh, lens=None):
    from ezaudio_b200 import _lib
    L = _lib.lib()
    out = torch.full((B, Lq, H * dh), 3.0, device="cuda", dtype=torch.bfloat16)
    if lens is None:
        _lib.check(L.ezb_test_attention(0, *[_lib.ptr(a) for a in args], _lib.ptr(mask), _lib.ptr(out), B, H, Lq, Lk, dh, impl, _lib.stream_ptr()))
    else:
        _lib.check(L.ezb_test_attention_lens(0, *[_lib.ptr(a) for a in args], _lib.ptr(lens), _lib.ptr(out), B, H, Lq, dh, impl, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out


def _inputs(B, H, Lq, Lk, dh, masked, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = (torch.randn(B, H, Lq, dh, device="cuda", generator=g) * 1.5).bfloat16().float()
    k = torch.randn(B, H, Lk, dh, device="cuda", generator=g) * 1.5
    v = torch.randn(B, H, Lk, dh, device="cuda", generator=g).bfloat16().float()
    if masked == "grow":   # scores grow by orders of magnitude from key block to key block: exercises the O rescale
        k = k * torch.linspace(0.2, 3.0, Lk, device="cuda")[None, None, :, None]
    k = k.bfloat16().float()
    mask = None
    if masked is True or masked == "one":
        mask = torch.zeros(B, Lk, dtype=torch.uint8, device="cuda")
        for i in range(B):
            mask[i, : (1 if (masked == "one" or i == B - 1) else min(Lk, 8 + 5 * i))] = 1
    return q, k, v, mask


SHAPES = [(8, 16, 500, 500, 72, False), (16, 16, 500, 500, 72, False), (4, 16, 1500, 1500, 72, False), (8, 16, 500, 100, 72, True),
          (8, 16, 256, 256, 64, False), (2, 3, 200, 385, 72, False), (3, 2, 130, 65, 72, True), (2, 2, 40, 12, 72, True), (2, 2, 37, 1, 64, False),
          (2, 3, 300, 129, 64, True), (3, 2, 100, 300, 72, "one"), (2, 5, 700, 700, 72, "grow"), (2, 3, 400, 512, 64, "grow")]


@pytest.mark.parametrize("row80", [False, True])
@pytest.mark.parametrize("B,H,Lq,Lk,dh,masked", SHAPES)
def test_gen8_accuracy(B, H, Lq, Lk, dh, masked, row80):
    """Max error against float64 on the bf16 operands: within 3e-2 and at most 1.25 x generation 6's on the same inputs.  Partial last key
    blocks (385, 65, 12, 1, 129 keys), Lq below one query tile, a single valid key, score growth, dh 64 / 72, both q / k row pitches."""
    q, k, v, mask = _inputs(B, H, Lq, Lk, dh, masked, Lq * 7 + Lk + dh)
    args = _layout(q, k, v, row80)
    ref = _ref(q, k, v, mask)
    off = 100 if row80 else 0
    e8 = (_run(8 + off, args, mask, B, H, Lq, Lk, dh).double() - ref).abs().max().item()
    e6 = (_run(6 + off, args, mask, B, H, Lq, Lk, dh).double() - ref).abs().max().item()
    assert math.isfinite(e8) and e8 < 3e-2, e8
    assert e8 <= 1.25 * e6, (e8, e6)


@pytest.mark.parametrize("B,H,Lq,Lk,dh,masked", [(8, 16, 500, 500, 72, False), (8, 16, 500, 100, 72, True), (16, 16, 500, 500, 72, False)])
def test_gen8_vs_gen6_xl(B, H, Lq, Lk, dh, masked):
    """The XL shapes in the product layout (80-element rows): only reordering-level differences from generation 6, a few bf16 ulps of O(1)
    outputs."""
    q, k, v, mask = _inputs(B, H, Lq, Lk, dh, masked, 11)
    args = _layout(q, k, v, True)
    d = (_run(108, args, mask, B, H, Lq, Lk, dh).float() - _run(106, args, mask, B, H, Lq, Lk, dh).float()).abs()
    print(f"gen8 vs gen6 {B}x{H} Lq {Lq} Lk {Lk}: max {d.max().item():.3e} mean {d.mean().item():.3e}")
    assert d.max().item() < 2e-2 and d.mean().item() < 1e-3


@pytest.mark.parametrize("row80", [False, True])
@pytest.mark.parametrize("dh", [72, 64])
def test_gen8_nan_past_lk(dh, row80):
    """V^T columns past Lk hold NaN: the tensor map's extent stops at Lk, so nothing of them reaches the output."""
    B, H, Lq, Lk = 2, 3, 300, 200
    q, k, v, mask = _inputs(B, H, Lq, Lk, dh, False, 5)
    out = _run(108 if row80 else 8, _layout(q, k, v, row80, fill=float("nan")), None, B, H, Lq, Lk, dh)
    err = (out.double() - _ref(q, k, v, None)).abs().max().item()
    assert math.isfinite(err) and err < 3e-2, err


LENS = [1, 63, 127, 128, 129, 317, 500]


@pytest.mark.parametrize("row80", [False, True])
@pytest.mark.parametrize("dh", [72, 64])
def test_gen8_lens_nan_padding(dh, row80):
    """A padded batch with NaN in every padded token of q, k and v: valid rows are finite and bit-identical to the run alone at L = lens[b],
    padded rows are zeros."""
    B, H, L = len(LENS), 2, 500
    q, k, v, _ = _inputs(B, H, L, L, dh, False, 3 + dh)
    qn, kn, vn = q.clone(), k.clone(), v.clone()
    for b, n in enumerate(LENS):
        qn[b, :, n:] = float("nan"); kn[b, :, n:] = float("nan"); vn[b, :, n:] = float("nan")
    impl = 108 if row80 else 8
    lens = torch.tensor(LENS, dtype=torch.int32, device="cuda")
    out = _run(impl, _layout(qn, kn, vn, row80, fill=float("nan")), None, B, H, L, L, dh, lens=lens)
    for b, n in enumerate(LENS):
        qs, ks, vs = q[b:b + 1, :, :n].contiguous(), k[b:b + 1, :, :n].contiguous(), v[b:b + 1, :, :n].contiguous()
        solo = _run(impl, _layout(qs, ks, vs, row80), None, 1, H, n, n, dh)
        assert torch.equal(out[b, :n], solo[0]), (b, n)
        assert bool((out[b, n:] == 0).all()), (b, n)
        err = (out[b:b + 1, :n].double() - _ref(qs, ks, vs, None)).abs().max().item()
        assert math.isfinite(err) and err < 3e-2, (b, n, err)


@pytest.mark.parametrize("masked", [False, True])
def test_gen8_batch_independent(masked):
    """Head (0, 0) gives the same bits at B*H = 1, 16, 128 and 256: tiles and key order do not depend on the number of heads."""
    H, Lq, Lk, dh = 16, 500, 500 if not masked else 100, 72
    q, k, v, mask = _inputs(16, H, Lq, Lk, dh, masked, 21)
    outs = []
    for B, Hh in ((1, 1), (1, 16), (8, 16), (16, 16)):
        m = None if mask is None else mask[:B].contiguous()
        outs.append(_run(108, _layout(q[:B, :Hh].contiguous(), k[:B, :Hh].contiguous(), v[:B, :Hh].contiguous(), True), m, B, Hh, Lq, Lk, dh)[0, :, :dh])
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_generation_selection():
    """Generation 8 runs by default for dh 64 / 72 and falls back to 6 for other head dims; a non-default attn6 / attn7, or attn8 = 0, selects
    the older generations."""
    from ezaudio_b200 import _lib
    L = _lib.lib()

    def launched(dh, **opts):
        for name, val in opts.items():
            _lib.check(L.ezb_set_option(name.encode(), val))
        try:
            q, k, v, _ = _inputs(1, 2, 64, 64, dh, False, 1)
            before = {g: L.ezb_attn_launch_count(g) for g in (4, 6, 7, 8)}
            _run(1, _layout(q, k, v, False), None, 1, 2, 64, 64, dh)
            return [g for g in (4, 6, 7, 8) if L.ezb_attn_launch_count(g) != before[g]]
        finally:
            _lib.check(L.ezb_set_option(b"attn6", ATTN6_DEFAULT))
            _lib.check(L.ezb_set_option(b"attn7", 0))
            _lib.check(L.ezb_set_option(b"attn8", 1))

    assert launched(72) == [8]
    assert launched(64) == [8]
    assert launched(40) == [6]
    assert launched(72, attn8=0) == [6]
    assert launched(72, attn6=1) == [6]
    assert launched(72, attn6=0) == [4]
    assert launched(72, attn7=1) == [7]
