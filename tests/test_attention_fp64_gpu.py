"""The DiT's attention kernels against fp64: generation 8 (attention_wgmma.cuh, impl 8 / 108), generation 6 (attention_mma.cuh, impl 6 /
106, the kernel for head dims other than 64 / 72) and the fp32 CUDA-core kernel (attention_simt.cuh, impl 0, and impl 3 = the bf16x3
[hi | lo | hi] rows the parity mode writes), launched through ezb_test_attention / ezb_test_attention_lens with the layouts Dit::attention
uses.  Inputs are drawn on the CPU from fixed seeds, so every precondition below holds for the exact values the kernels read.

Exact probes (bit for bit).
  Uniform: q = 0 and V integers in {+-1, +-2} with alternating signs along the keys.  Every valid key scores 0 and gets P = 1 exactly, so
    l = n and O = S, the integer column sum over the valid keys (every partial sum is an integer below 2^24: the tensor cores and the fma
    chain add it exactly).  The output is bf16(fl32(S) * fl32(1/n)) bit for bit (bf16x3: [hi | bf16(y - hi) | hi]); a row with no valid key
    is zeros.  With |S| < 128 (asserted) one missing or duplicated key always changes the bf16 result.  Masks: prefix, suffix, 30 % random
    holes, the first 64 / 128 / 256 keys masked (one or two whole leading key blocks of every kernel: a row with no valid key yet), only the
    last key, a single key at 63, 64, 65, 127, 128 or 129, no key, every key; Lk from 1 to 1500.  Padded batches: lens 0, 1, 63, 127, 128,
    129, 317, 500 and 600 at L = 500 -- the kernels clamp lens to [1, L], so 0 acts as 1 and 600 as 500.
  One-hot: K = bf16(u_j) for random unit vectors u_j and Q_i = bf16(alpha u_t(i)); the targets t(i) run over every key (a permutation per
    sample: the first and last key of every 64- and 128-key block, the block that straddles Lk and, with lens, the straddling block of each
    sample).  alpha is chosen so that, in fp64 on the bf16 operands, the target leads every other valid key by >= 60 in log2 units (asserted
    as a precondition).  Then P = 1 for the target and < 2^-60 elsewhere, and the output row is v_t exactly (the bf16 value for the tensor
    cores, bf16_rn(v) for the fp32 kernel, lo = bf16(v - hi) exactly for bf16x3); |v| >= 0.5 keeps the < 2^-60 weights below half an ulp.
    Block 0 always holds a local maximum of weight 1, so for every target past the first block the O rescale must shrink that key to below
    2^-60.  Masked variant: each masked key is 2 u_c of a valid key c, so on the rows that target c the masked key leads by >= 60 log2 units;
    the output must still be v_c.  These probes catch any Q row, K / V row or V^T column misindexing, a missing or wrong rescale, and a ring
    stage or phase mix-up.

Per-element bounds on random inputs, tensor-core kernels.  The reference is softmax(Q K^T / sqrt(dh)) V in fp64 on the bf16 operands, with
p_j its weights and ref its value.  The kernel's weights are P~_j / sum P~ with P~_j = p_j (1 + e_j): e_j holds the bf16 rounding of P
(|.| <= u = 2^-8) and the fp32 error of the score and its exponential (|.| <= d).  Because sum_j p_j (v_j - ref) = 0,
  y - ref = sum_j p_j e_j (v_j - ref) / (1 + e_bar),   so   |y - ref| <= (u + d) sum_j p_j |v_j - ref| (1 + 2^-7).
  d (natural-log units, per row) = (n_k + 1) 2^-23 sigma + 3 2^-22 sigma + 2^-22 + n_blk 2^-21:  n_k = DK / 16 k16 steps of the score
    accumulation, each truncating at most 2^-23 of a partial sum bounded by sigma = scale max_j sum_d |q_d k_jd|; the scale_log2 constant and
    product and the subtraction of the row maximum, three fp32 roundings of values up to 2 sigma log2(e); exp2f within 2 ulp; per key block
    (n_blk = ceil(Lk / 64)) one exp2f rescale factor and its products with O and l.
  l sums the same rounded P in fp32: ceil(Lk / 4) + n_blk + 2 roundings of a partial sum <= l, lambda = (ceil(Lk / 4) + n_blk + 2) 2^-24
    relative, plus 1 / l and O / l, 2^-23.  The P V accumulation truncates up to ceil(Lk / 16) + n_blk + 1 times at most 2^-23 of a
    partial sum bounded by sum_j p_j |v_j|: gamma.  The output is one bf16 rounding, u |ref|.
  Allowance:  A = (1 + 2^-7) ((u + d) sum p |v - ref| + (lambda + 2^-23) |ref| + gamma sum p |v|) + u |ref|.
  Mean bound: the roundings of P and of the output are independent with rms <= u / sqrt(3) relative, so per element
    E|y - ref| <= rms <= M = u / sqrt(3) (sqrt(sum p^2 (v - ref)^2) + |ref|) + d sum p |v - ref| + (lambda + 2^-23) |ref| + gamma sum p |v|,
  and the mean of |y - ref| over a tensor must stay under the mean of M (factor 1).  A systematic error fails it: the scale 1/sqrt(80) of
  the padded dh = 72 row instead of 1/sqrt(72) gives 6 to 12 times the mean of M (and 10 to 19 times A) in an emulation of the kernels'
  numerics at the xl_self, xl_cross and tiny_self shapes.
Per-element bounds, fp32 kernel (the T5 model of test_conditioning_gpu.py with the DiT's scale and -inf key masks): each score is a dh-long
fma chain of q * scale (one more rounding) and k, error ds = (dh + 3) 2^-24 scale max_j sum |q k|; a probability moves by up to twice
that relatively plus expf's 2 ulp, and the P V and l sums over Lk keys and the per-tile rescales add (Lk + 32) 2^-24 max |v|:
  slack = max|v| (4 ds + 16 2^-24 + (Lk + 32) 2^-24);  kmul 1: |y - ref| <= 2^-8 |ref| + (1 + 2^-7) slack;  kmul 3: hi + lo within
  2^-16 |ref| + (1 + 2^-7) slack and the third block bit-equal to the first.
Shapes: self-attention at B H = 8 x 16, L = 500 (four 10-s prompts with CFG) and 4 x 16, L = 1500 (30-s inpainting); cross-attention at
Lq 500, Lk 100 with per-sample prompt-length masks; the tiny models' dh 64 / 72; generation 6 also at dh 40 / 80 and the fp32 kernel at 96.
q / k are per-head LayerNorm-like rows (|q|, |k| ~ sqrt(dh)), also with 3x the gain (peaked rows) and with the key norms growing 15x along
the keys (every block raises the row maximum: the O rescale).
Measured on one H100 SXM (80 GB HBM3, 700 W limit), printed per case with pytest -s: max error / A up to 0.99 (xl_self_peaked, where the
output rounding alone reaches its worst case u |ref|; 0.30 at xl_self, 0.19 at inpaint_30s, 0.70 at xl_cross), mean error / mean M 0.17 to
0.47; the fp32 kernel's max error / allowance up to 0.91.  Generations 6 and 8 give the same ratios.  Framing: outputs are prefilled with the bf16 NaN pattern 0x7FAB plus one spare row; every element must be
written and the spare row keep it.  Padding the kernels must not read (q / k columns past dh, V^T rows past dh and keys past Lk, the tokens
past lens) holds NaN."""
import ctypes as C
import math

import pytest
import torch

gpu = pytest.mark.gpu

SENT = 0x7FAB
U16 = 2.0 ** -8     # bf16 unit roundoff
U = 2.0 ** -24      # fp32 unit roundoff
LOG2E = 1.0 / math.log(2.0)
SIMT, SIMT3 = 0, 3
EZB_ERR_ARG, EZB_ERR_SHAPE, EZB_ERR_UNSUPPORTED = -1, -2, -3
LEADS = 60.0        # log2 units by which a one-hot target must lead every other valid key

# (impl, dh) of every kernel in scope
GEN8 = [(8, 64), (8, 72), (108, 72)]
GEN6 = [(6, 40), (6, 64), (6, 72), (106, 72), (6, 80)]
FP32 = [(SIMT, 64), (SIMT, 72), (SIMT, 96), (SIMT3, 64), (SIMT3, 72), (SIMT3, 96)]
KERNELS = GEN8 + GEN6 + FP32
LENS = [0, 1, 63, 127, 128, 129, 317, 500, 600]   # L = 500: 0 acts as 1, 600 as 500
PROBE_LK = [1, 7, 8, 63, 64, 65, 127, 128, 129, 385, 500, 1500]


def _kid(kd):
    return f"impl{kd[0]}-dh{kd[1]}"


def _is_simt(impl):
    return impl in (SIMT, SIMT3)


def _generation(impl):
    return None if _is_simt(impl) else impl % 100


# ------------------------------------------------------------------------------------------------------------------------------ plumbing
def _tc_layout(q, k, v, row80):
    """[B, H, L, dh] -> bf16 q / k [B*H, L, dhp] and V^T [B*H, dvp, ceil8(Lk)] as the QKV epilogue writes them, every padding element NaN."""
    B, H, Lq, dh = q.shape
    Lk = k.shape[2]
    dhp = 80 if (row80 and dh == 72) else (dh + 63) // 64 * 64
    dvp, lkp = (dh + 15) // 16 * 16, (Lk + 7) // 8 * 8
    nan = float("nan")
    qb = torch.full((B * H, Lq, dhp), nan, device="cuda", dtype=torch.bfloat16)
    kb = torch.full((B * H, Lk, dhp), nan, device="cuda", dtype=torch.bfloat16)
    vt = torch.full((B * H, dvp, lkp), nan, device="cuda", dtype=torch.bfloat16)
    qb[:, :, :dh] = q.reshape(B * H, Lq, dh)
    kb[:, :, :dh] = k.reshape(B * H, Lk, dh)
    vt[:, :dh, :Lk] = v.reshape(B * H, Lk, dh).transpose(1, 2)
    return qb, kb, vt


def _launch(impl, q, k, v, mask=None, lens=None):
    """Runs kernel `impl` on fp32 [B, H, L, dh] tensors (bf16 values for the tensor cores) -> bf16 [B, Lq, kmul H dh]; checks the framing
    and that the requested generation ran."""
    from ezaudio_b200 import _lib
    Lib = _lib.lib()
    B, H, Lq, dh = q.shape
    Lk = k.shape[2]
    kmul = 3 if impl == SIMT3 else 1
    if _is_simt(impl):
        args = (q.cuda().contiguous(), k.cuda().contiguous(), v.cuda().contiguous())
    else:
        args = _tc_layout(q.cuda(), k.cuda(), v.cuda(), impl >= 100)
    out = torch.full((B * Lq + 1, kmul * H * dh), SENT, dtype=torch.int16, device="cuda")
    mask = None if mask is None else mask.cuda()
    lens = None if lens is None else lens.cuda()
    gen = _generation(impl)
    before = Lib.ezb_attn_launch_count(gen) if gen is not None else 0
    ptrs = [_lib.ptr(a) for a in args]
    if lens is None:
        rc = Lib.ezb_test_attention(0, *ptrs, _lib.ptr(mask), _lib.ptr(out), B, H, Lq, Lk, dh, impl, _lib.stream_ptr())
    else:
        rc = Lib.ezb_test_attention_lens(0, *ptrs, _lib.ptr(lens), _lib.ptr(out), B, H, Lq, dh, impl, _lib.stream_ptr())
    _lib.check(rc)
    torch.cuda.synchronize()
    if gen is not None:
        assert Lib.ezb_attn_launch_count(gen) == before + 1, f"impl {impl} did not run generation {gen}"
    assert bool((out[-1] == SENT).all()), "the spare row past the output was written"
    body = out[:-1]
    assert not bool((body == SENT).any()), f"{int((body == SENT).sum())} output elements left unwritten"
    return body.view(torch.bfloat16).view(B, Lq, kmul * H * dh)


def _valid_keys(B, Lq, Lk, mask=None, lens=None, device="cpu"):
    """-> bool [B, Lq, Lk]: key j counts for query row i of sample b (lens: clamped to [1, L]; rows past it have no key)."""
    if lens is not None:
        n = lens.clamp(1, Lk).to(device)
        j = torch.arange(Lk, device=device)
        i = torch.arange(Lq, device=device)
        return (j[None, None, :] < n[:, None, None]) & (i[None, :, None] < n[:, None, None])
    if mask is None:
        return torch.ones(B, Lq, Lk, dtype=torch.bool, device=device)
    return mask.to(device).bool()[:, None, :].expand(B, Lq, Lk)


def _split_rows(y, kmul):
    """fp32 [B, Lq, H, dh] -> the bf16 rows the kernel writes: [B, Lq, H dh] or [hi | lo | hi]."""
    B, Lq = y.shape[:2]
    y = y.reshape(B, Lq, -1)
    hi = y.bfloat16()
    if kmul == 1:
        return hi
    return torch.cat([hi, (y - hi.float()).bfloat16(), hi], -1)


def _assert_same(got, want, what):
    g, w = got.float().cpu(), want.float().cpu()
    bad = ~((g == w) | (g.isnan() & w.isnan()))
    if bool(bad.any()):
        i = tuple(int(x) for x in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ, first at {i}: got {float(g[i])!r}, want {float(w[i])!r}")


# ------------------------------------------------------------------------------------------------------------------------------ uniform probe
def _uniform_v(B, H, Lk, dh, g):
    """Integers in {+-1, +-2}, the sign alternating along the keys (partial sums stay small) with a random sign per column."""
    m = torch.randint(1, 3, (B, H, Lk, dh), generator=g).float()
    col = torch.randint(0, 2, (B, H, 1, dh), generator=g).float() * 2 - 1
    alt = 1.0 - 2.0 * (torch.arange(Lk) % 2).float()
    return m * col * alt[None, None, :, None]


def _uniform_want(v, valid, kmul):
    """bf16(fl32(S) fl32(1/n)) of the column sums S over the valid keys; zeros for a row without one."""
    S = torch.einsum("bqk,bhkd->bqhd", valid.double(), v.double())
    assert float(S.abs().max()) < 128, "precondition: |S| < 128"
    n = valid.sum(-1).float()[:, :, None, None]
    inv = torch.where(n > 0, 1.0 / n.clamp(min=1), torch.zeros_like(n))
    return _split_rows(S.float() * inv, kmul)


def _probe_masks(Lk, g):
    """One sample per mask pattern, [14, Lk] uint8."""
    rows = []

    def add(keys):
        m = torch.zeros(Lk, dtype=torch.uint8)
        m[keys] = 1
        rows.append(m)

    add(slice(0, max(1, 2 * Lk // 3)))                      # prefix (a prompt shorter than the context)
    add(slice(Lk // 3, Lk))                                  # suffix
    rows.append((torch.rand(Lk, generator=g) > 0.3).to(torch.uint8))   # 30 % holes
    for lead in (64, 128, 256):                              # whole leading key blocks masked (everything when Lk <= lead)
        add(slice(lead, Lk))
    add(slice(Lk - 1, Lk))                                   # the last key only
    for j in (63, 64, 65, 127, 128, 129):                    # a single key on a block edge (the last key when Lk is shorter)
        add(min(j, Lk - 1))
    add(slice(0, 0))                                         # no key at all
    add(slice(0, Lk))                                        # every key
    return torch.stack(rows)


def _probe_operands(impl, B, H, Lq, Lk, dh, g):
    q = torch.zeros(B, H, Lq, dh)
    k = torch.randn(B, H, Lk, dh, generator=g)
    if not _is_simt(impl):
        k = k.bfloat16().float()
    return q, k, _uniform_v(B, H, Lk, dh, g)


@gpu
@pytest.mark.parametrize("Lk", PROBE_LK)
@pytest.mark.parametrize("kd", KERNELS, ids=_kid)
def test_uniform_probe_masks(kd, Lk):
    impl, dh = kd
    g = torch.Generator().manual_seed(1000 * dh + Lk + impl)
    mask = _probe_masks(Lk, g)
    B, H, Lq = mask.shape[0], 2, 130
    q, k, v = _probe_operands(impl, B, H, Lq, Lk, dh, g)
    got = _launch(impl, q, k, v, mask=mask)
    want = _uniform_want(v, _valid_keys(B, Lq, Lk, mask=mask), 3 if impl == SIMT3 else 1)
    _assert_same(got, want, f"uniform probe impl {impl} dh {dh} Lk {Lk}")


@gpu
@pytest.mark.parametrize("kd", KERNELS, ids=_kid)
def test_uniform_probe_lens(kd):
    impl, dh = kd
    g = torch.Generator().manual_seed(77 * dh + impl)
    B, H, L = len(LENS), 2, 500
    lens = torch.tensor(LENS, dtype=torch.int32)
    q, k, v = _probe_operands(impl, B, H, L, L, dh, g)
    valid = _valid_keys(B, L, L, lens=lens)
    want = _uniform_want(v, valid, 3 if impl == SIMT3 else 1)
    qn, kn, vn = q.clone(), k.clone(), v.clone()
    for b, n in enumerate(lens.clamp(1, L).tolist()):   # NaN in every padded token
        qn[b, :, n:] = float("nan"); kn[b, :, n:] = float("nan"); vn[b, :, n:] = float("nan")
    got = _launch(impl, qn, kn, vn, lens=lens)
    _assert_same(got, want, f"uniform probe (lens) impl {impl} dh {dh}")


# ------------------------------------------------------------------------------------------------------------------------------ one-hot probe
def _onehot_case(impl, dh, targets, valid, g, copies=None):
    """targets long [B, Lq] (a valid key of each row that has one), valid bool [B, Lq, Lk] -> (q, k, v, want).
    copies: {b: {masked key m: valid key c}}, K_m = 2 u_c."""
    B, Lq = targets.shape
    Lk = valid.shape[-1]
    H = 2
    u = torch.randn(B, H, Lk, dh, generator=g, dtype=torch.float64)
    u = u / u.norm(dim=-1, keepdim=True)
    ku = u.clone()
    for b, cp in (copies or {}).items():
        for m, c in cp.items():
            ku[b, :, m] = 2.0 * u[b, :, c]
    scale = 1.0 / math.sqrt(dh)
    has = valid.any(-1)                                                   # [B, Lq]
    tsel = targets[:, None, :, None].expand(B, H, Lq, dh)
    ut = u.gather(2, tsel)                                                # [B, H, Lq, dh]

    def leads(qv, kv):
        s = (qv @ kv.transpose(-1, -2)) * scale * LOG2E                    # [B, H, Lq, Lk]
        st = s.gather(3, targets[:, None, :, None].expand(B, H, Lq, 1))[..., 0]
        other = valid[:, None].clone().expand(B, H, Lq, Lk).clone()
        other.scatter_(3, targets[:, None, :, None].expand(B, H, Lq, 1), False)
        rival = s.masked_fill(~other, float("-inf")).amax(-1)
        masked_best = s.masked_fill(valid[:, None], float("-inf")).amax(-1)
        return st - rival, masked_best - st

    lead1, _ = leads(ut, ku)
    lead1 = lead1[has[:, None].expand_as(lead1)]
    alpha = 1.0 if bool(torch.isinf(lead1).all()) else 1.05 * LEADS / float(lead1.min())
    q = (alpha * ut).float().bfloat16().float()
    k = ku.float().bfloat16().float()
    lead, over = leads(q.double(), k.double())
    rows = has[:, None].expand_as(lead)
    assert float(lead[rows].min()) >= LEADS, f"precondition: lead {float(lead[rows].min()):.1f} < {LEADS} log2 units"
    if copies:
        dom = over[rows] >= LEADS
        assert float(dom.double().mean()) >= 0.25, "precondition: too few rows where a masked key dominates"
    mag = 0.5 + torch.rand(B, H, Lk, dh, generator=g)
    v = torch.where(torch.rand(B, H, Lk, dh, generator=g) < 0.5, -mag, mag)
    if not _is_simt(impl):
        v = v.bfloat16().float()
    vt = v.gather(2, tsel).permute(0, 2, 1, 3)                              # [B, Lq, H, dh]
    y = torch.where(has[:, :, None, None], vt, torch.zeros_like(vt))
    return q, k, v, _split_rows(y, 3 if impl == SIMT3 else 1)


def _perm_targets(B, Lq, pools, g):
    """Row i of sample b targets pool_b[perm[i % len(pool_b)]]: every key of the pool is a target."""
    t = torch.zeros(B, Lq, dtype=torch.long)
    for b, pool in enumerate(pools):
        perm = pool[torch.randperm(len(pool), generator=g)]
        t[b] = perm[torch.arange(Lq) % len(pool)]
    return t


@gpu
@pytest.mark.parametrize("Lq,Lk", [(1, 1), (65, 65), (129, 129), (385, 385), (1500, 1500), (500, 100), (7, 500)])
@pytest.mark.parametrize("kd", KERNELS, ids=_kid)
def test_onehot_probe(kd, Lq, Lk):
    impl, dh = kd
    g = torch.Generator().manual_seed(31 * Lk + Lq + dh + impl)
    B = 2
    t = _perm_targets(B, Lq, [torch.arange(Lk)] * B, g)
    q, k, v, want = _onehot_case(impl, dh, t, _valid_keys(B, Lq, Lk), g)
    got = _launch(impl, q, k, v)
    _assert_same(got, want, f"one-hot probe impl {impl} dh {dh} Lq {Lq} Lk {Lk}")


@gpu
@pytest.mark.parametrize("Lq,Lk", [(385, 385), (500, 100), (300, 1500)])
@pytest.mark.parametrize("kd", KERNELS, ids=_kid)
def test_onehot_probe_masked_key_dominates(kd, Lq, Lk):
    impl, dh = kd
    g = torch.Generator().manual_seed(53 * Lk + Lq + dh + impl)
    B = 2
    mask = (torch.rand(B, Lk, generator=g) > 0.3).to(torch.uint8)
    mask[:, 0] = 1
    copies, pools = {}, []
    for b in range(B):
        ok, masked = mask[b].nonzero()[:, 0], (mask[b] == 0).nonzero()[:, 0]
        pick = ok[torch.randperm(len(ok), generator=g)][: len(masked)]
        copies[b] = {int(m): int(c) for m, c in zip(masked, pick)}
        pools.append(pick if Lq <= 2 * len(pick) else ok)   # rows target the copied keys first
    t = _perm_targets(B, Lq, pools, g)
    q, k, v, want = _onehot_case(impl, dh, t, _valid_keys(B, Lq, Lk, mask=mask), g, copies)
    got = _launch(impl, q, k, v, mask=mask)
    _assert_same(got, want, f"one-hot probe (masked key dominant) impl {impl} dh {dh} Lq {Lq} Lk {Lk}")


@gpu
@pytest.mark.parametrize("kd", KERNELS, ids=_kid)
def test_onehot_probe_lens(kd):
    impl, dh = kd
    g = torch.Generator().manual_seed(91 + dh + impl)
    B, L = len(LENS), 500
    lens = torch.tensor(LENS, dtype=torch.int32)
    n = lens.clamp(1, L)
    t = _perm_targets(B, L, [torch.arange(int(x)) for x in n], g)
    q, k, v, want = _onehot_case(impl, dh, t, _valid_keys(B, L, L, lens=lens), g)
    for b, nb in enumerate(n.tolist()):
        q[b, :, nb:] = float("nan"); k[b, :, nb:] = float("nan"); v[b, :, nb:] = float("nan")
    got = _launch(impl, q, k, v, lens=lens)
    _assert_same(got, want, f"one-hot probe (lens) impl {impl} dh {dh}")


# ------------------------------------------------------------------------------------------------------------------------------ fp64 bounds
def _ref_device():
    return "cuda" if torch.cuda.is_available() else "cpu"


def _fp64_stats(q, k, v, valid):
    """fp64 softmax(q k^T / sqrt(dh)) v on the given values (valid bool [B, Lq, Lk]; a row without a valid key is 0) -> dict of
    [B, Lq, H, dh] tensors ref, a1 = sum p |v - ref|, apv = sum p |v|, q2 = sum p^2 (v - ref)^2, and sigma [B, Lq, H]."""
    B, H, Lq, dh = q.shape
    Lk = k.shape[2]
    scale = 1.0 / math.sqrt(dh)
    dev = _ref_device()
    out = {n: torch.empty(B, Lq, H, dh, dtype=torch.float64, device=dev) for n in ("ref", "a1", "apv", "q2")}
    sigma = torch.empty(B, Lq, H, dtype=torch.float64, device=dev)
    rc = max(1, (1 << 27) // (Lk * dh))   # rows per chunk of the [rows, Lk, dh] temporary
    for b in range(B):
        ok = valid[b].to(dev)
        for h in range(H):
            qd, kd, vd = q[b, h].to(dev).double(), k[b, h].to(dev).double(), v[b, h].to(dev).double()
            s = (qd @ kd.T) * scale
            p = s.masked_fill(~ok, float("-inf")).softmax(-1).nan_to_num(0.0)
            ref = p @ vd
            p2 = p * p
            out["ref"][b, :, h] = ref
            out["apv"][b, :, h] = p @ vd.abs()
            out["q2"][b, :, h] = (p2 @ (vd * vd) - 2 * ref * (p2 @ vd) + ref * ref * p2.sum(-1, keepdim=True)).clamp(min=0)
            sigma[b, :, h] = ((qd.abs() @ kd.abs().T) * scale).masked_fill(~ok, 0).amax(-1)
            for i0 in range(0, Lq, rc):
                i1 = min(Lq, i0 + rc)
                dev_ = (vd[None] - ref[i0:i1, None]).abs()
                out["a1"][b, i0:i1, h] = torch.bmm(p[i0:i1, None], dev_)[:, 0]
    out["sigma"] = sigma
    return out


def _tc_allowance(st, dh, Lk):
    """-> (A, M) [B, Lq, H, dh]: the per-element allowance and the rms model of the module docstring."""
    DK = 64 if dh <= 64 else 80
    nblk = -(-Lk // 64)
    sig = st["sigma"][..., None]
    d = (DK // 16 + 1) * 2.0 ** -23 * sig + 3 * 2.0 ** -22 * sig + 2.0 ** -22 + nblk * 2.0 ** -21
    lam = (-(-Lk // 4) + nblk + 2) * U + 2.0 ** -23
    gam = (-(-Lk // 16) + nblk + 1) * 2.0 ** -23
    ref = st["ref"].abs()
    A = (1 + 2.0 ** -7) * ((U16 + d) * st["a1"] + lam * ref + gam * st["apv"]) + U16 * ref
    M = U16 / math.sqrt(3) * (st["q2"].sqrt() + ref) + d * st["a1"] + lam * ref + gam * st["apv"]
    return A, M


def _simt_slack(q, k, v, valid):
    """-> [B, Lq, H, dh]: the fp32 kernel's allowance beyond the output rounding (module docstring)."""
    B, H, Lq, dh = q.shape
    Lk = k.shape[2]
    scale = 1.0 / math.sqrt(dh)
    dev = _ref_device()
    qd, kd = q.to(dev).double(), k.to(dev).double()
    qk = torch.empty(B, H, Lq, dtype=torch.float64, device=dev)
    for b in range(B):
        qk[b] = ((qd[b].abs() @ kd[b].abs().transpose(-1, -2)) * scale).masked_fill(~valid[b].to(dev)[None], 0).amax(-1)
    ds = (dh + 3) * U * qk
    vmax = v.to(dev).double().abs().nan_to_num(0).amax((-1, -2))           # [B, H]
    s = vmax[:, :, None] * (4 * ds + 16 * U + (Lk + 32) * U)               # [B, H, Lq]
    return s.permute(0, 2, 1)[..., None].expand(B, Lq, H, dh)


def _ln_rows(B, H, L, dh, g, gain=1.0):
    """Per-head LayerNorm-like rows: zero mean, unit variance per row (|x| ~ sqrt(dh)), times a per-(head, column) gain around `gain`."""
    x = torch.randn(B, H, L, dh, generator=g)
    x = (x - x.mean(-1, keepdim=True)) / x.std(-1, unbiased=False, keepdim=True)
    return x * (gain * (1 + 0.2 * torch.randn(1, H, 1, dh, generator=g)))


# name: (B, H, Lq, Lk, masks, qk)    masks: None, "prompt" (per-sample prompt lengths) or "lens"
SHAPES = {
    "xl_self": (8, 16, 500, 500, None, "ln"),
    "xl_self_peaked": (8, 16, 500, 500, None, "peaked"),
    "xl_self_grow": (8, 16, 500, 500, None, "grow"),
    "inpaint_30s": (4, 16, 1500, 1500, None, "ln"),
    "xl_cross": (8, 16, 500, 100, "prompt", "ln"),
    "tiny_self": (2, 2, 40, 40, None, "ln"),
    "tiny_cross": (2, 2, 40, 12, "prompt", "ln"),
    "tiny64_self": (2, 4, 130, 130, None, "grow"),
    "tiny64_cross": (2, 4, 130, 100, "prompt", "peaked"),
    "lens": (len(LENS), 2, 500, 500, "lens", "ln"),
}


def _bound_inputs(name, impl, dh):
    B, H, Lq, Lk, masks, qk = SHAPES[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)) * 131 + dh)
    gain = 3.0 if qk == "peaked" else 1.0
    q, k = _ln_rows(B, H, Lq, dh, g, gain), _ln_rows(B, H, Lk, dh, g, gain)
    if qk == "grow":   # the key norms grow 15x along the keys: each block raises the row maximum
        k = k * torch.linspace(0.2, 3.0, Lk)[None, None, :, None]
    v = torch.randn(B, H, Lk, dh, generator=g)
    if not _is_simt(impl):
        q, k, v = q.bfloat16().float(), k.bfloat16().float(), v.bfloat16().float()
    mask = lens = None
    if masks == "prompt":   # per-sample prompt lengths, one sample with a single token
        n = torch.randint(1, Lk + 1, (B,), generator=g)
        n[0], n[-1] = Lk, 1
        mask = (torch.arange(Lk)[None] < n[:, None]).to(torch.uint8)
    elif masks == "lens":
        lens = torch.tensor(LENS, dtype=torch.int32)
    return q, k, v, mask, lens


def _bound_case(impl, dh, name):
    q, k, v, mask, lens = _bound_inputs(name, impl, dh)
    B, H, Lq, _ = q.shape
    Lk = k.shape[2]
    valid = _valid_keys(B, Lq, Lk, mask=mask, lens=lens)
    qn, kn, vn = q, k, v
    if lens is not None:   # NaN in the padded tokens the kernel gets; the reference sees zeros there
        qn, kn, vn = q.clone(), k.clone(), v.clone()
        for b, nb in enumerate(lens.clamp(1, Lq).tolist()):
            qn[b, :, nb:] = float("nan"); kn[b, :, nb:] = float("nan"); vn[b, :, nb:] = float("nan")
    got = _launch(impl, qn, kn, vn, mask=mask, lens=lens)
    st = _fp64_stats(q, k, v, valid)
    ref = st["ref"].reshape(B * Lq, H * dh)
    what = f"impl {impl} dh {dh} {name}"
    if _is_simt(impl):
        from tests.test_step_kernels_gpu import _check_bf16
        slack = _simt_slack(q, k, v, valid).reshape(B * Lq, H * dh)
        kmul = 3 if impl == SIMT3 else 1
        emax, qmax = _check_bf16(got.reshape(B * Lq, kmul * H * dh), ref, slack, kmul, what)
        print(f"\n{what}: max err {emax:.3e}, max err / allowance {qmax:.3f}")
        return
    A, M = _tc_allowance(st, dh, Lk)
    err = (got.double().reshape(B, Lq, H, dh) - st["ref"]).abs()
    r = err / (A + 1e-30)
    i = int(r.argmax())
    assert bool(torch.isfinite(err).all()), f"{what}: non-finite output"
    assert bool((err <= A).all()), f"{what}: err {float(err.flatten()[i]):.3e} > allowance {float(A.flatten()[i]):.3e} at flat index {i}"
    mean_ratio = float(err.mean()) / float(M.mean())
    assert mean_ratio <= 1.0, f"{what}: mean err {float(err.mean()):.3e} > mean rms model {float(M.mean()):.3e}"
    print(f"\n{what}: max err {float(err.max()):.3e}, max err / A {float(r.max()):.3f}, mean err / mean M {mean_ratio:.3f}")


@gpu
@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("impl", [8, 108, 6, 106, SIMT, SIMT3])
def test_bound_dh72(impl, name):
    _bound_case(impl, 64 if name.startswith("tiny64") else 72, name)


@gpu
@pytest.mark.parametrize("name", ["tiny64_self", "tiny64_cross", "tiny_cross", "lens"])
@pytest.mark.parametrize("kd", [(6, 40), (6, 80), (8, 64), (SIMT, 96), (SIMT3, 96)], ids=_kid)
def test_bound_other_head_dims(kd, name):
    _bound_case(kd[0], kd[1], name)


# ------------------------------------------------------------------------------------------------------------------------------ the hook
def test_attention_hook_rejects_bad_arguments():
    """Argument validation happens before any device work (this runs without a GPU)."""
    from ezaudio_b200 import _lib
    Lib = _lib.lib()
    buf = (C.c_float * 64)()
    p = C.c_void_p(C.addressof(buf))

    def rc(impl=8, dh=72, B=2, H=4, Lq=100, Lk=100, q=p, mask=None):
        return Lib.ezb_test_attention(0, q, p, p, mask, p, B, H, Lq, Lk, dh, impl, None)

    def rc_lens(impl=8, dh=72, B=2, H=4, L=100, lens=p):
        return Lib.ezb_test_attention_lens(0, p, p, p, lens, p, B, H, L, dh, impl, None)

    assert rc(q=None) == EZB_ERR_ARG
    for impl in (-1, 2, 5, 9, 100, 103, 105, 200, 208):
        assert rc(impl=impl) == EZB_ERR_ARG, impl
    for impl in (SIMT, SIMT3):
        for dh in (0, 2, 66, 100, 128):        # the fp32 kernel: multiples of 4 up to 96
            assert rc(impl=impl, dh=dh) == EZB_ERR_UNSUPPORTED, (impl, dh)
    for impl in (1, 6, 106):
        for dh in (0, 4, 36, 88, 96):           # tensor cores: multiples of 8 up to 80
            assert rc(impl=impl, dh=dh) == EZB_ERR_UNSUPPORTED, (impl, dh)
    for impl in (8, 108):
        for dh in (40, 56, 80):                 # generation 8: 64 or 72
            assert rc(impl=impl, dh=dh) == EZB_ERR_UNSUPPORTED, (impl, dh)
    for impl in (SIMT, 6, 8):
        dh = 64
        assert rc(impl=impl, dh=dh, B=0) == EZB_ERR_SHAPE
        assert rc(impl=impl, dh=dh, H=0) == EZB_ERR_SHAPE
        assert rc(impl=impl, dh=dh, Lq=0) == EZB_ERR_SHAPE
        assert rc(impl=impl, dh=dh, Lk=0) == EZB_ERR_SHAPE
        assert rc(impl=impl, dh=dh, B=4096, H=16) == EZB_ERR_SHAPE    # B H = 65536 CTA rows
        assert rc_lens(impl=impl, dh=dh, L=0) == EZB_ERR_SHAPE
    assert rc_lens(lens=None) == EZB_ERR_ARG
    assert rc_lens(impl=2) == EZB_ERR_ARG
