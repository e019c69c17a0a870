"""The DiT's linears on 128-wide N-tiles (csrc/gemm.cuh EpiLinear and EpiLinearScaled, on the single-CTA kernel gemm<128> and the 2-CTA
cluster kernel gemm2<128>), launched through ezb_test_linear as Dit::lin and the ControlNet zero-linears launch them, against fp64 references.

Exact operands.  The hook packs the fp32 weight W [N, K] as Dit::init packs it and returns the packed bf16 W'; the reference multiplies
exactly what the kernel reads, in fp64: A' [M, kmul K] and W' [N, kmul K] (bf16x3: A' = [hi | lo | hi], W' = [hi | hi | lo]).  Every
product is exact in fp32, so only the fp32 accumulation and the epilogue's few fp32 operations are left.

fp32 outputs, per element:  |out - ref| <= EPS * S,   S = |osc keep| (|A'| |W'|^T + |bias|) + |resid|,
  osc the uniform scale (1 when 0) or the per-sample scale, keep = 1 - gate (1 without a gate).  The wgmma accumulator is rounded once per
  16-term step (at most 2^-23 relative, truncation), n = K' / 16 steps for K' = kmul K <= 13 824 (n <= 864).  With incoherent term signs the
  partial sums grow like sqrt(j) and the rounding errors keep the sign of the partial sum, so the error is about 2^-23 * 0.2 sqrt(n) S
  <= 2^-20.4 S.  Bias add, scale, 1 - gate, the gate product and the residual add are five more fp32 roundings (<= 5 * 2^-24 S).  EPS = 2^-17,
  the VAE layers' value, keeps a margin of about 8.  The mean error of a tensor must stay under EPS / 4 * mean S: a systematic offset such
  as a missing bias or a neighbouring clip's gate does not.
bf16 outputs:  |got - want| <= 2^-8 |want| + (1 + 2^-7) prop,   want = act(ref),
  prop = |act'| EPS S + (SiLU only) 2^-21 |want|.  2^-8 |want| is the bf16 rounding; the rounding acts on the kernel's value, want + prop,
  hence the factor 1 + 2^-7.  |act'| <= 1 for none and <= 1.1 for SiLU (max silu' = 1.0998).  The kernel's silu(x) = x / (1 + expf(-x)):
  expf within 2 ulp (2^-22 relative), the add and the division one rounding each (2^-24), in all under 2^-21 |silu|.  The mean error must
  stay under 0.75 * 2^-8 mean |want| + mean prop (a bf16 rounding averages about 2^-9.5 relative).
bf16x3 (kmul 3):
  - split outputs: hi + lo within 2^-16 |want| + (1 + 2^-7) prop (lo = bf16(y - hi) rounds a value of at most 2^-8 |y|); the third block
    equals the first, bit for bit.
  - against the unrounded fp32 operands x (A's source) and W: with x = hi + lo + e, |e| <= 2^-16 |x| (the same for w), the kernel's three
    products differ from x w by x e_w + e_x w - e_x e_w + lo_x lo_w, and |lo| <= 2^-8 (1 + 2^-8) |x|, so per product by at most
    C3 |x| |w|,  C3 = (2 + (1 + 2^-8)^2 + 2^-16) 2^-16 < 3.01 * 2^-16.  Bound: |out - ref_src| <= |osc keep| C3 |x| |W|^T + EPS S for fp32
    outputs; for bf16 the same term times |act'| joins prop.
  - the packed weight: hi = bf16(w), the second block equal to the first, lo = bf16(w - hi), bit for bit.

Layout: outputs hold a spare row and spare columns filled with NaN (fp32) or the bf16 sentinel 0x7FAB; everything outside [M, N] (split:
outside the three N-column blocks) must still hold it, and everything inside must be written.  A's pitch lda may exceed kmul K; its pad
columns hold the sentinel too, and the kernel must not read them.

Cases: every dispatch code of EpiLinear::run on both kernels -- the fast paths bias -> f32, residual in place, gated residual in place,
bf16 and bf16 + SiLU, and the generic path (bf16x3 SiLU split as the context embedding's first layer, out_scale in {1, 0.5, -1.3} with 0
reading as 1, clips of 1, 5 and 31 rows, whose gate is looked up per row) -- and the two-clips-per-warp gate lookup (clips of 32, 33, 140 and
250 rows: boundaries on a warp's first row, inside a warp and on a 128-row tile edge).  M covers one row, partial warps and tiles, odd M-tile
counts (the cluster's empty padding tile) and 4000 / 8000 rows, where a persistent CTA walks several tiles and the ring and acc_free wrap;
N covers a single partial tile (8, 136) and 1024 / 1152 / 3456; K covers K' not a multiple of 64 (the TMA zero-fills the tail).
EpiLinearScaled runs per-sample scales {0, 1, 0.37, -1.3, 2.5} and must give, per sample, the bits of the uniform out_scale run with that
scale (exact zeros for 0).  A clip computed inside a batch equals the same clip computed alone, and the single-CTA and cluster kernels give
the same bits: both run the same k-ordered wgmma chain per tile and the same epilogue.  Kernel 0 must pick what Dit::lin picks."""
import ctypes as C
import math

import pytest
import torch

gpu = pytest.mark.gpu

SENT = 0x7FAB   # a bf16 NaN pattern no epilogue produces
EPS = 2.0 ** -17
C3 = (2 + (1 + 2.0 ** -8) ** 2 + 2.0 ** -16) * 2.0 ** -16
SILU_D = 1.1     # max |silu'(x)| = 1.0998
SILU_EPS = 2.0 ** -21
SINGLE, PAIR, SINGLE_SCALED, PAIR_SCALED = 1, 2, 3, 4
ACT_NONE, ACT_SILU = 0, 1
PADC = 8         # spare columns of every output


def _sentinel(*shape):
    return torch.full(shape, SENT, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous().view(torch.int16)


def _split(x, kmul):
    """fp32 [..., K] -> the bf16 operand the library stores: hi, or [hi | lo | hi]."""
    hi = x.bfloat16()
    if kmul == 1:
        return hi
    return torch.cat([hi, (x - hi.float()).bfloat16(), hi], -1)


def _p(t):
    return None if t is None else t.data_ptr()


def _call(A, W, *, M, N, K, kmul=1, lda=None, kernel=PAIR, bias=None, resid=None, ldr=0, gate=None, gate_bstride=0, rpb=0, out_f32=None,
          ld32=0, out_bf16=None, ld16=0, split=0, act=ACT_NONE, out_scale=0.0, scale=None, pair=1, swap_ab=1, m_select=0, w_packed=None,
          on_stream=True):
    """-> (status, kernel that ran).  Tensors are passed by pointer, ints as they are; on_stream False passes no stream (no CUDA needed)."""
    from ezaudio_b200 import _lib
    ran = C.c_int32(-1)
    a = _lib.TestLinearArgs(M=M, N=N, K=K, kmul=kmul, lda=kmul * K if lda is None else lda, ldr=ldr, gate_bstride=gate_bstride,
                            rows_per_batch=rpb, ld32=ld32, ld16=ld16, split=split, act=act, out_scale=out_scale, kernel=kernel, pair=pair,
                            swap_ab=swap_ab, m_select=m_select)
    a.A, a.W, a.w_packed, a.bias, a.resid, a.gate, a.out_f32, a.out_bf16, a.scale = map(
        _p, (A, W, w_packed, bias, resid, gate, out_f32, out_bf16, scale))
    a.ran = C.pointer(ran)
    rc = _lib.lib().ezb_test_linear(0, C.byref(a), _lib.stream_ptr() if on_stream else None)
    return rc, ran.value


class Problem:
    """Operands of one linear: fp32 sources x [M, K] (activations) and W [N, K], the bf16 A the kernel reads (pitch lda, sentinel pad
    columns), bias, and -- after the first launch -- the packed weight and the fp64 exact-operand product."""

    def __init__(self, M, N, K, kmul=1, lda_extra=0, seed=0):
        g = torch.Generator(device="cuda").manual_seed(seed * 7919 + M * 31 + N * 7 + K + kmul)
        self.M, self.N, self.K, self.kmul = M, N, K, kmul
        self.x = torch.randn(M, K, device="cuda", generator=g)
        self.W = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
        self.bias = 0.5 * torch.randn(N, device="cuda", generator=g)
        self.g = g
        self.lda = kmul * K + lda_extra
        self.A = _sentinel(M, self.lda)
        self.A[:, :kmul * K] = _split(self.x, kmul)
        self.Wp = None

    def run(self, **kw):
        """One launch; the first one also fetches and checks the packed weight.  -> kernel that ran."""
        from ezaudio_b200 import _lib
        first = self.Wp is None
        wp = _sentinel(self.N + 1, self.kmul * self.K) if first else None
        rc, ran = _call(self.A, self.W, M=self.M, N=self.N, K=self.K, kmul=self.kmul, lda=self.lda, w_packed=wp, **kw)
        _lib.check(rc)
        torch.cuda.synchronize()
        if first:
            self._check_packing(wp)
        return ran

    def _check_packing(self, wp):
        K, N = self.K, self.N
        assert torch.equal(_bits(wp[N]), _bits(_sentinel(1, self.kmul * K)[0])), "packed weight: a row past N was written"
        wp = wp[:N]
        hi = self.W.bfloat16()
        assert torch.equal(_bits(wp[:, :K]), _bits(hi)), "packed weight: hi != bf16(w)"
        if self.kmul == 3:
            assert torch.equal(_bits(wp[:, K:2 * K]), _bits(hi)), "packed weight: second hi block != hi"
            assert torch.equal(_bits(wp[:, 2 * K:]), _bits((self.W - hi.float()).bfloat16())), "packed weight: lo != bf16(w - hi)"
        self.Wp = wp
        a = self.A[:, :self.kmul * K].double()
        w = wp.double()
        self.acc = a @ w.t()                                  # exact-operand product
        self.S = a.abs() @ w.abs().t() + self.bias.double().abs()
        if self.kmul == 3:
            self.acc_src = self.x.double() @ self.W.double().t()
            self.S_src = self.x.double().abs() @ self.W.double().abs().t()

    def gate(self, rpb, seed=0):
        """(gate rows [B, 6N] fp32 in the model's modulation layout, the slice at column 2N the kernel reads, fp64 keep [M, N])."""
        B = (self.M + rpb - 1) // rpb
        full = 0.3 * torch.randn(B, 6 * self.N, device="cuda", generator=self.g)
        sl = full[:, 2 * self.N:]
        keep = (1 - sl[:, :self.N].double()).repeat_interleave(rpb, 0)[:self.M]
        return sl, keep


def _f32_out(M, N, init=None):
    """fp32 output with a spare row and PADC spare columns of NaN; [M, N] holds `init` (the residual of an in-place epilogue)."""
    o = _nan(M + 1, N + PADC)
    if init is not None:
        o[:M, :N] = init
    return o


def _check_layout_f32(o, M, N, tag):
    assert bool(torch.isfinite(o[:M, :N]).all()), f"{tag}: element of [M, N] not written"
    assert bool(torch.isnan(o[M]).all()) and bool(torch.isnan(o[:M, N:]).all()), f"{tag}: written outside [M, N]"


def _check_layout_bf16(o, M, width, tag):
    s = _bits(_sentinel(1, 1))[0, 0]
    assert not bool((_bits(o[:M, :width]) == s).any()), f"{tag}: element of the output not written"
    assert bool((_bits(o[M]) == s).all()) and bool((_bits(o[:M, width:]) == s).all()), f"{tag}: written outside the output"


def _check_f32(got, ref, S, tag, extra=None):
    """Per-element EPS * S (+ extra) and the mean bound; -> max error / allowance."""
    err = (got.double() - ref).abs()
    allow = EPS * S + (0 if extra is None else extra)
    i = int((err - allow).argmax())
    assert bool((err <= allow).all()), f"{tag}: err {float(err.flatten()[i]):.3e} > {float(allow.flatten()[i]):.3e} at {divmod(i, got.shape[1])}"
    assert float(err.mean()) <= EPS / 4 * float(S.mean()) + (0 if extra is None else float(extra.mean())), f"{tag}: mean err {float(err.mean()):.3e}"
    return float((err / allow).max())


def _check_bf16(o, N, split, ref, S, act, tag, extra=None):
    """bf16 (or split [hi | lo | hi]) output vs act(ref) in fp64, see the module docstring."""
    if act == ACT_SILU:
        want = ref * torch.sigmoid(ref)
        prop = SILU_D * EPS * S + SILU_EPS * want.abs()
        dact = SILU_D
    else:
        want, prop, dact = ref, EPS * S, 1.0
    if extra is not None:
        prop = prop + dact * extra
    hi = o[:, :N].double()
    if split:
        assert torch.equal(_bits(o[:, 2 * N:3 * N]), _bits(o[:, :N])), f"{tag}: third block != hi"
        got, rnd, mean_rnd = hi + o[:, N:2 * N].double(), 2.0 ** -16 * want.abs(), 0.75 * 2.0 ** -16
    else:
        got, rnd, mean_rnd = hi, 2.0 ** -8 * want.abs(), 0.75 * 2.0 ** -8
    err = (got - want).abs()
    allow = rnd + (1 + 2.0 ** -7) * prop
    i = int((err - allow).argmax())
    assert bool((err <= allow).all()), f"{tag}: err {float(err.flatten()[i]):.3e} > {float(allow.flatten()[i]):.3e} at {divmod(i, N)}"
    assert float(err.mean()) <= mean_rnd * float(want.abs().mean()) + float(prop.mean()), f"{tag}: mean err {float(err.mean()):.3e}"
    return float((err / allow).max())


# (M, N, K, rows per clip of the gated residual): one row, partial warps / tiles, odd M-tile counts (129, 257, 500, 511 -> the cluster's
# empty padding tile), several tiles per persistent CTA (4000, 8000; 3456 features at 8000 rows), N of one partial tile, K' % 64 != 0
SHAPES = [(1, 136, 72, 32), (31, 8, 264, 32), (33, 1024, 1152, 33), (128, 1152, 72, 32), (129, 136, 2304, 64), (257, 1152, 264, 140),
          (500, 1152, 1152, 250), (511, 1024, 4608, 250), (4000, 1152, 1152, 500), (8000, 1152, 2304, 250), (8000, 3456, 1152, 500)]


def _f32_cases(p, kernel, rpb, tag):
    """Fast-path fp32 codes: bias -> f32 (4), residual in place (5), gated residual in place (7).  -> {code: output [M, N]}."""
    M, N = p.M, p.N
    outs = {}
    o = _f32_out(M, N)
    assert p.run(kernel=kernel, bias=p.bias, out_f32=o, ld32=N + PADC) == kernel
    _check_layout_f32(o, M, N, f"{tag} bias->f32")
    ref = p.acc + p.bias.double()
    _check_f32(o[:M, :N], ref, p.S, f"{tag} bias->f32")
    if p.kmul == 3:
        _check_f32(o[:M, :N], p.acc_src + p.bias.double(), p.S, f"{tag} bias->f32 vs fp32 sources", extra=C3 * p.S_src)
    outs[4] = o[:M, :N].clone()
    x = torch.randn(M, N, device="cuda", generator=p.g)
    o = _f32_out(M, N, x)
    p.run(kernel=kernel, bias=p.bias, resid=o, ldr=N + PADC, out_f32=o, ld32=N + PADC)
    _check_layout_f32(o, M, N, f"{tag} residual")
    _check_f32(o[:M, :N], x.double() + ref, p.S + x.double().abs(), f"{tag} residual")
    outs[5] = o[:M, :N].clone()
    gate, keep = p.gate(rpb)
    o = _f32_out(M, N, x)
    p.run(kernel=kernel, bias=p.bias, resid=o, ldr=N + PADC, gate=gate, gate_bstride=6 * N, rpb=rpb, out_f32=o, ld32=N + PADC)
    _check_layout_f32(o, M, N, f"{tag} gated residual")
    _check_f32(o[:M, :N], x.double() + keep * ref, keep.abs() * p.S + x.double().abs(), f"{tag} gated residual")
    outs[7] = o[:M, :N].clone()
    return outs


@gpu
@pytest.mark.parametrize("kernel", [SINGLE, PAIR])
@pytest.mark.parametrize("M,N,K,rpb", SHAPES)
def test_linear_fast_paths(kernel, M, N, K, rpb):
    """Codes 4, 5, 7 (fp32) and 8, 8 | SiLU (bf16) of EpiLinear::run, bf16 operands."""
    p = Problem(M, N, K)
    tag = f"kernel {kernel} M {M} N {N} K {K}"
    _f32_cases(p, kernel, rpb, tag)
    ref = p.acc + p.bias.double()
    for act in (ACT_NONE, ACT_SILU):
        o = _sentinel(M + 1, N + PADC)
        p.run(kernel=kernel, bias=p.bias, out_bf16=o, ld16=N + PADC, act=act)
        _check_layout_bf16(o, M, N, f"{tag} bf16 act {act}")
        _check_bf16(o[:M], N, False, ref, p.S, act, f"{tag} bf16 act {act}")


@gpu
@pytest.mark.parametrize("kernel", [SINGLE, PAIR])
@pytest.mark.parametrize("M,N,K,rpb", [(33, 136, 264, 33), (500, 1152, 1152, 250), (4000, 1152, 4608, 500)])
def test_linear_bf16x3_residual_paths(kernel, M, N, K, rpb):
    """Parity mode's fp32-output linears (K' = 3K): the fast paths on [hi | lo | hi] x [hi | hi | lo], also against the fp32 sources."""
    _f32_cases(Problem(M, N, K, kmul=3), kernel, rpb, f"bf16x3 kernel {kernel} M {M} N {N} K {K}")


@gpu
@pytest.mark.parametrize("kernel", [SINGLE, PAIR])
@pytest.mark.parametrize("M,N,K,lda_extra", [(1, 136, 72, 0), (257, 1152, 1024, 8), (500, 1152, 1024, 0), (129, 1024, 4608, 64)])
def test_linear_bf16x3_silu_split(kernel, M, N, K, lda_extra):
    """The context embedding's first layer in parity mode: SiLU -> bf16 written [hi | lo | hi] (generic path), also with lda > 3K."""
    p = Problem(M, N, K, kmul=3, lda_extra=lda_extra)
    o = _sentinel(M + 1, 3 * N + PADC)
    p.run(kernel=kernel, bias=p.bias, out_bf16=o, ld16=3 * N + PADC, split=1, act=ACT_SILU)
    tag = f"kernel {kernel} M {M} N {N} K {K} lda {p.lda}"
    _check_layout_bf16(o, M, 3 * N, tag)
    _check_bf16(o[:M], N, True, p.acc + p.bias.double(), p.S, ACT_SILU, tag)
    _check_bf16(o[:M], N, True, p.acc_src + p.bias.double(), p.S, ACT_SILU, f"{tag} vs fp32 sources", extra=C3 * p.S_src)


@gpu
@pytest.mark.parametrize("kernel", [SINGLE, PAIR])
@pytest.mark.parametrize("M,N,K,kmul,lda_extra", [(129, 1152, 264, 1, 0), (500, 1152, 1152, 1, 8), (257, 136, 72, 3, 0)])
def test_linear_out_scale(kernel, M, N, K, kmul, lda_extra):
    """Uniform out_scale (the ControlNet zero-linears, generic path): bias -> f32 and the gated residual across clips of 250 rows; 0 reads
    as 1, bit for bit."""
    p = Problem(M, N, K, kmul=kmul, lda_extra=lda_extra)
    tag = f"kernel {kernel} M {M} N {N} K {K} kmul {kmul}"
    outs = {}
    for s in (0.0, 1.0, 0.5, -1.3):
        o = _f32_out(M, N)
        p.run(kernel=kernel, bias=p.bias, out_f32=o, ld32=N + PADC, out_scale=s)
        _check_layout_f32(o, M, N, f"{tag} scale {s}")
        ref = p.acc + p.bias.double()
        osc = s if s != 0 else 1.0
        _check_f32(o[:M, :N], osc * ref, abs(osc) * p.S, f"{tag} scale {s}")
        outs[s] = o[:M, :N].clone()
    assert torch.equal(_bits(outs[0.0]), _bits(outs[1.0])), f"{tag}: out_scale 0 differs from 1"
    rpb = 250
    gate, keep = p.gate(rpb)
    x = torch.randn(M, N, device="cuda", generator=p.g)
    o = _f32_out(M, N, x)
    p.run(kernel=kernel, bias=p.bias, resid=o, ldr=N + PADC, gate=gate, gate_bstride=6 * N, rpb=rpb, out_f32=o, ld32=N + PADC, out_scale=-1.3)
    _check_layout_f32(o, M, N, f"{tag} gated, scale -1.3")
    _check_f32(o[:M, :N], x.double() + keep * -1.3 * ref, 1.3 * keep.abs() * p.S + x.double().abs(), f"{tag} gated, scale -1.3")


@gpu
@pytest.mark.parametrize("kernel", [SINGLE, PAIR])
@pytest.mark.parametrize("rpb", [1, 5, 31, 32, 33, 140, 250])
def test_linear_gate_per_clip(kernel, rpb):
    """Gated residual in place across clip boundaries.  rpb < 32: the generic path looks up each row's gate; rpb >= 32: a warp's 32 rows
    span at most two clips (boundaries on a warp's first row for 32, which also puts them on 128-row tile edges; inside warps otherwise)."""
    M, N, K = 1000, 1152, 264
    p = Problem(M, N, K, seed=rpb)
    gate, keep = p.gate(rpb)
    x = torch.randn(M, N, device="cuda", generator=p.g)
    o = _f32_out(M, N, x)
    p.run(kernel=kernel, bias=p.bias, resid=o, ldr=N + PADC, gate=gate, gate_bstride=6 * N, rpb=rpb, out_f32=o, ld32=N + PADC)
    tag = f"kernel {kernel} rows per clip {rpb}"
    _check_layout_f32(o, M, N, tag)
    _check_f32(o[:M, :N], x.double() + keep * (p.acc + p.bias.double()), keep.abs() * p.S + x.double().abs(), tag)


@gpu
@pytest.mark.parametrize("kernel", [SINGLE_SCALED, PAIR_SCALED])
@pytest.mark.parametrize("rpb,M", [(1, 129), (31, 500), (250, 1250)])
def test_linear_scaled_per_sample(kernel, rpb, M):
    """EpiLinearScaled: per-request conditioning scales.  Each sample with scale s != 0 has the bits of the uniform out_scale = s run on the
    same kernel family; scale 0 gives exact zeros; all within the fp64 bound."""
    N, K = 1152, 1152
    p = Problem(M, N, K, seed=rpb)
    B = (M + rpb - 1) // rpb
    levels = (0.0, 1.0, 0.37, -1.3, 2.5)
    scale = torch.tensor([levels[b % len(levels)] for b in range(B)], device="cuda")
    o = _f32_out(M, N)
    assert p.run(kernel=kernel, bias=p.bias, out_f32=o, ld32=N + PADC, scale=scale, rpb=rpb) == kernel
    tag = f"kernel {kernel} rows per clip {rpb}"
    _check_layout_f32(o, M, N, tag)
    srow = scale.double().repeat_interleave(rpb)[:M].unsqueeze(1)
    _check_f32(o[:M, :N], srow * (p.acc + p.bias.double()), srow.abs() * p.S, tag)
    rows = torch.arange(M, device="cuda") // rpb % len(levels)
    assert bool((o[:M][rows == 0, :N] == 0).all()), f"{tag}: scale 0 gives non-zeros"
    for i, s in enumerate(levels[1:], 1):
        u = _f32_out(M, N)
        p.run(kernel=kernel - 2, bias=p.bias, out_f32=u, ld32=N + PADC, out_scale=s)
        assert torch.equal(_bits(o[:M][rows == i, :N]), _bits(u[:M][rows == i, :N])), f"{tag}: scale {s} differs from the uniform run"


@gpu
@pytest.mark.parametrize("kernel", [SINGLE, PAIR])
@pytest.mark.parametrize("rpb", [5, 250])
def test_linear_clip_in_batch_equals_alone(kernel, rpb):
    """A clip's rows inside a batch of three equal the clip computed alone, bit for bit (gated residual; rpb 5 takes the generic path)."""
    N, K, B = 1152, 1152, 3
    M = B * rpb
    p = Problem(M, N, K, seed=rpb)
    gate, _ = p.gate(rpb)
    x = torch.randn(M, N, device="cuda", generator=p.g)
    o = _f32_out(M, N, x)
    p.run(kernel=kernel, bias=p.bias, resid=o, ldr=N + PADC, gate=gate, gate_bstride=6 * N, rpb=rpb, out_f32=o, ld32=N + PADC)
    r0, r1 = rpb, 2 * rpb
    A1 = p.A[r0:r1].clone()
    o1 = _f32_out(rpb, N, x[r0:r1])
    from ezaudio_b200 import _lib
    rc, _ = _call(A1, p.W, M=rpb, N=N, K=K, kernel=kernel, bias=p.bias, resid=o1, ldr=N + PADC, gate=gate[1:], gate_bstride=6 * N, rpb=rpb,
                  out_f32=o1, ld32=N + PADC)
    _lib.check(rc)
    torch.cuda.synchronize()
    assert torch.equal(_bits(o[r0:r1, :N]), _bits(o1[:rpb, :N])), f"kernel {kernel} rpb {rpb}: clip 1 in the batch != alone"


@gpu
@pytest.mark.parametrize("M,N,K,kmul", [(500, 1152, 1152, 1), (8000, 1152, 1152, 1), (257, 136, 264, 3)])
def test_linear_single_and_cluster_kernels_agree(M, N, K, kmul):
    """gemm<128> and gemm2<128> give the same bits: the cluster only shares the W tile between the two CTAs of a pair."""
    p = Problem(M, N, K, kmul=kmul)
    gate, _ = p.gate(250)
    x = torch.randn(M, N, device="cuda", generator=p.g)
    outs = []
    for kernel in (SINGLE, PAIR):
        o = _f32_out(M, N, x)
        p.run(kernel=kernel, bias=p.bias, resid=o, ldr=N + PADC, gate=gate, gate_bstride=6 * N, rpb=250, out_f32=o, ld32=N + PADC)
        outs.append(o[:M, :N])
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), f"M {M} N {N} K {K} kmul {kmul}: single-CTA and cluster kernels differ"


@gpu
def test_linear_dispatch_matches_dit_lin():
    """Kernel 0 runs what Dit::lin runs: swap-AB for fp32-output bf16 linears of >= 512 tokens (m_select counts instead of M when set),
    the cluster kernel for fewer tokens, short clips, a uniform scale, bf16x3 and bf16 outputs, the single-CTA kernel without pairing."""
    N, K = 1152, 1152

    def ran(M, kmul=1, **kw):
        p = Problem(M, N, K, kmul=kmul)
        if kw.pop("bf16", False):
            kw.update(out_bf16=_sentinel(M + 1, N + PADC), ld16=N + PADC)
        else:
            kw.update(out_f32=_f32_out(M, N), ld32=N + PADC)
        r = p.run(kernel=0, bias=p.bias, **kw)
        if "out_f32" in kw and "scale" not in kw and "gate" not in kw:
            osc = kw.get("out_scale") or 1.0
            _check_f32(kw["out_f32"][:M, :N], osc * (p.acc + p.bias.double()), abs(osc) * p.S, f"kernel 0 M {M} -> {r}")
        return r

    assert ran(511) == PAIR
    assert ran(512) in (256, 288)
    assert ran(100, m_select=512) in (256, 288)
    assert ran(4000) in (256, 288)
    gate, _ = Problem(4000, N, K).gate(5)
    x = _f32_out(4000, N, torch.zeros(4000, N, device="cuda"))
    assert ran(4000, resid=x, ldr=N + PADC, gate=gate, gate_bstride=6 * N, rpb=5) == PAIR
    assert ran(4000, out_scale=0.5) == PAIR
    assert ran(4000, kmul=3) == PAIR
    assert ran(4000, bf16=True) == PAIR
    assert ran(4000, pair=0) == SINGLE
    assert ran(4000, swap_ab=0) == PAIR
    scale = torch.ones(16, device="cuda")
    assert ran(4000, scale=scale, rpb=250) == PAIR_SCALED
    assert ran(4000, scale=scale, rpb=250, pair=0) == SINGLE_SCALED


def test_linear_hook_rejects_bad_arguments():
    """Argument validation happens before any device work (this runs without a GPU)."""
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    p16 = (p + 15) // 16 * 16

    class P:   # a fake tensor: only its address is passed
        def __init__(self, a):
            self.a = a

        def data_ptr(self):
            return self.a

    t = P(p16)
    good = dict(M=64, N=128, K=128, kernel=PAIR, bias=t, out_f32=t, ld32=128)

    def rc(**over):
        kw = {**good, **over}
        A, W = kw.pop("A", t), kw.pop("W", t)
        return _call(A, W, on_stream=False, **kw)[0]

    EZB_ERR_ARG, EZB_ERR_SHAPE, EZB_ERR_UNSUPPORTED = -1, -2, -3
    assert rc(A=None) == EZB_ERR_ARG
    assert rc(W=None) == EZB_ERR_ARG
    assert rc(out_f32=None) == EZB_ERR_ARG                                   # no output at all
    assert rc(N=132) == EZB_ERR_SHAPE and rc(N=4, ld32=4) == EZB_ERR_SHAPE    # N % 8, N below 8
    assert rc(K=132) == EZB_ERR_SHAPE
    assert rc(lda=132) == EZB_ERR_SHAPE and rc(lda=120) == EZB_ERR_SHAPE     # lda % 8, lda < kmul K
    assert rc(kmul=2) == EZB_ERR_ARG
    assert rc(out_f32=None, out_bf16=t, ld16=3 * 128, split=1) == EZB_ERR_ARG   # split with kmul 1
    assert rc(scale=t, resid=t, ldr=128, kernel=0) == EZB_ERR_UNSUPPORTED
    assert rc(scale=t, resid=t, ldr=128, gate=t, gate_bstride=0, rpb=4, kernel=0) == EZB_ERR_UNSUPPORTED
    assert rc(scale=t, out_bf16=t, ld16=128, kernel=0) == EZB_ERR_UNSUPPORTED
    assert rc(scale=t, rpb=0, kernel=PAIR_SCALED) == EZB_ERR_SHAPE          # rows_per_batch < 1
    assert rc(resid=t, ldr=128, gate=t, gate_bstride=0, rpb=0) == EZB_ERR_SHAPE
    assert rc(kernel=5) == EZB_ERR_ARG and rc(kernel=-1) == EZB_ERR_ARG
    assert rc(kernel=PAIR, scale=t, rpb=1) == EZB_ERR_ARG                  # EpiLinear kernel with a per-sample scale
    assert rc(kernel=SINGLE_SCALED) == EZB_ERR_ARG                         # EpiLinearScaled without one
    assert rc(act=2) == EZB_ERR_ARG                                         # snake is the VAE's
    assert rc(gate=t, gate_bstride=0, rpb=4) == EZB_ERR_ARG                # a gate without a residual
    assert rc(ld32=120) == EZB_ERR_SHAPE                                    # output pitch narrower than N
    assert rc(A=P(p16 + 8)) == EZB_ERR_ARG                                  # A not 16-byte aligned (TMA)
