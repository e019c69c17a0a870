"""The two runtime options that replace a stand-alone LayerNorm launch, at kernel level, against float64 references of the operation:

* ln_fold -- the LayerNorm folded into the GEMMs on either side of it (csrc/gemm.cuh FoldIn / FoldOut, csrc/dit.cuh build_fold_tables):
      h W^T = rstd ((x g) W^T - mu u) + v,   u = g W^T,  v = c W^T (+ bias),   g = w (1 + scale),  c = b (1 + scale) + shift.
  The GEMM that writes x also writes A = bf16(x g) and per-row (sum x, sum x^2) partials per 32-feature slot; the GEMM behind the
  LayerNorm turns the partials into (mu, rstd) and applies the per-row affine to its accumulator.
* ln_tail -- the LayerNorm run as the tail phase of a one-wave swap-AB GEMM behind a grid barrier (csrc/gemm_ln.cuh).

Everything runs through ezb_test_fold (and ezb_test_gemm kinds 20 / 21 for the skip path's two-source fold), which launch the kernels
as Dit launches them.  u = 2^-24 below is the fp32 unit roundoff; bf16 rounds to nearest with |bf16(a) - a| <= 2^-8 |a|.

Tables (fold_gc_kernel, fold_uv_kernel).  G = w (1 + scale) is one fp32 add and one multiply, so it must equal torch's fp32 value bit for
bit; Cc = b (1 + scale) + shift is within 2u (|b (1 + scale)| + |shift|).  U[r, n] = sum_k W'[n, k] G[r, k] over the packed bf16 W' is
a lane's fp32 fma chain of ceil(K / 32) terms and a 5-level warp tree: |U - U64| <= (ceil(K / 32) + 5) u sum_k |W' G| (the first-order
gamma_n bound); V the same over Cc, plus one rounding u |V| for the added bias.

Statistics of the fold.  From the partials (s1_s, s2_s), s = 1..n, the kernel forms s1, s2 by n - 1 sequential fp32 adds, mean =
s1 inv_dim and var = s2 inv_dim - mean^2 (inv_dim = fl(1 / width)), rstd = rsqrtf(var + 1e-5) (2 ulp).  In fp64 from the same partials
(m, e2 = sum s2 / width, var64 = e2 - m^2):
    dm  = (n + 1) u sum |s1_s| / width,        dv = (n + 1) u e2 + 2 |m| dm + 2 u (e2 + m^2),
    er  = dv / (2 (var64 + 1e-5)) + 3 u        (relative error of rstd).
var = E[x^2] - mean^2 cancels: at |mean| / std = 30, e2 = 901 var and er grows 901-fold, which is why the statistics term is explicit.
Exact-operand bound of the pre-activation h = fmaf(acc, rstd, fmaf(-mean rstd, u_n, v_n)), acc the fp32 wgmma sum of A W'^T:
    eh = rstd EPS S + 2 (rstd |acc| er + |u_n| (rstd |m| er + rstd dm + u rstd |m|) + u (|t| + |h|)),   S = |A| |W'|^T,
EPS = 2^-17 the accumulator allowance of test_linear_gpu.py (margin about 8 on its own derivation), the factor 2 a margin for second-order
terms of the fp32 part.
True-LayerNorm bound: the reference is fp64 LayerNorm(x) g + c times W' (+ bias), from the fp32 x.  The fold adds
    rstd 2^-8 (|x| |g|) |W'|^T                 (A = bf16(x g) is rounded before the mean is removed: grows with 1 + |mean| / std),
    rstd |m| dU + dV                           (the tables' fp32 error, bound above),
and the statistics term is taken with n + 32 instead of n terms (forming a partial of 32 fp32 values, in any order).
GEGLU (kinds 1, 2): out = bf16(h gelu(g)) with geglu_fast (Abramowitz-Stegun erf, |err| <= 1.5e-7, MUFU rcp / ex2): the kernel's erf is
within 2^-21 of the true one, so gelu within 2^-22 |g| (bound 2^-19 |h g| with margin), the products a few u |out|.  Propagated:
    prop = |gelu(g)| eh_h + 1.13 (|h| + eh_h) eh_g + 2^-19 |h g| + 2^-21 |want|   (max |gelu'| = 1.129),
    |got - want| <= 2^-8 |want| + (1 + 2^-7) prop,   mean error <= 0.75 * 2^-8 mean |want| + mean prop.
Linear outputs (skip path): |got - want| <= eh + u |want| (the bias add), mean error <= mean allowance / 4.
Rows of x have |mean| / std of about 0, 3 and 30 (row r % 3).  The GEGLU test prints, per group, the fold's error next to the unfolded
path's (stand-alone LayerNorm kernel, then the GEGLU GEMM) against the same true-LayerNorm reference.

LayerNorm tail: the tail runs ln_row_reg (widths 1024 / 1152, one source) or ln_row_generic, the arithmetic of the stand-alone kernels
that ln_variant 0 selects, so its output must equal theirs bit for bit on the GEMM's own fp32 output; both are held to the step-kernel
LayerNorm bound of test_step_kernels_gpu.py, the GEMM output to test_linear_gpu.py's.  When the tiles exceed the SM count the launch
must fall back to the GEMM alone, report it, and leave the LayerNorm output untouched.  The grid barrier resets its count to 0 and
advances its generation once per launch, back to back and under CUDA-graph replay."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_linear_gpu import EPS, _bits, _check_f32, _nan, _sentinel

gpu = pytest.mark.gpu

U = 2.0 ** -24
GD = 1.13            # max |gelu'|
OFFSETS = (0.0, 3.0, 30.0)
EZB_ERR_ARG, EZB_ERR_SHAPE, EZB_ERR_UNSUPPORTED = -1, -2, -3


# ------------------------------------------------------------------------------------------------------------------------------ plumbing
def _fold_call(on_stream=True, **kw):
    from ezaudio_b200 import _lib
    a = _lib.TestFoldArgs()
    for k, v in kw.items():
        setattr(a, k, v.data_ptr() if torch.is_tensor(v) else v)
    rc = _lib.lib().ezb_test_fold(0, C.byref(a), _lib.stream_ptr() if on_stream else None)
    return rc, a


def _fold(**kw):
    from ezaudio_b200 import _lib
    rc, a = _fold_call(**kw)
    _lib.check(rc)
    torch.cuda.synchronize()
    return a


def _gemm(A, W, M, N, K, bn, kind, **epi):
    from ezaudio_b200 import _lib
    e = _lib.TestEpilogue()
    for k, v in epi.items():
        setattr(e, k, v.data_ptr() if torch.is_tensor(v) else v)
    _lib.check(_lib.lib().ezb_test_gemm(0, _lib.ptr(A), A.stride(0), _lib.ptr(W), W.stride(0), M, N, K, bn, kind, C.byref(e), 0, 0, 0, 0, 0, 0,
                                        _lib.stream_ptr()))
    torch.cuda.synchronize()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rows(M, D, g):
    """randn rows shifted by 0, 3 or 30 (row r % 3): |mean| / std of about 0, 3 and 30."""
    off = torch.tensor(OFFSETS, device="cuda")[torch.arange(M, device="cuda") % 3]
    return torch.randn(M, D, device="cuda", generator=g) + off[:, None]


def _partials(x, ld_st):
    """(sum, sum of squares) of x per 32-feature slot, float2 [slots][ld_st] (rows >= M NaN), as FoldOut lays them out."""
    M, D = x.shape
    slots = (D + 31) // 32
    xp = F.pad(x, (0, slots * 32 - D)).view(M, slots, 32)
    st = torch.full((slots, ld_st, 2), float("nan"), device="cuda")
    st[:, :M, 0] = xp.sum(2).t()
    st[:, :M, 1] = (xp * xp).sum(2).t()
    return st


def _stats(s1, s2, width, n):
    """fp64 (m, rstd) from summed partials and the bounds dm, er of the module docstring; s1 / s2: [n, M] partials."""
    m = s1.sum(0) / width
    e2 = s2.sum(0) / width
    var = e2 - m * m
    rstd = 1 / torch.sqrt(var + 1e-5)
    dm = (n + 1) * U * s1.abs().sum(0) / width
    dv = (n + 1) * U * e2 + 2 * m.abs() * dm + 2 * U * (e2 + m * m)
    er = dv / (2 * (var + 1e-5)) + 3 * U
    return m[:, None], rstd[:, None], dm[:, None], er[:, None]


def _fold_h(acc, S, m, rstd, dm, er, u, v):
    """h = rstd acc - rstd m u + v in fp64 and its fp32 allowance eh (module docstring)."""
    t = -m * rstd * u + v
    h = rstd * acc + t
    eh = rstd * EPS * S + 2 * (rstd * acc.abs() * er + u.abs() * (rstd * m.abs() * er + rstd * dm + U * rstd * m.abs()) + U * (t.abs() + h.abs()))
    return h, eh


def _unpack(t, bn):
    """[M, 2 inner] in the packed GEGLU column order (N-tiles of bn: bn / 2 hidden, then bn / 2 gate) -> (hidden, gate) [M, inner]."""
    M, N = t.shape
    t = t.reshape(M, N // bn, 2, bn // 2)
    return t[:, :, 0].reshape(M, -1), t[:, :, 1].reshape(M, -1)


def _check_geglu(got, h, eh, bn, tag, rows=None):
    """bf16 GEGLU output [M, inner] vs h gelu(g) from the packed pre-activations h (fp64) with allowance eh -> (max err, max err / allow)."""
    hh, hg = _unpack(h, bn)
    eh_h, eh_g = _unpack(eh, bn)
    want = hh * F.gelu(hg)
    prop = F.gelu(hg).abs() * eh_h + GD * (hh.abs() + eh_h) * eh_g + 2.0 ** -19 * (hh * hg).abs() + 2.0 ** -21 * want.abs()
    allow = 2.0 ** -8 * want.abs() + (1 + 2.0 ** -7) * prop
    err = (got.double() - want).abs()
    i = int((err - allow).argmax())
    assert bool((err <= allow).all()), f"{tag}: err {float(err.flatten()[i]):.3e} > {float(allow.flatten()[i]):.3e} at {divmod(i, want.shape[1])}"
    assert float(err.mean()) <= 0.75 * 2.0 ** -8 * float(want.abs().mean()) + float(prop.mean()), f"{tag}: mean err {float(err.mean()):.3e}"
    return err, float((err / allow).max())


def _check_lin(got, want, allow, tag):
    err = (got.double() - want).abs()
    i = int((err - allow).argmax())
    assert bool((err <= allow).all()), f"{tag}: err {float(err.flatten()[i]):.3e} > {float(allow.flatten()[i]):.3e} at {divmod(i, want.shape[1])}"
    assert float(err.mean()) <= float(allow.mean()) / 4, f"{tag}: mean err {float(err.mean()):.3e} vs allowance {float(allow.mean()):.3e}"
    return err, float((err / allow).max())


def _table_terms(G, Cc, Wp, K):
    """fp32 error bounds dU, dV [1, N] of the fold tables over the packed W' (module docstring; V without the bias rounding)."""
    n = math.ceil(K / 32) + 5
    Wa = Wp.double().abs()
    return n * U * (G.double().abs() @ Wa.t()), n * U * (Cc.double().abs() @ Wa.t())


# ------------------------------------------------------------------------------------------------------------------------------ tables
@gpu
@pytest.mark.parametrize("K", [144, 1024, 1152, 2304])
@pytest.mark.parametrize("R", [1, 3, 128])
def test_fold_tables(K, R):
    """fold_gc_kernel + fold_uv_kernel at the model's widths (2304: the skip path, every one of a lane's 72 registers in use) for 1, 3 and
    fold_T = 128 timesteps, with and without the added bias; rows past R and past N stay untouched."""
    N = 259                                       # a partial last block of 8 warps
    g = _gen(K * 131 + R)
    W = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
    w, b = 1 + 0.2 * torch.randn(K, device="cuda", generator=g), 0.2 * torch.randn(K, device="cuda", generator=g)
    ld_mod = 6 * K
    tab = 0.3 * torch.randn(R, ld_mod, device="cuda", generator=g)   # [t][6 K] as the model's modulation rows; site 3: shift 3K, scale 4K
    sh, sc = tab[:, 3 * K:4 * K], tab[:, 4 * K:5 * K]
    add = 0.3 * torch.randn(N, device="cuda", generator=g)
    for use_add in (False, True):
        wp = _sentinel(N + 1, K)
        G, Cc, u, v = _nan(R + 1, K), _nan(R + 1, K), _nan(R + 1, N), _nan(R + 1, N)
        _fold(kind=0, N=N, K=K, R=R, w=w, b=b, shift=sh, scale=sc, ld_mod=ld_mod, W=W, add_v=add if use_add else None, w_packed=wp, G=G, Cc=Cc,
              u=u, v=v)
        tag = f"tables K {K} R {R} add_v {use_add}"
        assert torch.equal(_bits(wp[:N]), _bits(W.bfloat16())) and bool((_bits(wp[N]) == _bits(_sentinel(1, K))[0]).all()), f"{tag}: packed W"
        for t, rows in ((G, R), (Cc, R), (u, R), (v, R)):
            assert bool(t[rows].isnan().all()), f"{tag}: a row past R written"
        assert torch.equal(_bits(G[:R]), _bits(w * (1 + sc))), f"{tag}: G != w (1 + scale)"
        c64 = b.double() * (1 + sc).double() + sh.double()
        assert bool(((Cc[:R].double() - c64).abs() <= 2 * U * ((b.double() * (1 + sc).double()).abs() + sh.double().abs())).all()), f"{tag}: Cc"
        Wd = wp[:N].double()
        U64, V64 = G[:R].double() @ Wd.t(), Cc[:R].double() @ Wd.t()
        n = math.ceil(K / 32) + 5
        aU = n * U * (G[:R].double().abs() @ Wd.abs().t())
        aV = n * U * (Cc[:R].double().abs() @ Wd.abs().t())
        if use_add:
            V64 = V64 + add.double()
            aV = aV + U * V64.abs()
        eu, ev = (u[:R].double() - U64).abs(), (v[:R].double() - V64).abs()
        assert bool((eu <= aU).all()), f"{tag}: U err {float(eu.max()):.3e}, {float((eu / aU).max()):.2f} of the allowance"
        assert bool((ev <= aV).all()), f"{tag}: V err {float(ev.max()):.3e}, {float((ev / aV).max()):.2f} of the allowance"
        print(f"[fold] {tag}: U {float((eu / aU).max()):.3f}, V {float((ev / aV).max()):.3f} of the allowance")


# ------------------------------------------------------------------------------------------------------------------------------ FoldIn GEGLU
class GegluFold:
    """One norm3 -> GEGLU site: rows x, LayerNorm w / b and one modulation row, W1 / b1 in the reference layout; A = bf16(x G) and the
    partials as FoldOut writes them."""

    def __init__(self, M, D, inner, seed):
        g = _gen(seed)
        self.M, self.D, self.inner = M, D, inner
        self.x = _rows(M, D, g)
        self.w, self.b = 1 + 0.2 * torch.randn(D, device="cuda", generator=g), 0.2 * torch.randn(D, device="cuda", generator=g)
        self.tab = 0.3 * torch.randn(1, 6 * D, device="cuda", generator=g)
        self.sh, self.sc = self.tab[:, 3 * D:4 * D], self.tab[:, 4 * D:5 * D]
        self.W = torch.randn(2 * inner, D, device="cuda", generator=g) / math.sqrt(D)
        self.bias = 0.2 * torch.randn(2 * inner, device="cuda", generator=g)
        self.G = (self.w * (1 + self.sc[0])).contiguous()     # fp32, as fold_gc_kernel
        self.A = (self.x * self.G).bfloat16()
        self.ld_st = M + 16
        self.st = _partials(self.x, self.ld_st)
        self.slots = self.st.shape[0]
        self.g = g

    def tables(self):
        return dict(R=1, w=self.w, b=self.b, shift=self.sh, scale=self.sc, ld_mod=6 * self.D, W=self.W, bias=self.bias, A=self.A, st=self.st,
                    slots=self.slots, ld_st=self.ld_st)

    def outs(self):
        D, N = self.D, 2 * self.inner
        return dict(w_packed=_sentinel(N, D), G=_nan(1, D), Cc=_nan(1, D), u=_nan(N), v=_nan(N))

    def exact(self, o, A=None):
        """Exact-operand reference: packed h (fp64) and eh from the kernel's tables, packed W' and the partials."""
        A = self.A if A is None else A
        Wp = o["w_packed"]
        assert torch.equal(_bits(o["G"][0]), _bits(self.G)), "G != w (1 + scale)"
        acc = A.double() @ Wp.double().t()
        S = A.double().abs() @ Wp.double().abs().t()
        m, rstd, dm, er = _stats(self.st[:, :self.M, 0].double(), self.st[:, :self.M, 1].double(), self.D, self.slots)
        return _fold_h(acc, S, m, rstd, dm, er, o["u"].double()[None], o["v"].double()[None])

    def true(self, o, bias_packed):
        """True-LayerNorm reference: fp64 LayerNorm(x) G + Cc times W' plus the packed bias, and its allowance (module docstring)."""
        x = self.x.double()
        Wp, G, Cc = o["w_packed"].double(), o["G"].double(), o["Cc"].double()
        mu = x.mean(1, keepdim=True)
        rs = 1 / torch.sqrt(((x - mu) ** 2).mean(1, keepdim=True) + 1e-5)
        h = ((x - mu) * rs * G + Cc) @ Wp.t() + bias_packed.double()
        acc = self.A.double() @ Wp.t()
        S = self.A.double().abs() @ Wp.abs().t()
        m, rstd, dm, er = _stats(self.st[:, :self.M, 0].double(), self.st[:, :self.M, 1].double(), self.D, self.slots + 32)
        dm = dm + 32 * U * x.abs().sum(1, keepdim=True) / self.D
        _, eh = _fold_h(acc, S, m, rstd, dm, er, o["u"].double()[None], o["v"].double()[None])
        dU, dV = _table_terms(o["G"], o["Cc"], o["w_packed"], self.D)
        eh = eh + rs * 2.0 ** -8 * ((x.abs() * G.abs()) @ Wp.abs().t()) + rs * mu.abs() * dU + dV + U * o["v"].double().abs()[None]
        return h, eh


def _pack_bias(bias, inner, bn):
    half = bn // 2
    return torch.stack([bias[:inner].view(-1, half), bias[inner:].view(-1, half)], 1).reshape(-1).contiguous()


def _unfolded(p, o, bn):
    """The path without the fold on the same inputs: the stand-alone LayerNorm kernel Dit::ln selects, then the GEGLU GEMM Dit::block
    dispatches (2-CTA gemm2_geglu for 256-wide tiles, single-CTA EpiGeglu<128> otherwise)."""
    from tests.test_step_kernels_gpu import AUTO, _ln_call
    act = _ln_call(p.M, p.D, 1, AUTO, p.x, w=p.w, b=p.b, sh=p.sh, sc=p.sc, mbs=0, rpb=1)
    out = torch.zeros(p.M, p.inner, device="cuda", dtype=torch.bfloat16)
    _gemm(act, o["w_packed"], p.M, 2 * p.inner, p.D, bn, 11 if bn == 256 else 1, bias=_pack_bias(p.bias, p.inner, bn), out_bf16=out, ld16=p.inner)
    return out


GEGLU_SITES = {"XL": (1152, 4608, 256), "L": (1024, 4096, 256), "tiny72": (144, 576, 128)}


@gpu
@pytest.mark.parametrize("site", list(GEGLU_SITES))
@pytest.mark.parametrize("M", [257, 1000, 4000])
def test_fold_geglu(site, M):
    """The FoldIn GEGLU Dit::block dispatches: gemm2<256, EpiGeglu<256, true>> (XL, L) and gemm<128, EpiGeglu<128, true>> (tiny72: inner
    576 is not a multiple of 128), W1 and its bias packed as the model packs them, v carrying the GEGLU bias once.  Exact-operand and
    true-LayerNorm bounds; the fold's error is printed next to the unfolded path's."""
    D, inner, bn = GEGLU_SITES[site]
    p = GegluFold(M, D, inner, seed=M + D)
    o = p.outs()
    out = _sentinel((M + 1) * inner)
    _fold(kind=1, M=M, K=D, inner=inner, geglu_bn=0, out=out, **p.tables(), **o)
    tag = f"fold GEGLU {site} M {M}"
    assert bool((_bits(out[M * inner:]) == _bits(_sentinel(1))[0]).all()), f"{tag}: rows >= M written"
    got = out[:M * inner].view(M, inner)
    bp = _pack_bias(p.bias, inner, bn)
    assert torch.equal(_bits(o["w_packed"]), _bits(_pack_rows(p.W, inner, bn).bfloat16())), f"{tag}: packed W1"
    h, eh = p.exact(o)
    _, q = _check_geglu(got, h, eh, bn, f"{tag} exact operands")
    ht, eht = p.true(o, bp)
    err, qt = _check_geglu(got, ht, eht, bn, f"{tag} true LayerNorm")
    uerr = (_unfolded(p, o, bn).double() - (lambda hh, hg: hh * F.gelu(hg))(*_unpack(ht, bn))).abs()
    grp = torch.arange(M, device="cuda") % 3
    for i, off in enumerate(OFFSETS):
        print(f"[fold] {tag} |mean|/std {off:>4}: fold max err {float(err[grp == i].max()):.3e}, unfolded max err {float(uerr[grp == i].max()):.3e}"
              f" (vs fp64 LayerNorm + GEGLU; {q:.2f} / {qt:.2f} of the exact-operand / true-LayerNorm allowance)")


def _pack_rows(W, inner, bn):
    half = bn // 2
    D = W.shape[1]
    return torch.stack([W[:inner].view(inner // half, half, D), W[inner:].view(inner // half, half, D)], 1).reshape(2 * inner, D)


# ------------------------------------------------------------------------------------------------------------------------------ skip path
@gpu
@pytest.mark.parametrize("kind,bn", [(21, 256), (21, 288), (20, 0)])
def test_fold_skip_path_two_sources(kind, bn):
    """The out-blocks' skip_norm over [x | skip] folded into skip_linear (K = 2 D = 2304): statistics from both halves' partials, the x
    half of the operand multiplied by snw[:D] and the skip half by snw[D:] as Dit::block_output_fold has the producing GEMMs write them.
    The producers are EpiLinearTF gated residuals with clips of 140 rows (boundaries inside a 288-token tile)."""
    D, M, Kp, L = 1152, 1000, 264, 140
    g = _gen(kind * 1000 + bn)
    snw, snb = 1 + 0.2 * torch.randn(2 * D, device="cuda", generator=g), 0.2 * torch.randn(2 * D, device="cuda", generator=g)
    Wsk = torch.randn(D, 2 * D, device="cuda", generator=g) / math.sqrt(2 * D)
    bsk = 0.2 * torch.randn(D, device="cuda", generator=g)
    g1 = torch.rand(D, device="cuda", generator=g) + 0.5
    cat = _sentinel(M, 2 * D)
    ld_st = M + 16
    nb = (M + L - 1) // L

    def produce(a_kw):   # x = x0 + (1 - gate) (A W^T + bias), folded out as given
        A = torch.randn(M, Kp, device="cuda", generator=g).bfloat16()
        W = (torch.randn(D, Kp, device="cuda", generator=g) / math.sqrt(Kp)).bfloat16()
        bias = torch.randn(D, device="cuda", generator=g)
        gate = 0.3 * torch.randn(nb, 6 * D, device="cuda", generator=g)
        x = _rows(M, D, g)
        st = torch.full((D // 32, ld_st, 2), float("nan"), device="cuda")
        _gemm(A, W, M, D, Kp, 288, 21, bias=bias, resid=x, ldr=D, out_f32=x, ld32=D, gate=gate[:, 5 * D:], gate_bstride=6 * D, rows_per_batch=L,
              fout_st=st, fout_ld_st=ld_st, **a_kw)
        return x, st

    act = _sentinel(M, D)
    xs, st_s = produce(dict(fout_a0=act, fout_ld0=D, fout_g0=g1, fout_a1=cat[:, D:], fout_ld1=2 * D, fout_g1=snw[D:]))   # in-block output
    xx, st_x = produce(dict(fout_a0=cat, fout_ld0=2 * D, fout_g0=snw))                                              # mid / out-block output
    tag = f"skip fold kind {kind} bn {bn}"
    assert torch.equal(_bits(cat[:, :D]), _bits((xx * snw[:D]).bfloat16())), f"{tag}: x half of the operand"
    assert torch.equal(_bits(cat[:, D:]), _bits((xs * snw[D:]).bfloat16())), f"{tag}: skip half of the operand"
    wp, G, Cc, u, v = _sentinel(D, 2 * D), _nan(1, 2 * D), _nan(1, 2 * D), _nan(D), _nan(D)
    _fold(kind=0, N=D, K=2 * D, R=1, w=snw, b=snb, W=Wsk, w_packed=wp, G=G, Cc=Cc, u=u, v=v)
    out = _nan(M + 1, D)
    act2 = _sentinel(M, D)
    st_o = torch.full((D // 32, ld_st, 2), float("nan"), device="cuda")
    _gemm(cat, wp, M, D, 2 * D, bn, kind, bias=bsk, out_f32=out, ld32=D, fin_st=st_x, fin_slots=D // 32, fin_ld_st=ld_st, fin_inv_dim=1.0 / (2 * D),
          fin_u=u, fin_v=v, fin_st1=st_s, fin_slots1=D // 32, fout_st=st_o, fout_ld_st=ld_st, fout_a0=act2, fout_ld0=D, fout_g0=g1)
    assert bool(out[M].isnan().all()), f"{tag}: row M written"
    got = out[:M]
    assert torch.equal(_bits(act2), _bits((got * g1).bfloat16())), f"{tag}: folded-out operand"
    # exact operands: the kernel's cat, partials and tables
    n = 2 * (D // 32)
    s1 = torch.cat([st_x[:, :M, 0], st_s[:, :M, 0]]).double()
    s2 = torch.cat([st_x[:, :M, 1], st_s[:, :M, 1]]).double()
    acc = cat.double() @ wp.double().t()
    S = cat.double().abs() @ wp.double().abs().t()
    m, rstd, dm, er = _stats(s1, s2, 2 * D, n)
    h, eh = _fold_h(acc, S, m, rstd, dm, er, u.double()[None], v.double()[None])
    want = h + bsk.double()
    _, q = _check_lin(got, want, eh + U * want.abs(), f"{tag} exact operands")
    # true LayerNorm over [x | skip]
    xc = torch.cat([xx, xs], 1).double()
    mu = xc.mean(1, keepdim=True)
    rs = 1 / torch.sqrt(((xc - mu) ** 2).mean(1, keepdim=True) + 1e-5)
    want_t = ((xc - mu) * rs * snw.double() + snb.double()) @ wp.double().t() + bsk.double()
    m, rstd, dm, er = _stats(s1, s2, 2 * D, n + 32)
    dm = dm + 32 * U * xc.abs().sum(1, keepdim=True) / (2 * D)
    _, eht = _fold_h(acc, S, m, rstd, dm, er, u.double()[None], v.double()[None])
    dU, dV = _table_terms(G, Cc, wp, 2 * D)
    eht = eht + rs * 2.0 ** -8 * ((xc.abs() * snw.double().abs()) @ wp.double().abs().t()) + rs * mu.abs() * dU + dV + U * v.double().abs()[None]
    err, qt = _check_lin(got, want_t, eht + U * want_t.abs(), f"{tag} true LayerNorm")
    grp = torch.arange(M, device="cuda") % 3
    print(f"[fold] {tag}: {q:.2f} / {qt:.2f} of the exact-operand / true-LayerNorm allowance; max err per |mean|/std "
          + ", ".join(f"{off}: {float(err[grp == i].max()):.3e}" for i, off in enumerate(OFFSETS)))


# ------------------------------------------------------------------------------------------------------------------------------ fused MLP
@gpu
@pytest.mark.parametrize("M,L", [(1000, 500), (4000, 500), (1000, 40)])
def test_fold_mlp_fused(M, L):
    """mlp_fused<EpiGeglu<256, true>, EpiLinearTF<256>> (the whole MLP as one persistent launch, LayerNorm folded in and out) gives the bits
    of the same two GEMMs as two fold launches, and both phases are within their fp64 bounds: the GEGLU's exact-operand bound, the gated
    residual's test_linear bound on the kernel's own mid, the folded-out operand and partials of the new x."""
    D, inner = 1152, 4608
    p = GegluFold(M, D, inner, seed=M + L)
    g = p.g
    W2 = (torch.randn(D, inner, device="cuda", generator=g) / math.sqrt(inner)).bfloat16()
    b2 = torch.randn(D, device="cuda", generator=g)
    nb = (M + L - 1) // L
    gate = 0.3 * torch.randn(nb, 6 * D, device="cuda", generator=g)
    g0 = torch.rand(D, device="cuda", generator=g) + 0.5
    bar = torch.zeros(2, dtype=torch.int32, device="cuda")
    ld_st = p.ld_st

    def run(variant):
        o = p.outs()
        x = p.x.clone()   # the residual stream is the LayerNorm's input, updated in place
        mid, a0 = _sentinel(M, inner), _sentinel(M, D)
        st = torch.full((D // 32, ld_st, 2), float("nan"), device="cuda")
        _fold(kind=2, variant=variant, M=M, K=D, inner=inner, out=mid, W2=W2, b2=b2, x=x, gate=gate[:, 5 * D:], gate_bstride=6 * D, rows_per_batch=L,
              fout_st=st, a0=a0, g0=g0, grid_barrier=bar, **p.tables(), **o)
        return o, x, mid, a0, st

    o, x2, mid2, a02, st2 = run(1)
    for i in range(2):
        gen = int(bar[1])
        _, xf, midf, a0f, stf = run(0)
        assert int(bar[0]) == 0 and int(bar[1]) == gen + 1, (i, bar.tolist())
        for a, b_ in ((xf, x2), (midf, mid2), (a0f, a02), (stf[:, :M], st2[:, :M])):
            assert torch.equal(_bits(a), _bits(b_)), f"M {M} L {L}: persistent launch {i} differs from the two-launch fold path"
    tag = f"fold MLP M {M} L {L}"
    h, eh = p.exact(o)
    _check_geglu(mid2, h, eh, 256, f"{tag} GEGLU")
    keep = 1 - gate[:, 5 * D:].double().repeat_interleave(L, 0)[:M]
    x0 = p.x.double()
    ref = x0 + keep * (mid2.double() @ W2.double().t() + b2.double())
    S = keep.abs() * (mid2.double().abs() @ W2.double().abs().t() + b2.double().abs()) + x0.abs()
    _check_f32(x2, ref, S, f"{tag} gated residual")
    assert torch.equal(_bits(a02), _bits((x2 * g0).bfloat16())), f"{tag}: folded-out operand"
    assert bool(st2[:, M:].isnan().all()), f"{tag}: partials past M written"
    part = x2.double().view(M, D // 32, 32)
    e1 = (st2[:, :M, 0].double() - part.sum(2).t()).abs()
    e2 = (st2[:, :M, 1].double() - (part * part).sum(2).t()).abs()
    assert bool((e1 <= 2 * 6 * U * part.abs().sum(2).t()).all()), f"{tag}: partial sums"
    assert bool((e2 <= 2 * 7 * U * (part * part).sum(2).t()).all()), f"{tag}: partial sums of squares"


# ------------------------------------------------------------------------------------------------------------------------------ LayerNorm tail
class Tail:
    """x = x0 + (1 - gate) (A W^T + bias) through ezb_test_fold kind 3, then the LayerNorm of [x | x2 (+ x3)]."""

    def __init__(self, M, N, K, seed, gate_rpb=None, mod_rpb=None, D2=0, x3=False):
        from tests.test_step_kernels_gpu import _ln_params, _mod_table
        g = _gen(seed)
        self.M, self.N, self.K, self.D2 = M, N, K, D2
        self.A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
        self.W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
        self.bias = torch.randn(N, device="cuda", generator=g)
        self.x0 = torch.randn(M, N, device="cuda", generator=g) + 2.0
        self.gate_rpb = gate_rpb
        self.gate = 0.3 * torch.randn((M + gate_rpb - 1) // gate_rpb, 6 * N, device="cuda", generator=g) if gate_rpb else None
        self.w, self.b = _ln_params(N + D2, g)
        self.tab, self.sh, self.sc, self.mbs, self.rpb = _mod_table(M, N, mod_rpb, g)
        if mod_rpb is None:
            self.rpb = gate_rpb or 1
        self.x2 = torch.randn(M, D2, device="cuda", generator=g) if D2 else None
        self.x3 = torch.randn(M, D2, device="cuda", generator=g) if x3 else None
        self.bar = torch.zeros(2, dtype=torch.int32, device="cuda")

    def run(self, bn=0, out=None, ln_out=None, sync=True):
        M, N = self.M, self.N
        out = _nan(M + 1, N) if out is None else out
        ln_out = _sentinel(M + 1, N + self.D2) if ln_out is None else ln_out
        kw = dict(kind=3, M=M, N=N, K=self.K, bn=bn, A=self.A, W16=self.W, bias=self.bias, resid=self.x0, out_f32=out, w=self.w, b=self.b,
                  shift=self.sh, scale=self.sc, ld_mod=self.mbs, rows_per_batch=self.rpb, x2=self.x2, x3=self.x3, D2=self.D2, ln_out=ln_out,
                  grid_barrier=self.bar)
        if self.gate is not None:
            kw.update(gate=self.gate[:, 2 * N:], gate_bstride=6 * N)
        if sync:
            a = _fold(**kw)
        else:
            from ezaudio_b200 import _lib
            rc, a = _fold_call(**kw)
            _lib.check(rc)
        return a, out, ln_out

    def check_gemm(self, out, tag):
        M, N = self.M, self.N
        assert bool(out[M].isnan().all()), f"{tag}: GEMM row M written"
        acc = self.A.double() @ self.W.double().t() + self.bias.double()
        S = self.A.double().abs() @ self.W.double().abs().t() + self.bias.double().abs()
        keep = 1 - self.gate[:, 2 * N:3 * N].double().repeat_interleave(self.gate_rpb, 0)[:M] if self.gate is not None else 1.0
        _check_f32(out[:M], self.x0.double() + keep * acc, keep.abs() * S + self.x0.double().abs() if self.gate is not None else S + self.x0.double().abs(), tag)

    def check_ln(self, out, ln_out, tag):
        """Bit-identical to the stand-alone kernel with the same arithmetic, and within the step-kernel LayerNorm bound."""
        from tests.test_step_kernels_gpu import GENERIC, REG1, _check_bf16, _ln_call, _ln_ref
        M, N = self.M, self.N
        assert bool((_bits(ln_out[M]) == _bits(_sentinel(1))[0]).all()), f"{tag}: LayerNorm row M written"
        x = out[:M]
        reg = self.x2 is None and N in (1024, 1152)
        alone = _ln_call(M, N, 1, REG1 if reg else GENERIC, x, x2=self.x2, x3=self.x3, D2=self.D2, w=self.w, b=self.b, sh=self.sh, sc=self.sc,
                         mbs=self.mbs, rpb=self.rpb)
        assert torch.equal(_bits(ln_out[:M]), _bits(alone)), f"{tag}: tail != stand-alone {'reg' if reg else 'generic'} LayerNorm"
        ref, slack = _ln_ref(x, self.x2, self.x3, w=self.w, b=self.b, tab=self.tab, mbs=self.mbs, rpb=self.rpb)
        e, q = _check_bf16(ln_out[:M], ref, slack, 1, tag)
        print(f"[tail] {tag}: LayerNorm max err {e:.3e}, {q:.2f} of the allowance")


@gpu
@pytest.mark.parametrize("N", [1152, 1024])
@pytest.mark.parametrize("bn", [0, 256, 288])
def test_ln_tail_register_widths(N, bn):
    """Widths 1152 / 1024 (ln_row_reg) with per-clip modulation after the gated-residual out-projection, clips of 250 rows."""
    t = Tail(1000, N, 1152, seed=N + bn, gate_rpb=250, mod_rpb=250)
    a, out, ln_out = t.run(bn=bn)
    tag = f"tail N {N} bn {bn}"
    assert a.ran_fused == 1 and a.ran_bn in (256, 288) and (bn == 0 or a.ran_bn == bn), (a.ran_fused, a.ran_bn)
    t.check_gemm(out, tag)
    t.check_ln(out, ln_out, tag)


@gpu
@pytest.mark.parametrize("M,N", [(1000, 768), (777, 144)])
def test_ln_tail_generic_width(M, N):
    """A width without a register variant (ln_row_generic), modulated per clip, with a ragged last tile."""
    t = Tail(M, N, 264, seed=M + N, mod_rpb=259)
    a, out, ln_out = t.run()
    assert a.ran_fused == 1
    t.check_gemm(out, f"tail generic M {M} N {N}")
    t.check_ln(out, ln_out, f"tail generic M {M} N {N}")


@gpu
@pytest.mark.parametrize("x3", [False, True])
def test_ln_tail_skip_concat(x3):
    """skip_norm over [x | skip (+ ControlNet skip)] after the skip linear (bias only): the generic branch with a second source."""
    t = Tail(1000, 1152, 2304, seed=7 + x3, D2=1152, x3=x3)
    a, out, ln_out = t.run()
    assert a.ran_fused == 1
    t.check_gemm(out, f"tail skip x3 {x3}")
    t.check_ln(out, ln_out, f"tail skip x3 {x3}")


@gpu
@pytest.mark.parametrize("bn", [256, 288])
def test_ln_tail_ragged_m(bn):
    t = Tail(777, 1024, 1152, seed=bn, gate_rpb=259, mod_rpb=259)
    a, out, ln_out = t.run(bn=bn)
    assert a.ran_fused == 1 and a.ran_bn == bn
    t.check_gemm(out, f"tail ragged bn {bn}")
    t.check_ln(out, ln_out, f"tail ragged bn {bn}")


@gpu
def test_ln_tail_one_wave_limit():
    """128 features (one feature tile): sms x 256 tokens is one full wave and runs the tail; one token more needs sms + 1 tiles, so the
    launch must run the GEMM alone, report fused = false, and leave the LayerNorm output holding its sentinel."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for M, fused in ((sms * 256, 1), (sms * 256 - 5, 1), (sms * 256 + 1, 0)):
        t = Tail(M, 128, 264, seed=M, mod_rpb=500)
        a, out, ln_out = t.run(bn=256)
        tag = f"tail M {M} ({sms} SMs)"
        assert a.ran_fused == fused and a.ran_bn == 256, (tag, a.ran_fused)
        t.check_gemm(out, tag)
        if fused:
            t.check_ln(out, ln_out, tag)
        else:
            assert bool((_bits(ln_out) == _bits(_sentinel(1))[0]).all()), f"{tag}: the fallback wrote the LayerNorm output"
        assert int(t.bar[0]) == 0 and int(t.bar[1]) == fused, (tag, t.bar.tolist())


@gpu
def test_ln_tail_barrier_reuse_and_graph_replay():
    """Two launches back to back on one GridBarrier, then a CUDA-graph capture of the launch and its replay: the same bits every time,
    the barrier's count back at 0 and its generation advanced once per executed launch."""
    t = Tail(1000, 1152, 1152, seed=11, gate_rpb=250, mod_rpb=250)
    _, out0, ln0 = t.run()
    t.check_gemm(out0, "tail reuse")
    t.check_ln(out0, ln0, "tail reuse")
    outs = [t.run(sync=False)[1:] for _ in range(2)]
    torch.cuda.synchronize()
    assert int(t.bar[0]) == 0 and int(t.bar[1]) == 3, t.bar.tolist()
    out_g, ln_g = _nan(1001, 1152), _sentinel(1001, 1152)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        t.run(out=out_g, ln_out=ln_g, sync=False)
    assert int(t.bar[1]) == 3, "capture executed the launch"
    graph.replay()
    torch.cuda.synchronize()
    assert int(t.bar[0]) == 0 and int(t.bar[1]) == 4, t.bar.tolist()
    for o, ln in outs + [(out_g, ln_g)]:
        assert torch.equal(_bits(o), _bits(out0)) and torch.equal(_bits(ln), _bits(ln0)), "a repeated launch differs"


# ------------------------------------------------------------------------------------------------------------------------------ validation
def test_fold_hook_rejects_bad_arguments():
    """Argument validation happens before any device work (this runs without a GPU)."""
    buf = (C.c_float * 64)()
    p = (C.addressof(buf) + 15) // 16 * 16

    def rc(base, **over):
        return _fold_call(on_stream=False, **{**base, **over})[0]

    tables = dict(kind=0, N=8, K=64, R=1, w=p, b=p, W=p, w_packed=p, G=p, Cc=p, u=p, v=p)
    assert rc(tables, K=2305) == EZB_ERR_UNSUPPORTED and rc(tables, K=2312) == EZB_ERR_UNSUPPORTED   # more than 72 x 32 columns
    assert rc(tables, K=60) == EZB_ERR_SHAPE
    assert rc(tables, kind=4) == EZB_ERR_ARG and rc(tables, kind=-1) == EZB_ERR_ARG
    assert rc(tables, w_packed=None) == EZB_ERR_ARG and rc(tables, u=None) == EZB_ERR_ARG
    assert rc(tables, shift=p) == EZB_ERR_ARG                                  # shift without scale
    assert rc(tables, R=3, shift=p, scale=p, ld_mod=32) == EZB_ERR_SHAPE       # modulation rows narrower than K
    assert rc(tables, R=0) == EZB_ERR_SHAPE and rc(tables, R=129) == EZB_ERR_SHAPE
    geglu = dict(tables, kind=1, M=4, inner=64, bias=p, A=p, st=p, slots=2, ld_st=4, out=p)
    assert rc(geglu, geglu_bn=256) == EZB_ERR_UNSUPPORTED                     # inner 64: no 256-wide tiles
    assert rc(geglu, geglu_bn=64) == EZB_ERR_ARG
    assert rc(geglu, inner=96) == EZB_ERR_SHAPE
    assert rc(geglu, ld_st=3) == EZB_ERR_SHAPE and rc(geglu, slots=0) == EZB_ERR_SHAPE
    assert rc(geglu, st=None) == EZB_ERR_ARG and rc(geglu, R=2) == EZB_ERR_ARG
    mlp = dict(geglu, kind=2, inner=128, W2=p, b2=p, x=p, fout_st=p, a0=p, g0=p, grid_barrier=p)
    assert rc(mlp, grid_barrier=None) == EZB_ERR_ARG
    assert rc(mlp, K=72) == EZB_ERR_SHAPE                                     # folded-out partials need whole 32-feature slots
    assert rc(mlp, gate=p, rows_per_batch=16) == EZB_ERR_SHAPE
    assert rc(mlp, variant=2) == EZB_ERR_ARG
    tail = dict(kind=3, M=4, N=128, K=64, A=p, W16=p, out_f32=p, ln_out=p, w=p, b=p, grid_barrier=p)
    assert rc(tail, bn=128) == EZB_ERR_ARG
    assert rc(tail, D2=4) == EZB_ERR_ARG and rc(tail, x3=p) == EZB_ERR_ARG   # x2 missing
    assert rc(tail, out_f32=p + 4) == EZB_ERR_ARG                             # LayerNorm input read as float4
    assert rc(tail, N=130) == EZB_ERR_SHAPE and rc(tail, K=60) == EZB_ERR_SHAPE
    assert rc(tail, gate=p, rows_per_batch=64) == EZB_ERR_ARG                 # a gate without a residual
    assert rc(tail, shift=p, scale=p, ld_mod=6, rows_per_batch=1) == EZB_ERR_ARG
    assert rc(tail, grid_barrier=None) == EZB_ERR_ARG
