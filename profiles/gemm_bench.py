"""GEMM micro-benchmark through the C-ABI test hooks: TFLOP/s per kernel variant on the DiT shapes, plus the cycle counters of CTA 0 of the
2-CTA cluster launches (gemm.cuh GemmShape::dbg; build with EZB_DEBUG=1 for them to count).
  python profiles/gemm_bench.py                  # both sections
  python profiles/gemm_bench.py heads            # only the fused Q/K/V-heads GEMMs (ezb_test_heads), or `linear` for the others
  python profiles/gemm_bench.py m=4000,8000      # only the DiT block's GEGLU / MLP-out / QKV / cross-Q GEMMs and their alternatives, per M"""
import ctypes as C
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import _lib  # noqa: E402

L = _lib.lib()
L.ezb_set_option(b"gemm_debug", 1)


def run(M, N, K, bn, kind, label, resid=False, reps=20):
    A = torch.randn(M, K, device="cuda").bfloat16()
    W = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda")
    e = _lib.TestEpilogue()
    e.bias = bias.data_ptr()
    geglu = kind in (1, 11, 12)
    if geglu:
        out = torch.empty(M, N // 2, device="cuda", dtype=torch.bfloat16)
        e.out_bf16, e.ld16 = out.data_ptr(), N // 2
    elif resid:
        x = torch.randn(M, N, device="cuda")
        gate = torch.randn(8, N, device="cuda")
        e.resid, e.ldr, e.gate, e.gate_bstride, e.rows_per_batch = x.data_ptr(), N, gate.data_ptr(), N, (M + 7) // 8
        e.out_f32, e.ld32 = x.data_ptr(), N
    else:
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        e.out_bf16, e.ld16 = out.data_ptr(), N
    st = _lib.stream_ptr()
    args = (0, _lib.ptr(A), K, _lib.ptr(W), K, M, N, K, bn, kind, C.byref(e), 0, 0, 0, 0, 0, 0, st)
    for _ in range(3):
        _lib.check(L.ezb_test_gemm(*args))
    dbg = (C.c_ulonglong * 8)()
    L.ezb_debug_read(dbg)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        L.ezb_test_gemm(*args)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / reps
    L.ezb_debug_read(dbg)
    d = [v / reps for v in dbg[:6]]
    tf = 2.0 * M * N * K / ms / 1e9
    print(f"{label:34s} M{M} N{N} K{K} bn{bn}: {ms * 1e3:7.1f} us  {tf:7.1f} TF/s | cta0 cycles: total {d[5]:.0f} mainloop {d[0]:.0f} "
          f"acc_wait {d[1]:.0f} prod_wait_empty {d[2]:.0f} epi_busy {d[4]:.0f}")


# heads_gemm variants (csrc/host.cuh HeadsVariant)
PACKED3, PACKED3_PARKED, PAIR, PAIR_PARKED, SINGLE = 0, 1, 3, 4, 5
HEADS_NAMES = {PACKED3: "packed-3", PACKED3_PARKED: "packed-3 parked", PAIR: "pair-2", PAIR_PARKED: "pair-2 parked", SINGLE: "single-CTA"}


def heads(B, Lt, H, dh, nsec, variant, label, reps=20):
    """One heads_gemm launch per ezb_test_heads call (the hook also packs W and synchronises, so the timing uses the per-launch CUDA events the
    GEMM launchers record around the kernel alone: ezb_prof_gemm_*).  FLOPs: 2 M N D with N = nsec D -- the zero pad columns of the packed
    tiles are not counted.  RoPE is the model's default (MUFU)."""
    D, M = H * dh, B * Lt
    g = torch.Generator(device="cuda").manual_seed(1)
    A = torch.randn(M, D, device="cuda", generator=g).bfloat16()
    W = torch.randn(nsec * D, D, device="cuda", generator=g) / math.sqrt(D)
    norm = torch.stack([torch.ones(dh, device="cuda"), torch.zeros(dh, device="cuda")]).contiguous()
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dh, 2, device="cuda", dtype=torch.float32) / dh))
    kinds = (0, 1, 2) if nsec == 3 else (0,)
    ld_qk, dvp, Lpad = (80 if dh == 72 else 64), (dh + 15) // 16 * 16, (Lt + 7) // 8 * 8
    q = torch.empty(B * H, Lt, ld_qk, device="cuda", dtype=torch.bfloat16)
    k = torch.empty_like(q)
    vt = torch.empty(B * H, dvp, Lpad, device="cuda", dtype=torch.bfloat16)
    a = _lib.TestHeadsArgs()
    a.B, a.L, a.D, a.H, a.dh, a.nsec = B, Lt, D, H, dh, nsec
    for i, kd in enumerate(kinds):
        a.kinds[i] = kd
    a.norm_q = a.norm_k = norm.data_ptr()
    a.inv_freq, a.rope = inv_freq.data_ptr(), 2 if nsec == 3 else 0
    a.q, a.k, a.vt = q.data_ptr(), k.data_ptr(), vt.data_ptr()
    a.ld_qk, a.dvp, a.Lpad, a.variant = ld_qk, dvp, Lpad, variant
    st = _lib.stream_ptr()
    for _ in range(3):
        _lib.check(L.ezb_test_heads(0, _lib.ptr(A), _lib.ptr(W), C.byref(a), st))
    dbg = (C.c_ulonglong * 8)()
    L.ezb_debug_read(dbg)
    _lib.check(L.ezb_prof_gemm_begin())
    for _ in range(reps):
        _lib.check(L.ezb_test_heads(0, _lib.ptr(A), _lib.ptr(W), C.byref(a), st))
    n, ms = C.c_int(0), C.c_double(0.0)
    _lib.check(L.ezb_prof_gemm_end(C.byref(n), None, C.byref(ms)))
    assert n.value == reps, n.value
    L.ezb_debug_read(dbg)
    us = ms.value / reps * 1e3
    tf = 2.0 * M * nsec * D * D / us / 1e6
    line = f"{label:24s} {HEADS_NAMES[variant]:22s} M{M} N{nsec * D} K{D}: {us:7.1f} us  {tf:6.1f} TF/s"
    d = [v / reps for v in dbg[:6]]
    if any(d):   # EZB_DEBUG=1 build
        line += (f" | cta0 cycles: total {d[5]:.0f} mainloop {d[0]:.0f} acc_wait {d[1]:.0f} prod_wait_empty {d[2]:.0f} epi_busy {d[4]:.0f}")
    print(line, flush=True)


SECTIONS = [a for a in sys.argv[1:] if a in ("linear", "heads")] or ["linear", "heads"]
# m=4000,8000: token counts of XL at Be = 8 and 16, L = 500; each block GEMM next to the alternatives its runtime options select
MS = next((list(map(int, a[2:].split(","))) for a in sys.argv[1:] if a.startswith("m=")), None)
if MS is not None:
    if "linear" in SECTIONS:
        for M in MS:
            run(M, 9216, 1152, 256, 11, "pair geglu 256")
            run(M, 9216, 1152, 256, 12, "pair geglu 256 parked")
            run(M, 1152, 4608, 256, 20, "swapAB mlp2 resid+gate", resid=True)
            run(M, 1152, 4608, 128, 10, "pair mlp2 resid+gate 128", resid=True)
    if "heads" in SECTIONS:
        for M in MS:
            heads(M // 500, 500, 16, 72, 3, PACKED3, "XL self-QKV")
            heads(M // 500, 500, 16, 72, 3, PACKED3_PARKED, "XL self-QKV")
            heads(M // 500, 500, 16, 72, 1, PAIR, "XL cross-Q")
            heads(M // 500, 500, 16, 72, 1, SINGLE, "XL cross-Q")
    SECTIONS = []
if "linear" in SECTIONS:
    M = 4000
    run(M, 9216, 1152, 256, 11, "pair geglu 256")
    run(M, 9216, 1152, 256, 10, "pair linear-bf16 256")
    run(M, 9216, 1152, 128, 10, "pair linear-bf16 128")
    run(M, 9216, 1152, 128, 0, "1cta linear-bf16 128")
    run(M, 9216, 1152, 256, 0, "1cta linear-bf16 256")
    run(M, 1152, 1152, 128, 10, "pair proj bf16 128")
    run(M, 1152, 1152, 128, 10, "pair proj resid+gate 128", resid=True)
    run(M, 1152, 4608, 128, 10, "pair mlp2 resid+gate 128", resid=True)
    run(M, 1152, 4608, 128, 0, "1cta mlp2 resid+gate 128", resid=True)
    run(M, 1152, 1152, 256, 20, "swapAB proj resid+gate", resid=True)
    run(M, 1152, 4608, 256, 20, "swapAB mlp2 resid+gate", resid=True)
    run(M, 1152, 2304, 256, 20, "swapAB skip resid", resid=True)
    run(8192, 8192, 8192, 256, 10, "pair 8192^3 bf16 256", reps=5)
    run(8192, 8192, 8192, 128, 0, "1cta 8192^3 bf16 128", reps=5)
if "heads" in SECTIONS:
    for B in (8, 16):   # XL self-attention QKV (Be = 8 / 16, L = 500)
        for v in (PACKED3, PACKED3_PARKED, PAIR, PAIR_PARKED, SINGLE):
            heads(B, 500, 16, 72, 3, v, "XL self-QKV")
    for v in (PAIR, PAIR_PARKED, SINGLE):
        heads(8, 500, 16, 72, 1, v, "XL cross-Q")
    for v in (PACKED3, PACKED3_PARKED, PAIR, PAIR_PARKED, SINGLE):   # EzAudio-L: D = 1024, dh = 64
        heads(8, 500, 16, 64, 3, v, "L self-QKV")
    for v in (PAIR, PAIR_PARKED, SINGLE):
        heads(8, 500, 16, 64, 1, v, "L cross-Q")
