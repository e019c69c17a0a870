"""GEMM micro-benchmark through the C-ABI test hook: TFLOP/s per kernel variant on the DiT shapes, plus the cycle counters of CTA 0 of the
2-CTA cluster launches (gemm.cuh GemmShape::dbg; build with EZB_DEBUG=1 for them to count)."""
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
    geglu = kind in (1, 11)
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
