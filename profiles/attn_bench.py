"""Attention micro-benchmark through the C-ABI test hook (attention_mma.cuh variants, q / k row pitch 128 vs 80 elements for dh = 72).  CUDA events
over 20 back-to-back launches; the algorithmic FLOPs (4 Lq Lk dh per head) are also given as a share of the dense bf16 tensor peak.
  python profiles/attn_bench.py [res_poly_pp_bits] [attn6] [attn7]        # no arguments: the product's default variant"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import _lib  # noqa: E402

L = _lib.lib()
PEAK = float(os.environ.get("PEAK_TFLOPS", 989.0))   # H100 SXM data sheet, dense bf16
print(torch.cuda.get_device_name(0))


def run(B, H, Lq, Lk, dh, masked, label, impl, reps=20):
    dhp = (dh + 63) // 64 * 64
    if impl >= 100 and dh == 72:
        dhp = 80
    dvp, lkp = (dh + 15) // 16 * 16, (Lk + 7) // 8 * 8
    q = torch.randn(B * H, Lq, dhp, device="cuda").bfloat16()
    k = torch.randn(B * H, Lk, dhp, device="cuda").bfloat16()
    vt = torch.randn(B * H, dvp, lkp, device="cuda").bfloat16()
    q[:, :, dh:] = 0
    k[:, :, dh:] = 0
    mask = None
    if masked:
        mask = torch.zeros(B, Lk, dtype=torch.uint8, device="cuda")
        mask[:, :20] = 1
    out = torch.empty(B, Lq, H * dh, device="cuda", dtype=torch.bfloat16)
    args = (0, _lib.ptr(q), _lib.ptr(k), _lib.ptr(vt), _lib.ptr(mask), _lib.ptr(out), B, H, Lq, Lk, dh, impl, _lib.stream_ptr())
    for _ in range(3):
        _lib.check(L.ezb_test_attention(*args))
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        L.ezb_test_attention(*args)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / reps
    fl = 4.0 * B * H * Lq * Lk * dh
    print(f"{label:14s} impl {impl:3d} B{B} H{H} Lq{Lq} Lk{Lk} dh{dh}: {ms * 1e3:7.1f} us  {fl / ms / 1e9:6.1f} TFLOP/s "
          f"({fl / ms / 1e9 / PEAK:.3f} of {PEAK:.0f})")


MMA2 = int(sys.argv[1]) if len(sys.argv) > 1 else 0
L.ezb_set_option(b"attn_res", (MMA2 >> 1) & 1)
L.ezb_set_option(b"attn_poly", (MMA2 >> 2) & 1)
L.ezb_set_option(b"attn_pp", (MMA2 >> 3) & 1)
A6 = int(sys.argv[2]) if len(sys.argv) > 2 else 5   # bit 0 generation 6 (else 4), +2 FMA-pipe exp2 on odd warps, +4 P V after each half block
L.ezb_set_option(b"attn6", A6)
A7 = int(sys.argv[3]) if len(sys.argv) > 3 else 0   # generation 7: 128-key blocks
L.ezb_set_option(b"attn7", A7)
print("attn6 =", A6, "attn7 =", A7)
print("attn_res =", (MMA2 >> 1) & 1, "attn_poly =", (MMA2 >> 2) & 1, "attn_pp =", (MMA2 >> 3) & 1)
for impl in (1, 101):
    run(8, 16, 500, 500, 72, False, "self XL", impl)
    run(8, 16, 500, 100, 72, True, "cross XL", impl)
    run(4, 16, 1500, 1500, 72, False, "self XL 30s", impl)
    run(16, 16, 500, 500, 72, False, "self XL C4", impl)
    if impl < 100:
        run(8, 16, 256, 256, 64, False, "self L", impl)
