"""Attention generations side by side: impl 1 (q / k rows of 128 elements) and 101 (80-element rows, the product's layout for dh = 72) of the
tensor-core test hook under each generation the options select (attention_mma.cuh / attention_wgmma.cuh), on the shapes of attn_bench.py.
CUDA events over back-to-back launches after a warm-up; the algorithmic FLOPs (4 Lq Lk dh per head) over the time, and as a share of the
dense bf16 data-sheet peak.  Prints the card, its power limit and its maximum SM clock first.
  python profiles/attn_gen_bench.py [generations, default 6,8]"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import _lib  # noqa: E402

L = _lib.lib()
PEAK = 989.0   # H100 SXM data sheet, dense bf16 TFLOP/s
OPTS = {4: {"attn6": 0}, 6: {"attn8": 0}, 7: {"attn7": 1}, 8: {}}
SHAPES = [(8, 16, 500, 500, 72, False, "self XL"), (8, 16, 500, 100, 72, True, "cross XL"), (4, 16, 1500, 1500, 72, False, "self XL 30s"),
          (16, 16, 500, 500, 72, False, "self XL C4"), (8, 16, 256, 256, 64, False, "self L")]


def run(B, H, Lq, Lk, dh, masked, impl, reps=50):
    dhp = 80 if (impl >= 100 and dh == 72) else (dh + 63) // 64 * 64
    dvp, lkp = (dh + 15) // 16 * 16, (Lk + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn(B * H, Lq, dhp, device="cuda", generator=g).bfloat16()
    k = torch.randn(B * H, Lk, dhp, device="cuda", generator=g).bfloat16()
    vt = torch.randn(B * H, dvp, lkp, device="cuda", generator=g).bfloat16()
    q[:, :, dh:] = 0
    k[:, :, dh:] = 0
    mask = None
    if masked:
        mask = torch.zeros(B, Lk, dtype=torch.uint8, device="cuda")
        mask[:, :20] = 1
    out = torch.empty(B, Lq, H * dh, device="cuda", dtype=torch.bfloat16)
    args = (0, _lib.ptr(q), _lib.ptr(k), _lib.ptr(vt), _lib.ptr(mask), _lib.ptr(out), B, H, Lq, Lk, dh, impl, _lib.stream_ptr())
    for _ in range(5):
        _lib.check(L.ezb_test_attention(*args))
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        L.ezb_test_attention(*args)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def main():
    gens = [int(x) for x in (sys.argv[1] if len(sys.argv) > 1 else "6,8").split(",")]
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", smi.stdout.strip() or torch.cuda.get_device_name(0))
    for impl in (1, 101):
        for B, H, Lq, Lk, dh, masked, label in SHAPES:
            for gen in gens:
                for name, val in OPTS[gen].items():
                    _lib.check(L.ezb_set_option(name.encode(), val))
                try:
                    ms = run(B, H, Lq, Lk, dh, masked, impl)
                finally:
                    _lib.check(L.ezb_set_option(b"attn6", 5))
                    _lib.check(L.ezb_set_option(b"attn7", 0))
                    _lib.check(L.ezb_set_option(b"attn8", 1))
                tf = 4.0 * B * H * Lq * Lk * dh / ms / 1e9
                print(f"{label:12s} impl {impl:3d} gen {gen}  B{B} H{H} Lq{Lq} Lk{Lk} dh{dh}: {ms * 1e3:7.1f} us  {tf:6.1f} TFLOP/s "
                      f"({tf / PEAK:.3f} of {PEAK:.0f})", flush=True)


if __name__ == "__main__":
    main()
