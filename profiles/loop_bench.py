"""Seamless loops on the GPU: generate_loop_audio against the linear calls of the same length, the circular window kernels next to the
linear ones, and the wrapped decode next to the tiled one.

End to end: EzAudio-XL with synthetic weights, one prompt, CFG 5 / rescale 0.75, 50 DDIM steps (eta 1), decode included, on an
EzAudio(max_batch=8) whose workspaces hold 10 s: generate_audio(10) against generate_loop_audio(10) (one window: the extra cost is the two
kernels per step and the decode's halo), and generate_long_audio(30) against generate_loop_audio(30) (10 s windows, 2 s overlap; 4 windows
each).  Host wall time around each call ending in a device synchronise; each configuration warmed once (graph capture), then timed
`--e2e-reps` times, alternating; the median is reported.
Kernels: ezb_loop_gather / ezb_window_gather (CFG, two copies) and ezb_loop_blend / ezb_window_blend at the 60 s plan (128 channels; 8
linear windows, 8 loop windows of 500 frames, offset 191), CUDA events around `--launches` back-to-back launches, `--reps` times, median.
Decode: decode_loop against decode_tiled of a 30 s latent on a 10 s workspace (max_batch 8), alternated `--reps` times (CUDA events).
The card's name and power limit are read in the same run.  Prints one JSON line.
  python profiles/loop_bench.py [--launches 200] [--reps 5] [--e2e-reps 3] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import _lib, api, synth, weights  # noqa: E402
from ezaudio_b200.inference import check_loop, long_plan  # noqa: E402
from ezaudio_b200.vae import OobleckDecoder  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--launches", type=int, default=200)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--e2e-reps", type=int, default=3)
ap.add_argument("--skip-e2e", action="store_true")
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "loop_bench needs a GPU"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "not reported"
    except (OSError, subprocess.SubprocessError):
        power = "not reported"
    return name, power


def event_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_times():
    N, Lw, O, C = 3000, 500, 100, 128
    lt, lw = long_plan([N], Lw, O)
    _, ct, cw = check_loop([N], 1, Lw, O, True, 64, Lw)
    Wl, Wc = len(lw), len(cw)
    plan_l = torch.tensor([e for row in lt for e in row], dtype=torch.int32, device="cuda")
    plan_c = torch.tensor([e for row in ct for e in row], dtype=torch.int32, device="cuda")
    offs = torch.tensor([191], dtype=torch.int32, device="cuda")
    lat = torch.randn(1, C, N, device="cuda")
    win = torch.randn(2 * max(Wl, Wc), C, Lw, device="cuda")
    out = torch.empty(1, C, N, device="cuda")
    L, st = _lib.lib(), _lib.stream_ptr()
    fns = {"window_gather_cfg": lambda: _lib.check(L.ezb_window_gather(0, _lib.ptr(lat), _lib.ptr(win), _lib.ptr(plan_l), 1, C, N, Wl, Lw, O, 2, st)),
           "loop_gather_cfg": lambda: _lib.check(L.ezb_loop_gather(0, _lib.ptr(lat), _lib.ptr(win), _lib.ptr(plan_c), _lib.ptr(offs), 1, C, N, Wc, Lw, O,
                                                                   2, st)),
           "window_blend": lambda: _lib.check(L.ezb_window_blend(0, _lib.ptr(win), _lib.ptr(out), _lib.ptr(plan_l), 1, C, N, Wl, Lw, O, st)),
           "loop_blend": lambda: _lib.check(L.ezb_loop_blend(0, _lib.ptr(win), _lib.ptr(out), _lib.ptr(plan_c), _lib.ptr(offs), 1, C, N, Wc, Lw, O, st))}
    for f in fns.values():
        event_ms(f, 10)
    ts = {k: [] for k in fns}
    for _ in range(a.reps):
        for k, f in fns.items():
            ts[k].append(event_ms(f, a.launches) * 1e3)
    res = {k: dict(us_per_launch=round(statistics.median(v), 2), min_us=round(min(v), 2), max_us=round(max(v), 2)) for k, v in ts.items()}
    res["shape"] = f"1 clip / loop of {N} frames, C {C}, windows of {Lw}: {Wl} linear, {Wc} circular"
    return res


def decode_times():
    dcfg = synth.VAE_DECODER
    sd = weights.synthetic_state_dict(weights.vae_decoder_param_shapes(dcfg), 6)
    dec = OobleckDecoder(precision="bf16", max_batch=8, max_latent_len=500, **dcfg).load_state_dict(sd)
    z = synth.synth_latents(1, 1500, seed=3).cuda()
    fns = {"decode_loop_30s": lambda: dec.decode_loop(z), "decode_tiled_30s": lambda: dec.decode_tiled(z)}
    for f in fns.values():
        event_ms(f, 2)
    ts = {k: [] for k in fns}
    for _ in range(a.reps):
        for k, f in fns.items():
            ts[k].append(event_ms(f, 3))
    out = {k: dict(ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3)) for k, v in ts.items()}
    out["clip"] = "1 x 30 s (1500 latent frames), bf16, 10 s workspace, max_batch 8"
    return out


name, power = card()
result = dict(gpu=name, power_limit_and_max_sm_clock=power)
result["kernels"] = kernel_times()
print(f"[kernels] {result['kernels']}", flush=True)
result["decode"] = decode_times()
print(f"[decode] {result['decode']}", flush=True)
torch.cuda.empty_cache()

if not a.skip_e2e:
    enc = api.SyntheticTextEncoder(2048, 100)
    ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=8)
    prompt = "steady rain on a tin roof"
    kw = dict(guidance_scale=5, guidance_rescale=0.75, ddim_steps=50, eta=1, random_seed=2024)
    configs = {"generate_audio 10 s": lambda: ez.generate_audio(prompt, length=10, **kw),
               "generate_loop_audio 10 s": lambda: ez.generate_loop_audio(prompt, length=10, window_length=10, overlap=2, **kw),
               "generate_long_audio 30 s": lambda: ez.generate_long_audio(prompt, length=30, window_length=10, overlap=2, **kw),
               "generate_loop_audio 30 s": lambda: ez.generate_loop_audio(prompt, length=30, window_length=10, overlap=2, **kw)}

    def run(f):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for f in configs.values():
        run(f)   # graph capture, tensor maps
    times = {k: [] for k in configs}
    for _ in range(a.e2e_reps):
        for k, f in configs.items():
            times[k].append(run(f))
    result["e2e"] = dict(workload="EzAudio-XL synthetic weights, 1 prompt, CFG 5 / rescale 0.75, 50 DDIM steps, incl. VAE decode",
                         seconds={k: dict(median=round(statistics.median(v), 3), all=[round(x, 3) for x in v]) for k, v in times.items()})
    print(f"[e2e] {result['e2e']}", flush=True)

line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "loop_bench.json"), "w") as f:
        f.write(line + "\n")
