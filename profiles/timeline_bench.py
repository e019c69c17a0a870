"""Timelines of prompts on the GPU: generate_timeline_audio against generate_long_audio of the same length, and the timeline kernels next
to the windowed ones they extend.

End to end: EzAudio-XL with synthetic weights, CFG 5 / rescale 0.75, 50 DDIM steps (eta 1), decode included, on one EzAudio(max_batch=10)
whose workspaces hold 10 s: a 60 s timeline of three 20 s segments (birds, traffic, rain; 1 s transitions) in 10 s windows with 2 s
overlap (8 windows, 11 conditioned rows + 8 unconditional rows = 19 DiT rows) against generate_long_audio(60) of one prompt (8 windows x 2 =
16 rows).  Host wall time around each call ending in a device synchronise; each configuration warmed once (graph capture), then timed
`--e2e-reps` times, alternating; the median is reported.
Kernels at the same 60 s plan (128 channels, windows of 500 frames): ezb_timeline_gather (19 rows) against ezb_window_gather (CFG, two
copies: 16 rows), ezb_timeline_guide (11 rows against 8 shared uncond rows, rescale 0.75) against the per-window guidance the linear loop
runs (ezb_cfg_ddim_step with coefficients (1, 0, 0, 1, 0) on 8 pairs), and ezb_timeline_blend (11 rows) against ezb_window_blend (8 rows).
CUDA events around `--launches` back-to-back launches, `--reps` times alternating, median.  One DiT forward at 16 .. 20 rows (L 500,
Lc 100; CUDA events around 10 forwards, `--reps` times, median) shows how the DiT's cost grows with its rows.
The card's name and power limit are read in the same run.  Prints one JSON line.
  python profiles/timeline_bench.py [--launches 200] [--reps 5] [--e2e-reps 3] [--out DIR]
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
from ezaudio_b200 import _lib, api  # noqa: E402
from ezaudio_b200.inference import _guide_windows, check_timeline  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--launches", type=int, default=200)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--e2e-reps", type=int, default=3)
ap.add_argument("--skip-e2e", action="store_true")
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "timeline_bench needs a GPU"

TIMELINE = [("birds at dawn in a forest", 0, 20), ("traffic builds up on a city street", 20, 40), ("rain on the street", 40, 60)]


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
    N, Lw, O, C, T, gs, gr = 3000, 500, 100, 128, 50, 5.0, 0.75
    segs = [[(s * 50, e * 50) for _, s, e in TIMELINE]]
    _, table, windows, rows, spans = check_timeline(segs, [N], 1, Lw, O, T, True, 64, Lw)
    W, R = len(windows), len(rows)
    dev = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    plan = dev([e for row in table for e in row])
    trows = dev([e for k, b, q in rows for e in (k, *segs[b][q], T)])
    tspans = dev([e for row in spans for e in row])
    rlens, wlens = dev([Lw] * R), dev([Lw] * W)
    lat = torch.randn(1, C, N, device="cuda")
    x_in = torch.randn(R + W, C, Lw, device="cuda")
    guided = torch.zeros(R, C, Lw, device="cuda")
    out = torch.empty(1, C, N, device="cuda")
    L, st = _lib.lib(), _lib.stream_ptr()
    fns = {"window_gather_cfg": lambda: _lib.check(L.ezb_window_gather(0, _lib.ptr(lat), _lib.ptr(x_in), _lib.ptr(plan), 1, C, N, W, Lw, O, 2, st)),
           "timeline_gather_cfg": lambda: _lib.check(L.ezb_timeline_gather(0, _lib.ptr(lat), _lib.ptr(x_in), _lib.ptr(plan), _lib.ptr(trows), 1, C, N,
                                                                           W, R, Lw, O, 1, st)),
           "guide_windows": lambda: _guide_windows(x_in, guided, W, C, Lw, gs, gr, wlens),
           "timeline_guide": lambda: _lib.check(L.ezb_timeline_guide(0, _lib.ptr(x_in), _lib.ptr(guided), _lib.ptr(trows), _lib.ptr(rlens), R, W, C,
                                                                      Lw, gs, gr, st)),
           "window_blend": lambda: _lib.check(L.ezb_window_blend(0, _lib.ptr(x_in), _lib.ptr(out), _lib.ptr(plan), 1, C, N, W, Lw, O, st)),
           "timeline_blend": lambda: _lib.check(L.ezb_timeline_blend(0, _lib.ptr(x_in), _lib.ptr(out), _lib.ptr(plan), _lib.ptr(trows), _lib.ptr(tspans),
                                                                     1, C, N, W, R, Lw, O, st))}
    for f in fns.values():
        event_ms(f, 10)
    ts = {k: [] for k in fns}
    for _ in range(a.reps):
        for k, f in fns.items():
            ts[k].append(event_ms(f, a.launches) * 1e3)
    res = {k: dict(us_per_launch=round(statistics.median(v), 2), min_us=round(min(v), 2), max_us=round(max(v), 2)) for k, v in ts.items()}
    res["shape"] = f"1 clip of {N} frames, C {C}, {W} windows of {Lw}, {R} timeline rows (T {T})"
    return res


name, power = card()
result = dict(gpu=name, power_limit_and_max_sm_clock=power)
result["kernels"] = kernel_times()
print(f"[kernels] {result['kernels']}", flush=True)
torch.cuda.empty_cache()

if not a.skip_e2e:
    enc = api.SyntheticTextEncoder(2048, 100)
    ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=10)
    kw = dict(window_length=10, overlap=2, guidance_scale=5, guidance_rescale=0.75, ddim_steps=50, eta=1, random_seed=2024)
    configs = {"generate_long_audio 60 s (16 rows)": lambda: ez.generate_long_audio(TIMELINE[0][0], length=60, **kw),
               "generate_timeline_audio 60 s, 3 segments (19 rows)": lambda: ez.generate_timeline_audio(TIMELINE, transition=1, **kw)}

    def run(f):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    dit = {}   # one DiT forward at the two plans' row counts (and neighbours), L 500, Lc 100: how the DiT's cost grows with its rows
    for rows in (16, 17, 18, 19, 20):
        x, ctx = torch.randn(rows, 128, 500, device="cuda"), torch.randn(rows, 100, 2048, device="cuda")
        out = torch.empty_like(x)
        ez.unet.set_context(ctx, torch.ones(rows, 100, dtype=torch.bool, device="cuda"))
        ez.unet.set_timesteps([999])
        fwd = lambda: ez.unet.forward_step(x, 0, out=out)   # noqa: E731
        event_ms(fwd, 3)
        dit[rows] = round(statistics.median(event_ms(fwd, 10) for _ in range(a.reps)), 3)
    result["dit_forward_ms_by_rows"] = dit
    print(f"[dit] {dit}", flush=True)
    for f in configs.values():
        run(f)   # graph capture, tensor maps
    times = {k: [] for k in configs}
    for _ in range(a.e2e_reps):
        for k, f in configs.items():
            times[k].append(run(f))
    result["e2e"] = dict(workload="EzAudio-XL synthetic weights, CFG 5 / rescale 0.75, 50 DDIM steps, incl. VAE decode, max_batch 10",
                         seconds={k: dict(median=round(statistics.median(v), 3), all=[round(x, 3) for x in v]) for k, v in times.items()})
    print(f"[e2e] {result['e2e']}", flush=True)

line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "timeline_bench.json"), "w") as f:
        f.write(line + "\n")
