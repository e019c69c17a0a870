"""DPM-Solver++ against DDIM on the GPU: the fused update kernels, and generate_audio end to end.

Kernel time: ezb_cfg_dpm_step (2M, order 2) against ezb_cfg_ddim_step (eta 1) at B = 4, C = 128, L = 500 and 1500 with CFG 5 / rescale 0.75,
CUDA events around `--launches` back-to-back launches, the two kernels alternated `--reps` times in this one process; the median per launch
is reported, with the bytes each kernel moves (compulsory DRAM traffic, from the shapes) over that time.
End to end: EzAudio-XL with synthetic weights, `--prompts` prompts x 10 s, generate_audio with 25 DPM-Solver++ 2M steps against 50 and 100
DDIM steps (guidance 5, rescale 0.75, eta 1 for DDIM), host wall time around the call ending in a device synchronise, each configuration
warmed once (graph capture) and then timed `--e2e-reps` times, alternating.  The card's name and power limit are read in the same run.
Prints one JSON line.
  python profiles/dpm_bench.py [--launches 200] [--reps 10] [--prompts 4] [--e2e-reps 3] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import _lib, api  # noqa: E402
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--launches", type=int, default=200)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--prompts", type=int, default=4)
ap.add_argument("--e2e-reps", type=int, default=3)
ap.add_argument("--skip-e2e", action="store_true")
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "dpm_bench needs a GPU"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "not reported"
    except (OSError, subprocess.SubprocessError):
        power = "not reported"
    return name, power


def kernel_times(L, B=4, Cc=128, gs=5.0, gr=0.75):
    L_ = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(L)
    mo = torch.randn(2 * B, Cc, L, device="cuda", generator=g)
    lat = torch.randn(B, Cc, L, device="cuda", generator=g)
    hist = torch.randn(B, Cc, L, device="cuda", generator=g)
    noise = torch.randn(B, Cc, L, device="cuda", generator=g)
    d = DDIMScheduler()
    d.set_timesteps(50)
    dcoef = (C.c_float * 5)(*d.step_coefficients(int(d.timesteps[20]), 1.0))
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(25)
    c, order = s.step_coefficients(10)
    pcoef = (C.c_float * 7)(*c)
    st = _lib.stream_ptr()

    def ddim():
        _lib.check(L_.ezb_cfg_ddim_step(0, _lib.ptr(mo), _lib.ptr(lat), _lib.ptr(noise), B, Cc, L, gs, gr, dcoef, st, None))

    def dpm():
        _lib.check(L_.ezb_cfg_dpm_step(0, _lib.ptr(mo), _lib.ptr(lat), _lib.ptr(hist), None, B, Cc, L, gs, gr, pcoef, order, st, None))

    res = {"ddim": [], "dpm": []}
    for f in (ddim, dpm):   # warm-up: module load, attributes
        for _ in range(20):
            f()
    torch.cuda.synchronize()
    for _ in range(a.reps):
        for name, f in (("ddim", ddim), ("dpm", dpm)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                f()
            e1.record()
            e1.synchronize()
            res[name].append(e0.elapsed_time(e1) * 1e3 / a.launches)
        lat.normal_(generator=g)   # keep the values in range
    n = B * Cc * L * 4
    # compulsory bytes: DDIM reads text + uncond + latents + noise, writes latents; DPM 2M reads text + uncond + latents + history and writes
    # latents + history (rescale reads text + uncond a second time; counted once, as L2 may serve it)
    bytes_ = {"ddim": 5 * n, "dpm": 6 * n}
    out = {}
    for k, v in res.items():
        med = statistics.median(v)
        out[k] = dict(us_per_launch=round(med, 2), min_us=round(min(v), 2), max_us=round(max(v), 2), gbytes_per_s=round(bytes_[k] / med / 1e3, 1))
    return out


name, power = card()
result = dict(gpu=name, power_limit_and_max_sm_clock=power, kernel={})
for L in (500, 1500):
    result["kernel"][f"B4_C128_L{L}"] = kernel_times(L)
    print(f"[kernel] L={L}: {result['kernel'][f'B4_C128_L{L}']}", flush=True)

if not a.skip_e2e:
    enc = api.SyntheticTextEncoder(2048, 100)
    ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=a.prompts)
    prompts = [f"prompt {i}: rain and a distant dog" for i in range(a.prompts)]
    ddim = ez.noise_scheduler
    dpm = DPMSolverMultistepScheduler(**ez.params["diff"])
    configs = [("dpmsolver++ 2M, 25 steps", dpm, 25), ("DDIM, 50 steps", ddim, 50), ("DDIM, 100 steps", ddim, 100)]

    def run(sched, steps):
        ez.noise_scheduler = sched
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ez.generate_audio(prompts, length=10, guidance_scale=5, guidance_rescale=0.75, ddim_steps=steps, eta=1, random_seed=2024)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for _, sched, steps in configs:
        run(sched, steps)   # graph capture, tensor maps
    times = {label: [] for label, _, _ in configs}
    for _ in range(a.e2e_reps):
        for label, sched, steps in configs:
            times[label].append(run(sched, steps))
    ez.noise_scheduler = ddim
    result["e2e"] = dict(workload=f"EzAudio-XL synthetic weights, {a.prompts} prompts x 10 s, CFG 5 / rescale 0.75, generate_audio incl. VAE decode",
                         seconds={k: dict(median=round(statistics.median(v), 3), all=[round(x, 3) for x in v]) for k, v in times.items()})
    print(f"[e2e] {result['e2e']}", flush=True)

line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "dpm_bench.json"), "w") as f:
        f.write(line + "\n")
