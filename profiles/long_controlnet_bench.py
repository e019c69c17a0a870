"""Long ControlNet clips on the GPU: EzAudio_ControlNet.generate_long_audio against generate_audio, and the ControlNet forward on the
condition cache against the forward that runs the stem.

EzAudio-XL + energy ControlNet with synthetic weights and the synthetic text encoder, one process:
  * Forward: ezb_controlnet_forward (the stem's four convolutions, then the trunk) against ezb_controlnet_forward_cached (the trunk on
    the condition cache) at effective batch 16, L 500, Lc 100, one timestep for the batch, scale 1: the shape of a 60 s reference in 10 s
    windows with 2 s overlap under CFG (8 windows x 2).  CUDA events over `--iters` calls, the two alternated `--reps` times; medians.
    Both outputs are compared bit for bit.  Their difference, times the step count, is what caching the stem saves a windowed call.
  * End to end: one prompt, CFG 3.5, 50 DDIM steps (eta 1), decode included, host wall time around each call ending in a device
    synchronise: generate_long_audio on 30 s and 60 s references (10 s windows, 2 s overlap, max_batch 8) against generate_audio on a 10 s
    reference, on one EzAudio_ControlNet.  Each configuration is warmed once (graph capture), then timed `--e2e-reps` times, alternated.
The card's name and power limit are read in the same run.  Prints one JSON line.
  python profiles/long_controlnet_bench.py [--iters 30] [--reps 5] [--e2e-reps 3] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import api, config, synth, weights  # noqa: E402
from ezaudio_b200.dit import DiTControlNet  # noqa: E402
from ezaudio_b200.scheduler import DDIMScheduler  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=30)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--e2e-reps", type=int, default=3)
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "long_controlnet_bench needs a GPU"
STEPS = 50


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


def forward_bench():
    cfg, cn = synth.model_cfg("xl"), synth.CONTROLNET
    Be, L, Lc = 16, 500, 100
    sd_cn = weights.synthetic_state_dict(weights.controlnet_param_shapes(cfg, cn), 3)
    net = DiTControlNet(precision="bf16", max_batch=Be, max_len=L, max_ctx_len=Lc, max_timesteps=1000, **cfg, **cn)
    net.load_state_dict(sd_cn, mask_embed=torch.zeros(cfg["out_chans"]))
    del sd_cn
    ctx, mask = synth.synth_context(Be, Lc, cfg["context_dim"])
    net.set_context(ctx.cuda(), mask.cuda())
    s = DDIMScheduler()
    s.set_timesteps(STEPS)
    net.set_timesteps([int(t) for t in s.timesteps])
    x = synth.synth_latents(Be, L).cuda()
    cond = torch.rand(Be, 1, 2 * L, generator=torch.Generator().manual_seed(9)).cuda()
    net.set_condition(cond)
    outs = {k: [torch.empty(Be, L, cfg["embed_dim"], device="cuda") for _ in range(net.half)] for k in ("stem", "cached")}
    paths = {"ezb_controlnet_forward": lambda: net.forward_step(x, 7, cond, 1.0, outs=outs["stem"]),
             "ezb_controlnet_forward_cached": lambda: net.forward_step(x, 7, conditioning_scale=1.0, outs=outs["cached"])}
    for f in paths.values():   # warm-up: tensor maps, function attributes
        event_ms(f, 3)
    torch.cuda.synchronize()
    same = all(torch.equal(p.view(torch.int32), q.view(torch.int32)) for p, q in zip(outs["stem"], outs["cached"]))
    ts = {k: [] for k in paths}
    for _ in range(a.reps):
        for k, f in paths.items():
            ts[k].append(event_ms(f, a.iters))
    res = {k: dict(ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3)) for k, v in ts.items()}
    saved = res["ezb_controlnet_forward"]["ms"] - res["ezb_controlnet_forward_cached"]["ms"]
    res["saved_ms_per_step"] = round(saved, 3)
    res["saved_ms_per_50_step_call"] = round(STEPS * saved, 1)
    res["bit_identical"] = bool(same)
    res["shape"] = f"XL bf16, Be {Be}, L {L}, Lc {Lc}, one timestep, scale 1"
    del net
    torch.cuda.empty_cache()
    return res


def clip(seconds, seed):
    """Noise bursts with a slow loudness contour, so the energy condition varies along the clip."""
    rng = np.random.default_rng(seed)
    n = int(seconds * 24000)
    env = np.abs(np.sin(np.linspace(0, seconds * np.pi / 2.5, n))) + 0.05
    return (0.3 * env * rng.standard_normal(n)).astype(np.float32)


def e2e_bench():
    params = dict(config.BUILTIN_CONTROLNET["energy"], model_name="EzAudio-XL", model=synth.XL_MODEL,
                  text_encoder=dict(model="google/flan-t5-xl", max_length=100, cfg=0.1))
    cn = api.EzAudio_ControlNet("energy", ckpt_path="synthetic:2", controlnet_path="synthetic:3", vae_path="synthetic:6",
                                text_encoder=api.SyntheticTextEncoder(2048, 100), max_batch=8, params=params)
    prompt = "footsteps on gravel"
    kw = dict(guidance_scale=3.5, guidance_rescale=0, ddim_steps=STEPS, eta=1, random_seed=2024)
    refs = {s: clip(s, s) for s in (10, 30, 60)}
    configs = {"generate_audio 10 s": lambda: cn.generate_audio(prompt, refs[10], **kw),
               "generate_long_audio 30 s": lambda: cn.generate_long_audio(prompt, refs[30], window_length=10, overlap=2, **kw),
               "generate_long_audio 60 s": lambda: cn.generate_long_audio(prompt, refs[60], window_length=10, overlap=2, **kw)}

    def run(f):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, w = f()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, w

    shapes = {}
    for k, f in configs.items():
        _, w = run(f)   # graph capture, tensor maps
        shapes[k] = dict(samples=int(w.shape[0]), finite=bool(np.isfinite(w).all()))
    times = {k: [] for k in configs}
    for _ in range(a.e2e_reps):
        for k, f in configs.items():
            times[k].append(run(f)[0])
    return dict(workload="EzAudio-XL + energy ControlNet, synthetic weights, 1 prompt, CFG 3.5, 50 DDIM steps (eta 1), incl. VAE decode; "
                         "long calls in 10 s windows with 2 s overlap on max_batch 8",
                outputs=shapes,
                seconds={k: dict(median=round(statistics.median(v), 3), all=[round(x, 3) for x in v]) for k, v in times.items()})


name, power = card()
result = dict(gpu=name, power_limit_and_max_sm_clock=power)
result["forward"] = forward_bench()
print(f"[forward] {result['forward']}", flush=True)
result["e2e"] = e2e_bench()
print(f"[e2e] {result['e2e']}", flush=True)
line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "long_controlnet_bench.json"), "w") as f:
        f.write(line + "\n")
