"""ControlNet serving: the cached stem per step, and a mixed request trace, sequential generate_audio calls against the continuous engine.

EzAudio-XL + energy ControlNet with synthetic weights and cached (synthetic) text embeddings, in one process:
  * `ControlNet.forward` at the C4 shape (effective batch 16, L 500, Lc 100), CUDA events over `--iters` calls each, the three paths
    alternated: ezb_controlnet_forward with one timestep for the batch (what generate_audio runs; it may take the folded-LayerNorm kernels),
    ezb_controlnet_forward with per-sample host indices (the same trunk kernels as the device-index path), and ezb_controlnet_forward_tdev
    on the cached stem.  The difference of the last two is what caching the stem saves per step.
  * A seeded trace of `--requests` ControlNet requests with Poisson arrivals (mean gap `--gap` s): each its own reference clip (1-12 s of
    noise bursts), conditioning scale 0.5 or 1, guidance 3.5 or 5, 25 or 50 steps, eta 0 or 1.  It is replayed in real time against
    sequential EzAudio_ControlNet.generate_audio calls (one request per call, in arrival order: the only way to serve them before the engine)
    and against engine.ContinuousEngine with 4 slots, alternated, `--rounds` times each after one untimed warm-up pass each.  Reported per
    path: latency p50 / p95 (arrival to waveform on the host), audio seconds per wall second (10 s per request over first arrival to last
    waveform) and the host time per denoising step spent outside the CUDA-graph replay and event waits.
The card's name and power limit are read in the same run.  Prints one JSON line.
  python profiles/controlnet_engine_bench.py [--requests 8] [--gap 1.0] [--rounds 2] [--iters 50] [--seed 0] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import api, config, engine, inference, synth, weights  # noqa: E402
from ezaudio_b200.dit import DiTControlNet  # noqa: E402
from ezaudio_b200.frontend import ControlRequest  # noqa: E402
from ezaudio_b200.scheduler import DDIMScheduler  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=8)
ap.add_argument("--gap", type=float, default=1.0, help="mean inter-arrival time (s)")
ap.add_argument("--rounds", type=int, default=2)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "controlnet_engine_bench needs a GPU"
SLOTS = 4


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "not reported"
    except (OSError, subprocess.SubprocessError):
        power = "not reported"
    return name, power


# ---------------------------------------------------------------- 1. the ControlNet forward at the C4 shape
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
    s.set_timesteps(50)
    net.set_timesteps([int(t) for t in s.timesteps])
    x = synth.synth_latents(Be, L).cuda()
    cond = torch.rand(Be, 1, 2 * L, generator=torch.Generator().manual_seed(9)).cuda()
    net.set_condition(cond)
    outs = [torch.empty(Be, L, cfg["embed_dim"], device="cuda") for _ in range(net.half)]
    rows = [(7 + b) % 50 for b in range(Be)]
    tix = torch.tensor(rows, dtype=torch.int32, device="cuda")
    scale = torch.ones(Be, device="cuda")
    paths = {"uniform_host_index": lambda: net._run(x, None, None, None, 7, cond, 1.0, outs),
             "per_sample_host_index": lambda: net._run(x, None, None, (C.c_int32 * Be)(*rows), 0, cond, 1.0, outs),
             "device_index_cached_stem": lambda: net.forward_step(x, t_index=tix, scale=scale, outs=outs)}
    for f in paths.values():   # warm-up: tensor maps, function attributes
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in paths}
    for _ in range(3):   # alternated blocks
        for k, f in paths.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                f()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / a.iters)
    del net, outs
    torch.cuda.empty_cache()
    res = {k: dict(ms_per_forward=round(float(np.median(v)), 4), blocks=[round(t, 4) for t in v]) for k, v in times.items()}
    res["stem_saving_ms"] = round(res["per_sample_host_index"]["ms_per_forward"] - res["device_index_cached_stem"]["ms_per_forward"], 4)
    return res


# ---------------------------------------------------------------- 2. the request trace
class HostClock:
    """Host time of per-step work outside CUDA-graph replays and event waits (see profiles/continuous_bench.py)."""

    def __init__(self):
        self.excl, self.replays, self.host_s, self.steps = 0.0, 0, 0.0, 0
        clock = self
        for cls, name in ((torch.cuda.CUDAGraph, "replay"), (torch.cuda.Event, "synchronize")):
            orig = getattr(cls, name)

            def timed(self_, *args, _orig=orig, _replay=name == "replay", **kw):
                t0 = time.perf_counter()
                r = _orig(self_, *args, **kw)
                clock.excl += time.perf_counter() - t0
                clock.replays += _replay
                return r
            setattr(cls, name, timed)

    def wrap(self, owner, name, steps):
        orig = getattr(owner, name)
        clock = self

        def timed(*args, **kw):
            e0, r0 = clock.excl, clock.replays
            t0 = time.perf_counter()
            r = orig(*args, **kw)
            dt = time.perf_counter() - t0 - (clock.excl - e0)
            if clock.replays > r0:
                clock.host_s += dt
                clock.steps += steps(args, kw)
            return r
        setattr(owner, name, timed)

    def take(self):
        v = (1e3 * self.host_s / self.steps) if self.steps else None
        self.host_s, self.steps = 0.0, 0
        return v


def reference_clip(rng, seconds):
    """Noise bursts with a slow envelope: something for the energy condition to follow."""
    n = int(seconds * 24000)
    env = np.repeat(rng.random(max(1, n // 4800) + 1), 4800)[:n]
    return (0.3 * env * rng.standard_normal(n)).astype(np.float32)


def make_trace(seed, n):
    rng = random.Random(seed)
    nrng = np.random.default_rng(seed)
    t, out = 0.0, []
    for i in range(n):
        t += rng.expovariate(1.0 / a.gap)
        out.append((t, ControlRequest(f"request {i}: {rng.choice(['rain', 'dog', 'engine', 'bird', 'crowd'])} sound",
                                      reference_clip(nrng, rng.choice([1.0, 4.0, 7.5, 10.0, 12.0])), surpass_noise=rng.choice([0.0, 0.01]),
                                      guidance_scale=rng.choice([3.5, 5.0]), ddim_steps=rng.choice([25, 50]), eta=rng.choice([0.0, 1.0]),
                                      conditioning_scale=rng.choice([0.5, 1.0]), random_seed=1000 + i)))
    return out


def run_sequential(cn, trace):
    nxt, done = 0, {}
    t0 = time.perf_counter()
    while nxt < len(trace):
        now = time.perf_counter() - t0
        if trace[nxt][0] > now:
            time.sleep(trace[nxt][0] - now)
        r = trace[nxt][1]
        cn.generate_audio(r.prompt, r.audio, surpass_noise=r.surpass_noise, guidance_scale=r.guidance_scale, guidance_rescale=r.guidance_rescale,
                          ddim_steps=r.ddim_steps, eta=r.eta, conditioning_scale=r.conditioning_scale, random_seed=r.random_seed)
        done[nxt] = time.perf_counter() - t0
        nxt += 1
    return done


def run_engine(eng, trace):
    nxt, done, tick = 0, {}, {}
    t0 = time.perf_counter()
    while len(done) < len(trace):
        now = time.perf_counter() - t0
        while nxt < len(trace) and trace[nxt][0] <= now:
            r = trace[nxt][1]
            tick[eng.submit(r.prompt, audio=r.audio, surpass_noise=r.surpass_noise, guidance_scale=r.guidance_scale,
                            guidance_rescale=r.guidance_rescale, ddim_steps=r.ddim_steps, eta=r.eta, conditioning_scale=r.conditioning_scale,
                            random_seed=r.random_seed)] = nxt
            nxt += 1
        if not eng.pending():
            time.sleep(max(0.0, trace[nxt][0] - now))
            continue
        for t, _, _ in eng.step():
            done[tick[t]] = time.perf_counter() - t0
    return done


def summary(trace, done, host_ms):
    lat = np.array([done[i] - trace[i][0] for i in range(len(trace))])
    span = max(done.values()) - trace[0][0]
    return dict(latency_p50_s=round(float(np.percentile(lat, 50)), 3), latency_p95_s=round(float(np.percentile(lat, 95)), 3),
                audio_s_per_s=round(10.0 * len(trace) / span, 3), host_ms_per_step=None if host_ms is None else round(host_ms, 3))


result = dict(gpu=None, power_limit=None, forward_c4_shape=forward_bench(), requests=a.requests, mean_gap_s=a.gap, rounds=a.rounds,
              sequential=[], engine=[])
params = dict(config.BUILTIN_CONTROLNET["energy"], model_name="EzAudio-XL", model=synth.XL_MODEL,
              text_encoder=dict(model="google/flan-t5-xl", max_length=100, cfg=0.1))
cn = api.EzAudio_ControlNet("energy", ckpt_path="synthetic:2", controlnet_path="synthetic:3", vae_path="synthetic:6",
                            text_encoder=api.SyntheticTextEncoder(2048, 100), max_batch=SLOTS, params=params)
eng = engine.ContinuousEngine(cn, slots=SLOTS, ddim_steps=(25, 50))
clock = HostClock()
clock.wrap(inference, "_sample_latents_on_device", lambda args, kw: int(args[11]))   # ddim_steps argument
clock.wrap(eng.backend, "step", lambda args, kw: 1)
trace = make_trace(a.seed, a.requests)
warm = make_trace(a.seed + 1, 4)
run_sequential(cn, warm)
run_engine(eng, warm)
clock.take()
for _ in range(a.rounds):
    result["sequential"].append(summary(trace, run_sequential(cn, trace), clock.take()))
    result["engine"].append(summary(trace, run_engine(eng, trace), clock.take()))
result["engine_step_graph_captures"] = eng.backend.captures
result["gpu"], result["power_limit"] = card()
line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "controlnet_engine_bench.json"), "w") as f:
        f.write(line + "\n")
