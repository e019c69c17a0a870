"""Serving edits: a mixed trace of edits and text-to-audio requests, sequential scalar calls against the continuous engine.

EzAudio-XL with synthetic weights and cached (synthetic) text embeddings.  A seeded trace of `--requests` requests with Poisson arrivals
(mean gap `--gap` s), half of them edits of synthetic clips (crops of 3 to 9.5 s, the mask in the middle of the crop with up to 1 s of
context either side) and half text-to-audio requests of 4 to 10 s; 50 or 100 DDIM steps, guidance 3.5 or 5, eta 0 or 1.  It is replayed in
real time against
  * sequential scalar calls, one request per call in arrival order (EzAudio.editing_audio / EzAudio.generate_audio): what a server without
    the engine runs (the list form would make every edit wait for the longest in its batch);
  * engine.ContinuousEngine with 4 slots and 10-s padding: arrived requests are submitted before every step.
The two alternate in one process, `--rounds` times each, after one untimed warm-up pass each.  Reported per path: latency p50 / p95
(arrival to waveform on the host), audio seconds per wall second (crop seconds for an edit, the clip length for a generation, over first
arrival to last waveform) and the host time per denoising step spent outside the CUDA-graph replay and event waits.  A last engine pass
times each edit's admission (prepare + VAE encode of the crop + the slot's rows) between device synchronises, and each step the same way,
which gives what an edit's admission adds to the step it joins.  The card's name and power limit are read in the same run.  Prints one JSON
line.
  python profiles/edit_engine_bench.py [--requests 12] [--gap 0.5] [--rounds 2] [--seed 0] [--out DIR]
"""
import argparse
import dataclasses
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import api, engine, inference  # noqa: E402
from ezaudio_b200.frontend import EditRequest, Request  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=12)
ap.add_argument("--gap", type=float, default=0.5, help="mean inter-arrival time (s)")
ap.add_argument("--rounds", type=int, default=2)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "edit_engine_bench needs a GPU"
SLOTS, SR = 4, 24000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "not reported"
    except (OSError, subprocess.SubprocessError):
        power = "not reported"
    return name, power


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


def synthetic_clip(nrng, seconds):
    """A few tones under noise with a slow envelope."""
    t = np.arange(int(seconds * SR)) / SR
    tones = sum(0.2 * np.sin(2 * np.pi * f * t) for f in nrng.uniform(110, 1760, 3))
    env = np.repeat(nrng.random(int(seconds * 5) + 2), SR // 5)[:len(t)]
    return ((0.5 + 0.5 * env) * tones + 0.02 * nrng.standard_normal(len(t))).astype(np.float32)


def make_trace(seed, n):
    rng, nrng = random.Random(seed), np.random.default_rng(seed)
    t, out = 0.0, []
    for i in range(n):
        t += rng.expovariate(1.0 / a.gap)
        kw = dict(guidance_scale=rng.choice([3.5, 5.0]), ddim_steps=rng.choice([50, 100]), eta=rng.choice([0.0, 1.0]), random_seed=1000 + i)
        prompt = f"request {i}: {rng.choice(['rain', 'dog', 'engine', 'bird', 'crowd'])} sound"
        if i % 2 == 0:
            crop = rng.randint(6, 19) / 2                     # 3 .. 9.5 s
            b = min(1.0, crop / 4)
            start = b + rng.randint(0, 20) / 10
            clip = synthetic_clip(nrng, start + crop - b + rng.randint(0, 20) / 10)
            out.append((t, EditRequest(prompt, b, clip, start, crop - 2 * b, **kw), crop))
        else:
            length = rng.randint(8, 20) / 2                   # 4 .. 10 s
            out.append((t, Request(prompt, length=length, guidance_rescale=0.75, **kw), length))
    return out


def run_sequential(ez, trace):
    nxt, done = 0, {}
    t0 = time.perf_counter()
    while nxt < len(trace):
        now = time.perf_counter() - t0
        if trace[nxt][0] > now:
            time.sleep(trace[nxt][0] - now)
        r = trace[nxt][1]
        kw = dict(guidance_scale=r.guidance_scale, guidance_rescale=r.guidance_rescale, ddim_steps=r.ddim_steps, eta=r.eta, random_seed=r.random_seed)
        if isinstance(r, EditRequest):
            ez.editing_audio(r.prompt, r.boundary, r.gt_file, r.mask_start, r.mask_length, **kw)
        else:
            ez.generate_audio(r.prompt, length=r.length, **kw)
        done[nxt] = time.perf_counter() - t0
        nxt += 1
    return done


def run_engine(eng, trace):
    nxt, done, tick = 0, {}, {}
    t0 = time.perf_counter()
    while len(done) < len(trace):
        now = time.perf_counter() - t0
        while nxt < len(trace) and trace[nxt][0] <= now:
            tick[eng.submit(**dataclasses.asdict(trace[nxt][1]))] = nxt
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
                audio_s_per_s=round(sum(s for _, _, s in trace) / span, 3), host_ms_per_step=None if host_ms is None else round(host_ms, 3))


def synchronised_ms(owner, name, into):
    orig = getattr(owner, name)

    def timed(*args, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = orig(*args, **kw)
        torch.cuda.synchronize()
        into.append(1e3 * (time.perf_counter() - t0))
        return r
    setattr(owner, name, timed)
    return orig


enc = api.SyntheticTextEncoder(2048, 100)
ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=SLOTS)
eng = engine.ContinuousEngine(ez, slots=SLOTS, max_length_s=10.0, ddim_steps=(50, 100))
clock = HostClock()
clock.wrap(inference, "_sample_latents_on_device", lambda args, kw: int(args[11]))   # ddim_steps argument
clock.wrap(eng.backend, "step", lambda args, kw: 1)
trace = make_trace(a.seed, a.requests)
warm = make_trace(a.seed + 1, 4)
run_sequential(ez, warm)
run_engine(eng, warm)
clock.take()
result = dict(gpu=None, power_limit=None, requests=a.requests, edits=sum(isinstance(r, EditRequest) for _, r, _ in trace), mean_gap_s=a.gap,
              rounds=a.rounds, audio_s=round(sum(s for _, _, s in trace), 2), sequential=[], engine=[])
for _ in range(a.rounds):
    result["sequential"].append(summary(trace, run_sequential(ez, trace), clock.take()))
    result["engine"].append(summary(trace, run_engine(eng, trace), clock.take()))
admit_ms, step_ms = [], []
orig_admit = synchronised_ms(eng.backend, "_admit_edit", admit_ms)
orig_step = synchronised_ms(eng.backend, "step", step_ms)
run_engine(eng, trace)
eng.backend._admit_edit, eng.backend.step = orig_admit, orig_step
result["edit_admission_ms"] = dict(median=round(float(np.median(admit_ms)), 2), max=round(float(np.max(admit_ms)), 2), n=len(admit_ms))
result["engine_step_ms_synchronised"] = dict(median=round(float(np.median(step_ms)), 2), n=len(step_ms))
result["engine_step_graph_captures"] = eng.backend.captures
result["gpu"], result["power_limit"] = card()
line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "edit_engine_bench.json"), "w") as f:
        f.write(line + "\n")
