"""Serving latency under a mixed arrival trace: the batching front-end against the continuous-batching engine.

EzAudio-XL with synthetic weights and cached (synthetic) text embeddings.  A seeded trace of requests with Poisson arrivals (default 12
requests, mean gap 0.4 s), 50 or 100 DDIM steps, guidance 3.5 or 5, eta 0 or 1 and lengths of 4 to 10 s is replayed in real time against
  * frontend.BatchingFrontEnd(max_batch 4, length buckets of 5 s): whenever it is idle it plans the requests that have arrived and runs the
    first batch of the plan as one generate_audio call (one CUDA graph for the whole schedule);
  * engine.ContinuousEngine(4 slots, 10 s): arrived requests are submitted before every step.
The two alternate in one process, `--rounds` times each, after one untimed warm-up pass each.  For each it reports per-request latency
(arrival to waveform on the host, which includes a device synchronise) p50 / p95, audio seconds per wall second (first arrival to last
waveform), and the host time per denoising step spent outside the CUDA-graph replay (the per-step host work: noise draws, copies, launch
of the replay; for the engine also its copy of the step inputs, excluding the wait for the previous step's copy).  The card's name and power
limit are read in the same run.  A front-end batch whose graph key (batch size, padded length, schedule, guidance constants) is not
cached captures a new graph, so few of its calls in the trace replay one: its host time per step is also taken on a steady workload (the
same batch of 4 run twice, the second call timed).  Prints one JSON line.
  python profiles/continuous_bench.py [--requests 12] [--gap 0.4] [--rounds 2] [--seed 0] [--out DIR]
"""
import argparse
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
from ezaudio_b200.frontend import BatchingFrontEnd, Request, plan_batches  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=12)
ap.add_argument("--gap", type=float, default=0.4, help="mean inter-arrival time (s)")
ap.add_argument("--rounds", type=int, default=2)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "continuous_bench needs a GPU"
SLOTS, BUCKET = 4, 5.0


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "not reported"
    except (OSError, subprocess.SubprocessError):
        power = "not reported"
    return name, power


class HostClock:
    """Host time of per-step work outside CUDA-graph replays: wraps `fn_owner.fn_name` (one call = `steps(args)` denoising steps) and
    subtracts the time spent inside CUDAGraph.replay and Event.synchronize during the call.  Calls without a replay (eager pass + capture)
    are not counted."""

    def __init__(self):
        self.excl = 0.0
        self.replays = 0
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
        self.host_s, self.steps = 0.0, 0

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


class CaptureCount:
    """Counts CUDA-graph captures (torch.cuda.graph blocks)."""

    def __init__(self):
        self.n = 0
        clock = self

        class Counted(torch.cuda.graph):
            def __enter__(self):
                clock.n += 1
                return super().__enter__()

        torch.cuda.graph = Counted

    def take(self):
        n, self.n = self.n, 0
        return n


def make_trace(seed):
    rng = random.Random(seed)
    t, out = 0.0, []
    for i in range(a.requests):
        t += rng.expovariate(1.0 / a.gap)
        out.append((t, Request(f"request {i}: {rng.choice(['rain', 'dog', 'engine', 'bird', 'crowd'])} sound", length=rng.randint(8, 20) / 2,
                               guidance_scale=rng.choice([3.5, 5.0]), guidance_rescale=0.75, ddim_steps=rng.choice([50, 100]),
                               eta=rng.choice([0.0, 1.0]), random_seed=1000 + i)))
    return out


def run_frontend(ez, trace):
    fe = BatchingFrontEnd(ez, max_batch=SLOTS, length_bucket_s=BUCKET)
    waiting, nxt, done = [], 0, {}
    t0 = time.perf_counter()
    while len(done) < len(trace):
        now = time.perf_counter() - t0
        while nxt < len(trace) and trace[nxt][0] <= now:
            waiting.append(nxt)
            nxt += 1
        if not waiting:
            time.sleep(max(0.0, trace[nxt][0] - now))
            continue
        first = plan_batches([trace[i][1] for i in waiting], SLOTS, BUCKET)[0]
        idx = [waiting[j] for j in first.tickets]
        fe.run([trace[i][1] for i in idx])   # waveforms come back on the host (synchronised)
        end = time.perf_counter() - t0
        for i in idx:
            done[i] = end
            waiting.remove(i)
    return done


def run_engine(eng, trace):
    nxt, done, tick = 0, {}, {}
    t0 = time.perf_counter()
    while len(done) < len(trace):
        now = time.perf_counter() - t0
        while nxt < len(trace) and trace[nxt][0] <= now:
            r = trace[nxt][1]
            tick[eng.submit(r.prompt, length=r.length, guidance_scale=r.guidance_scale, guidance_rescale=r.guidance_rescale,
                            ddim_steps=r.ddim_steps, eta=r.eta, random_seed=r.random_seed)] = nxt
            nxt += 1
        if not eng.pending():
            time.sleep(max(0.0, trace[nxt][0] - now))
            continue
        for t, _, _ in eng.step():
            done[tick[t]] = time.perf_counter() - t0
    return done


def summary(trace, done, host_ms, captures):
    lat = np.array([done[i] - trace[i][0] for i in range(len(trace))])
    span = max(done.values()) - trace[0][0]
    return dict(latency_p50_s=round(float(np.percentile(lat, 50)), 3), latency_p95_s=round(float(np.percentile(lat, 95)), 3),
                audio_s_per_s=round(sum(r.length for _, r in trace) / span, 3), host_ms_per_step=None if host_ms is None else round(host_ms, 3),
                graph_captures=captures)


enc = api.SyntheticTextEncoder(2048, 100)
ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=SLOTS)
eng = engine.ContinuousEngine(ez, slots=SLOTS, max_length_s=10.0, ddim_steps=(50, 100))
clock, caps = HostClock(), CaptureCount()
clock.wrap(inference, "_sample_latents_on_device", lambda args, kw: int(args[11]))   # ddim_steps argument
clock.wrap(eng.backend, "step", lambda args, kw: 1)
trace = make_trace(a.seed)
warm = make_trace(a.seed + 1)[:4]
run_frontend(ez, warm)
run_engine(eng, warm)
clock.take(), caps.take()
result = dict(gpu=None, power_limit=None, requests=a.requests, mean_gap_s=a.gap, rounds=a.rounds, audio_s=sum(r.length for _, r in trace),
              frontend=[], engine=[])
for _ in range(a.rounds):
    done = run_frontend(ez, trace)
    result["frontend"].append(summary(trace, done, clock.take(), caps.take()))
    done = run_engine(eng, trace)
    result["engine"].append(summary(trace, done, clock.take(), caps.take()))
steady = [Request(f"steady {i}", length=10, guidance_scale=5.0, guidance_rescale=0.75, ddim_steps=100, eta=1.0, random_seed=i) for i in range(SLOTS)]
fe = BatchingFrontEnd(ez, max_batch=SLOTS, length_bucket_s=BUCKET)
fe.run(steady)
clock.take()
fe.run(steady)
v = clock.take()
result["frontend_steady_host_ms_per_step"] = None if v is None else round(v, 3)
result["engine_step_graph_captures"] = eng.backend.captures
result["gpu"], result["power_limit"] = card()
line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "continuous_bench.json"), "w") as f:
        f.write(line + "\n")
