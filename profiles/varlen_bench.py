"""Mixed-length traffic through the batching front-end: exact-length grouping against length buckets (clips of different lengths padded
into one batch, per-sample lengths in device memory).

A seeded stream of requests (EzAudio-XL, synthetic weights, default 16 requests of 3 to 10 s in 0.5-s steps, 50 DDIM steps, CFG 5) is run
twice from a cold graph cache: once with today's grouping (one batch per exact length) and once with `length_bucket_s`.  For each plan it
prints audio seconds per second, the number of captured CUDA graphs and the time spent capturing them.  It also times one DiT step at
Be = 8, L = 500 replayed from a CUDA graph with lens = NULL and with lens = [500] * 8 (alternating), and reads the card's name and power
limit in the same run.  Prints one JSON line.
  python profiles/varlen_bench.py [--requests 16] [--steps 50] [--bucket 5] [--out DIR]
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
from ezaudio_b200 import _lib, api  # noqa: E402
from ezaudio_b200.frontend import BatchingFrontEnd, Request  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=16)
ap.add_argument("--steps", type=int, default=50)
ap.add_argument("--cfg", type=float, default=5.0)
ap.add_argument("--bucket", type=float, default=5.0)
ap.add_argument("--max-batch", type=int, default=4)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "varlen_bench needs a GPU"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "not reported"
    except (OSError, subprocess.SubprocessError):
        power = "not reported"
    return name, power


class CaptureClock:
    """Counts and times the CUDA-graph captures of the sampling loop (torch.cuda.graph blocks)."""

    def __init__(self):
        self.n, self.s = 0, 0.0
        self._orig = torch.cuda.graph
        clock = self

        class Timed(self._orig):
            def __enter__(self):
                torch.cuda.synchronize()
                self._t0 = time.perf_counter()
                return super().__enter__()

            def __exit__(self, *exc):
                r = super().__exit__(*exc)
                torch.cuda.synchronize()
                clock.n += 1
                clock.s += time.perf_counter() - self._t0
                return r

        torch.cuda.graph = Timed


enc = api.SyntheticTextEncoder(2048, 100)
ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=a.max_batch)
rng = random.Random(a.seed)
reqs = [Request(f"request {i}: {rng.choice(['rain', 'dog', 'engine', 'bird', 'crowd'])} sound", length=rng.randint(6, 20) / 2, guidance_scale=a.cfg,
                ddim_steps=a.steps, random_seed=1000 + i) for i in range(a.requests)]
audio_s = sum(r.length for r in reqs)
ez.generate_audio("warm up", length=1, ddim_steps=2, random_seed=0)   # module loads, tensor maps, function attributes
clock = CaptureClock()
result = dict(gpu=None, power_limit=None, requests=a.requests, steps=a.steps, cfg=a.cfg, audio_s=audio_s,
              lengths=sorted({r.length for r in reqs}), plans={})
wavs = {}
for plan, bucket in (("exact", None), (f"bucket_{a.bucket:g}s", a.bucket)):
    ez.unet.__dict__.pop("_loop_cache", None)   # every plan starts from a cold graph cache, like a fresh server
    fe = BatchingFrontEnd(ez, max_batch=a.max_batch, length_bucket_s=bucket)
    n0, s0 = clock.n, clock.s
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fe.run(reqs)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    wavs[plan] = [w for _, w in out]
    result["plans"][plan] = dict(wall_s=round(wall, 3), audio_s_per_s=round(audio_s / wall, 3), captures=clock.n - n0,
                                 capture_s=round(clock.s - s0, 3))
p0, p1 = list(wavs)
result["plans_max_abs_diff"] = float(max(np.abs(x - y).max() for x, y in zip(wavs[p0], wavs[p1])))

# one DiT step at Be = 8, L = 500 from a CUDA graph: lens = NULL against lens = [500] * 8
B, L = 4, 500
te, tm = enc([f"p{i} a b c d e f" for i in range(B)])
ue, um = enc([""])
ez.unet.set_context(torch.cat([te, ue.expand(B, -1, -1)], 0).cuda(), torch.cat([tm, um.expand(B, -1)], 0).cuda())
ez.unet.set_timesteps([999])
x = torch.randn(2 * B, 128, L, device="cuda")
out = torch.empty_like(x)
lens = torch.full((2 * B,), L, dtype=torch.int32, device="cuda")
graphs = {}
for name, ln in (("lens_null", None), ("lens_full", lens)):
    for _ in range(2):
        ez.unet.forward_step(x, 0, out=out, lengths=ln)
    g = torch.cuda.CUDAGraph()
    with clock._orig(g):
        ez.unet.forward_step(x, 0, out=out, lengths=ln)
    graphs[name] = g
step_ms = {k: [] for k in graphs}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for _ in range(5):
    for name, g in graphs.items():
        g.replay()
        e0.record()
        for _ in range(20):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        step_ms[name].append(round(e0.elapsed_time(e1) / 20, 3))
result["dit_step_ms_Be8_L500"] = step_ms
result["gpu"], result["power_limit"] = card()
line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "varlen_bench.json"), "w") as f:
        f.write(line + "\n")
