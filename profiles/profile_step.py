"""Profiling driver: XL, 4 prompts + CFG (effective batch 8), L=500: warm-up, then inside a cudaProfilerStart/Stop range
`--steps` denoiser steps (DiT forward + fused CFG/DDIM update) and one VAE decode of 4 clips.
  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file launches.csv \
      python profiles/profile_step.py --steps 1          (or nsys --capture-range=cudaProfilerApi; summarize.py reads the ncu csv)
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import api, synth  # noqa: E402
from ezaudio_b200.inference import _ddim_step  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=1)
ap.add_argument("--vae", type=int, default=1)
ap.add_argument("--batch", type=int, default=4)
ap.add_argument("--opt", action="append", default=[], help="name=value runtime switches (ezb_set_option)")
a = ap.parse_args()
B, L = a.batch, 500
from ezaudio_b200 import _lib  # noqa: E402
for kv in a.opt:
    k, v = kv.split("=")
    _lib.check(_lib.lib().ezb_set_option(k.encode(), int(v)))
enc = api.SyntheticTextEncoder(2048, 100)
ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=B)
te, tm = enc([f"p{i} a b c d e f" for i in range(B)])
ue, um = enc([""])
ctx = torch.cat([te, ue.expand(B, -1, -1)], 0).cuda()
msk = torch.cat([tm, um.expand(B, -1)], 0).cuda()
ez.unet.set_context(ctx, msk)
ez.noise_scheduler.set_timesteps(50)
ts = [int(t) for t in ez.noise_scheduler.timesteps]
ez.unet.set_timesteps(ts)
lat = torch.randn(B, 128, L, device="cuda")
x = torch.cat([lat, lat], 0).contiguous()
out = torch.empty_like(x)
nz = torch.randn_like(lat)


def step(i):
    ez.unet.forward_step(x, i, out=out)
    _ddim_step(out, lat, nz, B, 128, L, 5.0, 0.75, ez.noise_scheduler.step_coefficients(ts[i], 1.0))


for i in range(2):
    step(i)
ez.autoencoder(embedding=lat)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStart()
for i in range(a.steps):
    step(i)
for _ in range(a.vae):
    ez.autoencoder(embedding=lat)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStop()
# in-situ timing (no profiler): 20 back-to-back steps with CUDA events
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for i in range(20):
    step(i)
e1.record()
torch.cuda.synchronize()
eager_ms = e0.elapsed_time(e1) / 20
# VAE decode of the B clips (10 s each), 5 back-to-back decodes
e0.record()
for _ in range(5):
    ez.autoencoder(embedding=lat)
e1.record()
torch.cuda.synchronize()
print(f"opts {a.opt}: VAE decode of {B} x 10 s: {e0.elapsed_time(e1) / 5:.3f} ms")
# the same step replayed from a CUDA graph (what the sampling loop does): no host launch cost at all
g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g):
    step(0)
for _ in range(3):
    g.replay()
torch.cuda.synchronize()
e0.record()
for i in range(20):
    g.replay()
e1.record()
torch.cuda.synchronize()
print(f"opts {a.opt}: {eager_ms:.3f} ms per eager DiT step (+CFG/DDIM), {e0.elapsed_time(e1) / 20:.3f} ms per graph replay")
