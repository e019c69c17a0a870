"""Audio-to-audio variations on the GPU: the fused start latent, and variation_audio end to end.

Start latent: ezb_vae_encode_noised (the Oobleck encoder with the bottleneck sample, scale_shift and add_noise fused into its last pass)
against ezb_vae_encode followed by `(z + shift) * scale` and `a * x0 + s * eps` in PyTorch, on the full-size VAE with synthetic weights at
B = 4, L = 500 and 1500 latent frames (10 s and 30 s clips).  CUDA events around `--launches` back-to-back calls, the two alternated `--reps`
times in this one process; the median per call is reported, and the difference, which is the time the fusion saves.
End to end: EzAudio-XL with synthetic weights, `--prompts` clips x 10 s, CFG 5 / rescale 0.75, 100 DDIM steps (eta 1): variation_audio at
strengths 0.3 / 0.5 / 0.8 against generate_audio, host wall time around the call ending in a device synchronise, each configuration warmed
once (graph capture) and then timed `--e2e-reps` times, alternating.  The card's name and power limit are read in the same run.
Prints one JSON line.
  python profiles/variation_bench.py [--launches 20] [--reps 5] [--prompts 4] [--e2e-reps 3] [--out DIR]
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
from ezaudio_b200 import api, synth, weights  # noqa: E402
from ezaudio_b200.vae import OobleckDecoder  # noqa: E402


ap = argparse.ArgumentParser()
ap.add_argument("--launches", type=int, default=20)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--prompts", type=int, default=4)
ap.add_argument("--e2e-reps", type=int, default=3)
ap.add_argument("--skip-e2e", action="store_true")
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "variation_bench needs a GPU"
SCALE, SHIFT = 0.18, 0.5   # any pair; the arithmetic does not depend on the values


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "not reported"
    except (OSError, subprocess.SubprocessError):
        power = "not reported"
    return name, power


def start_latent_times(vae, L, B=4):
    g = torch.Generator(device="cuda").manual_seed(L)
    audio = 0.3 * torch.randn(B, 1, L * vae.hop, device="cuda", generator=g)
    noise = torch.randn(B, 128, L, device="cuda", generator=g)
    eps = torch.randn(B, 128, L, device="cuda", generator=g)
    ab_host = [[0.6, 0.8]] * B
    ab = torch.tensor(ab_host, device="cuda")
    a_col, s_col = ab[:, 0].view(B, 1, 1), ab[:, 1].view(B, 1, 1)

    def fused():
        return vae.encode_noised(audio, ab, eps, SCALE, SHIFT, noise=noise)

    def unfused():
        z = vae.encode(audio, noise=noise)
        return a_col * ((z + SHIFT) * SCALE) + s_col * eps

    same = torch.equal(fused(), unfused())   # the fused kernel rounds each op as PyTorch does
    res = {"fused": [], "unfused": []}
    for f in (fused, unfused):   # warm-up: module load, tensor maps
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    for _ in range(a.reps):
        for name, f in (("fused", fused), ("unfused", unfused)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                f()
            e1.record()
            e1.synchronize()
            res[name].append(e0.elapsed_time(e1) / a.launches)
    out = {k: dict(ms_per_call=round(statistics.median(v), 4), min_ms=round(min(v), 4), max_ms=round(max(v), 4)) for k, v in res.items()}
    out["saved_ms"] = round(out["unfused"]["ms_per_call"] - out["fused"]["ms_per_call"], 4)
    out["bit_identical"] = bool(same)
    return out


name, power = card()
result = dict(gpu=name, power_limit_and_max_sm_clock=power, start_latent={})
ecfg, dcfg = synth.VAE_ENCODER, synth.VAE_DECODER
sd = dict(weights.synthetic_state_dict(weights.vae_decoder_param_shapes(dcfg), 6))
sd.update(weights.synthetic_state_dict(weights.vae_encoder_param_shapes(ecfg), 8))
vae = OobleckDecoder(precision="bf16", max_batch=4, max_latent_len=1500, encoder_cfg=ecfg, **dcfg).load_state_dict(sd)
for L in (500, 1500):
    result["start_latent"][f"B4_L{L}"] = start_latent_times(vae, L)
    print(f"[start latent] L={L}: {result['start_latent'][f'B4_L{L}']}", flush=True)
del vae, sd
torch.cuda.empty_cache()

if not a.skip_e2e:
    enc = api.SyntheticTextEncoder(2048, 100)
    ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=a.prompts)
    prompts = [f"prompt {i}: rain and a distant dog" for i in range(a.prompts)]
    sr = ez.params["autoencoder"]["sr"]
    t = np.arange(10 * sr) / sr
    clips = [(0.3 * np.sin(2 * np.pi * (110 + 55 * i) * t)).astype(np.float32) for i in range(a.prompts)]
    kw = dict(guidance_scale=5, guidance_rescale=0.75, ddim_steps=100, eta=1, random_seed=2024)
    configs = [("generate_audio", None)] + [(f"variation_audio strength {s}", s) for s in (0.3, 0.5, 0.8)]

    def run(strength):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if strength is None:
            ez.generate_audio(prompts, length=10, **kw)
        else:
            ez.variation_audio(prompts, clips, strength=strength, **kw)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for _, s in configs:
        run(s)   # graph capture, tensor maps
    times = {label: [] for label, _ in configs}
    for _ in range(a.e2e_reps):
        for label, s in configs:
            times[label].append(run(s))
    base = statistics.median(times["generate_audio"])
    result["e2e"] = dict(workload=f"EzAudio-XL synthetic weights, {a.prompts} clips x 10 s, CFG 5 / rescale 0.75, 100 DDIM steps, incl. VAE "
                                  "encode (variations) and decode",
                         seconds={k: dict(median=round(statistics.median(v), 3), of_generate=round(statistics.median(v) / base, 3),
                                          all=[round(x, 3) for x in v]) for k, v in times.items()})
    print(f"[e2e] {result['e2e']}", flush=True)

line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "variation_bench.json"), "w") as f:
        f.write(line + "\n")
