"""Long edits on the GPU: EzAudio.editing_long_audio against editing_audio, and the tiled VAE encode against a one-shot encode.

EzAudio-XL with synthetic weights and the synthetic text encoder, one process:
  * Encode: OobleckDecoder.encode_tiled of a 60 s crop (3000 latent frames) on a 10 s workspace (max_batch 8: seven chunks of at most
    500 frames, one encode call) against a one-shot encode on a workspace that holds 60 s.  Both with the same given bottleneck noise;
    the outputs are compared bit for bit.  CUDA events over `--iters` calls, the two alternated `--reps` times; medians.  The difference is
    the cost of the halos (7 frames on each inner edge).
  * End to end: one prompt, CFG 3.5, 50 DDIM steps (eta 1), encode and decode included, host wall time around each call ending in a
    device synchronise, on EzAudio(max_batch=8) handles whose workspaces hold 10 s (one for the 8 s crops, one for the continuations):
      - editing_audio and editing_long_audio on the same 8 s crop (one window: the outputs must be identical, the times should match);
      - editing_long_audio continuing a 10 s clip by 20 s and by 50 s with 5 s of context (25 s and 55 s crops, 10 s windows, 2 s overlap).
    Each configuration is warmed once (graph capture), then timed `--e2e-reps` times, alternated.
The card's name and power limit are read in the same run.  Prints one JSON line.
  python profiles/long_edit_bench.py [--iters 10] [--reps 5] [--e2e-reps 3] [--out DIR]
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
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--e2e-reps", type=int, default=3)
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "long_edit_bench needs a GPU"


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


def clip(seconds, seed):
    rng = np.random.default_rng(seed)
    n = int(seconds * 24000)
    t = np.arange(n) / 24000
    return (0.2 * np.sin(2 * np.pi * 220 * t) * (0.6 + 0.4 * np.sin(t)) + 0.05 * rng.standard_normal(n)).astype(np.float32)


def encode_bench():
    sd = dict(weights.synthetic_state_dict(weights.vae_decoder_param_shapes(synth.VAE_DECODER), 6))
    sd.update(weights.synthetic_state_dict(weights.vae_encoder_param_shapes(synth.VAE_ENCODER), 8))
    kw = dict(precision="bf16", encoder_cfg=synth.VAE_ENCODER, **synth.VAE_DECODER)
    small = OobleckDecoder(max_batch=8, max_latent_len=500, **kw).load_state_dict(sd)
    big = OobleckDecoder(max_batch=1, max_latent_len=3000, **kw).load_state_dict(sd)
    del sd
    audio = torch.from_numpy(clip(60, 1)).view(1, 1, -1).cuda()
    noise = torch.randn(1, 128, 3000, generator=torch.Generator().manual_seed(2)).cuda()
    paths = {"encode_tiled on a 10 s workspace": lambda: small.encode_tiled(audio, noise=noise),
             "encode on a 60 s workspace": lambda: big.encode(audio, noise=noise)}
    outs = {k: f() for k, f in paths.items()}
    torch.cuda.synchronize()
    same = torch.equal(*outs.values())
    ts = {k: [] for k in paths}
    for _ in range(a.reps):
        for k, f in paths.items():
            ts[k].append(event_ms(f, a.iters))
    res = {k: dict(ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3)) for k, v in ts.items()}
    res["bit_identical"] = bool(same)
    res["crop"] = "1 x 60 s (3000 latent frames), bf16, given bottleneck noise"
    del small, big
    torch.cuda.empty_cache()
    return res


def e2e_bench():
    # the windowed loop keeps the graphs of two plan shapes per DiT handle: the continuations get their own EzAudio, so that alternating
    # the three long configurations replays their graphs instead of capturing them again on every call
    enc = api.SyntheticTextEncoder(2048, 100)
    ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=8)
    ez2 = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=enc, max_batch=8)
    prompt = "rain turns into a thunderstorm"
    kw = dict(guidance_scale=3.5, guidance_rescale=0, ddim_steps=50, eta=1, random_seed=2024)
    ten = clip(10, 3)
    mid = dict(boundary=2, gt_file=ten, mask_start=3, mask_length=4)   # an 8 s crop [1 s, 9 s)
    configs = {"editing_audio 8 s crop": lambda: ez.editing_audio(prompt, **mid, **kw),
               "editing_long_audio 8 s crop": lambda: ez.editing_long_audio(prompt, **mid, **kw),
               "editing_long_audio 10 s + 20 s": lambda: ez2.editing_long_audio(prompt, 5, ten, 10, 20, **kw),
               "editing_long_audio 10 s + 50 s": lambda: ez2.editing_long_audio(prompt, 5, ten, 10, 50, **kw)}

    def run(f):
        torch.manual_seed(7)   # the VAE bottleneck noise: the same draw for both 8 s calls
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, w = f()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, w

    shapes, outs = {}, {}
    for k, f in configs.items():
        _, w = run(f)   # graph capture, tensor maps
        outs[k] = w
        shapes[k] = dict(samples=int(w.shape[0]), finite=bool(np.isfinite(w).all()))
    times = {k: [] for k in configs}
    for _ in range(a.e2e_reps):
        for k, f in configs.items():
            times[k].append(run(f)[0])
    return dict(workload="EzAudio-XL, synthetic weights, 1 prompt, CFG 3.5, 50 DDIM steps (eta 1), incl. VAE encode and decode; "
                         "10 s windows with 2 s overlap on max_batch 8",
                outputs=shapes,
                eight_second_crop_identical=outs["editing_audio 8 s crop"].tobytes() == outs["editing_long_audio 8 s crop"].tobytes(),
                seconds={k: dict(median=round(statistics.median(v), 3), all=[round(x, 3) for x in v]) for k, v in times.items()})


name, power = card()
result = dict(gpu=name, power_limit_and_max_sm_clock=power)
result["encode"] = encode_bench()
print(f"[encode] {result['encode']}", flush=True)
result["e2e"] = e2e_bench()
print(f"[e2e] {result['e2e']}", flush=True)
line = json.dumps(result)
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "long_edit_bench.json"), "w") as f:
        f.write(line + "\n")
