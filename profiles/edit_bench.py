"""Edits (inpainting) of different crop lengths: scalar `editing_audio` calls in sequence against the list form in batches of four.

EzAudio-XL with synthetic weights, N edits (default 8) of synthetic 10-s clips whose crops are spread over 3 to 10 s, 50 DDIM steps, CFG 3.5.
The two plans alternate for `--rounds` rounds (default 2) after a warm-up pass of each (graph captures are counted over the whole run,
warm-up included); every wall time ends in a device synchronise.  Prints audio seconds (of crop) per second, the latency per edit, the graph
captures of each plan, the share of the wall time spent in VAE encode + decode (timed on a second, instrumented pass), and the card's name
and power limit read in the same run.  Prints one JSON line.
  python profiles/edit_bench.py [--edits 8] [--steps 50] [--rounds 2] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import api  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--edits", type=int, default=8)
ap.add_argument("--steps", type=int, default=50)
ap.add_argument("--cfg", type=float, default=3.5)
ap.add_argument("--rounds", type=int, default=2)
ap.add_argument("--batch", type=int, default=4)
ap.add_argument("--out", help="directory for the JSON result")
a = ap.parse_args()
assert torch.cuda.is_available(), "edit_bench needs a GPU"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "not reported"
    except (OSError, subprocess.SubprocessError):
        power = "not reported"
    return name, power


captures = [0]
_graph = torch.cuda.graph


class CountedGraph(_graph):
    def __enter__(self):
        captures[0] += 1
        return super().__enter__()


torch.cuda.graph = CountedGraph

sr = 24000
ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(2048, 100), max_batch=a.batch)
rng = np.random.default_rng(0)
clips = [(0.3 * rng.standard_normal(10 * sr)).astype(np.float32) for _ in range(a.edits)]
crop_s = [3 + 7 * i / max(a.edits - 1, 1) for i in range(a.edits)]            # crop = mask + 2 * boundary, 3 .. 10 s
edits = [dict(text=f"edit {i}: a bell rings", gt_file=clips[i], mask_start=(10 - c) / 2 + c / 4, mask_length=c / 2, boundary=c / 4,
              random_seed=100 + i) for i, c in enumerate(crop_s)]
order = [i for pair in zip(range(a.edits // 2), range(a.edits - 1, a.edits // 2 - 1, -1)) for i in pair] if a.edits % 2 == 0 else list(range(a.edits))
kw = dict(guidance_scale=a.cfg, ddim_steps=a.steps)

vae_s = [0.0]
dec = ez.autoencoder.decoder


def timed(fn):
    def f(*args, **kwargs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn(*args, **kwargs)
        torch.cuda.synchronize()
        vae_s[0] += time.perf_counter() - t0
        return r
    return f


def scalar():
    for e in edits:
        ez.editing_audio(**e, **kw)


def batched():   # short and long crops mixed in every batch, padded to the workspace length so all batches share one graph
    for j in range(0, a.edits, a.batch):
        grp = [edits[i] for i in order[j:j + a.batch]]
        ez.editing_audio(**{k: [e[k] for e in grp] for k in grp[0]}, **kw, pad_length=10)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


plans = {"scalar": scalar, f"batched_{a.batch}": batched}
res = {k: dict(wall_s=[], captures=0) for k in plans}
for name, fn in plans.items():   # warm-up: module loads, tensor maps, graph captures
    c0 = captures[0]
    fn()
    res[name]["captures"] += captures[0] - c0
for _ in range(a.rounds):
    for name, fn in plans.items():
        c0 = captures[0]
        res[name]["wall_s"].append(round(wall(fn), 3))
        res[name]["captures"] += captures[0] - c0
call, encode = type(dec).__call__, type(dec).encode
type(dec).__call__, type(dec).encode = timed(call), timed(encode)   # instrumented pass: the synchronises perturb the wall time, so it is separate
for name, fn in plans.items():
    vae_s[0] = 0.0
    w = wall(fn)
    res[name]["vae_share"] = round(vae_s[0] / w, 3)
type(dec).__call__, type(dec).encode = call, encode
audio_s = sum(crop_s)
for name, r in res.items():
    best = min(r["wall_s"])
    r["audio_s_per_s"] = round(audio_s / best, 3)
    r["latency_per_edit_s"] = round(best / a.edits, 3)
gpu, power = card()
line = json.dumps(dict(gpu=gpu, power_limit=power, edits=a.edits, steps=a.steps, cfg=a.cfg, crop_s=[round(c, 2) for c in crop_s], crop_audio_s=round(audio_s, 2),
                       plans=res))
print(line)
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "edit_bench.json"), "w") as f:
        f.write(line + "\n")
