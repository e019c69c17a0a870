"""One-process A/B sweep of the launch-time switches (ezb_set_option): XL, 4 prompts + CFG (effective batch 8), L = 500.  The model is built
once; for every option set one denoiser step (DiT forward + fused CFG/DDIM update) is captured into a CUDA graph and replayed 30 times between
CUDA events (what the sampling loop does; no host launch cost).  `skip=<mask>` sets do not launch a class of kernels (results are garbage): the
drop in step time is that class's in-situ cost.
  python profiles/ab_sweep.py                       # the built-in list
  python profiles/ab_sweep.py "attn_res=1" "attn_res=1,attn_poly=1"
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import _lib, api  # noqa: E402
from ezaudio_b200.inference import _ddim_step  # noqa: E402

DEFAULTS = {"attn7": 0, "w_prefetch": 0, "attn6": 5, "attn_pp": 0, "attn_res": 0, "attn_poly": 0, "cq_single": 0, "mlp2_pair": 0, "swap_mc": 0,
            "mlp_fused": 0, "ln_variant": 2, "ln_tail": 0, "skip": 0}
for a in sys.argv[1:]:
    if a.startswith("default:"):   # e.g. default:attn_res=1 changes the baseline every set is applied on top of
        k, v = a[8:].split("=")
        DEFAULTS[k] = int(v)
SETS = [a for a in sys.argv[1:] if not a.startswith("default:")] or [
    "", "attn_res=1", "attn_poly=1", "attn_res=1,attn_poly=1", "cq_single=1", "mlp2_pair=1", "swap_mc=1",
    "mlp_fused=1", "",
    "skip=1", "skip=2", "skip=4", "skip=8", "skip=16", "skip=31", ""]

B, L = 4, 500
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


e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for s in SETS:
    opts = dict(DEFAULTS)
    for kv in filter(None, s.split(",")):
        k, v = kv.split("=")
        opts[k] = int(v)
    for k, v in opts.items():
        _lib.check(_lib.lib().ezb_set_option(k.encode(), v))
    lat.normal_()
    for i in range(2):
        step(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step(0)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(30):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    print(f"opts [{s}]: {e0.elapsed_time(e1) / 30:.3f} ms per graph replay of one step", flush=True)
    del g
