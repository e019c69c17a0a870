#!/usr/bin/env python
"""Benchmark of the EzAudio hot path (BASELINE.json metric: audio-seconds generated per wall-second, EzAudio-XL,
50 DDIM steps, 10-s prompts).

  python bench.py --gpus N --steps K --warmup W           -> our arm (CUDA library), one JSON line from rank 0
  python bench.py --impl reference --gpus N --steps K ... -> the reference algorithm's CPU path (oracle port), same JSON

A "step" is one full pass of the hot path over one batch: 4 prompts per GPU x 10 s, 50 DDIM steps with classifier-free
guidance (effective batch 8; API defaults guidance 5 / rescale 0.75 / eta 1, api/ezaudio.py:102) + VAE decode (BASELINE configs C2/C3).
`value` times the loop with inputs resident in HBM; `e2e` times the public API call (`EzAudio.generate_audio`) with
host-resident cached T5 embeddings (pinned) copied in and the waveforms copied back out every step.

The same line also carries (N = 1; cheap legs, a few seconds each):
  parity   measured max / mean-abs of the BENCHMARKED precision on the reference's own golden output (tests/golden/dit_XL.npz, written by the
           unmodified reference), and the same two numbers plus the THROUGHPUT of --precision bf16x3 (the mode that meets the 1e-3 bound);
  configs  BASELINE configs C4 (XL + energy ControlNet, 8 prompts) and C5 (30-s inpainting, 100 steps, VAE encode + decode; two prompts per
           GPU, on ranks 0 and 1 when launched with >= 2 GPUs) through the public API, with their algorithmic TFLOP and roofline fraction.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

PROMPTS_PER_GPU = 4
SECONDS, STEPS_DDIM, LC = 10, 50, 100
GF_DIT_XL_L500 = 786.7e9    # SURVEY Appendix A: algorithmic FLOPs of one XL DiT forward per sample (L=500, Lc=100)
GF_VAE_10S = 499.4e9        # SURVEY Appendix C: VAE decode per 10-s clip
GF_CN_XL_L500 = 1167.8e9    # DiT + ControlNet (14 in-blocks + 14 zero-linears) per sample-forward (SURVEY 8d)
GF_DIT_XL_L1500 = 2528e9    # one XL forward per sample at L = 1500 (self-attention grows 9x)
GF_VAE_ENC_10S = 499.3e9


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(burst=d["bf16_tflops"], sustained=d["bf16_tflops_sustained"], hbm=d["hbm_gbs"], src="measured (MEASURED_PEAKS.json)")
    return dict(burst=989.0, sustained=989.0, hbm=3350.0, src="NVIDIA H100 SXM data sheet (dense BF16, HBM3; a ceiling, not a measured rate)")


class ClockSampler:
    def __init__(self, idx):
        q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.p = subprocess.Popen(["nvidia-smi", "-i", str(idx), f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "200"],
                                      stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except Exception:
            self.p = None

    def stop(self):
        if self.p is None:
            return None
        self.p.terminate()
        try:
            out = self.p.communicate(timeout=5)[0]
        except Exception:
            return None
        sm, mx, reasons = [], 0, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for line in out.strip().splitlines():
            f = [x.strip() for x in line.split(",")]
            if len(f) < 6:
                continue
            try:
                sm.append(float(f[0])); mx = max(mx, float(f[1]))
            except ValueError:
                continue
            for n, v in zip(names, f[2:6]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        if not sm:
            return None
        busy = [x for x in sm if x > 0.5 * max(sm)] or sm
        return dict(sm_mhz=statistics.median(busy), sm_max_mhz=mx, reasons=sorted(reasons), samples=len(sm))


def pick_threads():
    """'All the host threads it can use': the fastest of a few thread counts on a GEMM probe (oversubscribing a cgroup-limited box makes
    torch CPU slower, not faster)."""
    avail = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else os.cpu_count()
    a_ = torch.randn(2048, 1152)
    b_ = torch.randn(1152, 4608)
    best, threads = None, avail
    for n in sorted({8, 16, 32, 64, avail}):
        if n > avail:
            continue
        torch.set_num_threads(n)
        a_ @ b_
        t0 = time.perf_counter()
        for _ in range(3):
            a_ @ b_
        dt = time.perf_counter() - t0
        if best is None or dt < best:
            best, threads = dt, n
    return threads, avail


def cpu_reference_leg(steps=1, warmup=0, threads=None):
    """The reference algorithm's own CPU path (oracle port: torch fp32, all host threads).  One STEP = a bounded sample of the job: one XL
    DiT forward at effective batch 2 (one prompt with CFG) and one VAE decode of 2 s; the job cost is extrapolated from the mean sample
    (50 forwards + 5 x the 2-s decode per 10-s clip; the per-step cost does not depend on t).  `warmup` untimed samples, then `steps` timed."""
    from ezaudio_b200 import synth, weights
    from oracle import ezaudio_oracle as O
    avail = None
    if threads is None:
        threads, avail = pick_threads()
    torch.set_num_threads(threads)
    cfg = synth.model_cfg("xl")
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 2)
    vsd = weights.synthetic_state_dict(weights.vae_decoder_param_shapes(synth.VAE_DECODER), 6)
    x = synth.synth_latents(2, 500)
    ctx, mask = synth.synth_context(2, LC, cfg["context_dim"])
    t = torch.tensor(479)
    z = synth.synth_latents(1, 100, 128, seed=31)
    fw, va = [], []
    with torch.no_grad():
        O.maskdit_forward(sd, cfg, x[:1], t, ctx[:1], mask[:1])  # page-in (half a sample)
        for i in range(max(0, warmup) + max(1, steps)):
            t0 = time.perf_counter()
            O.maskdit_forward(sd, cfg, x, t, ctx, mask)
            t1 = time.perf_counter()
            O.vae_decode(vsd, z)
            t2 = time.perf_counter()
            if i >= warmup:
                fw.append(t1 - t0)
                va.append(t2 - t1)
    t_fwd, t_vae = statistics.mean(fw), statistics.mean(va) * (SECONDS * 50 / 100)
    total = STEPS_DDIM * t_fwd + t_vae
    return dict(value=SECONDS / total, unit="audio-s/s", cores=threads, cores_available=avail, kind="port",
                sample=f"{len(fw)} timed sample(s) after {warmup} warm-up: 1 XL DiT forward (B_eff=2, L=500) = {t_fwd:.2f}s x{STEPS_DDIM} + VAE decode 2 s x5 = "
                       f"{t_vae:.2f}s; oracle port (torch fp32 CPU, {threads} threads)",
                t_fwd_s=t_fwd, t_vae_10s_s=t_vae, sample_seconds=sum(fw) + sum(va))


def timed_ms(fn, reps, warm=1):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def dit_xl_parity(unet, dev):
    """max / mean-abs of one XL DiT forward against the UNMODIFIED reference's output on the same weights and inputs (tests/golden/dit_XL.npz,
    written by oracle/gen_golden.py from /root/reference; a committed fixture, nothing under oracle/ is touched here)."""
    import numpy as np
    from ezaudio_b200 import synth
    g = np.load(os.path.join(ROOT, "tests", "golden", "dit_XL.npz"))
    B, L, Lc = int(g["B"]), int(g["L"]), int(g["Lc"])
    x = synth.synth_latents(B, L)
    ctx, mask = synth.synth_context(B, Lc, 2048)
    mask[-1] = False
    mask[-1, 0] = True
    out, _ = unet(x.to(dev), torch.from_numpy(g["t"]), ctx.to(dev), context_mask=mask.to(dev))
    err = (out.cpu() - torch.from_numpy(g["out"])).abs()
    return dict(max_abs=float(err.max()), mean_abs=float(err.mean()), ref_std=float(torch.from_numpy(g["out"]).std()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--precision", default="bf16", choices=["bf16", "bf16x3"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-cfg", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip the parity / bf16x3 / C4 / C5 legs")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's waveforms (what the API returns) as DIR/wav.npy, float32")
    a = ap.parse_args()
    if a.steps < 1 or a.warmup < 0:
        ap.error("--steps must be at least 1 and --warmup at least 0")
    # stdout carries exactly ONE JSON line: library banners (e.g. "NCCL version ...") are sent to stderr
    sys.stdout.flush()
    real_stdout = os.dup(1)
    os.dup2(2, 1)

    def emit(line):
        sys.stdout.flush()
        os.write(real_stdout, (json.dumps(line) + "\n").encode())

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    config = dict(workload=f"C2/C3: EzAudio-XL, {STEPS_DDIM}-step DDIM, {SECONDS} s, {PROMPTS_PER_GPU} prompts/GPU, "
                           f"{'no CFG' if a.no_cfg else 'CFG 5.0 / rescale 0.75 (effective batch 8)'}, eta 1, cached T5 embeddings, + VAE decode",
                  prompts_per_gpu=PROMPTS_PER_GPU, global_prompts=PROMPTS_PER_GPU * max(world, a.gpus), parallelism=f"prompt-sharded dp{max(world, a.gpus)}",
                  weights="synthetic random-init (seed 2), all zero-init tensors re-drawn", cache="weights 1.75 GB bf16 streamed per DiT step >> 50 MB L2 (no flush needed)")
    base = dict(metric="audio-seconds generated per wall-second (EzAudio-XL, 50-step DDIM, 10 s)", unit="audio-s/s", n_gpus=max(world, a.gpus),
                steps=a.steps, warmup=a.warmup, higher_is_better=True, scaling="weak", vs_baseline=None, data="synthetic", config=config)

    if a.impl == "reference":
        if rank != 0:
            return
        cb = cpu_reference_leg(steps=a.steps, warmup=a.warmup)
        line = dict(base, impl="reference", value=cb["value"], ms_per_step=1e3 * cb["sample_seconds"] / max(1, a.steps), dtype="f32", cpu_baseline=cb,
                    projected_ms_per_job=1e3 * SECONDS / cb["value"],
                    e2e=dict(value=cb["value"], unit="audio-s/s", h2d_bytes_per_step=0, d2h_bytes_per_step=0), gpu_launches=0, n_gpus=max(world, a.gpus))
        emit(line)
        return

    from ezaudio_b200 import _lib, api, synth
    from ezaudio_b200.inference import inference, sample_latents
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    B = PROMPTS_PER_GPU
    # public API object (reference-facing): synthetic checkpoint + cached-T5 stand-in returning PINNED HOST tensors
    enc = api.SyntheticTextEncoder(2048, LC)

    def host_encoder(prompts):
        e, m = enc(prompts)
        return e.pin_memory(), m.pin_memory()

    ez = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", device=dev, text_encoder=host_encoder, precision=a.precision, max_batch=B,
                     max_length_s=SECONDS)
    prompts = [f"synthetic prompt number {rank * B + i} with a dog barking and rain" for i in range(B)]
    gs, gr = (None, 0.0) if a.no_cfg else (5, 0.75)
    L = SECONDS * 50
    te, tm = enc(prompts)
    ue, um = enc([""])
    te, tm, ue, um = te.to(dev), tm.to(dev), ue.to(dev), um.to(dev)

    def step_resident(model=None, use_graphs=True):
        m = model or ez
        lat = sample_latents(m.unet, m.noise_scheduler, te, tm, ue, um, None, None, L, gs, gr, STEPS_DDIM, 1, 2024 + rank * B, device=dev,
                             use_graphs=use_graphs)
        return m.autoencoder(embedding=lat)

    def step_e2e():
        if a.no_cfg:
            embeds = ez._text_embeds(prompts, [""])
            return inference(ez.autoencoder, ez.unet, None, None, None, None, ez.params, ez.noise_scheduler, prompts, None, L, None, 0.0, STEPS_DDIM, 1,
                             2024, dev, text_embeds=embeds).cpu().numpy()
        return ez.generate_audio(prompts, length=SECONDS, guidance_scale=5, guidance_rescale=0.75, ddim_steps=STEPS_DDIM, eta=1, random_seed=2024)

    def sync_all():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
            torch.cuda.synchronize()

    for _ in range(a.warmup):
        step_resident()
    sync_all()
    Lb = _lib.lib()
    n0 = Lb.ezb_launch_count()
    clocks = ClockSampler(local)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        wav = step_resident()
    e1.record()
    sync_all()
    ms = e0.elapsed_time(e1)
    clk = clocks.stop()
    launches = int(Lb.ezb_launch_count() - n0)
    assert torch.isfinite(wav).all()
    if a.dump_outputs and rank == 0:   # fixed seeds and synthetic weights: the same arguments give the same inputs on every run
        import numpy as np
        os.makedirs(a.dump_outputs, exist_ok=True)
        np.save(os.path.join(a.dump_outputs, "wav.npy"), wav.float().cpu().numpy())
    # ---- end to end through the public API (host buffers in / out)
    step_e2e()
    sync_all()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        step_e2e()
    sync_all()
    ms_e2e = (time.perf_counter() - t0) * 1e3
    if dist is not None:
        t = torch.tensor([ms, ms_e2e], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms, ms_e2e = float(t[0]), float(t[1])
    n_e = 1 if a.no_cfg else 2
    h2d = (B + 1) * LC * 2048 * 4 + (B + 1) * LC
    d2h = B * L * 480 * 4
    pk = peaks()
    reps = max(1, min(a.steps, 2))

    # ---- C5 (30-s inpainting): two prompts per GPU; with >= 2 GPUs ranks 0 and 1 run it side by side (BASELINE: batch 4 on 2 GPUs)
    c5 = None
    if not a.no_extras and (world == 1 or rank < 2):
        Bc, Lc5 = 2, 1500
        ez5 = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", device=dev, text_encoder=enc, precision=a.precision, max_batch=Bc,
                          max_length_s=30)
        audio = 0.1 * torch.randn(Bc, 1, 480 * Lc5, generator=torch.Generator().manual_seed(9 + rank)).to(dev)
        p5 = [f"synthetic prompt {rank * Bc + i}" for i in range(Bc)]
        embeds5 = ez5._text_embeds(p5, [""])

        def job5():
            gt = ez5.autoencoder(audio=audio)
            mask = torch.zeros(Bc, 128, Lc5, device=dev, dtype=torch.bool)
            mask[:, :, 250:1250] = True
            return inference(ez5.autoencoder, ez5.unet, gt, mask, None, None, ez5.params, ez5.noise_scheduler, p5, None, Lc5, 3.5, 0.0, 100, 1, 2024, dev,
                             text_embeds=embeds5).cpu()

        ms5, out5 = timed_ms(job5, reps)
        assert out5.shape == (Bc, 1, 480 * Lc5) and torch.isfinite(out5).all()
        c5 = ms5
        del ez5, out5
        torch.cuda.empty_cache()
    if dist is not None and not a.no_extras:
        t = torch.tensor([c5 if c5 is not None else 0.0], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        c5 = float(t[0])

    # ---- dominant kernel (wgmma GEMM): CUDA-event timed per launch over one instrumented generation on rank 0
    roof = None
    if rank == 0:
        _lib.check(Lb.ezb_prof_gemm_begin())
        step_resident(use_graphs=False)  # eager launches so that every GEMM passes the event-timing hook
        nl, fl, tms = C.c_int(), C.c_double(), C.c_double()
        _lib.check(Lb.ezb_prof_gemm_end(C.byref(nl), C.byref(fl), C.byref(tms)))
        ach_all = fl.value / (tms.value * 1e-3) / 1e12
        all_gemm = dict(achieved=ach_all, unit="TFLOP/s", frac=ach_all / pk["sustained"], launches=nl.value, gemm_share_of_step=tms.value / (ms / a.steps))
        # dominant kernel: the GEGLU MLP-in GEMM (largest launch: M = 8 x 500 tokens, N = 9216, K = 1152), 128 x 256 tiles in 2-CTA clusters
        gf = 2.0 * (B * n_e * L) * 9216 * 1152
        n2, f2, t2 = C.c_int(), C.c_double(), C.c_double()
        _lib.check(Lb.ezb_prof_gemm_stats(0.99 * gf, C.byref(n2), C.byref(f2), C.byref(t2)))
        ach = f2.value / (t2.value * 1e-3) / 1e12 if n2.value else 0.0
        roof = dict(bound="tensor", kernel="gemm_wgmma_kernel<256, EpiGeglu<256>, 2> (GEGLU MLP-in GEMM, 2-CTA clusters sharing the W tile: M=%d N=9216 K=1152)" % (B * n_e * L),
                    achieved=ach, peak=pk["sustained"], unit="TFLOP/s", frac=ach / pk["sustained"],
                    peak_source=pk["src"] + ", sustained figure (kernel timed inside a long step)",
                    compulsory_bytes="A 9.2 MB + W 21.2 MB read, 36.9 MB bf16 output written",
                    launches=n2.value, flops_per_launch=gf, ms_per_launch=t2.value / max(1, n2.value), share_of_step=t2.value / (ms / a.steps),
                    how="CUDA events around every GEMM launch on the launch stream during one extra instrumented (eager, non-graph) generation",
                    all_gemm_launches=all_gemm)
    if rank != 0:
        if dist is not None:
            dist.destroy_process_group()
        return
    total_audio = SECONDS * B * max(world, 1)
    value = total_audio * a.steps / (ms * 1e-3)
    job_flops = (STEPS_DDIM * n_e * B * GF_DIT_XL_L500 + B * GF_VAE_10S) * max(world, 1)
    line = dict(base, impl="ours", value=value, ms_per_step=ms / a.steps, dtype=a.precision,
                dit_step_ms=None, clocks=clk, gpu_launches=launches,
                e2e=dict(value=total_audio * a.steps / (ms_e2e * 1e-3), unit="audio-s/s", h2d_bytes_per_step=h2d, d2h_bytes_per_step=d2h,
                         api="EzAudio.generate_audio(list[str]) with pinned host T5 embeddings; waveform .cpu().numpy()"),
                roofline=roof,
                job_tensor_roofline_frac=job_flops * a.steps / (ms * 1e-3) / 1e12 / (pk["sustained"] * max(world, 1)),
                job_algorithmic_tflop_per_step=job_flops / 1e12)
    # DiT-step ms: one denoiser forward (+CFG/DDIM update) inside the loop
    ez.unet.set_context(torch.cat([te, ue.expand(B, -1, -1)], 0) if not a.no_cfg else te, torch.cat([tm, um.expand(B, -1)], 0) if not a.no_cfg else tm)
    ez.unet.set_timesteps([int(t) for t in ez.noise_scheduler.timesteps])
    xin = torch.randn(B * n_e, 128, L, device=dev)
    for _ in range(3):
        ez.unet.forward_step(xin, 0)
    torch.cuda.synchronize()
    e0.record()
    for i in range(10):
        ez.unet.forward_step(xin, i)
    e1.record()
    torch.cuda.synchronize()
    line["dit_step_ms"] = e0.elapsed_time(e1) / 10

    if not a.no_extras:
        cfgs = {}
        if c5 is not None:
            n5 = 2 if world >= 2 else 1
            tf5 = n5 * (100 * 4 * GF_DIT_XL_L1500 + 2 * (GF_VAE_10S + GF_VAE_ENC_10S) * 3) / 1e12
            cfgs["C5"] = dict(workload=f"XL inpainting (editing path), 30 s (L=1500), 100 steps, CFG 3.5, VAE encode + decode, host waveform out; 2 prompts per GPU on {n5} GPU(s)"
                                       + ("" if n5 == 2 else " (BASELINE quotes batch 4 on 2 GPUs: launch with --gpus >= 2 for that)"),
                              n_gpus=n5, ms_per_job=c5, audio_s_per_s=n5 * 60 / (c5 * 1e-3), algorithmic_tflop=tf5,
                              tensor_roofline_frac=tf5 / (c5 * 1e-3) / (pk["sustained"] * n5), reps=reps, timing="CUDA events, max over the participating ranks")
        if world == 1:
            # ---- parity block + bf16x3 throughput (the mode that meets north_star's 1e-3) on the same C2/C3 workload
            par = {a.precision: dict(dit_XL_vs_reference=dit_xl_parity(ez.unet, dev), audio_s_per_s=value)}
            other = "bf16x3" if a.precision == "bf16" else "bf16"
            del ez
            torch.cuda.empty_cache()
            ezo = api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", device=dev, text_encoder=enc, precision=other, max_batch=B,
                              max_length_s=SECONDS)
            po = dit_xl_parity(ezo.unet, dev)
            mso, wo = timed_ms(lambda: step_resident(ezo), reps)
            assert torch.isfinite(wo).all()
            par[other] = dict(dit_XL_vs_reference=po, audio_s_per_s=SECONDS * B / (mso * 1e-3), ms_per_job=mso, reps=reps)
            par["note"] = ("per-step DiT output vs the unmodified reference's fp32 output on identical weights / inputs (tests/golden/dit_XL.npz); "
                           "north_star's 1e-3 is met by bf16x3 (split-bf16 operands, 3x the GEMM work); plain bf16 operands sit at the dtype's floor "
                           "(the reference's own bf16-autocast path: 4.4e-2..5.5e-2 max-abs)")
            line["parity"] = par
            del ezo, wo
            torch.cuda.empty_cache()
            # ---- C4: XL + energy ControlNet, 8 prompts, CFG 3.5 (effective batch 16), through EzAudio_ControlNet.generate_audio (host in / out)
            import numpy as np
            from ezaudio_b200 import config as ezcfg
            B4 = 8
            params = dict(ezcfg.BUILTIN_CONTROLNET["energy"], model_name="EzAudio-XL", model=synth.XL_MODEL,
                          text_encoder=dict(model="google/flan-t5-xl", max_length=100, cfg=0.1))
            cn = api.EzAudio_ControlNet("energy", ckpt_path="synthetic:2", controlnet_path="synthetic:3", vae_path="synthetic:6", device=dev,
                                        text_encoder=enc, precision=a.precision, max_batch=B4, params=params)
            wave = (0.1 * torch.randn(240000, generator=torch.Generator().manual_seed(9))).numpy()
            p4 = [f"synthetic prompt {i}" for i in range(B4)]
            t0 = time.perf_counter()
            cn.generate_audio(p4, wave, guidance_scale=3.5, guidance_rescale=0, ddim_steps=50, eta=1, conditioning_scale=1, random_seed=2024)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(reps):
                out4 = cn.generate_audio(p4, wave, guidance_scale=3.5, guidance_rescale=0, ddim_steps=50, eta=1, conditioning_scale=1, random_seed=2024)
            torch.cuda.synchronize()
            ms4 = (time.perf_counter() - t0) * 1e3 / reps
            assert len(out4[1]) == B4 and all(np.isfinite(w).all() for w in out4[1])
            tf4 = (50 * 2 * B4 * GF_CN_XL_L500 + B4 * GF_VAE_10S) / 1e12
            cfgs["C4"] = dict(workload="XL + energy ControlNet, 50 steps, 8 prompts, CFG 3.5 (effective batch 16), 10 s, via EzAudio_ControlNet.generate_audio "
                                       "(host waveform in, host waveforms out; wall clock around the API call)",
                              n_gpus=1, ms_per_job=ms4, audio_s_per_s=10 * B4 / (ms4 * 1e-3), algorithmic_tflop=tf4,
                              tensor_roofline_frac=tf4 / (ms4 * 1e-3) / pk["sustained"], reps=reps)
            del cn
            torch.cuda.empty_cache()
        line["configs"] = cfgs
    if not a.no_cpu_baseline and world == 1:
        line["cpu_baseline"] = cpu_reference_leg()
    emit(line)
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
