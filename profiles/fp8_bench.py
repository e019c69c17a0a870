"""FP8 mode against bf16 on the C2 job (EzAudio-XL, 50-step DDIM with CFG 5 / rescale 0.75, 4 prompts x 10 s, + VAE decode), one JSON line.

Both modes are built in the same process from the same synthetic checkpoint and alternated `--reps` times each (other work shares the host and
the card), then:
  * audio-s/s of the whole job (CUDA events around sampling + decode, the same window as bench.py's resident leg) and the DiT step time
    (one forward at the job's effective batch 8, L = 500);
  * CUDA-event times of the two FP8 projection classes and their bf16 counterparts at M = 4000 and 8000 tokens (the kernels the model
    launches, through the test hooks; the library's per-GEMM events time the GEMM launch alone), with TFLOP/s on the tile FLOPs against the
    data-sheet dense peaks (989 bf16, 1979 FP8 TFLOP/s; ceilings, not measured rates);
  * the FP8 mode's max / mean error against the reference's golden XL forward (tests/golden/dit_XL.npz);
  * the card's name, power limit and SM clock, read in the same run.
    python profiles/fp8_bench.py [--reps 3] [--out fp8_bench.json]"""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK = {"bf16": 989.0, "fp8": 1979.0}
B, SECONDS, STEPS, LC = 4, 10, 50, 100


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout
        return dict(zip(q.split(","), [f.strip() for f in out.strip().splitlines()[0].split(",")]))
    except Exception as e:   # the numbers then lack their context: say so in the record
        return dict(error=repr(e))


def prof(fn, reps):
    """Mean CUDA-event time (ms) and tile FLOPs of the one GEMM launch fn() makes."""
    from ezaudio_b200 import _lib
    L = _lib.lib()
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    L.ezb_prof_gemm_begin()
    for _ in range(reps):
        fn()
    n, f, ms = C.c_int(), C.c_double(), C.c_double()
    _lib.check(L.ezb_prof_gemm_end(C.byref(n), C.byref(f), C.byref(ms)))
    assert n.value == reps, n.value
    return ms.value / reps, f.value / reps


def projections(M, reps):
    """GEGLU (D 1152 -> 2 x 4608) and packed QKV (D 1152, 16 heads of 72) at M tokens, bf16 and FP8 kernels."""
    from ezaudio_b200 import _lib
    from tests.test_heads_gpu import PACKED3, ROPE_MUFU, _dvp, _lpad
    L = _lib.lib()
    D, inner, H, dh = 1152, 4608, 16, 72
    Lc = 500 if M % 500 == 0 else M
    Bc = M // Lc
    g = torch.Generator(device="cuda").manual_seed(M)
    x = torch.randn(M, D, device="cuda", generator=g)
    ln_w, ln_b = torch.ones(D, device="cuda"), torch.zeros(D, device="cuda")
    q8 = torch.empty(M, D, dtype=torch.uint8, device="cuda")
    s8 = torch.empty(M, device="cuda")
    _lib.check(L.ezb_test_fp8(0, C.byref(_lib.TestFp8Args(kind=0, M=M, D=D, x=x.data_ptr(), weight=ln_w.data_ptr(), bias=ln_b.data_ptr(),
                                                           q=q8.data_ptr(), s=s8.data_ptr())), _lib.stream_ptr()))
    A16 = x.bfloat16()
    out = {}
    # GEGLU
    W1 = torch.randn(2 * inner, D, device="cuda", generator=g) / math.sqrt(D)
    b1 = torch.zeros(2 * inner, device="cuda")
    W1p = W1.bfloat16()   # layout does not matter for timing
    mid = torch.empty(M, inner, dtype=torch.bfloat16, device="cuda")
    e = _lib.TestEpilogue()
    e.bias, e.out_bf16, e.ld16 = b1.data_ptr(), mid.data_ptr(), inner
    st = _lib.stream_ptr()
    bf = prof(lambda: L.ezb_test_gemm(0, _lib.ptr(A16), D, _lib.ptr(W1p), D, M, 2 * inner, D, 256, 11, C.byref(e), 0, 0, 0, 0, 0, 0, st), reps)
    a8 = _lib.TestFp8Args(kind=1, M=M, D=D, q=q8.data_ptr(), s=s8.data_ptr(), inner=inner, w=W1.data_ptr(), b=b1.data_ptr(), out=mid.data_ptr())
    f8 = prof(lambda: L.ezb_test_fp8(0, C.byref(a8), st), reps)
    out["geglu"] = {k: dict(ms=v[0], tflops=v[1] / v[0] / 1e9, share_of_peak=v[1] / v[0] / 1e9 / PEAK[k]) for k, v in (("bf16", bf), ("fp8", f8))}
    # packed QKV with the heads epilogue
    W = torch.randn(3 * D, D, device="cuda", generator=g) / math.sqrt(D)
    nq = torch.stack([torch.ones(dh, device="cuda"), torch.zeros(dh, device="cuda")]).contiguous()
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dh, 2, device="cuda", dtype=torch.float32) / dh))
    qo = torch.empty(Bc * H, Lc, 80, dtype=torch.bfloat16, device="cuda")
    ko = torch.empty_like(qo)
    vt = torch.empty(Bc * H, _dvp(dh), _lpad(Lc), dtype=torch.bfloat16, device="cuda")
    h = _lib.TestHeadsArgs()
    h.B, h.L, h.D, h.H, h.dh, h.nsec = Bc, Lc, D, H, dh, 3
    for i in range(3):
        h.kinds[i] = i
    h.norm_q = h.norm_k = nq.data_ptr()
    h.inv_freq, h.rope = inv_freq.data_ptr(), ROPE_MUFU
    h.q, h.k, h.vt = qo.data_ptr(), ko.data_ptr(), vt.data_ptr()
    h.ld_qk, h.dvp, h.Lpad, h.variant = 80, _dvp(dh), _lpad(Lc), PACKED3
    bf = prof(lambda: L.ezb_test_heads(0, _lib.ptr(A16), _lib.ptr(W), C.byref(h), st), reps)
    a8 = _lib.TestFp8Args(kind=2, M=M, D=D, q=q8.data_ptr(), s=s8.data_ptr(), w=W.data_ptr(), B=Bc, L=Lc, H=H, dh=dh, norm_q=nq.data_ptr(),
                          norm_k=nq.data_ptr(), inv_freq=inv_freq.data_ptr(), rope=ROPE_MUFU, q_out=qo.data_ptr(), k_out=ko.data_ptr(),
                          vt_out=vt.data_ptr(), ld_qk=80, dvp=_dvp(dh), Lpad=_lpad(Lc))
    f8 = prof(lambda: L.ezb_test_fp8(0, C.byref(a8), st), reps)
    out["qkv"] = {k: dict(ms=v[0], tflops=v[1] / v[0] / 1e9, share_of_peak=v[1] / v[0] / 1e9 / PEAK[k]) for k, v in (("bf16", bf), ("fp8", f8))}
    for k in out:
        out[k]["fp8_speedup"] = out[k]["bf16"]["ms"] / out[k]["fp8"]["ms"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from ezaudio_b200 import api
    from ezaudio_b200.inference import sample_latents
    import bench
    dev = torch.device("cuda", 0)
    enc = api.SyntheticTextEncoder(2048, LC)
    ez = {p: api.EzAudio("s3_xl", ckpt_path="synthetic:2", vae_path="synthetic:6", device=dev, text_encoder=enc, precision=p, max_batch=B,
                         max_length_s=SECONDS) for p in ("bf16", "fp8")}
    prompts = [f"synthetic prompt number {i} with a dog barking and rain" for i in range(B)]
    te, tm = (t.to(dev) for t in enc(prompts))
    ue, um = (t.to(dev) for t in enc([""]))
    Lf = SECONDS * 50

    def job(p):
        m = ez[p]
        lat = sample_latents(m.unet, m.noise_scheduler, te, tm, ue, um, None, None, Lf, 5, 0.75, STEPS, 1, 2024, device=dev)
        return m.autoencoder(embedding=lat)

    def dit_step(p):
        return ez[p].unet.forward_step(x8, 0)

    for p in ez:
        job(p)
    torch.cuda.synchronize()
    card_before = card()
    runs = {p: [] for p in ez}
    for _ in range(a.reps):
        for p in ez:
            ms, wav = bench.timed_ms(lambda: job(p), 1, warm=0)
            assert torch.isfinite(wav).all()
            runs[p].append(B * SECONDS / (ms / 1e3))
    # one DiT forward at the job's shape (effective batch 8 = 4 prompts + 4 unconditional rows, L = 500)
    x8 = torch.randn(2 * B, 128, Lf, device=dev)
    ctx8 = torch.cat([te, ue.expand(B, -1, -1)]).contiguous()
    msk8 = torch.cat([tm, um.expand(B, -1)]).contiguous()
    step_ms = {}
    for p in ez:
        ez[p].unet.set_context(ctx8, msk8)
        ez[p].unet.set_timesteps([479])
        step_ms[p] = bench.timed_ms(lambda: dit_step(p), 20, warm=3)[0]
    proj = {M: projections(M, 20) for M in (4000, 8000)}
    parity = bench.dit_xl_parity(ez["fp8"].unet, dev)
    line = dict(workload="C2: EzAudio-XL, 50-step DDIM, CFG 5 / rescale 0.75, 4 prompts x 10 s, + VAE decode; synthetic weights (seed 2)",
                audio_s_per_s={p: dict(runs=runs[p], median=statistics.median(runs[p]), spread=max(runs[p]) - min(runs[p])) for p in runs},
                dit_step_ms=step_ms, projections_ms=proj, fp8_vs_dit_XL_golden=parity,
                peaks_tflops=dict(PEAK, src="NVIDIA H100 SXM data sheet, dense (a ceiling at 700 W, not a measured rate)"),
                card_before=card_before, card_after=card())
    s = json.dumps(line)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
