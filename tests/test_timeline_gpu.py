"""Timelines of prompts on the GPU: the timeline gather, guide and blend kernels against a torch index gather, ezb_cfg_ddim_step and fp64
(NaN wherever they must not read, sentinels wherever they must not write), a one-segment timeline against generate_long_audio (and
generate_audio when it fits one window), bit for bit, the loop against the oracle's DiT driven by an fp64 restatement of gather / guide /
blend / update, batches against solo calls, graph replay on new boundaries and prompts, and the row capacity."""
import ctypes
import gc

import numpy as np
import pytest
import torch

from ezaudio_b200 import _lib, synth, weights
from ezaudio_b200.inference import check_timeline, long_plan
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
from oracle import ezaudio_oracle as O

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
LW, OV = 40, 8   # the kernel tests' window and overlap


def _dev(rows):
    return torch.tensor([e for row in rows for e in row], dtype=torch.int32, device="cuda")


def _timeline(lens, Lw, O_, T, seed, extra=2):
    """Random timelines covering each clip: cuts in timeline order plus `extra` overlapping segments; returns the plan and device tables."""
    rng = np.random.default_rng(seed)
    segs = []
    for n in lens:
        cuts = sorted(set([0, n] + ([int(c) for c in rng.integers(1, n, size=3)] if n > 1 else [])))
        s = [(a, b) for a, b in zip(cuts, cuts[1:])]
        for _ in range(extra):
            a = int(rng.integers(0, n))
            s.append((a, int(rng.integers(a + 1, n + 1))))
        segs.append(s)
    lens, table, windows, rows, spans = check_timeline(segs, lens, len(lens), Lw, O_, T, True, 10 ** 6, Lw)
    trows = [(k, *segs[b][q], T) for k, b, q in rows]
    return segs, table, windows, rows, spans, trows


# ---------------------------------------------------------------- kernels
@pytest.mark.parametrize("C_", [16, 128])
def test_timeline_gather_against_index_gather(C_):
    Lw, O_, T = 40, 8, 5
    lens = [73, 37, 130, 40, 1]
    _, table, windows, rows, _, trows = _timeline(lens, Lw, O_, T, 1)
    B, W, R, N = len(lens), len(windows), len(rows), max(lens)
    g = torch.Generator().manual_seed(4)
    lat = torch.randn(B, C_, N, generator=g)
    for b, n in enumerate(lens):
        lat[b, :, n:] = float("nan")   # past a clip's end: never read
    lat_d, plan, rows_d = lat.cuda(), _dev(table), _dev(trows)
    L, st = _lib.lib(), _lib.stream_ptr()
    for uncond in (0, 1):
        n_out = R + W * uncond
        win = torch.full((n_out + 1, C_, Lw), 7.0, device="cuda")   # a sentinel row past the last written one
        _lib.check(L.ezb_timeline_gather(0, _lib.ptr(lat_d), _lib.ptr(win), _lib.ptr(plan), _lib.ptr(rows_d), B, C_, N, W, R, Lw, O_, uncond, st))
        got = win.cpu()
        src = [k for k, _, _ in rows] + (list(range(W)) if uncond else [])
        idx = torch.tensor([[b * N + s + j if j < ln else B * N for j in range(Lw)] for b, s, ln in (windows[k] for k in src)])
        flat = torch.cat([lat.transpose(0, 1).reshape(C_, -1), torch.zeros(C_, 1)], 1)   # (C, B * N + 1): the last column is the zero pad
        want = flat[:, idx].permute(1, 0, 2)
        assert torch.equal(got[:n_out], want), uncond
        assert torch.equal(got[n_out], torch.full((C_, Lw), 7.0))


def _ddim_pair(t, u, ln, gs, gr):
    """ezb_cfg_ddim_step with coefficients (1, 0, 0, 1, 0) on the pair [t | u] over ln frames: the guided v."""
    Cc, Lw = t.shape
    pair = torch.stack([t, u]).contiguous()
    x = torch.zeros(1, Cc, Lw, device="cuda")
    lens = torch.tensor([ln], dtype=torch.int32, device="cuda")
    coef = (1.0, 0.0, 0.0, 1.0, 0.0)
    _lib.check(_lib.lib().ezb_cfg_ddim_step(0, _lib.ptr(pair), _lib.ptr(x), None, 1, Cc, Lw, gs, gr, (ctypes.c_float * 5)(*coef), _lib.stream_ptr(),
                                            _lib.ptr(lens)))
    return x[0]


def _cfg64(t, u, gs, gr):
    t, u = t.double(), u.double()
    v = u + gs * (t - u)
    if gr > 0:
        v = gr * v * (t.std() / v.std()) + (1 - gr) * v
    return v


@pytest.mark.parametrize("gr", [0.0, 0.7])
def test_timeline_guide_equals_cfg_ddim_step_on_each_pair(gr):
    Lw, O_, T, C_, gs = 40, 8, 6, 128, 3.0
    lens = [73, 37, 25]   # the last two clips are one short window each: window lengths below Lw
    _, table, windows, rows, _, trows = _timeline(lens, Lw, O_, T, 2)
    W, R = len(windows), len(rows)
    assert R > W   # some windows' rows share an uncond row
    g = torch.Generator().manual_seed(9)
    out = torch.randn(R + W, C_, Lw, generator=g).cuda()
    wl = [windows[k][2] for k, _, _ in rows]
    assert min(wl) < Lw
    lens_d, rows_d = torch.tensor(wl, dtype=torch.int32, device="cuda"), _dev(trows)
    guided = torch.zeros(R + 1, C_, Lw, device="cuda")
    guided[R] = 7.0   # a sentinel row past R
    _lib.check(_lib.lib().ezb_timeline_guide(0, _lib.ptr(out), _lib.ptr(guided), _lib.ptr(rows_d), _lib.ptr(lens_d), R, W, C_, Lw, gs, gr,
                                             _lib.stream_ptr()))
    assert torch.equal(guided[R], torch.full((C_, Lw), 7.0, device="cuda"))
    worst = 0.0
    for r, (k, _, _) in enumerate(rows):
        ln = wl[r]
        want = _ddim_pair(out[r], out[R + k], ln, gs, gr)
        assert torch.equal(guided[r], want), r   # the same bits, zeros past the window's length included
        ref = _cfg64(out[r, :, :ln].cpu(), out[R + k, :, :ln].cpu(), gs, gr)
        scale = float((out[r, :, :ln].abs() + out[R + k, :, :ln].abs()).max())
        err = float((guided[r, :, :ln].cpu().double() - ref).abs().max())
        worst = max(worst, err / scale)
        assert err <= 8 * (1 + gs) * EPS * scale, (r, err)   # the CFG's roundings, the fp32 rescale ratio and its two products
    print(f"[timeline] guide vs fp64 CFG + rescale (gr {gr}): max-abs error {worst:.2e} x max(|t| + |u|)")


def _blend64(wins, table, windows, rows, trows, lens):
    """fp64 restatement: per clip, sum w_k(j) a(f) v_r(j) / sum w_k(j) a(f) over the rows covering f; and how many rows cover f."""
    res, cover, weight1 = [], [], []
    for b, (first, count, n) in enumerate(table):
        num, den, cnt = np.zeros((wins.shape[1], n)), np.zeros(n), np.zeros(n, dtype=int)
        one = np.zeros(n, dtype=bool)
        for r, ((k, rb, _), (_, s, e, T)) in enumerate(zip(rows, trows)):
            if rb != b:
                continue
            _, s0, ln = windows[k]
            j = np.arange(ln, dtype=np.float64)
            w = np.ones(ln)
            O1 = OV + 1
            if k > first:
                w = np.minimum(w, (j + 1) / O1)
            if k < first + count - 1:
                w = np.minimum(w, (LW - j) / O1)
            f = s0 + np.arange(ln)
            a = np.where((f >= s - T) & (f < e + T), np.minimum(1.0, np.minimum((f - s + T + 1) / (T + 1), (e + T - f) / (T + 1))), 0.0)
            pos = a > 0
            num[:, f[pos]] += (w * a)[pos] * wins[r, :, :ln][:, pos].astype(np.float64)
            den[f[pos]] += (w * a)[pos]
            cnt[f[pos]] += 1
            one[f[pos & (w * a == 1)]] = True
        res.append(num / den)
        cover.append(cnt)
        weight1.append(one & (cnt == 1))
    return res, cover, weight1


@pytest.mark.parametrize("C_,T", [(16, 5), (128, 5), (128, 0), (16, 40)])
def test_timeline_blend_against_fp64(C_, T):
    lens = [73, 37, 130, 40, 1]
    _, table, windows, rows, spans, trows = _timeline(lens, LW, OV, T, 3 + T)
    B, W, R, N = len(lens), len(windows), len(rows), max(lens)
    g = torch.Generator().manual_seed(5)
    wins = torch.randn(R, C_, LW, generator=g)
    for r, (k, _, _) in enumerate(rows):
        wins[r, :, windows[k][2]:] = float("nan")   # row frames past a window's length: never read
    out = torch.full((B, C_, N), 7.0, device="cuda")
    wins_d, plan, rows_d, spans_d = wins.cuda(), _dev(table), _dev(trows), _dev(spans)   # held until the launch has run
    _lib.check(_lib.lib().ezb_timeline_blend(0, _lib.ptr(wins_d), _lib.ptr(out), _lib.ptr(plan), _lib.ptr(rows_d), _lib.ptr(spans_d), B, C_, N, W,
                                             R, LW, OV, _lib.stream_ptr()))
    got = out.cpu()
    ref, cover, one = _blend64(wins.numpy(), table, windows, rows, trows, lens)
    vmax = float(np.nanmax(np.abs(wins.numpy())))
    worst, exact = 0, 0
    for b, n in enumerate(lens):
        assert torch.equal(got[b, :, n:], torch.full((C_, N - n), 7.0)), b   # past the clip's end: not written
        err = np.abs(got[b, :, :n].double().numpy() - ref[b])
        bound = (2 * cover[b] + 4) * EPS * vmax   # the fp32 weights and their product, a product and a sum per term, the division
        assert (err <= bound).all(), (b, float((err / bound).max()))
        worst = max(worst, float((err / (EPS * vmax)).max()))
        assert np.array_equal(got[b, :, :n].numpy()[:, one[b]], ref[b][:, one[b]].astype(np.float32)), b   # one row of weight 1: bit for bit
        exact += int(one[b].sum())
    assert exact > 0 or T >= LW   # a transition as long as the window leaves no frame to one row
    print(f"[timeline] blend (C {C_}, T {T}, up to {max(c.max() for c in cover)} rows per frame) vs fp64: {worst:.1f} ulp of max|v|")


@pytest.mark.parametrize("T", [0, 3, 100])
def test_one_segment_blend_equals_window_blend(T):
    C_, lens = 128, [73, 37, 130, 40, 1]
    table, windows = long_plan(lens, LW, OV)
    trows = [(k, 0, lens[b], T) for k, (b, _, _) in enumerate(windows)]
    spans = [(first, count) for first, count, _ in table]
    B, W, N = len(lens), len(windows), max(lens)
    wins = torch.randn(W, C_, LW, generator=torch.Generator().manual_seed(6)).cuda()
    a = torch.full((B, C_, N), 7.0, device="cuda")
    b_ = torch.full((B, C_, N), 7.0, device="cuda")
    L, st = _lib.lib(), _lib.stream_ptr()
    plan, rows_d, spans_d = _dev(table), _dev(trows), _dev(spans)
    _lib.check(L.ezb_window_blend(0, _lib.ptr(wins), _lib.ptr(a), _lib.ptr(plan), B, C_, N, W, LW, OV, st))
    _lib.check(L.ezb_timeline_blend(0, _lib.ptr(wins), _lib.ptr(b_), _lib.ptr(plan), _lib.ptr(rows_d), _lib.ptr(spans_d), B, C_, N, W, W, LW, OV, st))
    assert torch.equal(a, b_)


def test_timeline_kernels_reject_bad_arguments():
    L, st = _lib.lib(), _lib.stream_ptr()
    x = torch.zeros(64, device="cuda")
    p, rows, spans = _dev([(0, 1, 4)]), _dev([(0, 0, 4, 0), (0, 0, 4, 0)]), _dev([(0, 2)])
    lens = torch.full((2,), 4, dtype=torch.int32, device="cuda")
    ok = dict(B=1, C=1, N=4, W=1, R=2, Lw=4, O=1)

    def gather(rows_p=rows, uncond=1, **kw):
        a = {**ok, **kw}
        return L.ezb_timeline_gather(0, _lib.ptr(x), _lib.ptr(x), _lib.ptr(p), rows_p, a["B"], a["C"], a["N"], a["W"], a["R"], a["Lw"], a["O"],
                                     uncond, st)

    def blend(rows_p=rows, spans_p=spans, **kw):
        a = {**ok, **kw}
        return L.ezb_timeline_blend(0, _lib.ptr(x), _lib.ptr(x), _lib.ptr(p), rows_p, spans_p, a["B"], a["C"], a["N"], a["W"], a["R"], a["Lw"],
                                    a["O"], st)

    def guide(rows_p=rows, lens_p=lens, R=2, W=1, Lw=4):
        return L.ezb_timeline_guide(0, _lib.ptr(x), _lib.ptr(x), rows_p, _lib.ptr(lens_p) if lens_p is not None else None, R, W, 1, Lw, 3.0, 0.5,
                                    st)

    rp, sp = _lib.ptr(rows), _lib.ptr(spans)
    misaligned = ctypes.c_void_p(rows.data_ptr() + 4)
    assert gather(rp) == 0 and blend(rp, sp) == 0 and guide(rp) == 0
    torch.cuda.synchronize()
    for kw in (dict(O=0), dict(O=3), dict(W=0), dict(R=0), dict(B=2), dict(Lw=1), dict(C=0)):
        assert gather(rp, **kw) != 0 and blend(rp, sp, **kw) != 0, kw
    assert gather(rp, uncond=2) != 0 and gather(None) != 0 and gather(misaligned) != 0
    assert blend(rp, None) != 0 and blend(None, sp) != 0 and blend(misaligned, sp) != 0
    assert guide(None) != 0 and guide(rp, None) != 0 and guide(misaligned) != 0 and guide(rp, R=1, W=2) != 0 and guide(rp, Lw=0) != 0


# ---------------------------------------------------------------- the loop through the API
def _ez(monkeypatch, max_batch=8, precision="bf16"):
    from ezaudio_b200 import api, config
    from tests.test_api_gpu import _tiny_params
    tiny = _tiny_params()
    monkeypatch.setattr(config, "load_params", lambda name, path=None, table=None: tiny)
    return api.EzAudio("s3_xl", ckpt_path="synthetic:3", vae_path="synthetic:6", text_encoder=api.SyntheticTextEncoder(64, 16),
                       max_batch=max_batch, max_length_s=2, precision=precision)


SAMPLERS = [("ddim", 0.0), ("ddim", 1.0), ("dpmsolver++", 1.0), ("sde-dpmsolver++", 1.0)]


def _set_sampler(ez, alg):
    ez.noise_scheduler = DDIMScheduler(**ez.params["diff"]) if alg == "ddim" else DPMSolverMultistepScheduler(**ez.params["diff"], algorithm_type=alg)


@pytest.mark.parametrize("alg,eta", SAMPLERS)
def test_one_segment_timeline_equals_generate_long_audio(alg, eta, monkeypatch):
    gc.collect()
    ez = _ez(monkeypatch)
    _set_sampler(ez, alg)
    kw = dict(window_length=1, overlap=0.2, guidance_scale=5, guidance_rescale=0.75, ddim_steps=6, eta=eta, random_seed=17)
    for prompt, length in (("a dog barks", 2.5), ("rain on a roof", 0.9), ("", 2.5)):   # 3 windows; one window; no guidance
        sr, want = ez.generate_long_audio(prompt, length=length, **kw)
        sr2, got = ez.generate_timeline_audio([(prompt, 0, length)], transition=0.3, **kw)
        assert sr2 == sr and got.shape == want.shape == (480 * int(length * 50),)
        assert got.tobytes() == want.tobytes(), (alg, eta, prompt)
        if length <= 1:
            _, solo = ez.generate_audio(prompt, length=length, **{k: v for k, v in kw.items() if k not in ("window_length", "overlap")})
            assert solo.tobytes() == got.tobytes(), (alg, eta, prompt)


def test_batch_equals_solo_replay_and_moved_boundaries(monkeypatch):
    gc.collect()
    ez = _ez(monkeypatch, max_batch=12, precision="bf16x3")
    kw = dict(window_length=1, overlap=0.2, transition=0.1, guidance_scale=5, guidance_rescale=0.75, ddim_steps=5, eta=1)
    tls = [[("birds at dawn", 0, 1.2), ("traffic builds up", 1.2, 2.5)], [("engine hum", 0, 0.9)],
           [("crowd noise", 0, 1.0), ("rain on the street", 0.8, 2.0), ("", 1.9, 2.0)]]
    seeds = [5, 9, 13]
    sr, batch = ez.generate_timeline_audio(tls, random_seed=seeds, **kw)
    assert [w.shape for w in batch] == [(480 * 125,), (480 * 45,), (480 * 100,)]
    assert all(w.dtype == np.float32 and np.isfinite(w).all() for w in batch)
    for tl, s, w in zip(tls, seeds, batch):   # each solo call runs its own row count: bf16x3's bits do not depend on it
        _, solo = ez.generate_timeline_audio(tl, random_seed=s, **kw)
        assert solo.tobytes() == w.tobytes(), tl
    _, again = ez.generate_timeline_audio(tls, random_seed=seeds, **kw)   # a replay of the captured schedule
    assert all(a.tobytes() == b.tobytes() for a, b in zip(again, batch))
    # moved boundaries and new prompts on the same row layout (the same segments active in the same windows): the replay follows the
    # device tables, and equals an eager run of that timeline
    moved = [[("a choir sings", 0, 1.3), ("thunder rolls in", 1.3, 2.5)], [("a kettle whistles", 0, 0.9)],
             [("wind in the pines", 0, 1.05), ("", 0.85, 2.0), ("surf on a beach", 1.92, 2.0)]]
    from ezaudio_b200.inference import check_timeline
    def rows(t):
        segs = [[(round(s * 50), round(e * 50)) for _, s, e in c] for c in t]
        return [(k, b) for k, b, _ in check_timeline(segs, [125, 45, 100], 3, 50, 10, 5, True, 24, 100)[3]]
    assert rows(moved) == rows(tls)
    n0 = len(ez.unet.__dict__["_timeline_cache"])
    _, replay = ez.generate_timeline_audio(moved, random_seed=seeds, **kw)
    assert len(ez.unet.__dict__["_timeline_cache"]) == n0   # no new capture
    ez.unet.__dict__.pop("_timeline_cache")
    _, eager = ez.generate_timeline_audio(moved, random_seed=seeds, **kw)
    for a, b, c in zip(replay, eager, batch):
        assert a.tobytes() == b.tobytes() and a.tobytes() != c.tobytes()


def test_row_capacity_raises_and_leaves_the_handle_usable(monkeypatch):
    gc.collect()
    ez = _ez(monkeypatch, max_batch=4)   # 8 DiT rows
    kw = dict(window_length=1, overlap=0.2, transition=0.1, ddim_steps=3, random_seed=1)
    tl = [("birds at dawn", 0, 1.2), ("traffic builds up", 1.2, 2.5)]   # 3 windows, 4 conditioned rows + 3 uncond rows = 7
    _, a = ez.generate_timeline_audio(tl, **kw)
    with pytest.raises(ValueError, match="needs max_batch >= 5"):   # 6 conditioned rows + 4 uncond rows = 10
        ez.generate_timeline_audio([("birds at dawn", 0, 1.6), ("traffic builds up", 1.2, 3.3)], **kw)
    _, b = ez.generate_timeline_audio(tl, **kw)
    assert a.tobytes() == b.tobytes() and np.isfinite(a).all()


# ---------------------------------------------------------------- the loop against the oracle
@pytest.mark.parametrize("sampler", ["ddim", "dpmsolver++"])
def test_timeline_matches_oracle_dit_with_fp64_rows(sampler):
    from ezaudio_b200.dit import MaskDiT
    from ezaudio_b200.inference import sample_timeline_latents
    gc.collect()
    lens, Lw, O_, T, gs, gr, steps, eta, seed, Lc = [73, 89], 40, 8, 4, 3.0, 0.5, 4, 1.0, 11, 12
    segments = [[(0, 0, 30), (1, 30, 52), (2, 52, 73)], [(2, 0, 36), (0, 30, 66), (1, 66, 89)]]   # transitions cross window edges
    frames = [[(s, e) for _, s, e in c] for c in segments]
    _, table, windows, rows, spans = check_timeline(frames, lens, 2, Lw, O_, T, True, 64, Lw)
    assert [c for _, c, _ in table] == [3, 3] and len(rows) > len(windows)
    cfg = synth.tiny_model(72)
    sd = weights.synthetic_state_dict(weights.dit_param_shapes(cfg), 3)
    ctx, mask = synth.synth_context(3, Lc, cfg["context_dim"])
    uctx, umask = synth.synth_context(1, Lc, cfg["context_dim"], seed=8, uncond=True)
    m = MaskDiT(precision="bf16x3", max_batch=len(rows) + len(windows), max_len=Lw, max_ctx_len=Lc, max_timesteps=8, **cfg).load_state_dict(sd)
    sched = DDIMScheduler() if sampler == "ddim" else DPMSolverMultistepScheduler(algorithm_type=sampler)
    lat = sample_timeline_latents(m, sched, ctx, mask, uctx, umask, segments, lens, Lw, O_, T, gs, gr, steps, eta, seed).cpu()
    gens = [torch.Generator(device="cuda").manual_seed(seed + b) for b in range(2)]
    x = [torch.randn((1, 128, n), generator=g, device="cuda")[0].cpu().double() for g, n in zip(gens, lens)]
    step_noise = [[torch.empty((1, 128, n), device="cuda").normal_(generator=g)[0].cpu() for g, n in zip(gens, lens)] for _ in range(steps)] \
        if sampler == "ddim" else None
    sched.set_timesteps(steps)
    W, R = len(windows), len(rows)
    prompt = [segments[b][q][0] for _, b, q in rows]
    wctx, wmask = torch.cat([ctx[prompt], uctx.expand(W, -1, -1)]), torch.cat([mask[prompt], umask.expand(W, -1)])
    m1 = [None] * 2
    with torch.no_grad():
        for i, t in enumerate(sched.timesteps.tolist()):
            xw = torch.stack([x[b][:, s:s + ln] for b, s, ln in [windows[k] for k, _, _ in rows] + windows]).float()
            out, _ = O.maskdit_forward(sd, cfg, xw, torch.tensor(t), wctx, wmask)
            win_of = [k for k, _, _ in rows]
            vr = O.cfg_combine(out[:R], out[R:][win_of], gs, gr).double()
            v = []
            for b, (first, count, n) in enumerate(table):
                num, den = torch.zeros(128, n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
                for r, (k, rb, q) in enumerate(rows):
                    if rb != b:
                        continue
                    _, s0, ln = windows[k]
                    j = torch.arange(ln, dtype=torch.float64)
                    w = torch.ones(ln, dtype=torch.float64)
                    if k > first:
                        w = torch.minimum(w, (j + 1) / (O_ + 1))
                    if k < first + count - 1:
                        w = torch.minimum(w, (Lw - j) / (O_ + 1))
                    s, e = frames[b][q]
                    f = s0 + j
                    a = torch.clamp(torch.minimum((f - s + T + 1) / (T + 1), (e + T - f) / (T + 1)), 0.0, 1.0)
                    num[:, s0:s0 + ln] += w * a * vr[r, :, :ln]
                    den[s0:s0 + ln] += w * a
                v.append(num / den)
            for b in range(2):
                if sampler == "ddim":
                    c = [float(e) for e in sched.step_coefficients(t, eta)]
                    x0, eps = c[0] * x[b] - c[1] * v[b], c[0] * v[b] + c[1] * x[b]
                    x[b] = c[2] * x0 + c[3] * eps + c[4] * step_noise[i][b].double()
                else:
                    c, order = sched.step_coefficients(i)
                    m0 = c[0] * x[b] - c[1] * v[b]
                    p = c[2] * x[b] + c[3] * m0
                    if order == 2:
                        p = p + c[4] * (c[5] * (m0 - m1[b]))
                    x[b], m1[b] = p, m0
    for b, n in enumerate(lens):
        err = float((lat[b, :, :n].double() - x[b]).abs().max())
        print(f"[timeline] {sampler} clip {b} ({n} frames, {table[b][1]} windows, {spans[b][1]} rows): vs oracle DiT + fp64 rows max-abs {err:.2e}")
        assert err < 5e-3, (b, err)
        assert torch.equal(lat[b, :, n:], torch.zeros(128, max(lens) - n))
