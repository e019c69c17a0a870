"""Audio-to-audio variations on the host: the img2img start index, add_noise's coefficients against fp64 closed forms, DPM-Solver++ with a
begin index, the analytic Gaussian toy (a variation at strength 1 is the full run), and the continuous engine / batching front-end host logic
for variation requests (stub device backend)."""
import math

import numpy as np
import pytest

from ezaudio_b200.config import DIFF
from ezaudio_b200.engine import ContinuousEngine
from ezaudio_b200.frontend import BatchingFrontEnd, Request, VariationRequest
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler, start_index

ABAR = DDIMScheduler(**DIFF).alphas_cumprod.double().numpy()


@pytest.mark.parametrize("steps", [1, 2, 7, 10, 25, 50, 100, 1000])
@pytest.mark.parametrize("strength", [1e-3, 0.01, 0.05, 0.1, 0.3, 1 / 3, 0.5, 0.8, 0.999, 1.0])
def test_start_index_is_diffusers_img2img(steps, strength):
    # diffusers' StableDiffusionImg2ImgPipeline.get_timesteps: init_timestep = min(int(steps * strength), steps); t_start = steps - init_timestep
    n_run = min(int(steps * strength), steps)
    if n_run == 0:
        with pytest.raises(ValueError):
            start_index(steps, strength)
        return
    k = start_index(steps, strength)
    assert k == steps - n_run and 0 <= k < steps
    assert (k == 0) == (n_run == steps)


@pytest.mark.parametrize("strength", [0, 0.0, -0.1, 1.0001, 2, float("nan"), float("inf"), True, "0.5", None])
def test_start_index_rejects_strength_outside_0_1(strength):
    with pytest.raises(ValueError):
        start_index(100, strength)


def test_start_index_rejects_bad_step_counts():
    for steps in (0, -3, 2.5):
        with pytest.raises(ValueError):
            start_index(steps, 0.5)


def test_ddim_add_noise_coefficients_against_fp64():
    s = DDIMScheduler(**DIFF)
    for t in (0, 1, 10, 99, 250, 479, 500, 750, 998, 999):
        a, sg = s.add_noise_coefficients(t)
        abar = float(s.alphas_cumprod[t])   # the fp32 abar diffusers reads
        assert abs(a - math.sqrt(abar)) <= 2e-7 * max(1.0, math.sqrt(abar)) and abs(sg - math.sqrt(1 - abar)) <= 2e-7, t
        assert isinstance(a, float) and isinstance(sg, float)
        assert abs(a * a + sg * sg - 1) < 1e-6
        assert abs(abar - ABAR[t]) <= 1e-6
    assert s.add_noise_coefficients(999) == (0.0, 1.0)   # zero terminal SNR: abar_999 = 0 exactly, so x_999 = eps
    with pytest.raises(ValueError):
        s.add_noise_coefficients(1000)


@pytest.mark.parametrize("n", [10, 25, 100])
def test_dpm_add_noise_coefficients_against_fp64(n):
    s = DPMSolverMultistepScheduler(**DIFF)
    with pytest.raises(ValueError):
        s.add_noise_coefficients(999)   # no schedule yet
    s.set_timesteps(n)
    for i, t in enumerate(s.timesteps.tolist()):
        a, sg = s.add_noise_coefficients(t)
        sig = float(s.sigmas[i])
        want_a = 1 / math.sqrt(sig * sig + 1)
        assert abs(a - want_a) <= 1e-6 * want_a and abs(sg - sig * want_a) <= 1e-6, (i, t)
        if i > 0:   # away from the clamp the pair is DDIM's
            d = DDIMScheduler(**DIFF).add_noise_coefficients(t)
            assert abs(a - d[0]) < 1e-5 and abs(sg - d[1]) < 1e-5
    a, sg = s.add_noise_coefficients(999)
    assert a != 0.0 and abs(a - 2.0 ** -12) < 1e-10 and abs(sg - 1.0) < 1e-7   # the 2**-24 clamp: a = 2**-12, not 0
    with pytest.raises(ValueError):
        s.add_noise_coefficients(998)   # not in the schedule


@pytest.mark.parametrize("alg", ["dpmsolver++", "sde-dpmsolver++"])
@pytest.mark.parametrize("n", [10, 25, 100])
def test_dpm_begin_index(alg, n):
    s = DPMSolverMultistepScheduler(**DIFF, algorithm_type=alg)
    s.set_timesteps(n)
    for i in range(n):
        assert s.step_coefficients(i, begin_index=0) == s.step_coefficients(i)   # begin 0: today's values
    for k in (1, n // 3, n // 2, n - 2, n - 1):
        c, order = s.step_coefficients(k, begin_index=k)
        assert order == 1 and c[4] == 0.0 and c[5] == 0.0   # the first step taken has no history
        c0, o0 = s.step_coefficients(k)
        assert c[:4] == c0[:4] and c[6] == c0[6]   # only the second-order term goes
        for i in range(k + 1, n):
            assert s.step_coefficients(i, begin_index=k) == s.step_coefficients(i), (k, i)
        with pytest.raises(ValueError):
            s.step_coefficients(k - 1, begin_index=k)


def _gauss_v(x, t, mu, sd):
    a, sg = np.sqrt(ABAR[t]), np.sqrt(1 - ABAR[t])
    x0 = mu + a * sd * sd / (a * a * sd * sd + sg * sg) * (x - a * mu)
    return a * (x - a * x0) / sg - sg * x0


def _ddim_run(n, x, k, mu, sd):
    s = DDIMScheduler(**DIFF)
    s.set_timesteps(n)
    for t in s.timesteps.tolist()[k:]:
        c = s.step_coefficients(t, 0.0)
        v = _gauss_v(x, t, mu, sd)
        x0, e = c[0] * x - c[1] * v, c[0] * v + c[1] * x
        x = c[2] * x0 + c[3] * e
    return x


@pytest.mark.parametrize("n", [10, 25, 50, 100])
def test_analytic_gaussian_strength_one_is_the_full_run(n):
    """fp64, exact denoiser of N(mu, sd^2) data: DDIM (eta 0) from add_noise(x0, eps, t_k) with k = start_index(n, 1) is the run from eps;
    at strength < 1 it is the run from the noised clip, which lands closer to the clip."""
    rng = np.random.default_rng(n)
    eps, x0 = rng.standard_normal(4096), 0.3 + 0.7 * rng.standard_normal(4096)
    s = DDIMScheduler(**DIFF)
    s.set_timesteps(n)
    k = start_index(n, 1.0)
    assert k == 0
    a, sg = s.add_noise_coefficients(int(s.timesteps[k]))
    full = _ddim_run(n, eps, 0, 0.3, 0.7)
    var = _ddim_run(n, a * x0 + sg * eps, k, 0.3, 0.7)
    assert np.array_equal(var, full)
    k = start_index(n, 0.3)
    a, sg = s.add_noise_coefficients(int(s.timesteps[k]))
    part = _ddim_run(n, a * x0 + sg * eps, k, 0.3, 0.7)
    assert np.abs(part - x0).mean() < np.abs(full - x0).mean()


# ---- engine and front-end host logic (stub device backend)

class StubSlots:
    sr, latent_sr, hop, max_frames, max_timesteps = 24000, 50, 480, 500, 1000

    def __init__(self):
        self.calls = []

    def make_scheduler(self):
        return DDIMScheduler()

    def admit(self, k, prompt, seed, frames, **kw):
        self.calls.append(("admit", k, prompt, seed, frames, kw))

    def step(self, plan):
        self.calls.append(("step", list(plan)))

    def finish(self, k, frames):
        self.calls.append(("finish", k, frames))
        return ("wav", k, frames)


class StubControlSlots(StubSlots):
    control = True


def _clip(seconds=2.0, seed=0):
    return (0.1 * np.random.default_rng(seed).standard_normal(int(seconds * 24000))).astype(np.float32)


def _per_request_steps(be):
    """Every non-None SlotStep, per admitted request (in admission order)."""
    slot_req, seen, nxt = {}, {}, 0
    for c in be.calls:
        if c[0] == "admit":
            slot_req[c[1]] = nxt
            seen[nxt] = []
            nxt += 1
        elif c[0] == "step":
            for k, e in enumerate(c[1]):
                if e is not None:
                    seen[slot_req[k]].append(e)
    return seen


def test_variation_request_defaults_are_variation_audio_defaults():
    import inspect
    from ezaudio_b200.api import EzAudio
    sig = inspect.signature(EzAudio.variation_audio).parameters
    r = VariationRequest("rain", _clip())
    for name in ("strength", "guidance_scale", "guidance_rescale", "ddim_steps", "eta", "random_seed"):
        assert getattr(r, name) == sig[name].default, name
    assert r.strength == 0.8 and r.scheduler == "ddim"


@pytest.mark.parametrize("sched", ["ddim", "dpmsolver++", "sde-dpmsolver++"])
def test_engine_variation_runs_n_run_steps_from_its_start(sched):
    be = StubSlots()
    eng = ContinuousEngine(None, slots=2, ddim_steps=(10, 25), schedulers=("ddim", "dpmsolver++", "sde-dpmsolver++"), backend=be)
    wave = _clip(1.01)   # 24240 samples: 51 frames, the last one zero-padded
    reqs = [VariationRequest("rain", wave, strength=0.3, ddim_steps=25, random_seed=4, scheduler=sched),
            Request("wind", length=1, ddim_steps=10, random_seed=5),
            VariationRequest("a bell", wave, strength=1.0, ddim_steps=10, random_seed=6, scheduler=sched)]
    res = eng.run(reqs)
    assert len(res) == 3
    admits = [c for c in be.calls if c[0] == "admit"]
    seen = _per_request_steps(be)
    for j, r in enumerate(reqs):
        if isinstance(r, Request):
            assert admits[j][5] == {} and len(seen[j]) == r.ddim_steps
            continue
        n = r.ddim_steps
        k = start_index(n, r.strength)
        assert admits[j][4] == 51
        wv, ab = admits[j][5]["variation"]
        assert wv is wave or np.array_equal(wv, wave)
        s = DDIMScheduler() if sched == "ddim" else DPMSolverMultistepScheduler(algorithm_type=sched)
        s.set_timesteps(n)
        assert ab == s.add_noise_coefficients(int(s.timesteps[k]))
        got = seen[j]
        assert len(got) == n - k == min(int(n * r.strength), n)   # exactly n_run steps ...
        assert [eng.table[e.t_index] for e in got] == s.timesteps.tolist()[k:]   # ... from row k
        for i, e in enumerate(got, start=k):
            assert e.frames == 51 and e.cfg and e.guidance_scale == 5.0
            if sched == "ddim":
                assert not e.dpm and e.coef == s.step_coefficients(int(s.timesteps[i]), 1.0) and e.draw_noise
            else:
                coef, order = s.step_coefficients(i, begin_index=k)
                assert e.dpm and e.coef == coef and e.order == order
                if i == k:
                    assert order == 1   # DPM-Solver++'s first step taken is order 1
    if sched != "ddim":
        assert any(e.order == 2 for e in seen[0])


def test_engine_variation_validation():
    be = StubSlots()
    eng = ContinuousEngine(None, slots=2, ddim_steps=(10, 25), backend=be)
    bad = [dict(strength=0), dict(strength=1.5), dict(strength=float("nan")), dict(strength="0.5"), dict(strength=0.05, ddim_steps=10),
           dict(ddim_steps=30), dict(scheduler="dpmsolver++"), dict(random_seed=-1), dict(guidance_scale=float("inf")),
           dict(init_audio=np.zeros((2, 100), np.float32)), dict(init_audio=np.zeros(0, np.float32)),
           dict(init_audio=np.full(100, np.nan, np.float32)), dict(init_audio=_clip(10.5)), dict(init_audio=[0.1, 0.2]),
           dict(init_audio="/nonexistent/clip.wav")]
    for kw in bad:
        kw = dict(dict(init_audio=_clip(), ddim_steps=25, random_seed=1), **kw)
        with pytest.raises(ValueError):
            eng.submit("rain", **kw)
    assert eng.pending() == 0 and be.calls == []
    t = eng.submit("rain", init_audio=_clip(10.0), strength=0.04, ddim_steps=25)   # int(25 * 0.04) = 1 step; 500 frames fit
    assert t == 0 and eng.pending() == 1


def test_controlnet_engine_rejects_variations():
    be = StubControlSlots()
    eng = ContinuousEngine(None, slots=2, ddim_steps=(25,), backend=be)
    with pytest.raises(ValueError, match="variation"):
        eng.submit("rain", init_audio=_clip(), ddim_steps=25)
    with pytest.raises(ValueError):
        eng.run([VariationRequest("rain", _clip(), ddim_steps=25)])
    assert eng.pending() == 0 and be.calls == []


class StubBackend:
    def __init__(self):
        self.calls = []

    def generate_audio(self, text, **kw):
        self.calls.append((text, kw))
        return 24000, [("wav", p) for p in text]


def test_batching_front_end_rejects_variations():
    be = StubBackend()
    fe = BatchingFrontEnd(be, max_batch=4)
    with pytest.raises(ValueError):
        fe.submit("rain", init_audio=_clip(), strength=0.5)
    with pytest.raises(ValueError):
        fe.run([Request("rain", length=2), VariationRequest("wind", _clip())])
    from ezaudio_b200.frontend import ControlRequest, EditRequest
    with pytest.raises(ValueError):
        fe.run([EditRequest("rain", 1, _clip(), 0.5, 0.5)])
    with pytest.raises(ValueError):
        fe.run([ControlRequest("rain", _clip())])
    assert be.calls == []
    assert fe.submit("rain", length=2) == 0
    assert fe.run() == [(24000, ("wav", "rain"))]
