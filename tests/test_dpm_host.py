"""DPM-Solver++ multistep on the host: the scheduler's schedule, order plan and coefficients (against DDIM, and against the exact ODE solution
of an analytic Gaussian model in fp64), and the continuous engine / batching front-end host logic for requests that ask for it."""
import numpy as np
import pytest

from ezaudio_b200.config import DIFF
from ezaudio_b200.engine import ContinuousEngine
from ezaudio_b200.frontend import BatchingFrontEnd, Request
from ezaudio_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler

STEPS = (10, 20, 25, 50, 100)
ABAR = DDIMScheduler(**DIFF).alphas_cumprod.double().numpy()   # the training schedule a denoiser sees (abar[999] = 0)


@pytest.mark.parametrize("n", STEPS)
@pytest.mark.parametrize("alg", ["dpmsolver++", "sde-dpmsolver++"])
def test_schedule_timesteps_sigmas_and_order_plan(n, alg):
    s = DPMSolverMultistepScheduler(**DIFF, algorithm_type=alg)
    d = DDIMScheduler(**DIFF)
    s.set_timesteps(n)
    d.set_timesteps(n)
    assert s.timesteps.tolist() == d.timesteps.tolist()
    sig = s.sigmas.double().numpy()
    assert len(sig) == n + 1 and np.isfinite(sig).all() and sig[-1] == 0.0
    assert abs(sig[0] - np.sqrt((1 - 2.0 ** -24) / 2.0 ** -24)) < 1e-3 * sig[0]   # the zero-SNR clamp keeps the first sigma finite
    assert np.all(np.diff(sig) < 0)
    assert s.orders == [1] + [2] * (n - 2) + [1]
    for i in range(n):
        coef, order = s.step_coefficients(i)
        assert order == s.orders[i] and len(coef) == 7 and np.isfinite(coef).all()
        if order == 1:
            assert coef[4] == 0.0 and coef[5] == 0.0
        assert (coef[6] != 0.0) == (alg == "sde-dpmsolver++" and i < n - 1)
    last, _ = s.step_coefficients(n - 1)   # sigma_t = 0: x <- m0
    assert last[2] == 0.0 and last[3] == 1.0 and last[6] == 0.0
    assert s.draws_noise == (alg == "sde-dpmsolver++")
    o1 = DPMSolverMultistepScheduler(**DIFF, solver_order=1, algorithm_type=alg)
    o1.set_timesteps(n)
    assert o1.orders == [1] * n


@pytest.mark.parametrize("kw", [dict(solver_order=3), dict(solver_type="heun"), dict(use_karras_sigmas=True), dict(use_lu_lambdas=True),
                                dict(thresholding=True), dict(final_sigmas_type="sigma_min"), dict(algorithm_type="dpmsolver"),
                                dict(algorithm_type="sde-dpmsolver"), dict(prediction_type="epsilon"), dict(timestep_spacing="leading")])
def test_unsupported_configs_raise(kw):
    with pytest.raises(NotImplementedError):
        DPMSolverMultistepScheduler(**dict(DIFF, **kw))


def test_step_index_outside_the_schedule_raises():
    s = DPMSolverMultistepScheduler(**DIFF)
    with pytest.raises(ValueError):
        s.step_coefficients(0)   # no schedule yet
    s.set_timesteps(10)
    with pytest.raises(ValueError):
        s.step_coefficients(10)


def _ddim(x, v, c):
    x0 = c[0] * x - c[1] * v
    eps = c[0] * v + c[1] * x
    return c[2] * x0 + c[3] * eps


def _dpm(x, v, m1, c, order, z=None):
    m0 = c[0] * x - c[1] * v
    prev = c[2] * x + c[3] * m0
    if order == 2:
        prev = prev + c[4] * (c[5] * (m0 - m1))
    if z is not None:
        prev = prev + c[6] * z
    return prev, m0


@pytest.mark.parametrize("n", STEPS)
def test_order1_is_ddim_eta0(n):
    """dpmsolver++ of order 1 is DDIM with eta = 0: the same update in fp64 from the fp32 coefficients, to round-off, at every step after the
    first (where DDIM's abar is exactly 0 and DPM-Solver++'s is clamped to 2**-24)."""
    s = DPMSolverMultistepScheduler(**DIFF, solver_order=1)
    d = DDIMScheduler(**DIFF)
    s.set_timesteps(n)
    d.set_timesteps(n)
    rng = np.random.default_rng(n)
    x, v = rng.standard_normal(4096), rng.standard_normal(4096)
    for i, t in enumerate(d.timesteps.tolist()):
        if i == 0:
            continue
        c, order = s.step_coefficients(i)
        got, _ = _dpm(x, v, None, c, order)
        want = _ddim(x, v, d.step_coefficients(t, 0.0))
        assert np.abs(got - want).max() <= 2e-6 * (np.abs(x) + np.abs(v)).max(), (n, i)


def _gauss_v(x, t, mu, s):
    """The exact v-prediction of data N(mu, s^2) per element at training timestep t (the posterior mean of x0, turned into v)."""
    a, sg = np.sqrt(ABAR[t]), np.sqrt(1 - ABAR[t])
    x0 = mu + a * s * s / (a * a * s * s + sg * sg) * (x - a * mu)
    return a * (x - a * x0) / sg - sg * x0


def _run(sched, n, xT, mu, s):
    sched.set_timesteps(n)
    x, m1 = xT.copy(), None
    for i, t in enumerate(sched.timesteps.tolist()):
        v = _gauss_v(x, t, mu, s)
        if isinstance(sched, DDIMScheduler):
            x = _ddim(x, v, sched.step_coefficients(t, 0.0))
        else:
            c, order = sched.step_coefficients(i)
            x, m1 = _dpm(x, v, m1, c, order)
    return x


@pytest.mark.parametrize("n", STEPS)
def test_analytic_gaussian(n):
    """Analytic toy, not the model: with the exact posterior-mean denoiser of N(mu, s^2) data, the probability-flow ODE from x_T (abar = 0 at
    t = 999) ends at mu + s x_T.  Dirac data (s = 0) lands on mu; for s > 0 the 2M endpoint is closer to it than DDIM's (eta = 0)."""
    xT = np.random.default_rng(7).standard_normal(4096)
    mu = 0.3
    got = _run(DPMSolverMultistepScheduler(**DIFF), n, xT, mu, 0.0)
    assert np.abs(got - mu).max() < 1e-6
    for s in (0.3, 0.7, 1.5):
        exact = mu + s * xT
        e_ddim = np.abs(_run(DDIMScheduler(**DIFF), n, xT, mu, s) - exact).max()
        e_2m = np.abs(_run(DPMSolverMultistepScheduler(**DIFF), n, xT, mu, s) - exact).max()
        e_1 = np.abs(_run(DPMSolverMultistepScheduler(**DIFF, solver_order=1), n, xT, mu, s) - exact).max()
        assert e_2m < e_ddim, (n, s, e_2m, e_ddim)
        assert abs(e_1 - e_ddim) < 1e-2 * e_ddim   # order 1 is DDIM eta = 0 up to the clamped first step


# ---- engine and front-end host logic (stub device backend)

class StubSlots:
    sr, latent_sr, max_frames, max_timesteps = 24000, 50, 500, 1000

    def __init__(self):
        self.calls = []

    def make_scheduler(self):
        return DDIMScheduler()

    def admit(self, k, prompt, seed, frames):
        self.calls.append(("admit", k, prompt, seed, frames))

    def step(self, plan):
        self.calls.append(("step", list(plan)))

    def finish(self, k, frames):
        self.calls.append(("finish", k, frames))
        return ("wav", k, frames)


def test_engine_serves_ddim_and_dpm_requests_in_shared_slots():
    be = StubSlots()
    eng = ContinuousEngine(None, slots=2, ddim_steps=(10, 25), schedulers=("ddim", "dpmsolver++", "sde-dpmsolver++"), backend=be)
    ddim_only = ContinuousEngine(None, slots=2, ddim_steps=(10, 25), backend=StubSlots())
    assert eng.table == ddim_only.table   # DPM-Solver++ shares DDIM's timesteps: the table does not grow
    reqs = [Request("a", length=2, ddim_steps=10, scheduler="dpmsolver++", random_seed=1),
            Request("b", length=3, ddim_steps=25, eta=1, random_seed=2),
            Request("c", length=4, ddim_steps=10, scheduler="sde-dpmsolver++", random_seed=3)]
    res = eng.run(reqs)
    assert [w for _, w in res] == [("wav", 0, 100), ("wav", 1, 150), ("wav", 0, 200)]   # "c" takes the slot "a" freed
    slot_req, nxt, seen = {}, 0, {0: [], 1: [], 2: []}
    for c in be.calls:
        if c[0] == "admit":
            slot_req[c[1]] = nxt
            nxt += 1
        elif c[0] == "step":
            for k, e in enumerate(c[1]):
                if e is not None:
                    seen[slot_req[k]].append(e)
    for i, r in enumerate(reqs):
        got = seen[i]
        assert len(got) == r.ddim_steps
        if r.scheduler == "ddim":
            assert not any(e.dpm for e in got) and all(e.draw_noise for e in got)
            continue
        s = DPMSolverMultistepScheduler(algorithm_type=r.scheduler)
        s.set_timesteps(r.ddim_steps)
        assert [eng.table[e.t_index] for e in got] == s.timesteps.tolist()
        for j, e in enumerate(got):
            coef, order = s.step_coefficients(j)
            assert e.dpm and e.coef == coef and e.order == order
            assert e.draw_noise == (r.scheduler == "sde-dpmsolver++")   # eta is ignored
            assert e.cfg and e.guidance_scale == 5.0 and e.guidance_rescale == 0.75


def test_engine_rejects_schedulers_it_was_not_built_with():
    be = StubSlots()
    eng = ContinuousEngine(None, slots=2, ddim_steps=(25,), backend=be)
    assert eng.schedulers == ("ddim",)
    for kind in ("dpmsolver++", "sde-dpmsolver++", "euler"):
        with pytest.raises(ValueError):
            eng.submit("a dog barks", length=2, ddim_steps=25, scheduler=kind)
    assert eng.pending() == 0 and eng.step() == [] and be.calls == []
    eng2 = ContinuousEngine(None, slots=2, ddim_steps=(25,), schedulers=("dpmsolver++",), backend=be)
    with pytest.raises(ValueError):
        eng2.submit("a dog barks", length=2, ddim_steps=25)   # a DDIM request to a DPM-only engine
    with pytest.raises(ValueError):
        eng2.submit("a dog barks", length=2, ddim_steps=25, scheduler="sde-dpmsolver++")
    assert be.calls == []
    for bad in (("unipc",), (), "ddim"):
        with pytest.raises(ValueError):
            ContinuousEngine(None, slots=2, ddim_steps=(25,), schedulers=bad, backend=StubSlots())


class StubBackend:
    def __init__(self):
        self.calls = []

    def generate_audio(self, text, **kw):
        self.calls.append((text, kw))
        return 24000, [("wav", p) for p in text]


def test_batching_front_end_rejects_dpm_requests():
    be = StubBackend()
    fe = BatchingFrontEnd(be, max_batch=4)
    with pytest.raises(ValueError, match="DDIM"):
        fe.submit("rain", length=2, scheduler="dpmsolver++")
    with pytest.raises(ValueError, match="DDIM"):
        fe.run([Request("rain", length=2), Request("wind", length=2, scheduler="sde-dpmsolver++")])
    assert be.calls == []
    assert fe.submit("rain", length=2) == 0
    assert fe.run() == [(24000, ("wav", "rain"))]
