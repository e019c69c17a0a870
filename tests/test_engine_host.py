"""Continuous batching, host side: the scheduler of engine.ContinuousEngine driven with a stub device backend (admission order, per-request
schedules and constants, tickets, validation before any device work)."""
import pytest

from ezaudio_b200.engine import ContinuousEngine
from ezaudio_b200.frontend import Request
from ezaudio_b200.scheduler import DDIMScheduler


class StubSlots:
    """Records every call; the 'waveform' of a finished slot is (slot, frames)."""
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


def _engine(slots=2, ddim_steps=(25, 50, 100)):
    be = StubSlots()
    return ContinuousEngine(None, slots=slots, ddim_steps=ddim_steps, backend=be), be


def _schedule(n):
    s = DDIMScheduler()
    s.set_timesteps(n)
    return s, [int(t) for t in s.timesteps]


def test_table_is_the_union_of_the_allowed_schedules():
    eng, _ = _engine()
    _, t100 = _schedule(100)
    assert eng.table == sorted(t100)   # trailing spacing: the 25- and 50-step schedules are subsets of the 100-step one
    for n in (25, 50):
        assert set(_schedule(n)[1]) <= set(t100)
    with pytest.raises(ValueError):
        _engine(ddim_steps=(200,))       # 200 rows exceed the 128-row tables
    with pytest.raises(ValueError):
        _engine(ddim_steps=(0, 50))
    with pytest.raises(ValueError):
        _engine(slots=0)


def test_fifo_admission_into_freed_slots():
    eng, be = _engine(slots=2)
    steps = [25, 50, 25, 100, 25]
    tickets = [eng.submit(f"p{i}", ddim_steps=n, length=2, random_seed=i) for i, n in enumerate(steps)]
    assert tickets == [0, 1, 2, 3, 4]
    done = list(eng.stream())
    admits = [c for c in be.calls if c[0] == "admit"]
    # p2 takes slot 0 right after p0's 25 steps; after step 50 both slots are free and p3, p4 fill them in order
    assert [(c[1], c[2]) for c in admits] == [(0, "p0"), (1, "p1"), (0, "p2"), (0, "p3"), (1, "p4")]
    step_no, admitted_at = 0, {}
    for c in be.calls:
        if c[0] == "step":
            step_no += 1
        elif c[0] == "admit":
            admitted_at[c[2]] = step_no
    assert admitted_at == {"p0": 0, "p1": 0, "p2": 25, "p3": 50, "p4": 50}
    assert [t for t, _, _ in done] == [0, 2, 1, 4, 3]   # completion order
    assert eng.pending() == 0 and eng.step() == []


def test_each_request_runs_its_own_schedule_and_constants():
    eng, be = _engine(slots=3)
    reqs = [Request("a dog barks", length=4, guidance_scale=5, guidance_rescale=0.75, ddim_steps=50, eta=1, random_seed=3),
            Request("", length=10, guidance_scale=5, guidance_rescale=0.75, ddim_steps=25, eta=0, random_seed=4),
            Request("rain", length=7.5, guidance_scale=3.5, guidance_rescale=0, ddim_steps=100, eta=0.5),
            Request("wind", length=1, guidance_scale=None, ddim_steps=25, eta=1, random_seed=5)]
    for r in reqs:
        eng.submit(r.prompt, length=r.length, guidance_scale=r.guidance_scale, guidance_rescale=r.guidance_rescale, ddim_steps=r.ddim_steps,
                   eta=r.eta, random_seed=r.random_seed)
    slot_req = {}   # slot -> index of the request in it
    seen = {i: [] for i in range(len(reqs))}
    nxt = 0
    while eng.pending():
        eng.step()
    for c in be.calls:
        if c[0] == "admit":
            slot_req[c[1]] = nxt
            assert (c[2], c[3], c[4]) == (reqs[nxt].prompt, reqs[nxt].random_seed, int(reqs[nxt].length * 50))
            nxt += 1
        elif c[0] == "step":
            for k, e in enumerate(c[1]):
                if e is not None:
                    seen[slot_req[k]].append(e)
        elif c[0] == "finish":
            assert c[2] == int(reqs[slot_req[c[1]]].length * 50)
    for i, r in enumerate(reqs):
        sched, ts = _schedule(r.ddim_steps)
        got = seen[i]
        assert len(got) == r.ddim_steps
        assert [eng.table[e.t_index] for e in got] == ts
        cfg = bool(r.guidance_scale) and r.prompt != ""
        eta = float(r.eta or 0)
        for e, t in zip(got, ts):
            assert e.coef == sched.step_coefficients(t, eta)
            assert e.cfg == cfg and e.guidance_scale == (float(r.guidance_scale) if cfg else 0.0)
            assert e.guidance_rescale == float(r.guidance_rescale or 0) and e.draw_noise == (eta > 0)
            assert e.frames == int(r.length * 50)


def test_tickets_and_result_order():
    eng, be = _engine(slots=2)
    reqs = [Request(f"p{i}", length=1 + i, ddim_steps=n, random_seed=i) for i, n in enumerate([100, 25, 50])]
    res = eng.run(reqs)
    assert [w for _, w in res] == [("wav", k, (1 + i) * 50) for i, k in enumerate([0, 1, 1])]
    assert all(sr == 24000 for sr, _ in res)
    # queued requests (run() without arguments) come back in submission order too; tickets keep counting
    t = [eng.submit("x", ddim_steps=50, length=3), eng.submit("y", ddim_steps=25, length=2)]
    assert t == [3, 4]
    assert [w[2] for _, w in eng.run()] == [150, 100]


@pytest.mark.parametrize("kw", [dict(ddim_steps=30), dict(ddim_steps=50.5), dict(ddim_steps="50"), dict(length=0), dict(length=10.5),
                                dict(length=-1), dict(length=float("nan")), dict(random_seed=-1), dict(random_seed=2 ** 63),
                                dict(random_seed=1.5), dict(random_seed="7"), dict(eta=-1), dict(guidance_scale=float("inf"))])
def test_invalid_requests_rejected_before_device_work(kw):
    eng, be = _engine()
    args = dict(dict(ddim_steps=50, length=5, random_seed=1), **kw)
    with pytest.raises(ValueError):
        eng.submit("a dog barks", **args)
    assert eng.pending() == 0 and eng.step() == [] and be.calls == []
