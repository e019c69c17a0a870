"""Edits in the continuous-batching engine, host side: engine.ContinuousEngine with a stub backend that takes edits (EditRequest defaults,
validation before any device work, a ControlNet engine refusing edits, FIFO admission over a mixed queue, an edit's slot plan, request
types and result order through stream / run)."""
import dataclasses
import inspect

import numpy as np
import pytest

from ezaudio_b200.api import edit_plan
from ezaudio_b200.engine import ContinuousEngine
from ezaudio_b200.frontend import ControlRequest, EditRequest, Request
from ezaudio_b200.scheduler import DDIMScheduler


class StubSlots:
    """Records every call; the 'waveform' of a finished slot is (slot, frames)."""
    sr, latent_sr, hop, max_frames, max_timesteps = 24000, 50, 480, 500, 1000

    def __init__(self):
        self.calls = []

    def make_scheduler(self):
        return DDIMScheduler()

    def admit(self, k, prompt, seed, frames, edit=None):
        self.calls.append(("admit", k, prompt, seed, frames, edit))

    def step(self, plan):
        self.calls.append(("step", list(plan)))

    def finish(self, k, frames):
        self.calls.append(("finish", k, frames))
        return ("wav", k, frames)


class StubControlSlots(StubSlots):
    control = True


def _engine(slots=2, backend=StubSlots):
    be = backend()
    return ContinuousEngine(None, slots=slots, ddim_steps=(25, 50, 100), backend=be), be


def _clip(seconds=4.0, seed=0):
    return (0.1 * np.random.default_rng(seed).standard_normal(int(seconds * 24000))).astype(np.float32)


def _edit(**kw):
    return dict(dict(boundary=1, gt_file=_clip(), mask_start=1.5, mask_length=1.0, ddim_steps=50, random_seed=1), **kw)


def test_edit_request_defaults_are_editing_audio_defaults():
    from ezaudio_b200.api import EzAudio
    sig = inspect.signature(EzAudio.editing_audio).parameters
    fields = {f.name: f for f in dataclasses.fields(EditRequest)}
    params = [p for p in list(sig.values())[1:] if p.name != "randomize_seed" and p.kind is not inspect.Parameter.KEYWORD_ONLY]
    for p in params:
        f = fields["prompt" if p.name == "text" else p.name]
        if p.default is inspect.Parameter.empty:
            assert f.default is dataclasses.MISSING, p.name
        else:
            assert f.default == p.default and type(f.default) is type(p.default), p.name
    assert len(fields) == len(params)   # every argument but self, randomize_seed and the list form's pad_length


@pytest.mark.parametrize("kw", [dict(ddim_steps=30), dict(random_seed=-1), dict(random_seed=1.5), dict(eta=-1), dict(guidance_scale=float("nan")),
                                dict(guidance_rescale=float("inf")), dict(mask_start=-0.1), dict(mask_length=0), dict(mask_length=-1),
                                dict(boundary=-0.5), dict(mask_start=float("nan")), dict(mask_length="1"),
                                dict(gt_file="/nonexistent/clip.wav"), dict(gt_file=np.zeros((2, 100), np.float32)),
                                dict(gt_file=np.zeros(0, np.float32)), dict(gt_file=np.array([0.1, np.nan], np.float32)), dict(gt_file=[0.1, 0.2]),
                                dict(mask_start=1, mask_length=12, boundary=0),      # a 12-s crop: 600 frames, the engine serves 500
                                dict(gt_file=_clip(30), mask_start=2, mask_length=9, boundary=1)])   # 11-s crop of a long clip
def test_invalid_edits_rejected_before_device_work(kw):
    eng, be = _engine()
    with pytest.raises(ValueError):
        eng.submit("a bell", **_edit(**kw))
    assert eng.pending() == 0 and eng.step() == [] and be.calls == []


def test_controlnet_engine_refuses_edits():
    eng, be = _engine(backend=StubControlSlots)
    with pytest.raises(ValueError):
        eng.submit("a bell", **_edit())
    with pytest.raises(ValueError):
        eng.run([EditRequest("a bell", **_edit())])
    with pytest.raises(ValueError):   # and an EzAudio engine refuses ControlNet requests
        _engine()[0].run([ControlRequest("a siren", _clip())])
    assert eng.pending() == 0 and be.calls == []


def test_edit_clip_read_at_submit(tmp_path):
    from scipy.io import wavfile
    f = str(tmp_path / "clip.wav")
    wavfile.write(f, 24000, (_clip(3) * 32767).astype(np.int16))
    eng, be = _engine()
    eng.submit("a bell", **_edit(gt_file=f))
    assert be.calls == []
    eng.step()
    (_, k, prompt, seed, frames, (wave, plan)), = [c for c in be.calls if c[0] == "admit"]
    assert (k, prompt, seed) == (0, "a bell", 1)
    assert wave.dtype == np.float32 and wave.shape == (72000,)
    assert plan == edit_plan(72000, 24000, 50, 480, 1, 1.5, 1.0) and frames == plan["frames"]


def test_fifo_admission_over_a_mixed_queue():
    eng, be = _engine(slots=2)
    steps = [25, 50, 25, 100, 25]
    tickets = []
    for i, n in enumerate(steps):
        if i % 2:
            tickets.append(eng.submit(f"p{i}", **_edit(ddim_steps=n, random_seed=i)))
        else:
            tickets.append(eng.submit(f"p{i}", ddim_steps=n, length=2, random_seed=i))
    assert tickets == [0, 1, 2, 3, 4]
    done = list(eng.stream())
    admits = [c for c in be.calls if c[0] == "admit"]
    assert [(c[1], c[2]) for c in admits] == [(0, "p0"), (1, "p1"), (0, "p2"), (0, "p3"), (1, "p4")]
    assert [c[5] is not None for c in admits] == [False, True, False, True, False]
    assert [t for t, _, _ in done] == [0, 2, 1, 4, 3]
    assert eng.pending() == 0 and eng.step() == []


def test_each_edit_runs_its_own_plan_schedule_and_constants():
    eng, be = _engine(slots=3)
    reqs = [EditRequest("a dog barks", 1, _clip(4, 1), 1.5, 1.0, guidance_scale=5, guidance_rescale=0.75, ddim_steps=50, eta=1, random_seed=3),
            EditRequest("", 0.5, _clip(2, 2), 1.6, 1.0, ddim_steps=25, eta=0, random_seed=4),   # outpaints 0.6 s; "" runs without guidance
            Request("rain", length=7.5, guidance_scale=3.5, guidance_rescale=0, ddim_steps=100, eta=0.5),
            EditRequest("wind", 0.4, _clip(3, 3), 0.5, 0.6, guidance_scale=None, ddim_steps=25, random_seed=5)]
    res = eng.run(reqs)
    assert len(res) == 4
    slot_req, seen, nxt = {}, {i: [] for i in range(len(reqs))}, 0
    for c in be.calls:
        if c[0] == "admit":
            r = reqs[nxt]
            slot_req[c[1]] = nxt
            assert (c[2], c[3]) == (r.prompt, r.random_seed)
            if isinstance(r, EditRequest):
                wave, plan = c[5]
                assert np.array_equal(wave, r.gt_file)
                assert plan == edit_plan(len(r.gt_file), 24000, 50, 480, r.boundary, r.mask_start, r.mask_length)
                assert c[4] == plan["frames"]
            else:
                assert c[5] is None and c[4] == int(r.length * 50)
            nxt += 1
        elif c[0] == "step":
            for k, e in enumerate(c[1]):
                if e is not None:
                    seen[slot_req[k]].append(e)
    frames = {i: edit_plan(len(r.gt_file), 24000, 50, 480, r.boundary, r.mask_start, r.mask_length)["frames"] if isinstance(r, EditRequest)
              else int(r.length * 50) for i, r in enumerate(reqs)}
    assert frames == {0: 100, 1: 75, 2: 375, 3: 60}
    for i, r in enumerate(reqs):
        sched = DDIMScheduler()
        sched.set_timesteps(r.ddim_steps)
        ts = [int(t) for t in sched.timesteps]
        got = seen[i]
        assert len(got) == r.ddim_steps and [eng.table[e.t_index] for e in got] == ts
        cfg = bool(r.guidance_scale) and r.prompt != ""
        eta = float(r.eta or 0)
        for e, t in zip(got, ts):
            assert e.frames == frames[i]
            assert e.cfg == cfg and e.guidance_scale == (float(r.guidance_scale) if cfg else 0.0)
            assert e.guidance_rescale == float(r.guidance_rescale or 0)
            assert e.coef == sched.step_coefficients(t, eta) and e.draw_noise == (eta > 0)
    assert sorted(c[2] for c in be.calls if c[0] == "finish") == [60, 75, 100, 375]


def test_stream_and_run_keep_request_types_and_order():
    eng, be = _engine(slots=2)
    reqs = [EditRequest("a", 1, _clip(4), 1.5, 1.0, ddim_steps=100, random_seed=1),   # a 2-s crop: 100 frames
            Request("b", length=3, ddim_steps=25, random_seed=2),                        # 150 frames
            EditRequest("c", 0.4, _clip(3), 0.5, 0.6, ddim_steps=50, random_seed=3)]     # 60 frames
    res = eng.run(reqs)
    assert [w for _, w in res] == [("wav", 0, 100), ("wav", 1, 150), ("wav", 1, 60)]
    assert all(sr == 24000 for sr, _ in res)
    assert [c[5] is not None for c in be.calls if c[0] == "admit"] == [True, False, True]
    done = list(eng.stream(reqs[::-1]))
    assert sorted(t for t, _, _ in done) == [3, 4, 5]
    assert {t: w[2] for t, _, w in done} == {3: 60, 4: 150, 5: 100}
    # queued requests (run() without arguments) come back in submission order; submit() builds an edit from gt_file
    t = [eng.submit("x", **_edit(ddim_steps=100)), eng.submit("y", ddim_steps=25, length=3)]
    assert t == [6, 7]
    assert [w[2] for _, w in eng.run()] == [100, 150]
    assert [c[5] is not None for c in be.calls if c[0] == "admit"][-2:] == [True, False]
