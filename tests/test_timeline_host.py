"""Timelines of prompts on the host: the segment weights against an fp64 restatement, the timeline rows against an independent
restatement (active segments per window, row order, the worked 60 s example), and every refusal generate_timeline_audio makes before any
device work."""
from types import SimpleNamespace

import numpy as np
import pytest

from ezaudio_b200.api import EzAudio
from ezaudio_b200.inference import check_timeline, segment_weights, timeline_plan, window_plan


def _weights64(s, e, n, T):
    f = np.arange(n, dtype=np.float64)
    a = np.minimum(1.0, np.minimum((f - s + T + 1) / (T + 1), (e + T - f) / (T + 1)))
    return np.where((f >= s - T) & (f < e + T), a, 0.0)


SEGMENTS = [(0, 1000, 3000, 50), (1000, 2000, 3000, 50), (2000, 3000, 3000, 50), (0, 3000, 3000, 50), (10, 20, 40, 0), (0, 1, 40, 0),
            (39, 40, 40, 0), (0, 1, 40, 7), (39, 40, 40, 7), (17, 18, 40, 3), (5, 30, 40, 12), (0, 40, 40, 100), (3, 9, 12, 1)]


@pytest.mark.parametrize("s,e,n,T", SEGMENTS)
def test_segment_weights_match_fp64(s, e, n, T):
    a = segment_weights(s, e, n, T)
    assert a.dtype == np.float32 and a.shape == (n,)
    ref = _weights64(s, e, n, T)
    assert np.array_equal(a > 0, ref > 0)
    assert (a[s:e] == 1).all()                                        # 1 inside the segment
    assert (np.abs(a.astype(np.float64) - ref) <= 2.0 ** -24 * ref).all()   # one IEEE rounding of the exact ratio
    f = np.arange(n)   # each ratio is the correctly rounded fp32 quotient
    t1 = np.float32(T + 1)
    want = np.minimum(np.float32(1), np.minimum(np.float32(1) * (f - s + T + 1).astype(np.float32) / t1, (e + T - f).astype(np.float32) / t1))
    assert np.array_equal(a[ref > 0], want[ref > 0])


def test_segment_weights_crossfade_abutting_segments():
    n, T = 300, 20
    a, b = segment_weights(0, 150, n, T), segment_weights(150, 300, n, T)
    both = np.flatnonzero((a > 0) & (b > 0))
    assert both.tolist() == list(range(130, 170))                    # 2T frames centred on the boundary
    assert (a[130:150] == 1).all() and (np.diff(a[149:170]) < 0).all()   # each stays 1 in its own segment and tapers past it
    assert (b[150:170] == 1).all() and (np.diff(b[130:151]) > 0).all()
    share = a[both] / (a[both] + b[both])
    assert (np.diff(share) < 0).all() and share[0] > 0.5 > share[-1]
    hard = segment_weights(0, 150, n, 0)
    assert (hard[:150] == 1).all() and (hard[150:] == 0).all()       # T = 0: a hard switch


def _rows_restated(segments, lengths, window, overlap, T):
    """An independent restatement: every window of every clip (window_plan), then each segment in timeline order whose weight is
    positive somewhere inside the window."""
    rows, k = [], 0
    for b, n in enumerate(lengths):
        for s0, ln in window_plan(n, window, overlap):
            for q, (s, e) in enumerate(segments[b]):
                if segment_weights(s, e, n, T)[s0:s0 + ln].max() > 0:
                    rows.append((k, b, q))
            k += 1
    return rows


def test_timeline_plan_worked_example():
    """60 s in 10 s windows with 2 s overlap (8 windows); birds 0-20 s, traffic 20-40 s, rain 40-60 s, 1 s transition: 11 rows."""
    segs = [[(0, 1000), (1000, 2000), (2000, 3000)]]
    table, windows, rows, spans = timeline_plan(segs, [3000], 500, 100, 50)
    assert len(windows) == 8 and table == [(0, 8, 3000)]
    per_window = [sum(1 for k, _, _ in rows if k == w) for w in range(8)]
    assert per_window == [1, 1, 2, 1, 2, 2, 1, 1] and len(rows) == 11 and spans == [(0, 11)]
    assert [q for _, _, q in rows] == [0, 0, 0, 1, 1, 1, 2, 1, 2, 2, 2]
    assert rows == _rows_restated(segs, [3000], 500, 100, 50)
    lens, _, _, rows2, _ = check_timeline(segs, [3000], 1, 500, 100, 50, True, 20, 500)
    assert rows2 == rows and lens == [3000]   # 11 + 8 = 19 rows fit max_batch 10
    with pytest.raises(ValueError, match="needs max_batch >= 10"):
        check_timeline(segs, [3000], 1, 500, 100, 50, True, 16, 500)
    check_timeline(segs, [3000], 1, 500, 100, 50, False, 11, 500)   # without guidance: the 11 conditioned rows


@pytest.mark.parametrize("seed", range(6))
def test_timeline_plan_matches_restatement(seed):
    rng = np.random.default_rng(seed)
    window, overlap = int(rng.integers(20, 60)), 0
    overlap = int(rng.integers(1, window // 2 + 1))
    lengths = [int(rng.integers(1, 400)) for _ in range(int(rng.integers(1, 4)))]
    T = int(rng.integers(0, 30))
    segments = []
    for n in lengths:   # random cuts covering the clip, plus some overlapping extras, in any order
        cuts = sorted(set([0, n] + [int(c) for c in rng.integers(1, n, size=int(rng.integers(0, 5)))] if n > 1 else [0, n]))
        segs = [(a, b) for a, b in zip(cuts, cuts[1:])]
        for _ in range(int(rng.integers(0, 3))):
            s = int(rng.integers(0, n))
            segs.append((s, int(rng.integers(s + 1, n + 1))))
        rng.shuffle(segs)
        segments.append(segs)
    lens, table, windows, rows, spans = check_timeline(segments, lengths, len(lengths), window, overlap, T, True, 10 ** 6, window)
    assert rows == _rows_restated(segments, lengths, window, overlap, T)
    for b, (r0, cnt) in enumerate(spans):
        assert all(rb == b for _, rb, _ in rows[r0:r0 + cnt]) and (b == 0 or r0 == sum(spans[b - 1]))
    for b, n in enumerate(lengths):   # every frame gets a positive total weight from the rows covering it
        total = np.zeros(n)
        for k, rb, q in rows:
            if rb == b:
                _, s0, ln = windows[k]
                total[s0:s0 + ln] += segment_weights(*segments[b][q], n, T)[s0:s0 + ln]
        assert (total > 0).all()


@pytest.mark.parametrize("segs,lengths,T", [
    ([[(0, 10), (12, 40)]], [40], 2),      # a gap in coverage
    ([[(0, 40), (10, 10)]], [40], 2),      # an empty segment
    ([[(0, 40), (45, 40)]], [40], 2),      # a start past the end (its end clipped to the clip)
    ([[(0, 40)]], [40], -1),               # a negative transition
    ([[(-3, 40)]], [40], 0),               # a start before the clip
    ([[(0, 20)], [(0, 40)]], [40], 0),     # clip 0 not covered past frame 20
    ([[(0, 40)]], [40, 40], 0),            # one timeline per clip
    ([[]], [40], 0),                       # no segment
])
def test_check_timeline_refusals(segs, lengths, T):
    with pytest.raises(ValueError):
        check_timeline(segs, lengths, len(lengths), 20, 4, T, True, 100, 20)


class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device work before validation: {name}")


def _stub_ez(max_batch=4, max_length_s=10.0):
    """An EzAudio whose every device-facing member fails the test when touched; only the host-side attributes are real."""
    ez = object.__new__(EzAudio)
    ez.params = {"autoencoder": {"latent_sr": 50, "sr": 24000, "scale": 1.0, "shift": 0.0}}
    ez.max_length_s = max_length_s
    ez.unet = SimpleNamespace(_h=SimpleNamespace(desc=SimpleNamespace(max_batch=2 * max_batch, max_len=int(max_length_s * 50))))
    ez.autoencoder = _NoDevice()
    ez.noise_scheduler = _NoDevice()

    def enc(prompts):
        raise AssertionError("text encoder called before validation")
    ez.encode_text = enc
    return ez


BIRDS = [("birds at dawn", 0, 20), ("traffic builds up", 20, 40), ("rain on the street", 40, 60)]


@pytest.mark.parametrize("kw", [
    dict(timeline=[("birds", 0, 10), ("rain", 12, 30)]),                          # gap in coverage
    dict(timeline=[("birds", 0, 30), ("rain", 10, 10)]),                          # empty segment
    dict(timeline=[("birds", 0, 30), ("rain", 40, 50)], length=30),               # start past the end
    dict(timeline=[("birds", 0, 30)], transition=-0.5),                           # negative transition
    dict(timeline=[("birds", 0, 30)], window_length=12),                          # window past max_length_s
    dict(timeline=[("birds", 0, 30)], overlap=0),                                 # overlap below one frame
    dict(timeline=[("birds", 0, 30)], overlap=6),                                 # overlap past half the window
    dict(timeline=[("birds", 0, 30)], length=0),                                  # empty clip
    dict(timeline=[[("birds", 0, 30)], [("rain", 0, 30)]], length=[30, 20, 10]),  # one length per clip
    dict(timeline=[("birds", 0, 30, 1)]),                                         # not (prompt, start, end)
    dict(timeline=[]),                                                            # no segment
    dict(timeline=BIRDS),                                                         # 11 + 8 = 19 rows > 2 * max_batch (4)
])
def test_generate_timeline_audio_validates_before_device_work(kw):
    with pytest.raises(ValueError):
        _stub_ez().generate_timeline_audio(**kw)


def test_generate_timeline_audio_row_capacity_message():
    with pytest.raises(ValueError, match="needs max_batch >= 10"):
        _stub_ez(max_batch=8).generate_timeline_audio(BIRDS)
    with pytest.raises(ValueError, match="needs max_batch >= 6"):   # no guidance: the 11 conditioned rows alone
        _stub_ez(max_batch=4).generate_timeline_audio(BIRDS, guidance_scale=0)
    with pytest.raises(ValueError, match="needs max_batch >= 6"):   # every prompt empty: no guidance either
        _stub_ez(max_batch=4).generate_timeline_audio([("", 0, 20), ("", 20, 40), ("", 40, 60)])
