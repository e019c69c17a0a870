"""Seamless loops on the host: the circular window plan (coverage, overlap, weights against an fp64 restatement, the shift schedule), the
row-capacity check, the validation generate_loop_audio does before any device work, and decode_loop's wrapped chunk indices."""
from types import SimpleNamespace

import numpy as np
import pytest

from ezaudio_b200.api import EzAudio
from ezaudio_b200.inference import check_loop, loop_offsets, loop_plan, loop_starts, loop_stride, loop_weights
from ezaudio_b200.vae import loop_chunks

PLANS = [(7, 10, 2), (10, 10, 2), (11, 10, 2), (16, 10, 2), (24, 10, 2), (25, 10, 3), (73, 40, 8), (64, 40, 8), (41, 40, 20),
         (1500, 500, 100), (3000, 500, 100), (2, 40, 1), (99, 12, 6)]


def _weights64(count, length, o):
    j = np.arange(length, dtype=np.float64)
    if count == 1:
        return np.ones(length)
    return np.minimum(1.0, np.minimum((j + 1) / (o + 1), (length - j) / (o + 1)))


@pytest.mark.parametrize("n,lw,o", PLANS)
def test_loop_plan_covers_the_circle(n, lw, o):
    count, ln = loop_plan(n, lw, o)
    assert ln == min(lw, n)
    assert count == (1 if n <= lw else -(-n // (lw - o)))
    for r in (0, 1, n // 3, n - 1):
        starts = loop_starts(n, count, r)
        assert starts == [((k * n) // count + r) % n for k in range(count)]
        cover = np.zeros(n, dtype=int)
        total = np.zeros(n)
        for s in starts:
            f = (s + np.arange(ln)) % n
            cover[f] += 1
            total[f] += _weights64(count, ln, o)
        assert (cover >= 1).all() and (total > 0).all(), (n, lw, o, r)
        if count > 1:   # neighbours on the circle (the last one's neighbour is window 0) share at least o frames
            for k in range(count):
                a, b = starts[k], starts[(k + 1) % count]
                gap = (b - a) % n
                assert ln - gap >= o, (k, gap)
        else:
            assert ln == n


def test_loop_plan_examples_and_refusals():
    assert loop_plan(1500, 500, 100) == (4, 500)   # a 30 s loop in 10 s windows with 2 s overlap
    assert loop_plan(500, 500, 100) == (1, 500)
    assert loop_plan(501, 500, 100) == (2, 500)
    assert loop_plan(120, 500, 100) == (1, 120)
    for o in (0, 251):
        with pytest.raises(ValueError):
            loop_plan(1000, 500, o)
    with pytest.raises(ValueError):
        loop_plan(1, 500, 100)


@pytest.mark.parametrize("n,lw,o", PLANS)
def test_loop_weights_match_fp64(n, lw, o):
    count, ln = loop_plan(n, lw, o)
    w = loop_weights(count, ln, o)
    assert w.dtype == np.float32 and w.shape == (ln,)
    assert (w > 0).all() and (w <= 1).all()
    ref = _weights64(count, ln, o)
    assert np.abs(w.astype(np.float64) - ref).max() <= 2.0 ** -24 * ref.max()
    if count > 1:   # both ends taper, symmetrically
        assert np.array_equal(w, w[::-1]) and w[0] < 1 and w[-1] < 1


def test_loop_offsets_formula():
    for n in (2, 3, 7, 100, 500, 1500, 1501):
        R = int(np.floor(n * 0.3819660112501051 + 0.5))
        assert loop_stride(n) == R
    lens, steps = [1500, 7, 501], 50
    offs = loop_offsets(lens, steps)
    assert len(offs) == steps and all(len(row) == 3 for row in offs)
    for i in range(steps):
        for b, n in enumerate(lens):
            assert offs[i][b] == (i * loop_stride(n)) % n
    assert offs[0] == [0, 0, 0]
    assert loop_stride(1500) == 573 and offs[1] == [573, 3, 191]


def test_check_loop_row_capacity_names_max_batch():
    lens, table, windows = check_loop([1500], 1, 500, 100, True, 8, 500)   # 4 windows x 2 = 8 rows
    assert table == [(0, 4, 1500)] and windows == [(0, 0, 500)] * 4
    with pytest.raises(ValueError, match="needs max_batch >= 4"):
        check_loop([1500], 1, 500, 100, True, 6, 500)
    lens, table, windows = check_loop([400, 3000, 2], 3, 500, 100, False, 16, 500)   # no guidance: one row per window
    assert table == [(0, 1, 400), (1, 8, 3000), (9, 1, 2)] and windows[0] == (0, 0, 400) and windows[-1] == (2, 0, 2)
    with pytest.raises(ValueError, match="needs max_batch >= 10"):
        check_loop([400, 3000, 2], 3, 500, 100, True, 16, 500)
    check_loop([500], 1, 500, 100, True, 2, 500)   # one window: the rows generate_audio takes
    for bad in ([1], [0], [1.5], [10, 20]):
        with pytest.raises(ValueError):
            check_loop(bad, 1, 500, 100, True, 16, 500)
    with pytest.raises(ValueError):
        check_loop([1000], 1, 600, 100, True, 16, 500)


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


@pytest.mark.parametrize("kw", [
    dict(text="rain", length=30, window_length=12),                               # window past max_length_s
    dict(text="rain", length=30, overlap=0),                                      # overlap below one frame
    dict(text="rain", length=30, overlap=0.01),                                   # overlap rounds to 0 frames
    dict(text="rain", length=30, overlap=6),                                      # overlap past half the window
    dict(text="rain", length=5, overlap=6),                                       # ... also for a one-window loop
    dict(text="rain", length=0),                                                  # empty loop
    dict(text="rain", length=0.03),                                               # one frame: no loop
    dict(text="rain", length=-3),
    dict(text=["rain", "wind"], length=[30, 0.001]),
    dict(text=["rain", "wind"], length=[30, 20, 10]),                             # one length per prompt
    dict(text=["rain", ""], length=30),                                           # empty and non-empty prompts mixed
    dict(text="rain", length=60),                                                 # 8 windows x 2 rows > 2 * max_batch (4)
    dict(text=["rain", "wind"], length=[30, 30]),                                 # 2 x 4 windows x 2 = 16 rows > 8
    dict(text="rain", length=31, window_length=2, overlap=1),                     # many short windows
])
def test_generate_loop_audio_validates_before_device_work(kw):
    with pytest.raises(ValueError):
        _stub_ez().generate_loop_audio(**kw)


def test_generate_loop_audio_row_capacity_message():
    with pytest.raises(ValueError, match="needs max_batch >= 8"):
        _stub_ez(max_batch=4).generate_loop_audio("rain", length=60)


@pytest.mark.parametrize("lens,M,h", [([5], 40, 9), ([1], 40, 9), ([22], 40, 9), ([23], 40, 9), ([150, 61, 3, 44], 40, 9), ([9, 10], 20, 9)])
def test_loop_chunks_wrap(lens, M, h):
    chunks = loop_chunks(lens, M, h)
    core = M - 2 * h
    for b, n in enumerate(lens):
        mine = [c for c in chunks if c[0] == b]
        assert [c[1] for c in mine] == list(range(0, n, core))       # cores tile the loop in order
        assert mine[-1][2] == n and all(c[2] - c[1] <= core for c in mine)
        for _, c0, c1, frames in mine:
            assert len(frames) == c1 - c0 + 2 * h <= M
            assert frames == [(c0 - h + t) % n for t in range(c1 - c0 + 2 * h)]
            assert frames[h:h + c1 - c0] == list(range(c0, c1))   # the core sits after h halo frames
    with pytest.raises(ValueError):
        loop_chunks([10], 18, 9)


def test_loop_chunks_short_loop_wraps_more_than_once():
    (b, c0, c1, frames), = loop_chunks([4], 40, 9)
    assert (b, c0, c1) == (0, 0, 4)
    assert frames == [3, 0, 1, 2, 3, 0, 1, 2, 3] + [0, 1, 2, 3] + [0, 1, 2, 3, 0, 1, 2, 3, 0]
