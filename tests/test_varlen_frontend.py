"""Clips of different lengths in one batch, host side: front-end length buckets (stub backend), length validation, C-ABI export."""
import ctypes

import pytest

from ezaudio_b200.frontend import BatchingFrontEnd, Request, length_bucket_bin, plan_batches
from ezaudio_b200.inference import check_lengths


class StubBackend:
    """Records every call; the 'waveform' of a prompt is (prompt, seed, its length, pad_length)."""

    def __init__(self, max_length_s=None):
        if max_length_s is not None:
            self.max_length_s = max_length_s
        self.calls = []

    def generate_audio(self, text, length=10, guidance_scale=5, guidance_rescale=0.75, ddim_steps=100, eta=1, random_seed=None, **kw):
        self.calls.append(dict(text=list(text), length=length, seed=random_seed, **kw))
        seeds = random_seed if isinstance(random_seed, (list, tuple)) else [random_seed] * len(text)
        lens = length if isinstance(length, (list, tuple)) else [length] * len(text)
        return 24000, [(p, s, n, kw.get("pad_length")) for p, s, n in zip(text, seeds, lens)]


LENGTHS = [4, 6, 7.5, 10, 3, 5, 9, 4.5]


def test_bucket_bins():
    assert [length_bucket_bin(v, 5) for v in LENGTHS] == [1, 2, 2, 2, 1, 1, 2, 1]
    assert length_bucket_bin(1.1, 0.1) == 11 and length_bucket_bin(0.01, 5) == 1


def test_bucketed_plan_groups_by_bucket_and_pads_to_its_top():
    reqs = [Request(f"p{i}", length=v, ddim_steps=50) for i, v in enumerate(LENGTHS)]
    batches = plan_batches(reqs, max_batch=3, length_bucket_s=5)
    assert [b.tickets for b in batches] == [[0, 4, 5], [7], [1, 2, 3], [6]]
    assert [b.pad_length for b in batches] == [5, 5, 10, 10]
    for b in batches:
        assert all(r.length <= b.pad_length for r in b.requests)


def test_default_plan_is_unchanged():
    reqs = [Request(f"p{i}", length=v, ddim_steps=50) for i, v in enumerate(LENGTHS)]
    for b in plan_batches(reqs, max_batch=3):
        assert b.pad_length is None and len({r.length for r in b.requests}) == 1
        assert b.key == b.requests[0].group_key()
    be = StubBackend(max_length_s=10)
    res = BatchingFrontEnd(be, max_batch=3).run(reqs)
    assert [r[1][2] for r in res] == LENGTHS
    assert all(not isinstance(c["length"], list) and "pad_length" not in c for c in be.calls)


def test_bucketed_front_end_calls_with_lengths_and_capped_pad():
    be = StubBackend(max_length_s=8)
    fe = BatchingFrontEnd(be, max_batch=4, length_bucket_s=5)
    reqs = [Request(f"p{i}", length=v, ddim_steps=50, random_seed=100 + i) for i, v in enumerate([3, 7.5, 4, 6])]
    res = fe.run(reqs)
    assert [r[1][:3] for r in res] == [(f"p{i}", 100 + i, v) for i, v in enumerate([3, 7.5, 4, 6])]
    assert [(c["length"], c["pad_length"]) for c in be.calls] == [([3, 4], 5), ([7.5, 6], 8)]   # 10 capped at the backend's 8 s
    assert BatchingFrontEnd(StubBackend(), 4, length_bucket_s=5).run(reqs[1:2])[0][1][3] == 10   # no cap advertised


def test_bucketed_groups_still_split_guidance_and_empty_prompts():
    reqs = [Request("a", length=4), Request("", length=4), Request("b", length=3, guidance_scale=3)]
    assert len(plan_batches(reqs, 8, length_bucket_s=5)) == 3
    with pytest.raises(ValueError):
        plan_batches(reqs, 8, length_bucket_s=0)


def test_check_lengths():
    assert check_lengths([5, 1, 10], 3, 10) == [5, 1, 10]
    for bad, B in (([0, 5], 2), ([11, 5], 2), ([5], 2), ([5, 5, 5], 2), ([2.5, 5], 2)):
        with pytest.raises(ValueError):
            check_lengths(bad, B, 10)
    with pytest.raises(NotImplementedError):
        check_lengths([5], 1, 10, gt=object())
    with pytest.raises(NotImplementedError):
        check_lengths([5], 1, 10, controlnet=object())


def test_library_exports_the_lengths_abi():
    from ezaudio_b200 import _lib, build
    build.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    assert hasattr(L, "ezb_test_attention_lens") and "ezb_test_attention_lens" in _lib.EXPORTS
    assert _lib.lib().ezb_version() == 2
