"""Batched / streaming front-end for the hot path (SURVEY 8(f) row 4).

The reference API takes one prompt per call (api/ezaudio.py:101, batch hard-wired to 1 at src/inference.py:67).  A server sees a
stream of independent requests; this module groups the ones that can share a launch sequence (same clip length, step count and
guidance constants -> same captured CUDA graphs), cuts them into batches of at most `max_batch` prompts, assigns the batches to
ranks (prompts are independent units: `ezaudio_b200.shard`), runs them through `EzAudio.generate_audio(list[str], ...)` and hands
the waveforms back in completion order (`stream`) or in request order (`run`).  Per-request seeds are honoured: prompt i of a batch
draws from torch.Generator(seed_i), so a request's audio does not depend on what it was batched with.

With `length_bucket_s` set, requests of different lengths share a batch: they group by ceil(length / bucket) instead of the exact
length, and the batch is padded to its bucket's top (capped at the backend's `max_length_s`), so there is one graph shape per bucket.
The backend then gets `length=[per-request lengths]` and `pad_length=`, and each request still gets exactly its solo audio.

Pure host logic: the backend is any object with the reference-shaped `generate_audio(text, length=, guidance_scale=, guidance_rescale=,
ddim_steps=, eta=, random_seed=)`; tests drive it with a stub on CPU."""
from __future__ import annotations

import collections
import dataclasses
import math
from typing import Dict, Iterable, Iterator, List, Optional, Sequence, Tuple


@dataclasses.dataclass(frozen=True)
class Request:
    """One text-to-audio request: the arguments of api/ezaudio.py:101-103 (defaults included)."""
    prompt: str
    length: int = 10
    guidance_scale: float = 5
    guidance_rescale: float = 0.75
    ddim_steps: int = 100
    eta: float = 1
    random_seed: Optional[int] = None
    scheduler: str = "ddim"   # the continuous engine also serves "dpmsolver++" / "sde-dpmsolver++" when built with them (eta is then ignored)

    def group_key(self, length_bucket_s: Optional[float] = None) -> Tuple:
        # "" switches guidance off for the whole call (api/ezaudio.py:109-111): empty prompts only batch with empty prompts
        size = self.length if length_bucket_s is None else ("bucket", length_bucket_bin(self.length, length_bucket_s))
        return (size, float(self.guidance_scale or 0.0), float(self.guidance_rescale or 0.0), int(self.ddim_steps), float(self.eta or 0.0),
                self.prompt == "")


@dataclasses.dataclass(frozen=True)
class ControlRequest:
    """One ControlNet request: the arguments of api/controlnet.py:113-118 (defaults included).  `audio` is the reference clip: a path, or a
    float32 mono waveform at the model's sample rate.  The clip is 10 s long, like the reference's; its waveform is trimmed to the length of
    the reference clip."""
    prompt: str
    audio: object
    surpass_noise: float = 0
    guidance_scale: float = 3.5
    guidance_rescale: float = 0
    ddim_steps: int = 50
    eta: float = 1
    conditioning_scale: float = 1
    random_seed: Optional[int] = None
    # as Request.scheduler; an init-only argument, so that the fields stay one per argument of EzAudio_ControlNet.generate_audio
    scheduler: dataclasses.InitVar[str] = "ddim"

    def __post_init__(self, scheduler):
        object.__setattr__(self, "scheduler", scheduler)


@dataclasses.dataclass(frozen=True)
class EditRequest:
    """One edit (inpainting / outpainting): the arguments of `EzAudio.editing_audio` for one clip (defaults included).  `gt_file` is the
    clip: a path, or a float32 mono waveform at the model's sample rate.  The result is the whole edited clip, as editing_audio returns it:
    the normalised original with the regenerated span spliced in, extended to the mask's end when the mask runs past the clip."""
    prompt: str
    boundary: float
    gt_file: object
    mask_start: float
    mask_length: float
    guidance_scale: float = 3.5
    guidance_rescale: float = 0
    ddim_steps: int = 100
    eta: float = 1
    random_seed: Optional[int] = None
    # as Request.scheduler; an init-only argument, so that the fields stay one per argument of EzAudio.editing_audio
    scheduler: dataclasses.InitVar[str] = "ddim"

    def __post_init__(self, scheduler):
        object.__setattr__(self, "scheduler", scheduler)


@dataclasses.dataclass(frozen=True)
class VariationRequest:
    """One audio-to-audio variation: the arguments of `EzAudio.variation_audio` for one clip (defaults included).  `init_audio` is the clip:
    a path, or a float32 mono waveform at the model's sample rate.  The result has the clip's length in samples."""
    prompt: str
    init_audio: object
    strength: float = 0.8
    guidance_scale: float = 5
    guidance_rescale: float = 0.75
    ddim_steps: int = 100
    eta: float = 1
    random_seed: Optional[int] = None
    # as Request.scheduler; an init-only argument, so that the fields stay one per argument of EzAudio.variation_audio
    scheduler: dataclasses.InitVar[str] = "ddim"

    def __post_init__(self, scheduler):
        object.__setattr__(self, "scheduler", scheduler)


def length_bucket_bin(length: float, length_bucket_s: float) -> int:
    """Bucket index of a clip length: ceil(length / bucket), so bucket k holds lengths in ((k - 1) * bucket, k * bucket]."""
    return max(1, math.ceil(length / length_bucket_s - 1e-9))


@dataclasses.dataclass
class Batch:
    key: Tuple
    tickets: List[int]
    requests: List[Request]
    pad_length: Optional[float] = None   # bucketed plans: the top of the bucket (seconds)


def plan_batches(requests: Sequence[Request], max_batch: int, length_bucket_s: Optional[float] = None) -> List[Batch]:
    """Stable grouping: requests keep their arrival order inside a group; groups are emitted in order of their first request.
    `length_bucket_s`: group lengths by bucket instead of exactly (see the module docstring); None keeps exact-length grouping."""
    if max_batch < 1:
        raise ValueError("max_batch must be >= 1")
    if length_bucket_s is not None and not length_bucket_s > 0:
        raise ValueError("length_bucket_s must be positive")
    groups: Dict[Tuple, List[int]] = collections.OrderedDict()
    for i, r in enumerate(requests):
        groups.setdefault(r.group_key(length_bucket_s), []).append(i)
    out: List[Batch] = []
    for key, idx in groups.items():
        for s in range(0, len(idx), max_batch):
            part = idx[s:s + max_batch]
            reqs = [requests[i] for i in part]
            pad = None if length_bucket_s is None else length_bucket_bin(reqs[0].length, length_bucket_s) * length_bucket_s
            out.append(Batch(key, part, reqs, pad))
    return out


def batches_of_rank(batches: Sequence[Batch], world: int, rank: int) -> List[Batch]:
    """Whole batches are dealt round-robin: every rank replays the same graph shapes, no collective is needed (SURVEY 8e)."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError("bad world/rank")
    return [b for i, b in enumerate(batches) if i % world == rank]


class BatchingFrontEnd:
    def __init__(self, backend, max_batch: int = 4, world: int = 1, rank: int = 0, length_bucket_s: Optional[float] = None):
        self.backend, self.max_batch, self.world, self.rank = backend, int(max_batch), int(world), int(rank)
        self.length_bucket_s = length_bucket_s
        self._queue: List[Request] = []

    @staticmethod
    def _check(r: Request) -> Request:
        if isinstance(r, (EditRequest, VariationRequest, ControlRequest)):
            raise ValueError(f"the batching front-end serves text-to-audio requests, got {type(r).__name__}; serve edits, variations and "
                             "ControlNet requests with engine.ContinuousEngine")
        if r.scheduler != "ddim":
            raise ValueError(f"the batching front-end runs DDIM only, got scheduler={r.scheduler!r}; serve DPM-Solver++ requests with "
                             "engine.ContinuousEngine(schedulers=...) or set EzAudio.noise_scheduler")
        return r

    def submit(self, prompt: str, **kw) -> int:
        """Queues a request; returns its ticket (index in submission order).  Requests for another scheduler than DDIM, and variations
        (`init_audio=`), raise ValueError."""
        if "init_audio" in kw:
            raise ValueError("the batching front-end serves no variations (init_audio); serve them with engine.ContinuousEngine")
        self._queue.append(self._check(Request(prompt, **kw)))
        return len(self._queue) - 1

    def _run_batch(self, b: Batch):
        r0 = b.requests[0]
        seeds = [r.random_seed for r in b.requests]
        seed_arg = seeds if any(s is not None for s in seeds) else None
        if seed_arg is not None and any(s is None for s in seeds):
            raise ValueError("a batch mixes seeded and unseeded requests: give every request a seed or none")
        kw = dict(guidance_scale=r0.guidance_scale, guidance_rescale=r0.guidance_rescale, ddim_steps=r0.ddim_steps, eta=r0.eta, random_seed=seed_arg)
        if b.pad_length is None:
            sr, wavs = self.backend.generate_audio([r.prompt for r in b.requests], length=r0.length, **kw)
        else:
            cap = getattr(self.backend, "max_length_s", None)
            pad = b.pad_length if cap is None else min(b.pad_length, cap)
            pad = max(pad, max(r.length for r in b.requests))
            sr, wavs = self.backend.generate_audio([r.prompt for r in b.requests], length=[r.length for r in b.requests], pad_length=pad, **kw)
        if len(wavs) != len(b.requests):
            raise RuntimeError("backend returned a different number of waveforms than prompts")
        return sr, wavs

    def stream(self, requests: Optional[Iterable[Request]] = None) -> Iterator[Tuple[int, int, object]]:
        """Yields (ticket, sample_rate, waveform) batch by batch, as soon as each batch of THIS rank has finished."""
        reqs = [self._check(r) for r in requests] if requests is not None else self._queue
        if requests is None:
            self._queue = []
        for b in batches_of_rank(plan_batches(reqs, self.max_batch, self.length_bucket_s), self.world, self.rank):
            sr, wavs = self._run_batch(b)
            for t, w in zip(b.tickets, wavs):
                yield t, sr, w

    def run(self, requests: Optional[Iterable[Request]] = None) -> List[Optional[Tuple[int, object]]]:
        """All requests of this rank, in request order: result[i] = (sr, waveform), or None for requests served by other ranks."""
        reqs = list(requests) if requests is not None else list(self._queue)
        if requests is None:
            self._queue = []
        out: List[Optional[Tuple[int, object]]] = [None] * len(reqs)
        for t, sr, w in self.stream(reqs):
            out[t] = (sr, w)
        return out
