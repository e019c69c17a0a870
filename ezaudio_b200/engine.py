"""Continuous batching for text-to-audio, edits and ControlNet: requests join a running batch at step boundaries.

`ContinuousEngine` keeps `slots` requests in flight in one padded, CFG-doubled batch (effective batch 2 * slots, clips padded to
`max_length_s`).  Each denoising step is one replay of one captured CUDA graph: the CFG-doubling copy, the DiT forward with per-sample
timestep rows read from device memory (`MaskDiT.forward_step(t_index=)`) and the fused CFG + rescale + DDIM update with per-sample
constants (ezb_cfg_ddim_step_slots).  Between steps the host admits queued requests into free slots, first come first served -- it
encodes the prompt, replaces that slot's text context row (`MaskDiT.set_context_rows`), seeds its generator and draws its initial noise
-- and decodes each request that finished its schedule alone at its own length.

Every request keeps its own step count (one of `ddim_steps`), guidance scale, rescale, eta, length and seed: the denoiser's timestep table
holds the sorted union of the allowed schedules (with trailing spacing the 25- and 50-step schedules are subsets of the 100-step one).  A
request's audio does not depend on what it shares the batch with.  Requests have the semantics of `EzAudio.generate_audio` for one prompt
(`frontend.Request`); the empty prompt "" runs without guidance, as it does there.

The same engine serves edits (`frontend.EditRequest`), with the semantics of `EzAudio.editing_audio` for one clip, next to text-to-audio
requests.  Every step passes the DiT a per-slot inpainting latent and a per-frame mask byte (rows k and slots + k for slot k): an edit's
rows hold its crop's VAE latent and its mask (1 on the regenerated frames and past the crop's end), every other slot's rows hold zeros and
an all-ones mask, which the DiT's input packing turns into exactly the operand it builds without an inpainting latent -- so text-to-audio
audio is unchanged, and one graph serves every mix.  Admitting an edit peak-normalises and pads its clip on the device and encodes its crop
alone (`Autoencoder(audio=)`, the scalar call's encode); finishing it pastes the kept frames of the latent back after the rescale, decodes
the crop alone and splices it into the normalised clip.  The encode draws the VAE bottleneck noise from the global torch RNG when the edit
is admitted (in queue order within a step), the draw editing_audio makes; text-to-audio admissions do not touch the global RNG.  So an
edit's audio depends on its own arguments, its seed and the global RNG state at its admission, not on its co-tenants.

Given an `api.EzAudio_ControlNet`, the engine serves `frontend.ControlRequest`s, with the semantics of `EzAudio_ControlNet.generate_audio`
for one prompt and one reference clip: 10-s clips, each with its own reference audio, noise gate and conditioning scale besides the
per-request constants above.  Admission also runs the clip's energy condition through the ControlNet stem once, into that slot's rows of
the ControlNet's condition cache (`DiTControlNet.set_condition_rows`); each step runs the ControlNet with per-sample timestep rows and
scales (`DiTControlNet.forward_step(t_index=, scale=)`) before the DiT.  A ControlNet engine serves no edits (the ControlNet API has no
editing call).  The FP8 mode is not served.

Built with `schedulers=` listing "dpmsolver++" and / or "sde-dpmsolver++" besides (or instead of) "ddim", the engine also serves requests with
`scheduler=` one of those (`scheduler.DPMSolverMultistepScheduler`, second order): each step then launches the fused CFG + DPM-Solver++
update with per-sample constants (ezb_cfg_dpm_step_slots) after the DDIM one, each kernel skipping the other kind's slots, and every slot
keeps its previous x0 prediction in a history buffer.  Such a request's audio equals `generate_audio` with that scheduler, one prompt and the
same seed.  The default engine (DDIM only) captures exactly the step graph it always has.

The same engine serves audio-to-audio variations (`frontend.VariationRequest`), with the semantics of `EzAudio.variation_audio` for one
clip.  Admitting one draws its start noise from the slot's generator (the draw a text-to-audio request makes), peak-normalises and pads
its clip on the device and encodes it alone straight into the noised start latent of slot k's row (`OobleckDecoder.encode_noised`, at the
request's start timestep; the bottleneck noise comes from the global torch RNG at admission, as for an edit); its schedule then begins at
`scheduler.start_index(ddim_steps, strength)`, with DPM-Solver++ taking that step at order 1.  Its inpainting rows and mask bytes are a
text-to-audio slot's, so the step graph does not change.

The host logic (admission, schedules, DDIM / DPM coefficients, tickets) is `ContinuousEngine`; the device work is `CudaSlots` (`ControlSlots`),
which tests replace with a stub."""
from __future__ import annotations

import collections
import dataclasses
import math
import numbers
import os
from typing import Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, post
from .frontend import ControlRequest, EditRequest, Request, VariationRequest
from .inference import scale_shift_re
from .scheduler import DDIMScheduler, DPMSolverMultistepScheduler, start_index

MAX_TABLE = 128   # rows of the denoiser's per-timestep LayerNorm tables (csrc/dit.cuh gc_T / fold_T)


@dataclasses.dataclass
class SlotStep:
    """What one active slot does in one step."""
    t_index: int              # row of the timestep table
    frames: int
    guidance_scale: float     # 0 without guidance
    guidance_rescale: float
    coef: List[float]         # DDIMScheduler.step_coefficients (DPM: DPMSolverMultistepScheduler.step_coefficients)
    cfg: bool
    draw_noise: bool          # eta > 0 (DPM: sde-dpmsolver++): the slot's generator draws this step's (1, C, frames) noise
    conditioning_scale: float = 1.0   # ControlNet requests: the factor of the ControlNet skips
    dpm: bool = False         # the update is DPM-Solver++ (ezb_cfg_dpm_step_slots) rather than DDIM
    order: int = 1            # DPM: the solver order of this step


@dataclasses.dataclass
class _Active:
    ticket: int
    req: object               # Request, EditRequest, VariationRequest or ControlRequest
    frames: int
    timesteps: List[int]
    sched: object             # DDIMScheduler or DPMSolverMultistepScheduler
    step: int = 0
    begin: int = 0            # the first step of the schedule it runs (a variation's start index)


class ContinuousEngine:
    """Continuous-batching server for `ez` (an `api.EzAudio`, or an `api.EzAudio_ControlNet`): `submit` requests, then `step` / `stream` /
    `run` them (see the module docstring).  An EzAudio engine serves text-to-audio requests and edits in one queue; a ControlNet engine
    serves ControlNet requests.

    slots: requests in flight (the denoiser runs 2 * slots samples; ez must have been built with max_batch >= slots).
    max_length_s: the padded clip length (at most ez.max_length_s); longer requests, and edits whose crop is longer, are rejected.
    ControlNet clips are 10 s.
    ddim_steps: the step counts requests may ask for; the union of their schedules must fit the timestep table.
    schedulers: the samplers requests may ask for (`Request.scheduler`): "ddim", "dpmsolver++", "sde-dpmsolver++"."""

    SCHEDULERS = ("ddim", "dpmsolver++", "sde-dpmsolver++")

    def __init__(self, ez, slots: int = 4, max_length_s: float = 10.0, ddim_steps: Sequence[int] = (25, 50, 100),
                 schedulers: Sequence[str] = ("ddim",), *, backend=None):
        self.control = bool(getattr(backend, "control", False)) if backend is not None else hasattr(ez, "controlnet")
        self.slots = int(slots)
        if self.slots < 1:
            raise ValueError("slots must be >= 1")
        if any(isinstance(n, bool) or int(n) != n for n in ddim_steps):
            raise ValueError(f"ddim_steps must list positive step counts, got {list(ddim_steps)}")
        allowed = sorted({int(n) for n in ddim_steps})
        if not allowed or allowed[0] < 1:
            raise ValueError(f"ddim_steps must list positive step counts, got {list(ddim_steps)}")
        if isinstance(schedulers, str) or not schedulers or any(k not in self.SCHEDULERS for k in schedulers):
            raise ValueError(f"schedulers must list some of {list(self.SCHEDULERS)}, got {schedulers!r}")
        self.schedulers = tuple(k for k in self.SCHEDULERS if k in schedulers)
        make = backend.make_scheduler if backend is not None else (lambda: DDIMScheduler(**ez.params["diff"]))
        diff = ez.params["diff"] if ez is not None else {}
        self._scheds = {}   # (scheduler, steps) -> a scheduler set to that many steps
        for kind in self.schedulers:
            for n in allowed:
                s = make() if kind == "ddim" else DPMSolverMultistepScheduler(**diff, algorithm_type=kind)
                s.set_timesteps(n)
                self._scheds[kind, n] = s
        # DPM-Solver++ uses DDIM's trailing timesteps: the table does not grow
        self._timesteps = {n: [int(t) for t in s.timesteps] for (_, n), s in self._scheds.items()}
        table = sorted({t for ts in self._timesteps.values() for t in ts})
        max_t = backend.max_timesteps if backend is not None else ez.unet._h.desc.max_timesteps
        if len(table) > min(max_t, MAX_TABLE):
            raise ValueError(f"the schedules of ddim_steps {allowed} hold {len(table)} distinct timesteps; the table holds at most "
                             f"{min(max_t, MAX_TABLE)}")
        self.ddim_steps = tuple(allowed)
        self.table = table
        self._row = {t: i for i, t in enumerate(table)}
        if backend is None:
            dpm = any(k != "ddim" for k in self.schedulers)
            backend = ControlSlots(ez, self.slots, table, dpm=dpm) if self.control else CudaSlots(ez, self.slots, max_length_s, table, dpm=dpm)
        self.backend = backend
        self._queue: collections.deque = collections.deque()
        self._active: List[Optional[_Active]] = [None] * self.slots
        self._tickets = 0

    # ---- requests
    def _frames(self, r: Request) -> int:
        self._check_common(r)
        if not isinstance(r.length, numbers.Real) or isinstance(r.length, bool) or not math.isfinite(r.length) or r.length <= 0:
            raise ValueError(f"length must be a positive number of seconds, got {r.length!r}")
        frames = int(r.length * self.backend.latent_sr)
        if not 1 <= frames <= self.backend.max_frames:
            raise ValueError(f"length {r.length} s is {frames} frames; this engine serves 1..{self.backend.max_frames}")
        return frames

    def _check_common(self, r):
        if not isinstance(r.ddim_steps, numbers.Integral) or isinstance(r.ddim_steps, bool) or int(r.ddim_steps) not in self.ddim_steps:
            raise ValueError(f"ddim_steps {r.ddim_steps} is not one of this engine's step counts {list(self.ddim_steps)}")
        if r.scheduler not in self.schedulers:
            raise ValueError(f"scheduler {r.scheduler!r} is not one this engine was built with {list(self.schedulers)}")
        s = r.random_seed
        if s is not None and (not isinstance(s, numbers.Integral) or isinstance(s, bool) or not 0 <= int(s) < 2 ** 63):
            raise ValueError(f"random_seed must be None or an integer in [0, 2**63), got {s!r}")
        for name in ("guidance_scale", "guidance_rescale", "eta"):
            v = getattr(r, name)
            if v is not None and (not isinstance(v, numbers.Real) or isinstance(v, bool) or not math.isfinite(v)):
                raise ValueError(f"{name} must be a finite number or None, got {v!r}")
        if (r.eta or 0) < 0:
            raise ValueError(f"eta must be >= 0, got {r.eta}")

    def _read_clip(self, a, what: str) -> np.ndarray:
        """A clip given as a path (read here, resampled to the model's rate) or as a float32 mono waveform; checked on the host."""
        if isinstance(a, (str, os.PathLike)):
            from .api import _load_audio
            try:
                a = _load_audio(os.fspath(a), self.backend.sr)
            except (OSError, ValueError) as e:
                raise ValueError(f"cannot read the {what} {a!r}: {e}") from e
        elif isinstance(a, np.ndarray):
            a = np.asarray(a, dtype=np.float32)
        else:
            raise ValueError(f"the {what} must be a path or a float32 mono waveform, got {type(a).__name__}")
        if a.ndim != 1 or a.size < 1 or not np.isfinite(a).all():
            raise ValueError(f"the {what} must be a non-empty, finite mono waveform, got shape {a.shape}")
        return a

    def _control_wave(self, r: ControlRequest) -> np.ndarray:
        """Checks a ControlNet request and loads its reference clip (host only)."""
        self._check_common(r)
        for name in ("surpass_noise", "conditioning_scale"):
            v = getattr(r, name)
            if not isinstance(v, numbers.Real) or isinstance(v, bool) or not math.isfinite(v):
                raise ValueError(f"{name} must be a finite number, got {v!r}")
        if r.surpass_noise < 0:
            raise ValueError(f"surpass_noise must be >= 0, got {r.surpass_noise}")
        return self._read_clip(r.audio, "reference clip")

    def _edit(self, r: EditRequest) -> Tuple[int, Tuple[np.ndarray, dict]]:
        """Checks an edit and loads its clip (host only); returns (crop frames, (clip, api.edit_plan of the edit))."""
        from .api import edit_plan
        self._check_common(r)
        for name in ("mask_start", "mask_length", "boundary"):
            v = getattr(r, name)
            if not isinstance(v, numbers.Real) or isinstance(v, bool) or not math.isfinite(v):
                raise ValueError(f"{name} must be a finite number of seconds, got {v!r}")
        if r.mask_start < 0 or r.mask_length <= 0 or r.boundary < 0:
            raise ValueError(f"mask_start and boundary must be >= 0 and mask_length > 0, got {r.mask_start}, {r.mask_length}, {r.boundary}")
        wave = self._read_clip(r.gt_file, "clip to edit")
        plan = edit_plan(len(wave), self.backend.sr, self.backend.latent_sr, self.backend.hop, r.boundary, r.mask_start, r.mask_length)
        if not 1 <= plan["frames"] <= self.backend.max_frames:
            raise ValueError(f"the edit's crop is {plan['frames']} frames; this engine serves 1..{self.backend.max_frames}")
        return plan["frames"], (wave, plan)

    def _variation(self, r: VariationRequest) -> Tuple[int, Tuple[np.ndarray, int]]:
        """Checks a variation and loads its clip (host only); returns (clip frames, (clip, start index))."""
        self._check_common(r)
        v = r.strength
        if not isinstance(v, numbers.Real) or isinstance(v, bool) or not math.isfinite(v):
            raise ValueError(f"strength must be a finite number, got {v!r}")
        k = start_index(int(r.ddim_steps), v)
        wave = self._read_clip(r.init_audio, "clip to vary")
        frames = -(-len(wave) // self.backend.hop)
        if not 1 <= frames <= self.backend.max_frames:
            raise ValueError(f"the clip is {frames} frames; this engine serves 1..{self.backend.max_frames}")
        return frames, (wave, k)

    def submit(self, prompt: str, **kw) -> int:
        """Queues a request and returns its ticket: an edit (the keyword arguments of `frontend.EditRequest`) when `gt_file` is given, a
        variation (`frontend.VariationRequest`) when `init_audio` is, otherwise a `frontend.Request`, or a `frontend.ControlRequest` for a
        ControlNet engine.  Invalid requests raise ValueError here, before any device work; a clip given as a path is read here."""
        if "gt_file" in kw:
            return self._enqueue(EditRequest(prompt, **kw))
        if "init_audio" in kw:
            return self._enqueue(VariationRequest(prompt, **kw))
        return self._enqueue(ControlRequest(prompt, **kw) if self.control else Request(prompt, **kw))

    def _enqueue(self, r) -> int:
        if isinstance(r, EditRequest):
            if self.control:
                raise ValueError("a ControlNet engine serves no edits (EzAudio_ControlNet has no editing call)")
            item = (r,) + self._edit(r)
        elif isinstance(r, VariationRequest):
            if self.control:
                raise ValueError("a ControlNet engine serves no variations (EzAudio_ControlNet has no variation call)")
            item = (r,) + self._variation(r)
        elif isinstance(r, ControlRequest) and self.control:
            item = (r, self.backend.max_frames, self._control_wave(r))
        elif isinstance(r, Request) and not self.control:
            item = (r, self._frames(r), None)
        else:
            raise ValueError(f"this {'ControlNet' if self.control else 'EzAudio'} engine does not serve {type(r).__name__}")
        t = self._tickets
        self._tickets += 1
        self._queue.append((t,) + item)
        return t

    def pending(self) -> int:
        """Requests queued or in flight."""
        return len(self._queue) + sum(a is not None for a in self._active)

    # ---- scheduling
    def _admit(self):
        for k in range(self.slots):
            if self._active[k] is None and self._queue:
                t, r, frames, extra = self._queue.popleft()
                seed = None if r.random_seed is None else int(r.random_seed)
                n, begin = int(r.ddim_steps), 0
                sched = self._scheds[r.scheduler, n]
                if self.control:
                    self.backend.admit(k, r.prompt, seed, frames, audio=extra, surpass_noise=float(r.surpass_noise))
                elif isinstance(r, EditRequest):
                    self.backend.admit(k, r.prompt, seed, frames, edit=extra)
                elif isinstance(r, VariationRequest):
                    wave, begin = extra
                    ab = sched.add_noise_coefficients(self._timesteps[n][begin])
                    self.backend.admit(k, r.prompt, seed, frames, variation=(wave, ab))
                else:
                    self.backend.admit(k, r.prompt, seed, frames)
                self._active[k] = _Active(t, r, frames, self._timesteps[n], sched, step=begin, begin=begin)

    def step(self) -> List[Tuple[int, int, object]]:
        """Admits queued requests into free slots, runs one denoising step of every request in flight and returns (ticket, sample_rate,
        waveform) of those that finished their schedule with it."""
        self._admit()
        if not any(a is not None for a in self._active):
            return []
        plan: List[Optional[SlotStep]] = []
        for a in self._active:
            if a is None:
                plan.append(None)
                continue
            r, t = a.req, a.timesteps[a.step]
            eta = float(r.eta or 0.0)
            cfg = bool(r.guidance_scale) and r.prompt != ""   # "" switches guidance off (api/ezaudio.py:109-111)
            gs, gr, cs = float(r.guidance_scale) if cfg else 0.0, float(r.guidance_rescale or 0.0), float(r.conditioning_scale) if self.control else 1.0
            if r.scheduler == "ddim":
                plan.append(SlotStep(self._row[t], a.frames, gs, gr, a.sched.step_coefficients(t, eta), cfg, eta > 0, cs))
            else:   # eta is ignored, as generate_audio ignores it with this scheduler
                coef, order = a.sched.step_coefficients(a.step, begin_index=a.begin)
                plan.append(SlotStep(self._row[t], a.frames, gs, gr, coef, cfg, a.sched.draws_noise, cs, dpm=True, order=order))
        self.backend.step(plan)
        done = []
        for k, a in enumerate(self._active):
            if a is None:
                continue
            a.step += 1
            if a.step == len(a.timesteps):
                wav = self.backend.finish(k, a.frames)
                self._active[k] = None
                done.append((a.ticket, self.backend.sr, wav))
        return done

    def stream(self, requests: Optional[Iterable[object]] = None) -> Iterator[Tuple[int, int, object]]:
        """Submits `requests` (if given: Request / EditRequest / VariationRequest objects, or ControlRequest objects for a ControlNet engine) and yields
        (ticket, sample_rate, waveform) in completion order until nothing is queued or in flight."""
        if requests is not None:
            for r in requests:
                self._enqueue(r)
        while self.pending():
            yield from self.step()

    def run(self, requests: Optional[Iterable[object]] = None) -> List[Tuple[int, object]]:
        """`requests` (default: the queued ones), in request order: result[i] = (sample_rate, waveform)."""
        if requests is not None:
            tickets = [self._enqueue(r) for r in requests]
        else:
            tickets = [q[0] for q in self._queue]
        pos = {t: i for i, t in enumerate(tickets)}
        out: List[Optional[Tuple[int, object]]] = [None] * len(tickets)
        for t, sr, w in self.stream():
            if t in pos:
                out[pos[t]] = (sr, w)
        return out


class CudaSlots:
    """Device side of ContinuousEngine: the slot buffers, the captured step graph and the per-slot generators of one `api.EzAudio`.

    The inpainting rows (`gt` [2 * slots, C, L] fp32, `gt_mask` [2 * slots, L] uint8, rows k and slots + k for slot k) go to every step:
    zeros and all ones for a free or text-to-audio slot, an edit's crop latent and mask while it is in flight (`admit(edit=)`); `finish`
    pastes, decodes and splices an edit, and puts its rows back.

    Between steps the engine owns the denoiser's context and timestep table: a generate_audio call on the same EzAudio replaces them, and the
    next step restores them (set_context of the whole batch, set_timesteps of the table)."""

    def __init__(self, ez, slots: int, max_length_s: float, table: Sequence[int], dpm: bool = False):
        p = ez.params["autoencoder"]
        self.ez, self.unet, self.S, self.table = ez, ez.unet, int(slots), [int(t) for t in table]
        self.sr, self.latent_sr, self.hop = int(p["sr"]), int(p["latent_sr"]), int(ez.autoencoder.decoder.hop)
        self.max_frames = int(round(max_length_s * self.latent_sr))
        desc = self.unet._h.desc
        self.max_timesteps = int(desc.max_timesteps)
        if getattr(self.unet, "precision", "bf16") == "fp8":
            raise NotImplementedError("the continuous engine serves the bf16 and bf16x3 precisions")
        if 2 * self.S > desc.max_batch:
            raise ValueError(f"{self.S} slots need a denoiser batch of {2 * self.S}; this EzAudio holds {desc.max_batch} (max_batch {desc.max_batch // 2})")
        if max_length_s > ez.max_length_s or self.max_frames > desc.max_len or self.max_frames < 1:
            raise ValueError(f"max_length_s {max_length_s} must lie in (0, {ez.max_length_s}] (the EzAudio's max_length_s)")
        if ez.encode_text is None:
            raise RuntimeError("no text encoder available: pass text_encoder=<callable> to EzAudio")
        self.C = int(self.unet.cfg["out_chans"])
        S, Be, C, L = self.S, 2 * self.S, self.C, self.max_frames
        self.device = torch.device("cuda", self.unet._h.dev_index)
        with torch.cuda.device(self.device):
            d = dict(device=self.device, dtype=torch.float32)
            self.lat, self.noise = torch.zeros(S, C, L, **d), torch.zeros(S, C, L, **d)   # padded frames stay zero
            self.hist = torch.zeros(S, C, L, **d) if dpm else None   # DPM-Solver++ slots: the previous step's x0 prediction
            self.x_in, self.out = torch.zeros(Be, C, L, **d), torch.zeros(Be, C, L, **d)
            self.gt = torch.zeros(Be, C, L, **d)
            self.gt_mask = torch.ones(Be, L, device=self.device, dtype=torch.uint8)   # 1: the DiT regenerates the frame
            # per-step inputs as one int32 block, staged through pinned memory: t_index [Be] | lens [Be] | ezb_ddim_slot [S] (8 words each)
            # [| ezb_dpm_slot [S] (10 words each) when DPM-Solver++ is served]
            words = 2 * Be + 8 * S + (10 * S if dpm else 0)
            self._h = torch.zeros(words, dtype=torch.int32, pin_memory=True)
            self._d = torch.zeros(words, dtype=torch.int32, device=self.device)
            self._copied = None
            self.t_index, self.lens, self.slots_dev = self._d[:Be], self._d[Be:2 * Be], self._d[2 * Be:2 * Be + 8 * S]
            self.dpm_slots_dev = self._d[2 * Be + 8 * S:] if dpm else None
            uemb, umask = ez.encode_text([""])   # the uncond rows: the "" embedding, once
            self.Lc = int(uemb.shape[1])
            self.ctx = uemb.to(**d).expand(Be, -1, -1).contiguous()
            self.cmask = umask.to(self.device).bool().expand(Be, -1).contiguous()
        self.gens: List[Optional[torch.Generator]] = [None] * S
        self.edits: List[Optional[Tuple[torch.Tensor, int, int]]] = [None] * S   # an edit's (normalised clip, s0, n_paste)
        self.trim: List[Optional[int]] = [None] * S   # a variation's clip length in samples
        self.graph, self._key, self._launches = None, None, 0
        self.captures = 0   # step graphs captured so far
        self._ctx_epoch = None

    def _own_denoiser(self):
        """Puts the engine's timestep table and context back if something else replaced them since the last step."""
        self.unet.set_timesteps(self.table)   # no device work when the table is already loaded
        h = self.unet._h
        if self._ctx_epoch != h.ctx_epoch:
            self.unet.set_context(self.ctx, self.cmask)
            self._ctx_epoch = h.ctx_epoch

    def admit(self, k: int, prompt: str, seed: Optional[int], frames: int, edit: Optional[Tuple[np.ndarray, dict]] = None,
              variation: Optional[Tuple[np.ndarray, Tuple[float, float]]] = None):
        """Starts slot k.  `edit`: (clip, api.edit_plan of the edit) for an edit, whose crop is `frames` latent frames long.  `variation`:
        (clip, (a, s) of add_noise at the start timestep) for a variation of a clip of `frames` latent frames."""
        with torch.cuda.device(self.device):
            if edit is not None:
                self._admit_edit(k, frames, *edit)
            self._own_denoiser()
            emb, mask = self.ez.encode_text([prompt])
            if tuple(emb.shape[1:]) != tuple(self.ctx.shape[1:]):
                raise ValueError(f"the text encoder returned {tuple(emb.shape)}, the engine's context rows are {tuple(self.ctx.shape[1:])}")
            self.ctx[k:k + 1].copy_(emb)
            self.cmask[k:k + 1].copy_(mask)
            self.unet.set_context_rows(self.ctx[k:k + 1], self.cmask[k:k + 1], k)
            g = torch.Generator(device=self.device)
            if seed is None:
                g.seed()
            else:
                g.manual_seed(seed)
            self.gens[k] = g
            self.lat[k].zero_()
            self.lat[k, :, :frames] = torch.randn((1, self.C, frames), generator=g, device=self.device)[0]   # the draw of a solo run
            if variation is not None:
                self._admit_variation(k, frames, *variation)

    def _admit_variation(self, k: int, frames: int, wave: np.ndarray, ab: Tuple[float, float]):
        """variation_audio's start of one clip (api.py): normalise and pad the clip on the device, then encode it alone and noise it with
        the start noise in slot k's latent row, in one pass -- the bottleneck noise comes from the global RNG."""
        clip = post.prepare_wave(torch.from_numpy(wave).to(self.device).unsqueeze(0), frames * self.hop, normalize=True)
        p = self.ez.params["autoencoder"]
        x_t = self.ez.autoencoder.decoder.encode_noised(clip.view(1, 1, -1), [ab], self.lat[k:k + 1, :, :frames], p["scale"], p["shift"])
        self.lat[k, :, :frames] = x_t[0]
        self.trim[k] = len(wave)

    def _admit_edit(self, k: int, frames: int, wave: np.ndarray, p: dict):
        """editing_audio's preparation of one clip (api.py): normalise and pad the clip on the device, encode the crop alone -- the
        bottleneck noise comes from the global RNG -- and write slot k's inpainting rows."""
        clip = post.prepare_wave(torch.from_numpy(wave).to(self.device).unsqueeze(0), p["n_total"], normalize=True)[0]
        z = self.ez.autoencoder(audio=clip[p["s0"]:p["s1"]].clone().view(1, 1, -1))
        if tuple(z.shape) != (1, self.C, frames):
            raise RuntimeError(f"the VAE encoded the crop to {tuple(z.shape)}, expected (1, {self.C}, {frames})")
        S = self.S
        self.gt[k].zero_()
        self.gt[k, :, :frames] = z[0]
        self.gt_mask[k].zero_()
        self.gt_mask[k, p["m0"]:p["m1"]] = 1
        self.gt_mask[k, frames:] = 1   # past the crop's end nothing of gt is used
        self.gt[S + k].copy_(self.gt[k])
        self.gt_mask[S + k].copy_(self.gt_mask[k])
        self.edits[k] = (clip, int(p["s0"]), int(p["n_paste"]))

    def _launch_step(self):
        S = self.S
        self.x_in[:S].copy_(self.lat)
        self.x_in[S:].copy_(self.lat)
        self.unet.forward_step(self.x_in, 0, gt=self.gt, gt_mask_u8=self.gt_mask, out=self.out, lengths=self.lens, t_index=self.t_index)
        self._launch_update(self.lens[:S])

    def _launch_update(self, lens):
        """The DDIM slots' update, then (when served) the DPM-Solver++ slots' one; each kernel leaves the other kind's slots alone."""
        S = self.S
        _lib.check(_lib.lib().ezb_cfg_ddim_step_slots(self.device.index, _lib.ptr(self.out), _lib.ptr(self.lat), _lib.ptr(self.noise),
                                                      _lib.ptr(self.slots_dev), S, self.C, self.max_frames, _lib.stream_ptr(), _lib.ptr(lens)))
        if self.hist is not None:
            _lib.check(_lib.lib().ezb_cfg_dpm_step_slots(self.device.index, _lib.ptr(self.out), _lib.ptr(self.lat), _lib.ptr(self.hist),
                                                         _lib.ptr(self.noise), _lib.ptr(self.dpm_slots_dev), S, self.C, self.max_frames,
                                                         _lib.stream_ptr(), _lib.ptr(lens)))

    def step(self, plan: Sequence[Optional[SlotStep]]):
        S, Be = self.S, 2 * self.S
        with torch.cuda.device(self.device):
            self._own_denoiser()
            if self._copied is not None:
                self._copied.synchronize()   # the previous step's copy has read the pinned block
            h = self._h.numpy()
            tix, lens = h[:Be], h[Be:2 * Be]
            words = h[2 * Be:2 * Be + 8 * S].reshape(S, 8)
            fl = words.view(np.float32)
            dwords = h[2 * Be + 8 * S:].reshape(S, 10) if self.hist is not None else None
            for k, e in enumerate(plan):
                if dwords is not None:
                    dwords[k] = 0   # inactive for the DPM kernel unless it is a DPM slot
                if e is None:   # inactive: one frame, no update
                    tix[k] = tix[S + k] = 0
                    lens[k] = lens[S + k] = 1
                    words[k] = 0
                    continue
                tix[k] = tix[S + k] = e.t_index
                lens[k] = lens[S + k] = e.frames
                flags = _lib.SLOT_ACTIVE | (_lib.SLOT_CFG if e.cfg else 0)
                if e.dpm:
                    if dwords is None:
                        raise RuntimeError("a DPM-Solver++ step on slots built without DPM-Solver++")
                    words[k] = 0   # inactive for the DDIM kernel
                    dfl = dwords.view(np.float32)
                    dfl[k, 0], dfl[k, 1] = e.guidance_scale, e.guidance_rescale
                    dfl[k, 2:9] = e.coef
                    dwords[k, 9] = flags | (_lib.SLOT_ORDER2 if e.order == 2 else 0)
                else:
                    fl[k, 0], fl[k, 1] = e.guidance_scale, e.guidance_rescale
                    fl[k, 2:7] = e.coef
                    words[k, 7] = flags
                if e.draw_noise:   # the draw a solo run makes at this step: a contiguous (1, C, frames) tensor from the slot's generator
                    self.noise[k, :, :e.frames] = torch.empty((1, self.C, e.frames), device=self.device).normal_(generator=self.gens[k])[0]
            self._d.copy_(self._h, non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record()
            key = (S, self.max_frames, self.Lc, int(_lib.lib().ezb_option_epoch()))
            L_ = _lib.lib()
            if self.graph is not None and key == self._key:
                self.graph.replay()
                L_.ezb_launch_count_add(self._launches)
                return
            self._launch_step()   # eager pass: this step's result, and warm caches for the capture
            snap = self.lat.clone()
            g = torch.cuda.CUDAGraph()
            n0 = L_.ezb_launch_count()
            with torch.cuda.graph(g):
                self._launch_step()
            self._launches = int(L_.ezb_launch_count() - n0)
            self.graph, self._key = g, key
            self.captures += 1
            self.lat.copy_(snap)   # capture does not execute; keep the eager result

    def finish(self, k: int, frames: int):
        """Decodes slot k alone at its own length (as inference() does) and frees it; returns the float32 waveform (hop * frames,), for a
        variation trimmed to its clip's length, or for an edit the whole edited clip (n_total,), as editing_audio returns it."""
        with torch.cuda.device(self.device):
            p = self.ez.params["autoencoder"]
            pred = scale_shift_re(self.lat[k:k + 1, :, :frames], p["scale"], p["shift"])
            edit = self.edits[k]
            if edit is not None:   # src/inference.py:104-105: the kept frames are the crop's latent, after the rescale
                regen = self.gt_mask[k, :frames].bool().view(1, 1, frames)
                pred = torch.where(regen, pred, self.gt[k:k + 1, :, :frames])
            wav = self.ez.autoencoder(embedding=pred.contiguous())
            self.lat[k].zero_()
            self.gens[k] = None
            if edit is None:
                n, self.trim[k] = self.trim[k], None
                return wav[0, 0, :n].cpu().numpy()
            clip, s0, n = edit
            post.splice_wave(clip, wav[0, 0], s0, n)
            for row in (k, self.S + k):
                self.gt[row].zero_()
                self.gt_mask[row].fill_(1)
            self.edits[k] = None
            return clip.cpu().numpy()


class ControlSlots(CudaSlots):
    """Device side of ContinuousEngine for an `api.EzAudio_ControlNet`: CudaSlots plus the ControlNet's context rows, condition cache and
    per-sample conditioning scales.  Every clip is 10 s long (the reference's), so the step runs without per-sample lengths.

    Between steps the engine also owns the ControlNet's context, timestep table and condition cache; the next step restores whatever a
    generate_audio call replaced."""
    control = True

    def __init__(self, ez, slots: int, table: Sequence[int], dpm: bool = False):
        super().__init__(ez, slots, 10.0, table, dpm=dpm)
        self.cn = ez.controlnet
        p = ez.params["autoencoder"]
        self.num_samples = int(10 * self.sr)
        if round(self.num_samples / self.sr * p["latent_sr"]) != self.max_frames:
            raise ValueError("the ControlNet clip length does not match the padded length")
        self.cond_kw = {k: v for k, v in ez.params["conditioner"].items() if k != "condition_type"}
        S, Be, L, D = self.S, 2 * self.S, self.max_frames, int(self.unet.cfg["embed_dim"])
        with torch.cuda.device(self.device):
            self.cond = torch.zeros(Be, 1, 2 * L, device=self.device)   # rows k and S + k: slot k's condition (the CFG rows repeat it)
            self._sh = torch.zeros(Be, dtype=torch.float32, pin_memory=True)
            self.scale = torch.zeros(Be, dtype=torch.float32, device=self.device)
            self.skips = [torch.empty(Be, L, D, device=self.device) for _ in range(self.cn.half)]
        self.n_samples: List[int] = [0] * S
        self._cn_ctx_epoch = self._cond_epoch = None

    def _own_denoiser(self):
        super()._own_denoiser()
        self.cn.set_timesteps(self.table)
        h = self.cn._h
        if self._cn_ctx_epoch != h.ctx_epoch:
            self.cn.set_context(self.ctx, self.cmask)
            self._cn_ctx_epoch = h.ctx_epoch
        if self._cond_epoch != self.cn.cond_epoch:
            self.cn.set_condition(self.cond)
            self._cond_epoch = self.cn.cond_epoch

    def admit(self, k: int, prompt: str, seed: Optional[int], frames: int, audio=None, surpass_noise: float = 0.0):
        from .api import energy_condition
        super().admit(k, prompt, seed, frames)   # the DiT's context row, the generator and the initial noise
        with torch.cuda.device(self.device):
            self.cn.set_context_rows(self.ctx[k:k + 1], self.cmask[k:k + 1], k)
            # normalise, noise-gate and pad / crop to 10 s, then the energy condition: generate_audio's preparation of one clip
            wave = post.prepare_wave(torch.from_numpy(audio).to(self.device).unsqueeze(0), self.num_samples, normalize=True, gate=surpass_noise)
            c = energy_condition(wave, **self.cond_kw)
            for row in (k, self.S + k):
                self.cond[row:row + 1].copy_(c)
                self.cn.set_condition_rows(self.cond[row:row + 1], row)
            self.n_samples[k] = len(audio)

    def _launch_step(self):
        S = self.S
        self.x_in[:S].copy_(self.lat)
        self.x_in[S:].copy_(self.lat)
        sk = self.cn.forward_step(self.x_in, t_index=self.t_index, scale=self.scale, outs=self.skips)
        self.unet.forward_step(self.x_in, 0, controlnet_skips=sk, out=self.out, t_index=self.t_index)
        self._launch_update(None)

    def step(self, plan: Sequence[Optional[SlotStep]]):
        with torch.cuda.device(self.device):
            if self._copied is not None:
                self._copied.synchronize()   # the previous step's copies have read the pinned blocks
            sh = self._sh.numpy()
            for k, e in enumerate(plan):
                sh[k] = sh[self.S + k] = 0.0 if e is None else e.conditioning_scale
            self.scale.copy_(self._sh, non_blocking=True)   # ordered before the event CudaSlots.step records after its own copy
        super().step(plan)

    def finish(self, k: int, frames: int):
        """As CudaSlots.finish, trimmed to the reference clip's length (api/controlnet.py:159)."""
        return super().finish(k, frames)[:self.n_samples[k]]
