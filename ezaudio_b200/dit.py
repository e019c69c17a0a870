"""Host-side mirror of the reference's denoiser modules, backed by libezb200.so.

`MaskDiT` keeps the call contract of src/models/conditioners.py:123-183 (and `.model` the one of
src/models/udit.py:281-362); `DiTControlNet` the one of src/models/controlnet.py:252-315.  They ingest
the reference state-dict unchanged (SURVEY Appendix D).  Tensors in, tensors out; all math runs in the
CUDA library -- there is no PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import torch

from . import _lib, weights

# "fp8": the QKV and GEGLU up-projections of every block on e4m3 operands (per-row scales), the rest as "bf16" (include/ezb200.h)
PRECISIONS = {"bf16": 0, "bf16x3": 1, "fp8": 2}


def check_fp8_config(cfg: dict):
    """The FP8 mode runs the packed three-heads-per-tile QKV kernel and the 256-wide GEGLU kernel only: configurations those cannot hold
    are rejected here, before any device work."""
    D, H = cfg["embed_dim"], cfg["num_heads"]
    dh = D // H
    if dh not in (64, 72) or H % 2 or D > 1152:
        raise ValueError(f"precision 'fp8' needs head dim 64 or 72 with an even head count and embed_dim <= 1152 "
                         f"(embed_dim {D}, heads {H}); use 'bf16' or 'bf16x3'")


def _as_f32c(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(dtype=torch.float32).contiguous()


class _Handle:
    """Owns one ezb_dit handle (a DiT or a ControlNet)."""
    _serial = 0

    def __init__(self, cfg: dict, controlnet: Optional[dict], precision: str, max_batch: int, max_len: int,
                 max_ctx_len: int, max_timesteps: int, device):
        weights.check_dit_config(cfg)
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {list(PRECISIONS)}")
        if precision == "fp8":
            check_fp8_config(cfg)
        self.cfg, self.cn = dict(cfg), (dict(controlnet) if controlnet else None)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.EzbError("ezaudio_b200 runs on CUDA devices only (no CPU path)")
        self.dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        D = cfg["embed_dim"]
        d = _lib.DitDesc(embed_dim=D, num_heads=cfg["num_heads"], depth=cfg["depth"], context_dim=cfg["context_dim"],
                         inner_dim=int(D * cfg["mlp_ratio"]), ada_rank=cfg["ada_sola_rank"],
                         ada_scaling=float(cfg["ada_sola_alpha"]) / float(cfg["ada_sola_rank"]),
                         latent_chans=cfg["out_chans"], is_controlnet=1 if controlnet else 0,
                         cond_c0=controlnet["cond_blocks"][0] if controlnet else 0,
                         cond_c1=controlnet["cond_blocks"][1] if controlnet else 0,
                         max_batch=max_batch, max_len=max_len, max_ctx_len=max_ctx_len, max_timesteps=max_timesteps,
                         precision=PRECISIONS[precision])
        if cfg["in_chans"] != 2 * cfg["out_chans"] + 1:
            raise NotImplementedError("in_chans must be 2*out_chans+1 (MaskDiT concat)")
        if controlnet and (len(controlnet["cond_blocks"]) != 2 or controlnet["cond_in"] != 1 or not controlnet.get("cond_mask", False)):
            raise NotImplementedError("controlnet stem: only cond_in=1, two cond_blocks, cond_mask=true")
        self.desc = d
        self.h = C.c_void_p()
        with torch.cuda.device(self.dev_index):
            _lib.check(_lib.lib().ezb_dit_create(C.byref(self.h), C.byref(d), self.dev_index))
        self.loaded = False
        self._ctx_key = None
        self.ctx_epoch = 0
        self._ts: List[int] = []
        _Handle._serial += 1
        self.serial = _Handle._serial   # identifies this handle in graph-cache keys (id() values are recycled)

    def __del__(self):
        try:
            if getattr(self, "h", None) and self.h.value:
                _lib.lib().ezb_dit_destroy(self.h)
                self.h = C.c_void_p()
        except Exception:
            pass

    def load_state_dict(self, sd: Dict[str, torch.Tensor], extra: Optional[Dict[str, torch.Tensor]] = None):
        L = _lib.lib()
        items = dict(sd)
        if extra:
            items.update(extra)
        with torch.cuda.device(self.dev_index):
            st = _lib.stream_ptr()
            for k, v in items.items():
                t = _as_f32c(v).to(self.device, non_blocking=True)
                shape = (C.c_int64 * t.dim())(*t.shape)
                _lib.check(L.ezb_dit_load_weight(self.h, k.encode(), _lib.ptr(t), shape, t.dim(), st))
                del t
            torch.cuda.current_stream().synchronize()
            _lib.check(L.ezb_dit_finalize_weights(self.h, st))
        self.loaded = True
        self._ts, self._ctx_key = [], None   # tables derived from the previous weights are stale

    # ---- step-invariant precompute
    def set_context(self, context: torch.Tensor, context_mask: Optional[torch.Tensor]):
        B, Lc, _ = context.shape
        ctx = _as_f32c(context).to(self.device)
        if context_mask is None:
            context_mask = torch.ones(B, Lc, dtype=torch.bool, device=self.device)
        m = context_mask.to(self.device).to(torch.uint8).contiguous()
        with torch.cuda.device(self.dev_index):
            _lib.check(_lib.lib().ezb_dit_set_context(self.h, _lib.ptr(ctx), _lib.ptr(m), B, Lc, _lib.stream_ptr()))
        self._keep = (ctx, m)
        self._ctx_key = None   # a direct set_context invalidates whatever ensure_context cached
        self.ctx_epoch += 1    # lets a holder of context rows (engine.ContinuousEngine) see that the layout was replaced

    def set_context_rows(self, context: torch.Tensor, context_mask: Optional[torch.Tensor], row0: int):
        n, Lc, _ = context.shape
        ctx = _as_f32c(context).to(self.device)
        if context_mask is None:
            context_mask = torch.ones(n, Lc, dtype=torch.bool, device=self.device)
        m = context_mask.to(self.device).to(torch.uint8).contiguous()
        with torch.cuda.device(self.dev_index):
            _lib.check(_lib.lib().ezb_dit_set_context_rows(self.h, _lib.ptr(ctx), _lib.ptr(m), int(row0), n, Lc, _lib.stream_ptr()))
        self._keep_rows = (ctx, m)
        self._ctx_key = None

    def set_timesteps(self, ts: Sequence[int]):
        ts = [int(t) for t in ts]
        if ts == self._ts:   # the tables depend on the weights and the timestep values only: a repeated schedule (every job of a server) reuses them
            return
        arr = (C.c_int64 * len(ts))(*ts)
        with torch.cuda.device(self.dev_index):
            _lib.check(_lib.lib().ezb_dit_set_timesteps(self.h, arr, len(ts), _lib.stream_ptr()))
        self._ts = ts

    # ---- generic-call conveniences (module-compatible path: recompute only what changed)
    def ensure_context(self, context, context_mask):
        key = (context.data_ptr(), context._version, tuple(context.shape),
               None if context_mask is None else (context_mask.data_ptr(), context_mask._version))
        if key != self._ctx_key:
            self.set_context(context, context_mask)
            self._ctx_key = key
            self._ctx_refs = (context, context_mask)   # keep the originals alive: the key is made of their addresses

    def ensure_timesteps(self, timesteps: torch.Tensor, B: int):
        tv = [int(timesteps)] * B if timesteps.dim() == 0 else [int(v) for v in timesteps.tolist()]
        if any(t not in self._ts for t in tv):
            self.set_timesteps(sorted(set(tv)))
        return [self._ts.index(t) for t in tv]

    @staticmethod
    def _mask_u8(gt_mask, B, L, device):
        if gt_mask is None:
            return None
        m = gt_mask.to(device)
        if m.dim() == 3:
            if m.shape[1] > 1 and not bool((m == m[:, :1]).all()):
                raise NotImplementedError("mae_mask_infer must be identical across channels (api/ezaudio.py:179-182)")
            m = m[:, 0]
        return m.reshape(B, L).to(torch.uint8).contiguous()


class UDiTView:
    """`unet.model(x257, t, context, context_mask=, controlnet_skips=)` of the reference (udit.py:281)."""

    def __init__(self, owner: "MaskDiT"):
        self._o = owner

    def __call__(self, x, timesteps, context, x_mask=None, context_mask=None, cls_token=None, controlnet_skips=None):
        Cc = self._o.cfg["out_chans"]
        if x.shape[1] != 2 * Cc + 1:
            raise ValueError("UDiT input must be the 2C+1 channel concat produced by MaskDiT(forward_model=False)")
        return self._o._forward_raw(x[:, :Cc], x[:, Cc:2 * Cc], x[:, 2 * Cc] > 0.5, timesteps, context, context_mask,
                                    controlnet_skips, gt_is_final=True)


class MaskDiT:
    """Drop-in for src/models/conditioners.py::MaskDiT (inference branches)."""

    def __init__(self, precision: str = "bf16", max_batch: int = 8, max_len: int = 512, max_ctx_len: int = 128,
                 max_timesteps: int = 128, device="cuda", **cfg):
        self.cfg = dict(cfg)
        self._h = _Handle(cfg, None, precision, max_batch, max_len, max_ctx_len, max_timesteps, device)
        self.device = self._h.device
        self.precision = precision
        self.model = UDiTView(self)
        self._mask_embed = None

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def load_state_dict(self, sd, strict: bool = True):
        self._h.load_state_dict(sd)
        self._mask_embed = _as_f32c(sd["mask_embed"]).to(self.device)
        return self

    # fast path used by the sampling loop
    def set_context(self, context, context_mask):
        self._h.set_context(context, context_mask)

    def set_timesteps(self, ts):
        self._h.set_timesteps(ts)

    def set_context_rows(self, context, context_mask, row0: int):
        """Replaces the text context of samples [row0, row0 + n) (context (n,Lc,ctx), context_mask (n,Lc)) in the layout of the last
        set_context, without recomputing the other rows; Lc must be that call's.  The rows come out as set_context of the whole updated
        batch computes them."""
        self._h.set_context_rows(context, context_mask, row0)

    def forward_step(self, x, step_index: int, gt=None, gt_mask_u8=None, controlnet_skips=None, out=None, lengths=None, t_index=None):
        """One denoiser forward at table row `step_index` (all samples share it).  x (Be,C,L) fp32 cuda.
        `lengths`: None, or a cuda int32 tensor (Be,) of clip lengths in 1..L (padded batch): frames < lengths[b] of sample b come out as a
        forward of that clip alone computes them; frames past it are not written.  The values are read on the device when the kernels run
        (so a captured graph follows later copies into the tensor) and are not checked here: the caller validates them.
        `t_index`: None, or a cuda int32 tensor (Be,) of per-sample table rows used instead of `step_index`; read on the device like
        `lengths` (out-of-range rows are clamped, the caller validates them)."""
        Be, Cc, L = x.shape
        if lengths is not None:
            if controlnet_skips is not None:
                raise NotImplementedError("per-sample lengths with ControlNet skips")
            if gt is not None and gt_mask_u8 is None:   # the padded frames of gt must be marked as regenerated, which takes a mask
                raise NotImplementedError("per-sample lengths with inpainting (gt) need gt_mask_u8, set past each clip's end")
            if lengths.dtype != torch.int32 or not lengths.is_cuda or tuple(lengths.shape) != (Be,) or not lengths.is_contiguous():
                raise ValueError(f"lengths must be a contiguous cuda int32 tensor of shape ({Be},)")
        if t_index is not None and (t_index.dtype != torch.int32 or not t_index.is_cuda or tuple(t_index.shape) != (Be,) or not t_index.is_contiguous()):
            raise ValueError(f"t_index must be a contiguous cuda int32 tensor of shape ({Be},)")
        out = torch.empty_like(x) if out is None else out
        sk = None
        if controlnet_skips is not None:
            sk = (C.c_void_p * len(controlnet_skips))(*[s.data_ptr() for s in controlnet_skips])
        with torch.cuda.device(self._h.dev_index):
            if t_index is not None:
                _lib.check(_lib.lib().ezb_dit_forward_tdev(self._h.h, _lib.ptr(x), _lib.ptr(gt), _lib.ptr(gt_mask_u8), _lib.ptr(t_index), sk,
                                                           _lib.ptr(out), Be, L, _lib.stream_ptr(), _lib.ptr(lengths)))
            else:
                _lib.check(_lib.lib().ezb_dit_forward(self._h.h, _lib.ptr(x), _lib.ptr(gt), _lib.ptr(gt_mask_u8), None, int(step_index),
                                                      sk, _lib.ptr(out), Be, L, _lib.stream_ptr(), _lib.ptr(lengths)))
        return out

    def _forward_raw(self, x, gt, gt_mask, timesteps, context, context_mask, controlnet_skips, gt_is_final=False):
        h = self._h
        Be, Cc, L = x.shape
        x = _as_f32c(x).to(self.device)
        h.ensure_context(context, context_mask)
        tidx = h.ensure_timesteps(timesteps if torch.is_tensor(timesteps) else torch.tensor(timesteps), Be)
        gtc = None if gt is None else _as_f32c(gt).to(self.device)
        m8 = None
        if gt is not None:
            m8 = h._mask_u8(gt_mask, Be, L, self.device) if gt_mask is not None else torch.zeros(Be, L, dtype=torch.uint8, device=self.device)
            if gt_is_final:  # gt already holds mask_embed where masked: channel mask only feeds the mask channel
                pass
        out = torch.empty_like(x)
        arr = (C.c_int32 * Be)(*tidx)
        sk = None
        if controlnet_skips:
            sks = [_as_f32c(s).to(self.device) for s in controlnet_skips]   # converted copies are kept alive until the next call
            sk = (C.c_void_p * len(sks))(*[s.data_ptr() for s in sks])
            self._keep_sk = sks
        with torch.cuda.device(h.dev_index):
            _lib.check(_lib.lib().ezb_dit_forward(h.h, _lib.ptr(x), _lib.ptr(gtc), _lib.ptr(m8), arr, 0, sk, _lib.ptr(out), Be, L,
                                                  _lib.stream_ptr(), None))
        return out

    def __call__(self, x, timesteps, context, x_mask=None, context_mask=None, cls_token=None, gt=None, mae_mask_infer=None,
                 forward_model=True):
        """conditioners.py:156-183.  Returns (out, mae_mask)."""
        if x_mask is not None or cls_token is not None:
            raise NotImplementedError("x_mask / cls_token are not used by the shipped configs")
        if gt is not None and mae_mask_infer is None:
            raise NotImplementedError("training-time random masking (mae_mask_infer=None with gt) is out of scope")
        mae_mask = torch.ones_like(x) if gt is None else mae_mask_infer.expand_as(gt).type_as(gt)
        if not forward_model:  # pure data movement (conditioners.py:150-153,174-176)
            me = self._mask_embed.view(1, -1, 1).to(x.dtype)
            g = me.expand_as(x) if gt is None else torch.where(mae_mask_infer.expand_as(gt), me.expand_as(gt), gt)
            return torch.cat([x, g, mae_mask[:, 0:1, :]], dim=1), mae_mask
        out = self._forward_raw(x, gt, mae_mask_infer, timesteps, context, context_mask, None)
        return out, mae_mask

    forward = __call__


class DiTControlNet:
    """Drop-in for src/models/controlnet.py::DiTControlNet (eval path).  `mask_embed` of the paired MaskDiT is needed
    because the library rebuilds the 2C+1 channel input itself."""

    def __init__(self, precision: str = "bf16", max_batch: int = 8, max_len: int = 512, max_ctx_len: int = 128,
                 max_timesteps: int = 128, device="cuda", cond_in=1, cond_blocks=None, cond_mask=True, cond_mask_prob=None,
                 cond_mask_ratio=None, cond_mask_span=None, **cfg):
        self.cfg = dict(cfg)
        self.cn = dict(cond_in=cond_in, cond_blocks=list(cond_blocks), cond_mask=cond_mask)
        self._h = _Handle(cfg, self.cn, precision, max_batch, max_len, max_ctx_len, max_timesteps, device)
        self.device = self._h.device
        self.half = cfg["depth"] // 2
        self.cond_epoch = 0

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def load_state_dict(self, sd, mask_embed: torch.Tensor, strict: bool = True):
        self._h.load_state_dict(sd, extra={"mask_embed": mask_embed})
        return self

    def set_context(self, context, context_mask):
        self._h.set_context(context, context_mask)

    def set_timesteps(self, ts):
        self._h.set_timesteps(ts)

    def set_context_rows(self, context, context_mask, row0: int):
        """As MaskDiT.set_context_rows."""
        self._h.set_context_rows(context, context_mask, row0)

    def _cond(self, condition, n: int, L: int) -> torch.Tensor:
        cond = _as_f32c(condition).to(self.device)
        if tuple(cond.shape) != (n, 1, 2 * L):
            raise ValueError(f"condition must be (n,1,2L)={(n, 1, 2 * L)}, got {tuple(cond.shape)}")
        return cond

    def set_condition(self, condition):
        """Runs the stem of condition (Be,1,2L) once into the handle's condition cache, which `forward_step(t_index=, scale=)` reads; this fixes
        the cache layout (Be, L).  ezb_controlnet_forward (the other call paths) neither reads nor writes the cache."""
        Be, L = int(condition.shape[0]), int(condition.shape[-1]) // 2
        cond = self._cond(condition, Be, L)
        with torch.cuda.device(self._h.dev_index):
            _lib.check(_lib.lib().ezb_controlnet_set_condition(self._h.h, _lib.ptr(cond), Be, L, _lib.stream_ptr()))
        self._keep_cond = cond
        self.cond_epoch += 1   # lets a holder of condition rows (engine.ContinuousEngine) see that the layout was replaced

    def set_condition_rows(self, condition, row0: int):
        """Replaces the cached condition of samples [row0, row0 + n) (condition (n,1,2L), L that of the last set_condition) without
        recomputing the other rows; they come out as set_condition of the whole updated batch computes them."""
        n, L = int(condition.shape[0]), int(condition.shape[-1]) // 2
        cond = self._cond(condition, n, L)
        with torch.cuda.device(self._h.dev_index):
            _lib.check(_lib.lib().ezb_controlnet_set_condition_rows(self._h.h, _lib.ptr(cond), int(row0), n, L, _lib.stream_ptr()))
        self._keep_cond_rows = cond

    def _run(self, x, gt, m8, tidx_arr, tall, condition, scale, outs):
        Be, Cc, L = x.shape
        D = self.cfg["embed_dim"]
        if outs is None:
            outs = [torch.empty(Be, L, D, device=self.device, dtype=torch.float32) for _ in range(self.half)]
        arr = (C.c_void_p * self.half)(*[o.data_ptr() for o in outs])
        cond = _as_f32c(condition).to(self.device)
        if cond.shape != (Be, 1, 2 * L):
            raise ValueError(f"condition must be (B,1,2L)={(Be, 1, 2 * L)}, got {tuple(cond.shape)}")
        with torch.cuda.device(self._h.dev_index):
            _lib.check(_lib.lib().ezb_controlnet_forward(self._h.h, _lib.ptr(x), _lib.ptr(gt), _lib.ptr(m8), tidx_arr, tall, _lib.ptr(cond),
                                                         float(scale), arr, Be, L, _lib.stream_ptr()))
        return outs

    def forward_step(self, x, step_index=0, condition=None, conditioning_scale=1.0, gt=None, gt_mask_u8=None, outs=None, t_index=None, scale=None):
        """One ControlNet forward at table row `step_index` on `condition` (Be,1,2L) with one `conditioning_scale`; returns depth/2 skips
        (Be,L,D) fp32 (written into `outs` when given).
        Without `condition` (and without `t_index` / `scale`) it reads the condition cache of set_condition instead, whose layout (Be, L) x
        must match (EzbError otherwise): the skips are bit-identical to passing the condition that was cached, and the stem, which does not
        depend on the step, does not run again (ezb_controlnet_forward_cached).
        With `t_index` and `scale` -- contiguous cuda int32 / fp32 tensors of shape (Be,), read on the device when the kernels run, like
        MaskDiT.forward_step's t_index -- sample b runs at table row t_index[b] on the cached condition of set_condition with its skips times
        scale[b] (0 gives zeros); `condition`, `gt` and `gt_mask_u8` are then not accepted."""
        if t_index is None and scale is None and condition is not None:
            return self._run(x, gt, gt_mask_u8, None, int(step_index), condition, conditioning_scale, outs)
        Be, Cc, L = x.shape
        if t_index is None and scale is None:
            if outs is None:
                outs = [torch.empty(Be, L, self.cfg["embed_dim"], device=self.device, dtype=torch.float32) for _ in range(self.half)]
            arr = (C.c_void_p * self.half)(*[o.data_ptr() for o in outs])
            with torch.cuda.device(self._h.dev_index):
                _lib.check(_lib.lib().ezb_controlnet_forward_cached(self._h.h, _lib.ptr(x), _lib.ptr(gt), _lib.ptr(gt_mask_u8), None, int(step_index),
                                                                    float(conditioning_scale), arr, Be, L, _lib.stream_ptr()))
            return outs
        if t_index is None or scale is None:
            raise ValueError("t_index and scale go together")
        if condition is not None or gt is not None or gt_mask_u8 is not None:
            raise ValueError("forward_step(t_index=, scale=) reads the condition cache of set_condition and takes no gt")
        for name, v, dt in (("t_index", t_index, torch.int32), ("scale", scale, torch.float32)):
            if v.dtype != dt or not v.is_cuda or tuple(v.shape) != (Be,) or not v.is_contiguous():
                raise ValueError(f"{name} must be a contiguous cuda {dt} tensor of shape ({Be},)")
        if outs is None:
            outs = [torch.empty(Be, L, self.cfg["embed_dim"], device=self.device, dtype=torch.float32) for _ in range(self.half)]
        arr = (C.c_void_p * self.half)(*[o.data_ptr() for o in outs])
        with torch.cuda.device(self._h.dev_index):
            _lib.check(_lib.lib().ezb_controlnet_forward_tdev(self._h.h, _lib.ptr(x), _lib.ptr(t_index), _lib.ptr(scale), arr, Be, L,
                                                              _lib.stream_ptr()))
        return outs

    def __call__(self, x, timesteps, context, x_mask=None, context_mask=None, cls_token=None, condition=None, cond_mask_infer=None,
                 conditioning_scale=1.0):
        """x is the 2C+1 channel concat from MaskDiT(forward_model=False) (src/inference_controlnet.py:89-96)."""
        Cc = self.cfg["out_chans"]
        Be, _, L = x.shape
        h = self._h
        h.ensure_context(context, context_mask)
        tidx = h.ensure_timesteps(timesteps if torch.is_tensor(timesteps) else torch.tensor(timesteps), Be)
        xs, gt = _as_f32c(x[:, :Cc]).to(self.device), _as_f32c(x[:, Cc:2 * Cc]).to(self.device)
        m8 = (x[:, 2 * Cc] > 0.5).to(torch.uint8).contiguous()
        # gt already carries mask_embed at masked positions; the library re-applies the same substitution (idempotent)
        return self._run(xs, gt, m8, (C.c_int32 * Be)(*tidx), 0, condition, conditioning_scale, None)

    forward = __call__
