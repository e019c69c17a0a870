"""DDIM scheduler (host-side control logic) -- restatement of `diffusers.DDIMScheduler` for the configuration the
reference instantiates (api/ezaudio.py:92-97 with ckpts/ezaudio-xl.yml:52-60; call sites src/inference.py:64,71,98-100).
diffusers is a third-party, un-pinned, un-vendored dependency of the reference (requirements.txt:2) and is absent from this
image, so the algorithm is restated from its published form (SURVEY Appendix B); parity at this boundary is unpinned
upstream and is checked by closed-form invariants (tests/test_scheduler.py).

Only the scalar schedule lives here; the tensor update runs in the fused CUDA kernel `ezb_cfg_ddim_step`.
"""
from __future__ import annotations

from typing import List, Tuple

import numpy as np
import torch


def _betas(num_train_timesteps, beta_start, beta_end, rescale_betas_zero_snr):
    """The scaled-linear betas, rescaled to zero terminal SNR when asked (fp32, diffusers op order)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    if rescale_betas_zero_snr:
        abar_sqrt = torch.cumprod(1.0 - betas, dim=0).sqrt()
        s0, sT = abar_sqrt[0].clone(), abar_sqrt[-1].clone()
        abar_sqrt = (abar_sqrt - sT) * (s0 / (s0 - sT))
        abar = abar_sqrt ** 2
        alphas = torch.cat([abar[0:1], abar[1:] / abar[:-1]])
        betas = 1 - alphas
    return betas


def trailing_timesteps(num_train_timesteps: int, num_inference_steps: int) -> torch.Tensor:
    """Trailing timestep spacing: num_train - 1 down to num_train / steps - 1."""
    if num_inference_steps > num_train_timesteps:
        raise ValueError("num_inference_steps exceeds num_train_timesteps")
    step_ratio = num_train_timesteps / num_inference_steps
    return torch.from_numpy(np.round(np.arange(num_train_timesteps, 0, -step_ratio)).astype(np.int64) - 1)


def start_index(num_inference_steps: int, strength: float) -> int:
    """First schedule index of an audio-to-audio variation, in diffusers' img2img convention: the last n_run = min(int(steps * strength),
    steps) steps run, from index steps - n_run.  strength outside (0, 1], or one that leaves no step to run, raises ValueError."""
    steps = int(num_inference_steps)
    if steps < 1 or steps != num_inference_steps:
        raise ValueError(f"num_inference_steps must be a positive step count, got {num_inference_steps!r}")
    if isinstance(strength, bool) or not isinstance(strength, (int, float, np.integer, np.floating)) or not 0 < strength <= 1:
        raise ValueError(f"strength must lie in (0, 1], got {strength!r}")
    n_run = min(int(steps * strength), steps)
    if n_run == 0:
        raise ValueError(f"strength {strength} runs no step of a {steps}-step schedule (int(steps * strength) = 0)")
    return steps - n_run


class DDIMScheduler:
    kind = "ddim"   # what sample_latents and the continuous engine dispatch on

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing", clip_sample=False,
                 set_alpha_to_one=True, **unused):
        if beta_schedule != "scaled_linear" or prediction_type != "v_prediction" or clip_sample or timestep_spacing != "trailing":
            raise NotImplementedError("only the shipped diffusion config (scaled_linear, v_prediction, trailing, no clipping)")
        self.num_train_timesteps = num_train_timesteps
        self.betas = betas = _betas(num_train_timesteps, beta_start, beta_end, rescale_betas_zero_snr)
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))
        self.num_inference_steps = None

    def set_timesteps(self, num_inference_steps: int):
        self.timesteps = trailing_timesteps(self.num_train_timesteps, num_inference_steps)
        self.num_inference_steps = num_inference_steps

    def scale_model_input(self, sample, timestep=None):
        return sample

    def add_noise_coefficients(self, timestep: int) -> Tuple[float, float]:
        """(a, s) of diffusers' add_noise at training timestep t, noisy = a * x0 + s * eps: (sqrt(abar_t), sqrt(1 - abar_t)) in fp32.  Under
        zero terminal SNR abar_999 is 0, so t = 999 gives exactly (0, 1)."""
        t = int(timestep)
        if not 0 <= t < self.num_train_timesteps:
            raise ValueError(f"timestep {timestep} outside 0..{self.num_train_timesteps - 1}")
        a = self.alphas_cumprod[t]
        return float(a ** 0.5), float((1 - a) ** 0.5)

    def step_coefficients(self, timestep: int, eta: float) -> List[float]:
        """[sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-sigma^2), sigma] of DDIMScheduler.step (fp32, diffusers op order):
        x0 = sqrt(a) x - sqrt(1-a) v ; eps = sqrt(a) v + sqrt(1-a) x ; prev = sqrt(a_prev) x0 + sqrt(1-a_prev-s^2) eps + s z."""
        t = int(timestep)
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        a = self.alphas_cumprod[t]
        ap = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        b = 1 - a
        variance = ((1 - ap) / b) * (1 - a / ap)
        sigma = eta * variance ** 0.5
        dirc = (1 - ap - sigma ** 2).clamp_min(0) ** 0.5  # radicand is >= 0 for the shipped schedule (tested); clamp guards round-off
        return [float(a ** 0.5), float(b ** 0.5), float(ap ** 0.5), float(dirc), float(sigma)]


class DPMSolverMultistepScheduler:
    """DPM-Solver++ multistep (Lu et al. 2022, arXiv:2211.01095) -- restatement of `diffusers.DPMSolverMultistepScheduler` for the shipped
    diffusion config (the constructor takes params['diff'] like DDIMScheduler) with solver_order 1 or 2, algorithm_type "dpmsolver++" or
    "sde-dpmsolver++", the midpoint second-order form, lower_order_final and final_sigmas_type "zero".  diffusers is absent, so the
    algorithm is restated from its published form and parity with diffusers itself is unpinned; the tests check it against the ODE solution
    of an analytic Gaussian model and against DDIM (order 1 is DDIM with eta = 0).  Everything else (order 3, the heun solver, Karras / Lu
    sigmas, thresholding, a non-zero final sigma) raises NotImplementedError.

    Timesteps are DDIMScheduler's (trailing spacing).  sigma_i = sqrt((1 - abar) / abar) at the timesteps, then a final sigma of 0; under
    zero terminal SNR abar[-1] is clamped to 2**-24 so that the first sigma is finite.  With alpha = 1 / sqrt(sigma^2 + 1) and
    sigma_t = sigma * alpha, step i turns the guided v-prediction v into m0 = alpha_s x - sigma_s v (the x0 prediction) and updates
        x <- kx x + k0 m0 + k1 (r (m0 - m1)) + kz z
    where m1 is the previous step's m0 and z a fresh Gaussian (sde-dpmsolver++ only).  Only the scalars live here; the tensor update runs in
    the fused CUDA kernel `ezb_cfg_dpm_step`, which keeps m0 per sample for the next step.  eta is ignored (diffusers' step() has none)."""

    kind = "dpm"

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing", solver_order=2,
                 algorithm_type="dpmsolver++", solver_type="midpoint", lower_order_final=True, euler_at_final=False, use_karras_sigmas=False,
                 use_lu_lambdas=False, final_sigmas_type="zero", thresholding=False, variance_type=None, **unused):
        if beta_schedule != "scaled_linear" or prediction_type != "v_prediction" or timestep_spacing != "trailing":
            raise NotImplementedError("only the shipped diffusion config (scaled_linear, v_prediction, trailing)")
        if solver_order not in (1, 2):
            raise NotImplementedError(f"solver_order {solver_order}: orders 1 and 2 are implemented")
        if algorithm_type not in ("dpmsolver++", "sde-dpmsolver++"):
            raise NotImplementedError(f"algorithm_type {algorithm_type!r}: dpmsolver++ and sde-dpmsolver++ are implemented")
        if solver_type != "midpoint":
            raise NotImplementedError(f"solver_type {solver_type!r}: the midpoint form is implemented")
        if use_karras_sigmas or use_lu_lambdas or thresholding or variance_type is not None:
            raise NotImplementedError("Karras / Lu sigmas, thresholding and learned variances are not implemented")
        if final_sigmas_type != "zero":
            raise NotImplementedError(f"final_sigmas_type {final_sigmas_type!r}: only 'zero' is implemented")
        self.num_train_timesteps = num_train_timesteps
        self.solver_order, self.algorithm_type = int(solver_order), algorithm_type
        self.lower_order_final, self.euler_at_final = bool(lower_order_final), bool(euler_at_final)
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, rescale_betas_zero_snr)
        self.alphas_cumprod = torch.cumprod(1.0 - self.betas, dim=0)
        if rescale_betas_zero_snr:
            self.alphas_cumprod[-1] = 2 ** -24   # keeps the first sigma finite
        self.init_noise_sigma = 1.0
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))
        self.num_inference_steps = None
        self.sigmas = None
        self.orders: List[int] = []

    @property
    def draws_noise(self) -> bool:
        """Whether every step takes a fresh Gaussian (sde-dpmsolver++): drawn at every step, the last one included, as diffusers does."""
        return self.algorithm_type == "sde-dpmsolver++"

    def set_timesteps(self, num_inference_steps: int):
        self.timesteps = trailing_timesteps(self.num_train_timesteps, num_inference_steps)
        self.num_inference_steps = n = num_inference_steps
        all_sigmas = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        sig = all_sigmas[self.timesteps.numpy()]
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        # order 1 at the first step (no history) and at the last (the final sigma is zero); solver_order in between
        self.orders = [1 if (i == 0 or i == n - 1 or self.solver_order == 1) else 2 for i in range(n)]

    def scale_model_input(self, sample, timestep=None):
        return sample

    @staticmethod
    def _alpha_sigma(sigma):
        alpha = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha, sigma * alpha

    def add_noise_coefficients(self, timestep: int) -> Tuple[float, float]:
        """(a, s) of diffusers' add_noise at timestep t of the schedule, noisy = a * x0 + s * eps: (alpha_t, sigma_t) of its sigma, fp32.
        At t = 999 the 2**-24 clamp gives a = 2**-12, not 0."""
        if self.sigmas is None:
            raise ValueError("call set_timesteps first")
        hit = (self.timesteps == int(timestep)).nonzero()
        if len(hit) == 0:
            raise ValueError(f"timestep {timestep} is not in the {self.num_inference_steps}-step schedule")
        alpha, sigma = self._alpha_sigma(self.sigmas[int(hit[0, 0])])
        return float(alpha), float(sigma)

    def step_coefficients(self, step_index: int, begin_index: int = 0):
        """(coef, order) of step `step_index`: coef = [alpha_s, sigma_s, kx, k0, k1, r, kz] of the update in the class docstring
        (k1 = r = 0 at order 1, kz = 0 without noise), fp32 in diffusers' order of operations.  At the last step lambda_t is infinite
        (sigma_t = 0); exp(-h) is then 0 and every coefficient is finite.  begin_index: the first step a run takes (an audio-to-audio
        variation starts part-way, diffusers' set_begin_index); that step has no history and is order 1.  An argument, not state, so that
        one scheduler serves runs that begin at different steps."""
        i, k = int(step_index), int(begin_index)
        if self.sigmas is None or not 0 <= i < len(self.orders):
            raise ValueError(f"step index {step_index} outside the schedule; call set_timesteps first")
        if not 0 <= k <= i:
            raise ValueError(f"begin index {begin_index} must lie in 0..{i} (the step index)")
        order = 1 if i == k else self.orders[i]
        alpha_t, sigma_t = self._alpha_sigma(self.sigmas[i + 1])
        alpha_s0, sigma_s0 = self._alpha_sigma(self.sigmas[i])
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)   # +inf at the last step
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        k1 = r = torch.tensor(0.0)
        kz = torch.tensor(0.0)
        if self.algorithm_type == "dpmsolver++":
            kx = sigma_t / sigma_s0
            k0 = -(alpha_t * (torch.exp(-h) - 1.0))
            if order == 2:
                k1 = -(0.5 * (alpha_t * (torch.exp(-h) - 1.0)))
        else:
            kx = sigma_t / sigma_s0 * torch.exp(-h)
            k0 = alpha_t * (1 - torch.exp(-2.0 * h))
            if order == 2:
                k1 = 0.5 * (alpha_t * (1 - torch.exp(-2.0 * h)))
            kz = sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h))
        if order == 2:
            alpha_s1, sigma_s1 = self._alpha_sigma(self.sigmas[i - 1])
            lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
            r0 = (lambda_s0 - lambda_s1) / h
            r = 1.0 / r0
        coef = [float(v) for v in (alpha_s0, sigma_s0, kx, k0, k1, r, kz)]
        if not all(np.isfinite(coef)):
            raise FloatingPointError(f"non-finite DPM-Solver++ coefficients at step {i}: {coef}")
        return coef, order
