"""Schedulers of the sampling pipeline.

`DDIMScheduler` holds the constants of the released MV-VDM (configs/inference/inference.yaml:36-42 of the reference: linear
betas 0.00085..0.012, 1000 train steps, leading spacing, steps_offset 1).  Its update runs in the a3d_ddim_step /
a3d_ddim_cfg_step kernel fused with classifier-free guidance and the frame-0 re-injection of pipeline.py:1023-1031; this
class owns the per-step coefficients that kernel is given.

`DPMSolverMultistepScheduler`, `EulerDiscreteScheduler` and `EulerAncestralDiscreteScheduler` are the other schedulers the
reference pipeline's constructor takes (pipeline.py:315-322), with diffusers 0.28.0 names, constructor arguments, attributes
and arithmetic (DESIGN section 4, "parity unpinned").  In the pipeline their update runs in the a3d_sampler_step kernel;
`next_step(t)` gives that kernel's scalars, computed in fp32 in diffusers' order of operations, and advances the step
counter.  `step()` is the same update in torch for callers outside the pipeline.  `from_config` takes a scheduler or its
`config`, so `DPMSolverMultistepScheduler.from_config(pipe.scheduler.config)` works as with diffusers."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

SAMPLER_DPMPP, SAMPLER_EULER = 0, 1          # a3d_sampler_step_args.kind


class _ConfigMixin:
    """diffusers' ConfigMixin surface: `config` (a dict of the constructor arguments, plus `_class_name`) and
    `from_config(config_or_scheduler, **overrides)`, which ignores keys the class does not take."""

    @classmethod
    def from_config(cls, config=None, **kwargs):
        cfg = dict(getattr(config, "config", config) or {})
        cfg.update(kwargs)
        return cls(**{k: v for k, v in cfg.items() if not k.startswith("_")})

    def _register(self, **kw):
        self.config = {"_class_name": type(self).__name__, **kw}


def _only(cls_name: str, option: str, value, allowed) -> None:
    if value not in allowed:
        raise NotImplementedError(f"{cls_name}: {option}={value!r} is not supported (supported: "
                                  f"{', '.join(repr(a) for a in allowed)})")


class DDIMScheduler(_ConfigMixin):
    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="linear",
                 steps_offset=1, clip_sample=False, set_alpha_to_one=True, **unused):
        if beta_schedule != "linear" or clip_sample:
            raise NotImplementedError("only the released configuration (linear betas, no clipping) is supported")
        self._register(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                       beta_schedule=beta_schedule, trained_betas=None, clip_sample=clip_sample,
                       set_alpha_to_one=set_alpha_to_one, steps_offset=steps_offset, prediction_type="epsilon",
                       thresholding=False, timestep_spacing="leading", rescale_betas_zero_snr=False)
        betas = np.linspace(beta_start, beta_end, num_train_timesteps, dtype=np.float32)
        self.alphas_cumprod = np.cumprod((1.0 - betas).astype(np.float32), dtype=np.float32)
        self.final_alpha_cumprod = np.float32(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_train_timesteps = num_train_timesteps
        self.steps_offset = steps_offset
        self.init_noise_sigma = 1.0
        self.order = 1
        self.timesteps = None
        self.num_inference_steps = None

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.num_train_timesteps // num_inference_steps
        self.timesteps = (np.arange(0, num_inference_steps) * ratio).round()[::-1].astype(np.int64) + self.steps_offset
        return self.timesteps

    def get_timesteps(self, num_inference_steps, strength):
        """The last int(n * strength) of the n steps (reference pipeline.py:667-674, after retrieve_timesteps).  The
        schedule keeps n steps, so prev_t of every step keeps the stride num_train_timesteps // n."""
        self.set_timesteps(num_inference_steps)
        init = min(int(num_inference_steps * strength), num_inference_steps)
        return self.timesteps[max(num_inference_steps - init, 0):]

    def _alphas(self, t: int):
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        return self.alphas_cumprod[t], self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod

    def alphas_for(self, t: int):
        a_t, a_p = self._alphas(t)
        return float(a_t), float(a_p)

    def step_coefficients(self, t: int, eta: float = 0.0):
        """(alpha_t, alpha_prev, dir_coef, std_dev) of DDIMScheduler.step(eps, t, x, eta) (diffusers 0.28.0), in fp32 and in
        its order of operations: variance = (1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev), std_dev = eta sqrt(variance),
        dir_coef = sqrt(1 - a_prev - std_dev^2).  x' = sqrt(a_prev) x0 + dir_coef eps + std_dev z."""
        a_t, a_p = self._alphas(t)
        one = np.float32(1.0)
        variance = ((one - a_p) / (one - a_t)) * (one - a_t / a_p)
        std_dev = np.float32(eta) * np.sqrt(variance)
        dir_coef = np.sqrt(one - a_p - std_dev * std_dev)
        return float(a_t), float(a_p), float(dir_coef), float(std_dev)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps) -> torch.Tensor:
        """sqrt(a_t) x + sqrt(1 - a_t) noise, with `timesteps` one per sample (or one for all) broadcast over the trailing
        dimensions (diffusers DDIMScheduler.add_noise; SURVEY Appendix B.10)."""
        ac = torch.from_numpy(self.alphas_cumprod).to(device=original_samples.device, dtype=original_samples.dtype)
        a = ac[torch.as_tensor(timesteps, device=original_samples.device).long()].flatten()
        while a.ndim < original_samples.ndim:
            a = a.unsqueeze(-1)
        return a ** 0.5 * original_samples + (1 - a) ** 0.5 * noise

    def scale_model_input(self, sample, t=None):
        return sample


# ------------------------------------------------------------------------------------------------ sigma-space schedulers
@dataclass(frozen=True)
class SolverStep:
    """The scalars of one a3d_sampler_step launch (include/a3d.h), each an fp32 value.  DPM-Solver++: m0 = (x - sigma_s0 eps)
    / alpha_s0, x' = c_x x - c_m0 m0 (+ c_d1 inv_r0 (m0 - m1) at order 2).  Euler: x' = x + d dt (+ sigma_up z)."""
    kind: int
    index: int                   # step index into `sigmas`
    order: int = 1
    alpha_s0: float = 1.0
    sigma_s0: float = 0.0
    c_x: float = 0.0
    c_m0: float = 0.0
    inv_r0: float = 0.0
    c_d1: float = 0.0
    sigma: float = 0.0
    dt: float = 0.0
    sigma_up: float = 0.0


@dataclass
class SchedulerOutput:
    prev_sample: torch.Tensor


def _check_common(name, beta_schedule, trained_betas, prediction_type, timestep_spacing, rescale_betas_zero_snr):
    _only(name, "beta_schedule", beta_schedule, ("linear",))
    _only(name, "trained_betas", trained_betas, (None,))
    _only(name, "prediction_type", prediction_type, ("epsilon",))
    _only(name, "timestep_spacing", timestep_spacing, ("linspace", "leading", "trailing"))
    _only(name, "rescale_betas_zero_snr", rescale_betas_zero_snr, (False,))


def _linear_alphas_cumprod(num_train_timesteps, beta_start, beta_end) -> torch.Tensor:
    betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    return torch.cumprod(1.0 - betas, dim=0)


def _train_sigmas(alphas_cumprod: torch.Tensor) -> np.ndarray:
    """sigma of every train timestep, ((1 - a) / a)^0.5 in fp32."""
    return (((1 - alphas_cumprod) / alphas_cumprod) ** 0.5).numpy()


def _sigma_to_t(sigma: np.ndarray, log_sigmas: np.ndarray) -> np.ndarray:
    """Fractional train timestep of each sigma by linear interpolation in log sigma (diffusers `_sigma_to_t`)."""
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    return ((1 - w) * low_idx + w * high_idx).reshape(sigma.shape)


def _truncated(scheduler, num_inference_steps, strength):
    """The last int(n * strength) timesteps of the n-step schedule (reference pipeline.py:667-674 after retrieve_timesteps;
    order 1).  The scheduler keeps the whole schedule, and its step index starts at the first kept timestep."""
    scheduler.set_timesteps(num_inference_steps)
    init = min(int(num_inference_steps * strength), num_inference_steps)
    return scheduler.timesteps[max(num_inference_steps - init, 0) * scheduler.order:]


class DPMSolverMultistepScheduler(_ConfigMixin):
    """diffusers 0.28.0 DPMSolverMultistepScheduler, algorithm "dpmsolver++", epsilon prediction, order 1 or 2."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear", trained_betas=None,
                 solver_order=2, prediction_type="epsilon", thresholding=False, dynamic_thresholding_ratio=0.995,
                 sample_max_value=1.0, algorithm_type="dpmsolver++", solver_type="midpoint", lower_order_final=True,
                 euler_at_final=False, use_karras_sigmas=False, use_lu_lambdas=False, final_sigmas_type="zero",
                 lambda_min_clipped=-float("inf"), variance_type=None, timestep_spacing="linspace", steps_offset=0,
                 rescale_betas_zero_snr=False, **unused):
        name = type(self).__name__
        _check_common(name, beta_schedule, trained_betas, prediction_type, timestep_spacing, rescale_betas_zero_snr)
        _only(name, "algorithm_type", algorithm_type, ("dpmsolver++",))
        _only(name, "solver_order", solver_order, (1, 2))
        _only(name, "solver_type", solver_type, ("midpoint", "heun"))
        _only(name, "final_sigmas_type", final_sigmas_type, ("zero", "sigma_min"))
        _only(name, "thresholding", thresholding, (False,))
        _only(name, "use_lu_lambdas", use_lu_lambdas, (False,))
        _only(name, "variance_type", variance_type, (None,))
        _only(name, "lambda_min_clipped", lambda_min_clipped, (-float("inf"),))
        self._register(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                       beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
                       prediction_type=prediction_type, thresholding=thresholding,
                       dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
                       algorithm_type=algorithm_type, solver_type=solver_type, lower_order_final=lower_order_final,
                       euler_at_final=euler_at_final, use_karras_sigmas=use_karras_sigmas, use_lu_lambdas=use_lu_lambdas,
                       final_sigmas_type=final_sigmas_type, lambda_min_clipped=lambda_min_clipped,
                       variance_type=variance_type, timestep_spacing=timestep_spacing, steps_offset=steps_offset,
                       rescale_betas_zero_snr=rescale_betas_zero_snr)
        self.num_train_timesteps = num_train_timesteps
        self.alphas_cumprod = _linear_alphas_cumprod(num_train_timesteps, beta_start, beta_end)
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.sigmas = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5
        self.init_noise_sigma = 1.0
        self.order = 1
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps,
                                                      dtype=np.float32)[::-1].copy())
        self.model_outputs = [None] * solver_order
        self.lower_order_nums = 0
        self._step_index = None

    @property
    def step_index(self):
        return self._step_index

    def set_timesteps(self, num_inference_steps, device=None):
        """The n-step schedule (int64 timesteps, n + 1 fp32 sigmas); clears the solver history."""
        cfg, T, n = self.config, self.num_train_timesteps, num_inference_steps
        if cfg["timestep_spacing"] == "linspace":
            timesteps = np.linspace(0, T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif cfg["timestep_spacing"] == "leading":
            step_ratio = T // (n + 1)
            timesteps = (np.arange(0, n + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
            timesteps += cfg["steps_offset"]
        else:                                                                            # trailing
            timesteps = np.arange(T, 0, -T / n).round().copy().astype(np.int64) - 1
        sigmas = _train_sigmas(self.alphas_cumprod)
        if cfg["use_karras_sigmas"]:
            log_sigmas = np.log(sigmas)
            flipped = np.flip(sigmas).copy()
            sigma_min, sigma_max = flipped[-1].item(), flipped[0].item()
            rho = 7.0
            ramp = np.linspace(0, 1, n)
            min_inv_rho, max_inv_rho = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
            sigmas = (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho
            timesteps = _sigma_to_t(sigmas, log_sigmas).round()
        else:
            sigmas = np.interp(timesteps, np.arange(0, len(sigmas)), sigmas)
        sigma_last = _train_sigmas(self.alphas_cumprod)[0] if cfg["final_sigmas_type"] == "sigma_min" else 0
        self.sigmas = torch.from_numpy(np.concatenate([sigmas, [sigma_last]]).astype(np.float32))
        self.timesteps = torch.from_numpy(timesteps).to(device=device, dtype=torch.int64)
        self.num_inference_steps = len(timesteps)
        self.model_outputs = [None] * cfg["solver_order"]
        self.lower_order_nums = 0
        self._step_index = None
        return self.timesteps

    def index_for_timestep(self, timestep, schedule_timesteps=None) -> int:
        """Index of `timestep` in the schedule: the second match if there are several, the last index if there is none."""
        if schedule_timesteps is None:
            schedule_timesteps = self.timesteps
        cand = (schedule_timesteps == torch.as_tensor(timestep).to(schedule_timesteps.device)).nonzero()
        if len(cand) == 0:
            return len(self.timesteps) - 1
        return cand[1 if len(cand) > 1 else 0].item()

    def _init_step_index(self, timestep):
        self._step_index = self.index_for_timestep(timestep)

    def get_timesteps(self, num_inference_steps, strength):
        return _truncated(self, num_inference_steps, strength)

    def scale_model_input(self, sample, timestep=None):
        return sample

    @staticmethod
    def _sigma_to_alpha_sigma_t(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def _coefficients(self, i: int, order: int) -> SolverStep:
        """fp32 torch scalars of step i in the order of diffusers' dpm_solver_first_order_update /
        multistep_dpm_solver_second_order_update.  sigma_next = 0 gives lambda_t = +inf, c_x = 0 and c_m0 = -1: x' = m0."""
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(self.sigmas[i + 1])
        alpha_s0, sigma_s0 = self._sigma_to_alpha_sigma_t(self.sigmas[i])
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        c_x = sigma_t / sigma_s0
        c_m0 = alpha_t * (torch.exp(-h) - 1.0)
        inv_r0 = c_d1 = 0.0
        if order == 2:
            alpha_s1, sigma_s1 = self._sigma_to_alpha_sigma_t(self.sigmas[i - 1])
            lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
            r0 = (lambda_s0 - lambda_s1) / h
            inv_r0 = float(1.0 / r0)
            if self.config["solver_type"] == "midpoint":
                c_d1 = -float(0.5 * (alpha_t * (torch.exp(-h) - 1.0)))        # x' = ... - 0.5 a_t (e^-h - 1) D1
            else:
                c_d1 = float(alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0))
        return SolverStep(SAMPLER_DPMPP, i, order, alpha_s0=float(alpha_s0), sigma_s0=float(sigma_s0), c_x=float(c_x),
                          c_m0=float(c_m0), inv_r0=inv_r0, c_d1=c_d1)

    def next_step(self, timestep) -> SolverStep:
        """The scalars of the step at `timestep`, and the step counter advanced as `step()` advances it: first order on the
        first step since set_timesteps and on a final step that asks for it (final_sigmas_type "zero", euler_at_final, or
        lower_order_final with fewer than 15 steps)."""
        if self._step_index is None:
            self._init_step_index(timestep)
        i, n, cfg = self._step_index, len(self.timesteps), self.config
        lower_order_final = i == n - 1 and (cfg["euler_at_final"] or (cfg["lower_order_final"] and n < 15)
                                            or cfg["final_sigmas_type"] == "zero")
        order = 1 if cfg["solver_order"] == 1 or self.lower_order_nums < 1 or lower_order_final else 2
        s = self._coefficients(i, order)
        if self.lower_order_nums < cfg["solver_order"]:
            self.lower_order_nums += 1
        self._step_index += 1
        return s

    def step(self, model_output, timestep, sample, generator=None, variance_noise=None, return_dict=True):
        """DPMSolverMultistepScheduler.step in torch; no noise is drawn."""
        s = self.next_step(timestep)
        sample = sample.to(torch.float32)
        m0 = (sample - s.sigma_s0 * model_output) / s.alpha_s0
        self.model_outputs = self.model_outputs[1:] + [m0]
        x = s.c_x * sample - s.c_m0 * m0
        if s.order == 2:
            x = x + s.c_d1 * (s.inv_r0 * (m0 - self.model_outputs[-2]))
        x = x.to(model_output.dtype)
        return SchedulerOutput(x) if return_dict else (x,)

    def add_noise(self, original_samples, noise, timesteps):
        """alpha x + sigma~ noise at the sigma of each timestep's index (index_for_timestep)."""
        sigmas = self.sigmas.to(device=original_samples.device, dtype=original_samples.dtype)
        schedule = self.timesteps.to(original_samples.device)
        ts = torch.as_tensor(timesteps).to(original_samples.device).reshape(-1)
        sigma = sigmas[[self.index_for_timestep(t, schedule) for t in ts]].flatten()
        while sigma.ndim < original_samples.ndim:
            sigma = sigma.unsqueeze(-1)
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma)
        return alpha_t * original_samples + sigma_t * noise


class _EulerBase(_ConfigMixin):
    """Schedule, input scaling and noising shared by the two Euler schedulers (diffusers 0.28.0)."""

    def _setup(self, num_train_timesteps, beta_start, beta_end):
        self.num_train_timesteps = num_train_timesteps
        self.alphas_cumprod = _linear_alphas_cumprod(num_train_timesteps, beta_start, beta_end)
        sigmas = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).flip(0)
        self.sigmas = torch.cat([sigmas, torch.zeros(1)])
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps,
                                                      dtype=float)[::-1].copy()).to(torch.float32)
        self.num_inference_steps = None
        self.order = 1
        self._step_index = None

    @property
    def step_index(self):
        return self._step_index

    @property
    def init_noise_sigma(self):
        max_sigma = self.sigmas.max()
        if self.config["timestep_spacing"] in ("linspace", "trailing"):
            return max_sigma
        return (max_sigma ** 2 + 1) ** 0.5

    def set_timesteps(self, num_inference_steps, device=None):
        """The n-step schedule: fp32 (possibly fractional) timesteps, n + 1 fp32 sigmas ending in 0."""
        cfg, T, n = self.config, self.num_train_timesteps, num_inference_steps
        self.num_inference_steps = n
        if cfg["timestep_spacing"] == "linspace":
            timesteps = np.linspace(0, T - 1, n, dtype=np.float32)[::-1].copy()
        elif cfg["timestep_spacing"] == "leading":
            timesteps = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.float32)
            timesteps += cfg["steps_offset"]
        else:                                                                            # trailing
            timesteps = np.arange(T, 0, -T / n).round().copy().astype(np.float32)
            timesteps -= 1
        sigmas = np.interp(timesteps, np.arange(0, T), _train_sigmas(self.alphas_cumprod))
        self.sigmas = torch.from_numpy(np.concatenate([sigmas, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(timesteps.astype(np.float32)).to(device=device)
        self._step_index = None
        return self.timesteps

    def index_for_timestep(self, timestep, schedule_timesteps=None) -> int:
        """Index of `timestep` in the schedule (the second match if there are several).  A timestep outside the schedule
        raises ValueError; diffusers raises IndexError there."""
        if schedule_timesteps is None:
            schedule_timesteps = self.timesteps
        idx = (schedule_timesteps == torch.as_tensor(timestep).to(schedule_timesteps.device)).nonzero()
        if len(idx) == 0:
            raise ValueError(f"{type(self).__name__}: timestep {float(timestep)} is not in the schedule")
        return idx[1 if len(idx) > 1 else 0].item()

    def _init_step_index(self, timestep):
        self._step_index = self.index_for_timestep(timestep)

    def get_timesteps(self, num_inference_steps, strength):
        return _truncated(self, num_inference_steps, strength)

    def scale_model_input(self, sample, timestep):
        """sample / (sigma^2 + 1)^0.5 at the current step."""
        if self._step_index is None:
            self._init_step_index(timestep)
        sigma = self.sigmas[self._step_index]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def _update(self, i: int) -> SolverStep:
        raise NotImplementedError

    def next_step(self, timestep) -> SolverStep:
        """The scalars of the step at `timestep`; advances the step counter as `step()` does."""
        if isinstance(timestep, int) or (isinstance(timestep, torch.Tensor) and not timestep.is_floating_point()):
            raise ValueError(f"{type(self).__name__}.step takes a timestep of `scheduler.timesteps`, not an integer index")
        if self._step_index is None:
            self._init_step_index(timestep)
        s = self._update(self._step_index)
        self._step_index += 1
        return s

    def _euler(self, s: SolverStep, model_output, sample, noise):
        sample = sample.to(torch.float32)
        x0 = sample - s.sigma * model_output
        d = (sample - x0) / s.sigma
        x = sample + d * s.dt
        if s.sigma_up != 0.0:
            x = x + noise * s.sigma_up
        return x.to(model_output.dtype)

    def add_noise(self, original_samples, noise, timesteps):
        """x + sigma noise at the sigma of each timestep's index."""
        sigmas = self.sigmas.to(device=original_samples.device, dtype=original_samples.dtype)
        schedule = self.timesteps.to(original_samples.device)
        ts = torch.as_tensor(timesteps).to(original_samples.device).reshape(-1)
        sigma = sigmas[[self.index_for_timestep(t, schedule) for t in ts]].flatten()
        while sigma.ndim < original_samples.ndim:
            sigma = sigma.unsqueeze(-1)
        return original_samples + noise * sigma


def _randn_like_output(model_output, generator):
    rand_device = generator.device if generator is not None else model_output.device
    return torch.randn(model_output.shape, generator=generator, device=rand_device,
                       dtype=model_output.dtype).to(model_output.device)


class EulerDiscreteScheduler(_EulerBase):
    """diffusers 0.28.0 EulerDiscreteScheduler with epsilon prediction, linear sigma interpolation and s_churn = 0.  Every
    step draws one normal sample of the model output's shape from the generator, as diffusers does (unused at gamma 0)."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear", trained_betas=None,
                 prediction_type="epsilon", interpolation_type="linear", use_karras_sigmas=False, sigma_min=None,
                 sigma_max=None, timestep_spacing="linspace", timestep_type="discrete", steps_offset=0,
                 rescale_betas_zero_snr=False, **unused):
        name = type(self).__name__
        _check_common(name, beta_schedule, trained_betas, prediction_type, timestep_spacing, rescale_betas_zero_snr)
        _only(name, "interpolation_type", interpolation_type, ("linear",))
        _only(name, "use_karras_sigmas", use_karras_sigmas, (False,))
        _only(name, "sigma_min", sigma_min, (None,))
        _only(name, "sigma_max", sigma_max, (None,))
        _only(name, "timestep_type", timestep_type, ("discrete",))
        self._register(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                       beta_schedule=beta_schedule, trained_betas=trained_betas, prediction_type=prediction_type,
                       interpolation_type=interpolation_type, use_karras_sigmas=use_karras_sigmas, sigma_min=sigma_min,
                       sigma_max=sigma_max, timestep_spacing=timestep_spacing, timestep_type=timestep_type,
                       steps_offset=steps_offset, rescale_betas_zero_snr=rescale_betas_zero_snr)
        self._setup(num_train_timesteps, beta_start, beta_end)

    def _update(self, i: int) -> SolverStep:
        sigma = self.sigmas[i]
        sigma_hat = sigma * (0.0 + 1)                                     # gamma = 0 (s_churn = 0)
        dt = self.sigmas[i + 1] - sigma_hat
        return SolverStep(SAMPLER_EULER, i, sigma=float(sigma_hat), dt=float(dt))

    def step(self, model_output, timestep, sample, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"), s_noise=1.0, generator=None,
             return_dict=True):
        _only(type(self).__name__, "s_churn", s_churn, (0.0,))
        s = self.next_step(timestep)
        _randn_like_output(model_output, generator)                       # drawn and unused at gamma 0, as in diffusers
        x = self._euler(s, model_output, sample, None)
        return SchedulerOutput(x) if return_dict else (x,)


class EulerAncestralDiscreteScheduler(_EulerBase):
    """diffusers 0.28.0 EulerAncestralDiscreteScheduler with epsilon prediction: an Euler step to sigma_down, then
    sigma_up times one normal sample of the model output's shape drawn from the generator."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear", trained_betas=None,
                 prediction_type="epsilon", timestep_spacing="linspace", steps_offset=0, rescale_betas_zero_snr=False,
                 **unused):
        name = type(self).__name__
        _check_common(name, beta_schedule, trained_betas, prediction_type, timestep_spacing, rescale_betas_zero_snr)
        self._register(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                       beta_schedule=beta_schedule, trained_betas=trained_betas, prediction_type=prediction_type,
                       timestep_spacing=timestep_spacing, steps_offset=steps_offset,
                       rescale_betas_zero_snr=rescale_betas_zero_snr)
        self._setup(num_train_timesteps, beta_start, beta_end)

    def _update(self, i: int) -> SolverStep:
        sigma_from, sigma_to = self.sigmas[i], self.sigmas[i + 1]
        sigma_up = (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5
        sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
        dt = sigma_down - sigma_from
        return SolverStep(SAMPLER_EULER, i, sigma=float(sigma_from), dt=float(dt), sigma_up=float(sigma_up))

    def step(self, model_output, timestep, sample, generator=None, return_dict=True):
        s = self.next_step(timestep)
        noise = _randn_like_output(model_output, generator)
        x = self._euler(s, model_output, sample, noise)
        return SchedulerOutput(x) if return_dict else (x,)


SOLVER_SCHEDULERS = (DPMSolverMultistepScheduler, EulerDiscreteScheduler, EulerAncestralDiscreteScheduler)
SCHEDULERS = {c.__name__: c for c in (DDIMScheduler, DPMSolverMultistepScheduler, EulerDiscreteScheduler,
                                      EulerAncestralDiscreteScheduler)}


def as_engine_scheduler(scheduler):
    """The engine's scheduler for `scheduler`: ours as they are; an instance of diffusers' class of the same name (or of
    any class with that name and a `config`) rebuilt from its config.  Anything else is returned unchanged."""
    if scheduler is None or isinstance(scheduler, tuple(SCHEDULERS.values())):
        return scheduler
    cls = SCHEDULERS.get(type(scheduler).__name__)
    if cls is not None and hasattr(scheduler, "config"):
        return cls.from_config(scheduler.config)
    return scheduler
