"""Test-side oracle of the DPM-Solver++, Euler and Euler-ancestral schedulers in the sampling pipeline (reference
animatediff/pipelines/pipeline.py:315-322, 580-590, 667-733, 939-1047).  diffusers 0.28.0 is not installed here: its
`DPMSolverMultistepScheduler` (dpmsolver++, orders 1-2), `EulerDiscreteScheduler` (s_churn 0) and
`EulerAncestralDiscreteScheduler` are restated from its published source, "parity unpinned" (DESIGN section 4).  Built on
oracle/ and tests/sampler_oracle.py without changing them.

* `DPMSolverOracle`, `EulerOracle`, `EulerAncestralOracle` -- the schedulers as diffusers writes them: schedules, per-step
  tensor arithmetic with the model-output history, index lookup, add_noise, init_noise_sigma, scale_model_input.
* `sampler` -- the reference `__call__` loop around the fp32 oracle UNet for any of them, with FreeInit and the similarity
  init; every random draw goes through the caller's generator.
* `sampler_step` -- float64 restatement of `a3d_sampler_step` with a per-element bound in the style of
  sampler_oracle.ddim_step: the update is at most 13 fp32 operations (3 of the CFG combine, 3 of m0, 7 of the order-2
  update; Euler: 3 + 8), so the bound is 13 u32 times the value of the same expression over the absolute values of its
  terms, times SLACK.  Frame 0 is an exact copy."""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import abi_oracle as A
from oracle import unet_oracle as U
from oracle.scheduler_oracle import butterworth_lpf, cfg_pipeline, freeinit_mix

DPMPP, EULER = 0, 1


def _alphas_cumprod(T=1000, beta_start=0.0001, beta_end=0.02):
    betas = torch.linspace(beta_start, beta_end, T, dtype=torch.float32)
    return torch.cumprod(1.0 - betas, dim=0)


# ------------------------------------------------------------------------------------------------ DPM-Solver++
class DPMSolverOracle:
    def __init__(self, beta_start=0.0001, beta_end=0.02, solver_order=2, solver_type="midpoint", lower_order_final=True,
                 euler_at_final=False, use_karras_sigmas=False, final_sigmas_type="zero", timestep_spacing="linspace",
                 steps_offset=0, num_train_timesteps=1000):
        self.T = num_train_timesteps
        self.alphas_cumprod = _alphas_cumprod(self.T, beta_start, beta_end)
        self.solver_order, self.solver_type = solver_order, solver_type
        self.lower_order_final, self.euler_at_final = lower_order_final, euler_at_final
        self.use_karras_sigmas, self.final_sigmas_type = use_karras_sigmas, final_sigmas_type
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        self.init_noise_sigma = 1.0
        self.order = 1

    def set_timesteps(self, n):
        T = self.T
        if self.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif self.timestep_spacing == "leading":
            ratio = T // (n + 1)
            ts = (np.arange(0, n + 1) * ratio).round()[::-1][:-1].copy().astype(np.int64) + self.steps_offset
        else:
            ts = np.arange(T, 0, -T / n).round().copy().astype(np.int64) - 1
        train = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        log_sigmas = np.log(train)
        if self.use_karras_sigmas:
            s = np.flip(train).copy()
            lo, hi = s[-1].item() ** (1 / 7.0), s[0].item() ** (1 / 7.0)
            sig = (hi + np.linspace(0, 1, n) * (lo - hi)) ** 7.0
            ts = np.array([self._sigma_to_t(x, log_sigmas) for x in sig]).round()
        else:
            sig = np.interp(ts, np.arange(0, len(train)), train)
        last = ((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5 if self.final_sigmas_type == "sigma_min" else 0
        self.sigmas = torch.from_numpy(np.concatenate([sig, [last]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts).to(torch.int64)
        self.model_outputs = [None] * self.solver_order
        self.lower_order_nums = 0
        self.step_index = None
        return self.timesteps

    @staticmethod
    def _sigma_to_t(sigma, log_sigmas):
        log_sigma = np.log(np.maximum(sigma, 1e-10))
        dists = log_sigma - log_sigmas[:, np.newaxis]
        low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
        high_idx = low_idx + 1
        low, high = log_sigmas[low_idx], log_sigmas[high_idx]
        w = np.clip((low - log_sigma) / (low - high), 0, 1)
        return ((1 - w) * low_idx + w * high_idx).reshape(np.shape(sigma))

    def get_timesteps(self, n, strength):
        self.set_timesteps(n)
        init = min(int(n * strength), n)
        return self.timesteps[max(n - init, 0):]

    def index_for_timestep(self, t):
        cand = (self.timesteps == t).nonzero()
        if len(cand) == 0:
            return len(self.timesteps) - 1
        return cand[1].item() if len(cand) > 1 else cand[0].item()

    @staticmethod
    def alpha_sigma(sigma):
        alpha = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha, sigma * alpha

    def order_of_next_step(self):
        i, n = self.step_index, len(self.timesteps)
        final = i == n - 1 and (self.euler_at_final or (self.lower_order_final and n < 15) or self.final_sigmas_type == "zero")
        return 1 if self.solver_order == 1 or self.lower_order_nums < 1 or final else 2

    def step(self, eps, t, x, generator=None):
        if self.step_index is None:
            self.step_index = self.index_for_timestep(t)
        order = self.order_of_next_step()
        i = self.step_index
        alpha_s0, sigma_s0 = self.alpha_sigma(self.sigmas[i])
        m0 = (x - sigma_s0 * eps) / alpha_s0                                             # convert_model_output
        self.model_outputs = self.model_outputs[1:] + [m0]
        alpha_t, sigma_t = self.alpha_sigma(self.sigmas[i + 1])
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        if order == 1:
            out = (sigma_t / sigma_s0) * x - (alpha_t * (torch.exp(-h) - 1.0)) * m0
        else:
            m1 = self.model_outputs[-2]
            alpha_s1, sigma_s1 = self.alpha_sigma(self.sigmas[i - 1])
            lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
            r0 = (lambda_s0 - lambda_s1) / h
            D1 = (1.0 / r0) * (m0 - m1)
            out = (sigma_t / sigma_s0) * x - (alpha_t * (torch.exp(-h) - 1.0)) * m0
            if self.solver_type == "midpoint":
                out = out - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1
            else:
                out = out + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self.step_index += 1
        return out

    def scale_model_input(self, x, t):
        return x

    def add_noise(self, x, noise, timesteps):
        sigma = self.sigmas[[self.index_for_timestep(t) for t in timesteps]].flatten()
        while sigma.ndim < x.ndim:
            sigma = sigma[..., None]
        alpha, sig = self.alpha_sigma(sigma)
        return alpha * x + sig * noise


# ------------------------------------------------------------------------------------------------ Euler
class EulerOracle:
    ancestral = False

    def __init__(self, beta_start=0.0001, beta_end=0.02, timestep_spacing="linspace", steps_offset=0, num_train_timesteps=1000):
        self.T = num_train_timesteps
        self.alphas_cumprod = _alphas_cumprod(self.T, beta_start, beta_end)
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        self.order = 1

    def set_timesteps(self, n):
        T = self.T
        if self.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n, dtype=np.float32)[::-1].copy()
        elif self.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.float32) + self.steps_offset
        else:
            ts = np.arange(T, 0, -T / n).round().copy().astype(np.float32) - 1
        train = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        sig = np.interp(ts, np.arange(0, len(train)), train)
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts.astype(np.float32))
        self.step_index = None
        return self.timesteps

    get_timesteps = DPMSolverOracle.get_timesteps

    @property
    def init_noise_sigma(self):
        m = self.sigmas.max()
        return m if self.timestep_spacing in ("linspace", "trailing") else (m ** 2 + 1) ** 0.5

    def index_for_timestep(self, t):
        idx = (self.timesteps == t).nonzero()
        return idx[1 if len(idx) > 1 else 0].item()                 # IndexError outside the schedule, as diffusers

    def scale_model_input(self, x, t):
        if self.step_index is None:
            self.step_index = self.index_for_timestep(t)
        return x / ((self.sigmas[self.step_index] ** 2 + 1) ** 0.5)

    def step(self, eps, t, x, generator=None):
        if self.step_index is None:
            self.step_index = self.index_for_timestep(t)
        sigma, sigma_next = self.sigmas[self.step_index], self.sigmas[self.step_index + 1]
        if not self.ancestral:
            noise = torch.randn(eps.shape, generator=generator, dtype=eps.dtype)    # drawn, unused at gamma 0
            sigma_hat = sigma * (0.0 + 1)
            x0 = x - sigma_hat * eps
            out = x + ((x - x0) / sigma_hat) * (sigma_next - sigma_hat)
        else:
            x0 = x - sigma * eps
            sigma_up = (sigma_next ** 2 * (sigma ** 2 - sigma_next ** 2) / sigma ** 2) ** 0.5
            sigma_down = (sigma_next ** 2 - sigma_up ** 2) ** 0.5
            out = x + ((x - x0) / sigma) * (sigma_down - sigma)
            noise = torch.randn(eps.shape, generator=generator, dtype=eps.dtype)
            out = out + noise * sigma_up
        self.step_index += 1
        return out

    def add_noise(self, x, noise, timesteps):
        sigma = self.sigmas[[self.index_for_timestep(t) for t in timesteps]].flatten()
        while sigma.ndim < x.ndim:
            sigma = sigma[..., None]
        return x + noise * sigma


class EulerAncestralOracle(EulerOracle):
    ancestral = True


# ------------------------------------------------------------------------------------------------ reference loop
def sampler(sd, cfg, first, prompt_embeds, negative_prompt_embeds, image_embeds, num_frames, num_inference_steps,
            guidance_scale, sched, generator, similarity=None, free_init_iters=1, scale_input=True, model=None):
    """The reference `__call__` (pipeline.py:929-1047, i2v_cond_time_zero off) on the CPU with the fp32 oracle UNet and the
    oracle scheduler `sched`: set_timesteps (or get_timesteps + the similarity init), initial noise times init_noise_sigma,
    FreeInit (add_noise at t = 999 of the previous schedule, a z_rand draw, the low-pass mix, set_timesteps), then per step
    scale_model_input on the CFG-doubled input, the UNet at t, CFG, scheduler.step with the generator and the frame-0
    re-injection.  `model(x, t, pe, cam, ie, nv)` replaces the oracle UNet when given; `scale_input=False` drops
    scale_model_input (a negative control)."""
    nv, c, _, h, w = first.shape
    do_cfg = guidance_scale > 1
    if similarity is None:
        timesteps = sched.set_timesteps(num_inference_steps)
        rest = torch.randn((nv, c, num_frames - 1, h, w), generator=generator, dtype=torch.float32)
        rest = rest * sched.init_noise_sigma
    else:
        timesteps = sched.get_timesteps(num_inference_steps, similarity["strength"])
        mask = torch.rand((nv, 1, num_frames - 1, h, w), generator=generator, dtype=torch.float32) < similarity["origin_prob"]
        cond = first.repeat_interleave(num_frames - 1, dim=2)
        noise = torch.randn((nv, c, num_frames - 1, h, w), generator=generator, dtype=torch.float32)
        blurred = sched.add_noise(cond, noise, timesteps[:1].repeat(nv))
        rest = mask.float() * cond + (1 - mask.float()) * blurred
    pe = torch.cat([negative_prompt_embeds, prompt_embeds]) if do_cfg else prompt_embeds
    ie = torch.cat([torch.zeros_like(image_embeds), image_embeds]) if do_cfg else image_embeds
    cam = U.get_camera(nv)
    cam = torch.cat([cam, cam]) if do_cfg else cam
    lat = torch.cat([first, rest], dim=2)
    initial = None
    for it in range(free_init_iters):
        if free_init_iters > 1:                                          # FreeInitMixin._apply_free_init on frames 1..
            rest = lat[:, :, 1:]
            if it == 0:
                initial = rest.clone()
            else:
                z_t = sched.add_noise(rest, initial, torch.full((nv,), sched.T - 1, dtype=torch.long))
                z_rand = torch.randn(rest.shape, generator=generator, dtype=torch.float32)
                rest = freeinit_mix(z_t, z_rand, butterworth_lpf(rest.shape)).float()
            timesteps = sched.set_timesteps(num_inference_steps)
            lat = torch.cat([first, rest], dim=2)
        for t in timesteps:
            x = torch.cat([lat, lat]) if do_cfg else lat
            if scale_input:
                x = sched.scale_model_input(x, t)
            elif sched.step_index is None:
                sched.step_index = sched.index_for_timestep(t)
            with torch.no_grad():
                eps = model(x, t, pe, cam, ie, nv) if model is not None else U.unet_forward(sd, cfg, x, t, pe, cam, ie, nv)
            if do_cfg:
                eps = cfg_pipeline(eps, guidance_scale)
            lat = sched.step(eps, t, lat, generator)
            lat = torch.cat([first, lat[:, :, 1:]], dim=2)
    return lat


# ------------------------------------------------------------------------------------------------ kernel oracle
def sampler_step(latents, noise_pred, first_frame, noise, history_out, history_in, bn, c, f, hw, cfg_mode, guidance,
                 step) -> tuple:
    """float64 a3d_sampler_step with the scalars of `step` (scheduler.SolverStep).  `latents` is the state before the step,
    `history_in` the m1 buffer.  Returns (Ref of the new latents, Ref of m0 or None)."""
    n = bn * c * f * hw
    shape = (bn, c, f, hw)
    x = A.flat(latents, n).to(A.F64).view(shape)
    if cfg_mode == 0:
        eps = A.flat(noise_pred, n).to(A.F64).view(shape)
        eps_abs = eps.abs()
    else:
        e2 = A.flat(noise_pred, 2 * n).to(A.F64).view(2 * bn, c, f, hw)
        ea, eb = e2[:bn], e2[bn:]
        eps = ea + guidance * (eb - ea) if cfg_mode == 1 else ea + guidance * (ea - eb)
        eps_abs = ea.abs() + abs(guidance) * (eb.abs() + ea.abs())
    m0_ref = None
    if step.kind == DPMPP:
        m0 = (x - step.sigma_s0 * eps) / step.alpha_s0
        m0_abs = (x.abs() + abs(step.sigma_s0) * eps_abs) / abs(step.alpha_s0)
        v = step.c_x * x - step.c_m0 * m0
        r_abs = abs(step.c_x) * x.abs() + abs(step.c_m0) * m0_abs
        if step.order == 2:
            m1 = A.flat(history_in, n).to(A.F64).view(shape)
            v = v + step.c_d1 * (step.inv_r0 * (m0 - m1))
            r_abs = r_abs + abs(step.c_d1 * step.inv_r0) * (m0_abs + m1.abs())
        if history_out is not None:
            e_m0 = 6 * A.U32 * m0_abs
            m0_ref = _ref(m0.clone(), e_m0, first_frame, None, shape)
    else:
        x0 = x - step.sigma * eps
        x0_abs = x.abs() + abs(step.sigma) * eps_abs
        d = (x - x0) / step.sigma
        v = x + d * step.dt
        r_abs = x.abs() + abs(step.dt / step.sigma) * (x.abs() + x0_abs)
        if step.sigma_up != 0.0:
            z = A.flat(noise, n).to(A.F64).view(shape)
            v = v + z * step.sigma_up
            r_abs = r_abs + abs(step.sigma_up) * z.abs()
    e = 13 * A.U32 * r_abs
    return _ref(v, e, first_frame, first_frame, shape), m0_ref


def _ref(v, e, first_frame, copy_from, shape):
    """Ref over [bn, c, f, hw]; with a first frame, frame 0 is `copy_from` exactly (None: the kernel leaves it alone, which
    the caller checks separately, so its bound is infinite)."""
    bn, c, f, hw = shape
    if first_frame is not None:
        if copy_from is not None:
            v[:, :, 0] = A.flat(copy_from, bn * c * hw).to(A.F64).view(bn, c, hw)
            e[:, :, 0] = 0
        else:
            e[:, :, 0] = math.inf
    bound = A.SLACK * A._store(v, e, True)
    return A.Ref(v.reshape(-1), bound.reshape(-1),
                 lambda i: "[bn, c, f, hw] index %s" % (tuple(int(t) for t in torch.unravel_index(torch.tensor(i), shape)),))
