"""DDIM scheduler constants of the released MV-VDM (configs/inference/inference.yaml:36-42 of the reference: linear betas
0.00085..0.012, 1000 train steps, leading spacing, steps_offset 1).  The update itself runs in the a3d_ddim_step /
a3d_ddim_cfg_step kernel fused with classifier-free guidance and the frame-0 re-injection of pipeline.py:1023-1031; this
class owns the per-step coefficients that kernel is given."""
from __future__ import annotations

import numpy as np
import torch


class DDIMScheduler:
    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="linear",
                 steps_offset=1, clip_sample=False, set_alpha_to_one=True, **unused):
        if beta_schedule != "linear" or clip_sample:
            raise NotImplementedError("only the released configuration (linear betas, no clipping) is supported")
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
