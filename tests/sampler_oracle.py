"""Test-side oracle of the sampler options the released configuration leaves at their defaults: stochastic DDIM (eta > 0),
sampling without classifier-free guidance and the `i2v_similarity_init` start (reference animatediff/pipelines/
pipeline.py:580-590, 667-733, 929-1047).  diffusers 0.28.0 `DDIMScheduler.step(..., eta, variance_noise)` is not installed
here: restated beside SURVEY.md Appendix B.10, "parity unpinned" like the rest of B.10.  Built on oracle/scheduler_oracle.py
and oracle/abi_oracle.py without changing them.

* `DDIMEtaOracle` -- `DDIMOracle` with `step(eps, t, x, eta, variance_noise)` and the reference's `get_timesteps`.
* `similarity_init` -- prepare_latents' similarity branch (pipeline.py:707-724).
* `sampler` -- the reference `__call__` loop (FreeInit off) around the fp32 oracle UNet.
* `ddim_step` -- float64 restatement of `a3d_ddim_step` with a per-element bound in the style of abi_oracle.py: the
  update is nine fp32 operations on the absolute values of its terms (the eight of ddim_cfg_step, where the kernel's
  sqrt(1 - a_prev) is replaced by the given dir_coef, plus the variance-noise FMA): 9 u32 R_abs, times SLACK.  Frame 0
  is an exact copy."""
from __future__ import annotations

import math

import torch

from oracle import abi_oracle as A
from oracle import unet_oracle as U
from oracle.scheduler_oracle import DDIMOracle, cfg_pipeline


class DDIMEtaOracle(DDIMOracle):
    def step(self, eps, t, x, eta=0.0, variance_noise=None):
        """DDIMScheduler.step with eta (fp32, diffusers' order): returns (prev_sample, pred_original_sample)."""
        prev_t = t - self.T // self.n
        a_t = self.alphas_cumprod[t]
        a_p = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        x0 = (x - (1 - a_t).sqrt() * eps) / a_t.sqrt()
        variance = ((1 - a_p) / (1 - a_t)) * (1 - a_t / a_p)
        std = eta * variance.sqrt()
        prev = a_p.sqrt() * x0 + (1 - a_p - std ** 2).sqrt() * eps
        if eta > 0:
            prev = prev + std * variance_noise
        return prev, x0

    def get_timesteps(self, n, strength):
        """pipeline.py:667-674 on the n-step schedule (which keeps its stride)."""
        self.set_timesteps(n)
        init = min(int(n * strength), n)
        return self.timesteps[max(n - init, 0):]


def similarity_init(first, num_frames, latent_timestep, origin_prob, sched: DDIMOracle, generator):
    """pipeline.py:707-724 with batch = the views: mask, then noise, then the blend."""
    nv, c, _, h, w = first.shape
    binary_mask = torch.rand((nv, 1, num_frames, h, w), generator=generator, dtype=torch.float32)
    binary_mask = binary_mask < origin_prob
    latent_cond_image = first.repeat_interleave(num_frames, dim=2)
    noise = torch.randn((nv, c, num_frames, h, w), generator=generator, dtype=torch.float32)
    blurred = sched.add_noise(latent_cond_image, noise, latent_timestep)
    return binary_mask.float() * latent_cond_image + (1 - binary_mask.float()) * blurred


def sampler(sd, cfg, first, prompt_embeds, negative_prompt_embeds, image_embeds, num_frames, num_inference_steps,
            guidance_scale, eta, generator, similarity=None):
    """The reference `__call__` (pipeline.py:929-1047, FreeInit off, i2v_cond_time_zero off) on the CPU: fp32 oracle UNet,
    CFG only when guidance_scale > 1, DDIM with eta, frame-0 re-injection.  Every random draw goes through `generator`:
    the initial noise (or the similarity mask and noise), then one variance-noise draw per step when eta > 0."""
    nv, c, _, h, w = first.shape
    do_cfg = guidance_scale > 1
    sched = DDIMEtaOracle()
    if similarity is None:
        timesteps = sched.set_timesteps(num_inference_steps)
        rest = torch.randn((nv, c, num_frames - 1, h, w), generator=generator, dtype=torch.float32)
    else:
        timesteps = sched.get_timesteps(num_inference_steps, similarity["strength"])
        rest = similarity_init(first, num_frames - 1, timesteps[:1].repeat(nv), similarity["origin_prob"], sched, generator)
    pe = torch.cat([negative_prompt_embeds, prompt_embeds]) if do_cfg else prompt_embeds
    ie = torch.cat([torch.zeros_like(image_embeds), image_embeds]) if do_cfg else image_embeds
    cam = U.get_camera(nv)
    cam = torch.cat([cam, cam]) if do_cfg else cam
    lat = torch.cat([first, rest], dim=2)
    for t in timesteps.tolist():
        x = torch.cat([lat, lat]) if do_cfg else lat
        with torch.no_grad():
            eps = U.unet_forward(sd, cfg, x, t, pe, cam, ie, nv)
        if do_cfg:
            eps = cfg_pipeline(eps, guidance_scale)
        noise = torch.randn(eps.shape, generator=generator, dtype=torch.float32) if eta > 0 else None
        lat, _ = sched.step(eps, t, lat, eta, noise)
        lat = torch.cat([first, lat[:, :, 1:]], dim=2)
    return lat


def ddim_step(latents, noise_pred, first_frame, variance_noise, bn, c, f, hw, cfg_mode, guidance, alpha_t, alpha_prev, dir_coef,
              std_dev) -> A.Ref:
    """`latents` is the state before the step."""
    n = bn * c * f * hw
    x = A.flat(latents, n).to(A.F64).view(bn, c, f, hw)
    if cfg_mode == 0:
        eps = A.flat(noise_pred, n).to(A.F64).view(bn, c, f, hw)
        eps_abs = eps.abs()
    else:
        e2 = A.flat(noise_pred, 2 * n).to(A.F64).view(2 * bn, c, f, hw)
        ea, eb = e2[:bn], e2[bn:]
        eps = ea + guidance * (eb - ea) if cfg_mode == 1 else ea + guidance * (ea - eb)
        eps_abs = ea.abs() + abs(guidance) * (eb.abs() + ea.abs())
    sa, sp = math.sqrt(alpha_t), math.sqrt(alpha_prev)
    x0 = (x - math.sqrt(1 - alpha_t) * eps) / sa
    v = sp * x0 + dir_coef * eps
    r_abs = sp / sa * (x.abs() + math.sqrt(1 - alpha_t) * eps_abs) + abs(dir_coef) * eps_abs
    if variance_noise is not None:
        z = A.flat(variance_noise, n).to(A.F64).view(bn, c, f, hw)
        v = v + std_dev * z
        r_abs = r_abs + abs(std_dev) * z.abs()
    e = 9 * A.U32 * r_abs
    if first_frame is not None:
        v[:, :, 0] = A.flat(first_frame, bn * c * hw).to(A.F64).view(bn, c, hw)
        e[:, :, 0] = 0
    return A.Ref(v.reshape(-1), (A.SLACK * A._store(v, e, True)).reshape(-1),
                 lambda i: "[bn, c, f, hw] index %s" % (tuple(int(t) for t in torch.unravel_index(torch.tensor(i), (bn, c, f, hw))),))
