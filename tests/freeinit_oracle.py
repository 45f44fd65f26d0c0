"""Test-side oracle of FreeInit's filters and coarse-to-fine sampling and of per-view generator lists in the reference's
sampling loop (reference animatediff/pipelines/pipeline.py:699-733, 975, 987-1047; diffusers 0.28.0 `FreeInitMixin`,
`randn_tensor`, `DDIMScheduler.step` and `EulerAncestralDiscreteScheduler.step` with a list of generators).  diffusers is
not installed here: restated from its published source, "parity unpinned" (DESIGN section 4).  Built on oracle/ and
tests/sampler_oracle.py, tests/solver_oracle.py without changing them.

* `free_init_freq_filter` -- FreeInitMixin._get_free_init_freq_filter as it is written (the per-entry Python loop).
* `free_init_num_steps` -- the step count _apply_free_init sets on one iteration (coarse-to-fine sampling).
* `randn_tensor` -- diffusers' randn_tensor, generator lists included.
* `DDIMLoop` -- `DDIMEtaOracle` behind the solver oracles' `step(eps, t, x, generator)`: eta > 0 draws the variance
  noise of the model output's shape with `randn_tensor` after the UNet call, as DDIMScheduler.step does.
* `EulerAncestralLists` -- `EulerAncestralOracle` whose per-step noise goes through `randn_tensor`, so a list of
  generators draws view by view.
* `sampler` -- the reference `__call__` loop (i2v_cond_time_zero off, no similarity init) with FreeInit as
  `enable_free_init` configures it: every filter method, order, stop frequencies and coarse-to-fine sampling; every random
  draw goes through `randn_tensor` with the caller's generator or list of generators.  Returns the latents and the number
  of UNet calls."""
from __future__ import annotations

import math

import torch

import sampler_oracle as SO
import solver_oracle as SV
from oracle import unet_oracle as U
from oracle.scheduler_oracle import cfg_pipeline, freeinit_mix

FREE_INIT_DEFAULTS = dict(num_iters=3, use_fast_sampling=False, method="butterworth", order=4, spatial_stop_frequency=0.25,
                          temporal_stop_frequency=0.25)


def free_init_freq_filter(shape, filter_type="butterworth", order=4, spatial_stop_frequency=0.25,
                          temporal_stop_frequency=0.25):
    """FreeInitMixin._get_free_init_freq_filter (diffusers 0.28.0) as it is written: a float32 tensor of `shape` filled
    entry by entry over (t, h, w) with a Python-float value; ideal compares d² with 2 d_s."""
    time, height, width = shape[-3], shape[-2], shape[-1]
    mask = torch.zeros(shape)
    if spatial_stop_frequency == 0 or temporal_stop_frequency == 0:
        return mask
    if filter_type == "butterworth":
        def retrieve_mask(x):
            return 1 / (1 + (x / spatial_stop_frequency ** 2) ** order)
    elif filter_type == "gaussian":
        def retrieve_mask(x):
            return math.exp(-1 / (2 * spatial_stop_frequency ** 2) * x)
    elif filter_type == "ideal":
        def retrieve_mask(x):
            return 1 if x <= spatial_stop_frequency * 2 else False
    else:
        raise NotImplementedError("`filter_type` must be one of gaussian, butterworth or ideal")
    for t in range(time):
        for h in range(height):
            for w in range(width):
                d_square = (((spatial_stop_frequency / temporal_stop_frequency) * (2 * t / time - 1)) ** 2
                            + (2 * h / height - 1) ** 2 + (2 * w / width - 1) ** 2)
                mask[..., t, h, w] = retrieve_mask(d_square)
    return mask


def free_init_num_steps(num_inference_steps, num_iters, free_init_iteration, use_fast_sampling):
    """The step count FreeInitMixin._apply_free_init sets the schedule to on one iteration (coarse-to-fine sampling)."""
    if use_fast_sampling:
        return max(1, int(num_inference_steps / num_iters * (free_init_iteration + 1)))
    return num_inference_steps


def randn_tensor(shape, generator=None, device=None, dtype=None):
    """diffusers 0.28.0 `randn_tensor` (utils/torch_utils.py): a list of generators draws item i of dim 0 from
    generator[i]; a CPU generator draws on the CPU and moves the result; a CUDA generator for another device raises."""
    rand_device = device
    batch_size = shape[0]
    device = torch.device(device) if device is not None else torch.device("cpu")
    if generator is not None:
        gen_device_type = generator.device.type if not isinstance(generator, list) else generator[0].device.type
        if gen_device_type != device.type and gen_device_type == "cpu":
            rand_device = "cpu"
        elif gen_device_type != device.type and gen_device_type == "cuda":
            raise ValueError(f"Cannot generate a {device} tensor from a generator of type {gen_device_type}.")
    if isinstance(generator, list) and len(generator) == 1:
        generator = generator[0]
    if isinstance(generator, list):
        shape = (1,) + tuple(shape[1:])
        latents = [torch.randn(shape, generator=generator[i], device=rand_device, dtype=dtype) for i in range(batch_size)]
        return torch.cat(latents, dim=0).to(device)
    return torch.randn(shape, generator=generator, device=rand_device, dtype=dtype).to(device)


class DDIMLoop(SO.DDIMEtaOracle):
    init_noise_sigma = 1.0

    def __init__(self, eta=0.0, **kw):
        super().__init__(**kw)
        self.eta = eta

    def scale_model_input(self, x, t):
        return x

    def step(self, eps, t, x, generator=None):
        noise = randn_tensor(eps.shape, generator, eps.device, eps.dtype) if self.eta > 0 else None
        return super().step(eps, int(t), x, self.eta, noise)[0]


class EulerAncestralLists(SV.EulerAncestralOracle):
    def step(self, eps, t, x, generator=None):
        if self.step_index is None:
            self.step_index = self.index_for_timestep(t)
        sigma, sigma_next = self.sigmas[self.step_index], self.sigmas[self.step_index + 1]
        x0 = x - sigma * eps
        sigma_up = (sigma_next ** 2 * (sigma ** 2 - sigma_next ** 2) / sigma ** 2) ** 0.5
        sigma_down = (sigma_next ** 2 - sigma_up ** 2) ** 0.5
        out = x + ((x - x0) / sigma) * (sigma_down - sigma)
        out = out + randn_tensor(eps.shape, generator, eps.device, eps.dtype) * sigma_up
        self.step_index += 1
        return out


def sampler(first, prompt_embeds, negative_prompt_embeds, image_embeds, num_frames, num_inference_steps, guidance_scale,
            sched, generator, model, free_init=None):
    """The reference loop on the CPU in fp32 around `model(x, t, pe, cam, ie, nv)`.  `free_init` is None (FreeInit off) or
    the keyword arguments of enable_free_init.  Per FreeInit iteration (FreeInitMixin._apply_free_init on frames 1..): the
    first keeps its noise; the others noise the previous result to t = 999 with the scheduler's add_noise on the previous
    schedule, draw z_rand and mix the two through the filter built at (1, C, F-1, h, w); then every iteration sets the
    schedule to its step count."""
    nv, c, _, h, w = first.shape
    do_cfg = guidance_scale > 1
    timesteps = sched.set_timesteps(num_inference_steps)
    rest = randn_tensor((nv, c, num_frames - 1, h, w), generator, first.device, torch.float32) * sched.init_noise_sigma
    pe = torch.cat([negative_prompt_embeds, prompt_embeds]) if do_cfg else prompt_embeds
    ie = torch.cat([torch.zeros_like(image_embeds), image_embeds]) if do_cfg else image_embeds
    cam = U.get_camera(nv)
    cam = torch.cat([cam, cam]) if do_cfg else cam
    lat = torch.cat([first, rest], dim=2)
    fi = dict(FREE_INIT_DEFAULTS, **free_init) if free_init is not None else None
    iters = fi["num_iters"] if fi is not None else 1
    calls, initial = 0, None
    for it in range(iters):
        if fi is not None:
            rest = lat[:, :, 1:]
            if it == 0:
                initial = rest.clone()
            else:
                z_t = sched.add_noise(rest, initial, torch.full((nv,), sched.T - 1, dtype=torch.long)).float()
                z_rand = randn_tensor(rest.shape, generator, rest.device, torch.float32)
                lpf = free_init_freq_filter((1, *rest.shape[1:]), fi["method"], fi["order"], fi["spatial_stop_frequency"],
                                            fi["temporal_stop_frequency"])
                rest = freeinit_mix(z_t, z_rand, lpf).float()
            timesteps = sched.set_timesteps(free_init_num_steps(num_inference_steps, iters, it, fi["use_fast_sampling"]))
            lat = torch.cat([first, rest], dim=2)
        for t in timesteps:
            x = torch.cat([lat, lat]) if do_cfg else lat
            x = sched.scale_model_input(x, t)
            with torch.no_grad():
                eps = model(x, t, pe, cam, ie, nv)
            calls += 1
            if do_cfg:
                eps = cfg_pipeline(eps, guidance_scale)
            lat = sched.step(eps, t, lat, generator)
            lat = torch.cat([first, lat[:, :, 1:]], dim=2)
    return lat, calls
