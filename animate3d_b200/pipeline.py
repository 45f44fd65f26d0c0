"""Host-side mirror of the reference's sampling pipeline `AnimateDiffMVI2VPipeline` (animatediff/pipelines/pipeline.py:274-1062)
for the denoising hot loop: FreeInit outer loop (987-999) x DDIM loop (1006-1047) with classifier-free guidance (1008,
1023-1025), scheduler step (1028) and first-frame re-injection (1031).

The UNet evaluation, CFG combine, DDIM update and frame-0 re-injection all run as CUDA kernels of liba3d.so.  The VAE and
the CLIP text / image encoders (SURVEY section 8(f), "next" rows) are injected as opaque callables or bypassed with
pre-computed embeddings / latents, exactly as the reference's own `prompt_embeds`, `ip_adapter_image_embeds` and
`latents` arguments allow (pipeline.py:770-778)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, List, Optional

import torch

from . import ops
from .scheduler import (MULTISTEP_SCHEDULERS, RING, SOLVER_SCHEDULERS, DDIMScheduler, DPMSolverMultistepScheduler,
                        PNDMScheduler, as_engine_scheduler)
from .unet import MVUNetMotionModel


@dataclass
class AnimateDiffMVI2VPipelineOutput:
    frames: object


def get_camera(num_views: int, elevation: float = 15.0, azimuth_start: float = 0.0, azimuth_span: float = 360.0) -> torch.Tensor:
    """Camera conditioning of pipeline.py:127-190: c2w of `num_views` cameras on a circle at `elevation`, translation
    normalised to the unit sphere, flattened to [num_views, 16]."""
    out = []
    gap = azimuth_span / num_views
    for i in range(num_views):
        e = math.radians(elevation)
        a = math.radians(azimuth_start + i * gap)
        pos = torch.tensor([math.cos(e) * math.cos(a), math.cos(e) * math.sin(a), math.sin(e)], dtype=torch.float32)
        look = -pos / pos.norm()
        right = torch.linalg.cross(look, torch.tensor([0.0, 0.0, 1.0]))
        right = right / right.norm()
        up = torch.linalg.cross(right, look)
        up = up / up.norm()
        c2w = torch.eye(4)
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2] = right, up, -look
        c2w[:3, 3] = pos / (pos.norm() + 1e-8)
        out.append(c2w.flatten())
    return torch.stack(out, 0)


def tensor2vid(video: torch.Tensor, processor=None, output_type: str = "np"):
    """pipeline.py:237-255: [B, C, F, H, W] in [-1, 1] -> per-batch frame lists.  `processor` (diffusers VaeImageProcessor) is
    optional: its postprocess for these three output types is (x / 2 + 0.5).clamp(0, 1) -> NHWC (-> uint8 PIL)."""
    import numpy as np
    outputs = []
    for b in range(video.shape[0]):
        frames = video[b].permute(1, 0, 2, 3)                                 # [F, C, H, W]
        if processor is not None:
            outputs.append(processor.postprocess(frames, output_type))
            continue
        img = (frames / 2 + 0.5).clamp(0, 1)
        if output_type == "pt":
            outputs.append(img)
        else:
            arr = img.detach().cpu().permute(0, 2, 3, 1).float().numpy()
            if output_type == "np":
                outputs.append(arr)
            elif output_type == "pil":
                from PIL import Image
                outputs.append([Image.fromarray((a * 255).round().astype("uint8")) for a in arr])
            else:
                raise ValueError(f"{output_type} does not exist. Please choose one of ['np', 'pt', 'pil']")
    if output_type == "np":
        outputs = np.stack(outputs)
    elif output_type == "pt":
        outputs = torch.stack(outputs)
    return outputs


def _butterworth_lpf(shape, order=4, d_s=0.25, d_t=0.25, device="cpu"):
    T, H, W = shape[-3], shape[-2], shape[-1]
    t = torch.arange(T, device=device)[:, None, None].float()
    h = torch.arange(H, device=device)[None, :, None].float()
    w = torch.arange(W, device=device)[None, None, :].float()
    d2 = ((d_s / d_t) * (2 * t / T - 1)) ** 2 + (2 * h / H - 1) ** 2 + (2 * w / W - 1) ** 2
    return 1.0 / (1.0 + (d2 / d_s ** 2) ** order)


FREE_INIT_METHODS = ("butterworth", "gaussian", "ideal")


def free_init_filter(shape, method="butterworth", order=4, d_s=0.25, d_t=0.25, device="cpu") -> torch.Tensor:
    """FreeInit's low-pass filter over the last three dimensions (T, H, W) of `shape`, as a float32 [T, H, W] tensor
    (diffusers 0.28.0 FreeInitMixin._get_free_init_freq_filter, which loops over the entries).  With
    d² = ((d_s/d_t)(2t/T − 1))² + (2h/H − 1)² + (2w/W − 1)²: butterworth 1 / (1 + (d²/d_s²)^order), gaussian
    exp(−d² / (2 d_s²)), ideal 1 where d² <= 2 d_s (diffusers compares d² with 2 d_s, not d_s²) and 0 elsewhere; all
    zeros when d_s or d_t is 0.  diffusers evaluates every entry in Python floats and stores it in float32: the gaussian
    and ideal filters are evaluated the same way, in float64 rounded once, while the butterworth filter keeps its float32
    arithmetic (`_butterworth_lpf`), a few ulps from diffusers'."""
    if method not in FREE_INIT_METHODS:
        raise NotImplementedError("`filter_type` must be one of gaussian, butterworth or ideal")
    T, H, W = shape[-3], shape[-2], shape[-1]
    if d_s == 0 or d_t == 0:
        return torch.zeros((T, H, W), device=device)
    if method == "butterworth":
        return _butterworth_lpf(shape, order, d_s, d_t, device)
    t = torch.arange(T, device=device, dtype=torch.float64)[:, None, None]
    h = torch.arange(H, device=device, dtype=torch.float64)[None, :, None]
    w = torch.arange(W, device=device, dtype=torch.float64)[None, None, :]
    d2 = ((d_s / d_t) * (2 * t / T - 1)) ** 2 + (2 * h / H - 1) ** 2 + (2 * w / W - 1) ** 2
    mask = torch.exp(-1 / (2 * d_s ** 2) * d2) if method == "gaussian" else (d2 <= d_s * 2).double()
    return mask.float()


def randn_tensor(shape, generator, device) -> torch.Tensor:
    """diffusers' randn_tensor: fp32 normal noise of `shape` on `device`.  `generator` is None, one torch.Generator, or a
    list of them, one per item along dim 0 (a list of one is that one generator).  Every draw runs on its generator's
    device, so a CPU generator gives the same stream whatever `device` is, and the result moves to `device`; a CUDA
    generator cannot fill a tensor on another device type (ValueError, as diffusers raises)."""
    device = torch.device(device)
    gens = generator if isinstance(generator, list) else [generator]
    for g in gens:
        if g is not None and g.device.type == "cuda" and device.type != "cuda":
            raise ValueError(f"cannot draw a {device} tensor from a {g.device} generator")
    if isinstance(generator, list) and len(generator) == 1:
        generator = generator[0]
    if isinstance(generator, list):
        item = (1,) + tuple(shape[1:])
        return torch.cat([torch.randn(item, generator=generator[i], device=generator[i].device,
                                      dtype=torch.float32).to(device) for i in range(shape[0])], 0)
    rand_device = generator.device if generator is not None else device
    return torch.randn(shape, generator=generator, device=rand_device, dtype=torch.float32).to(device)


def similarity_init_latents(first_frame_latents: torch.Tensor, num_frames: int, t_first, origin_prob: float,
                            scheduler, generator: Optional[torch.Generator]) -> torch.Tensor:
    """`i2v_similarity_init` latents of frames 1.. (reference prepare_latents, pipeline.py:707-724): each pixel of each
    frame is the first-frame latent with probability `origin_prob`, else that latent noised to the first timestep.  Draws
    the mask (uniform, [Nv, 1, num_frames, h, w]) and then the noise ([Nv, C, num_frames, h, w]) with `generator`, on its
    device.  `t_first` is a schedule entry (an int, or a 0-dim tensor of the scheduler's timesteps).  No init_noise_sigma
    scaling (pipeline.py:727-729).  A list of generators raises ValueError: the reference draws the mask with torch.rand,
    which takes one generator, and fails there with TypeError."""
    if isinstance(generator, list):
        raise ValueError("i2v_similarity_init draws its mask with one generator (torch.rand): pass a single "
                         "torch.Generator, not a list")
    nv, c, _, h, w = first_frame_latents.shape
    dev = first_frame_latents.device
    rand_device = generator.device if generator is not None else dev
    mask = torch.rand((nv, 1, num_frames, h, w), generator=generator, device=rand_device, dtype=torch.float32).to(dev)
    mask = (mask < origin_prob).float()
    noise = randn_tensor((nv, c, num_frames, h, w), generator, dev)
    cond = first_frame_latents.repeat_interleave(num_frames, dim=2)
    noised = scheduler.add_noise(cond, noise, torch.as_tensor(t_first).reshape(1).repeat(nv))
    return mask * cond + (1 - mask) * noised


class AnimateDiffMVI2VPipeline:
    """`AnimationPipeline` of north_star == this class (alias below).  Constructor keeps the reference's argument names
    (pipeline.py:308-325); everything except `unet` and `scheduler` is optional.  `scheduler` is a DDIMScheduler (the
    default), DPMSolverMultistepScheduler, EulerDiscreteScheduler, EulerAncestralDiscreteScheduler, PNDMScheduler or
    LMSDiscreteScheduler of scheduler.py, or diffusers' class of one of those names (rebuilt from its config); it may be
    replaced at any time, as with the reference:
    `pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config)`."""

    _free_init_method = "butterworth"
    _free_init_use_fast_sampling = False
    _free_init_filter = None                    # (key, filter) of the last filter built: one per (shape, options, device)

    def __init__(self, vae=None, text_encoder=None, tokenizer=None, unet: MVUNetMotionModel = None, motion_adapter=None,
                 scheduler: DDIMScheduler = None, feature_extractor=None, image_encoder=None):
        if unet is None:
            raise ValueError("unet is required")
        self.vae, self.text_encoder, self.tokenizer = vae, text_encoder, tokenizer
        self.unet, self.scheduler = unet, scheduler or DDIMScheduler()
        self.feature_extractor, self.image_encoder = feature_extractor, image_encoder
        self.free_init_enabled = False
        self._free_init_num_iters = 1
        self.device = unet.device

    @property
    def scheduler(self):
        return self._scheduler

    @scheduler.setter
    def scheduler(self, scheduler):
        self._scheduler = as_engine_scheduler(scheduler)

    def to(self, device):
        return self

    def enable_free_init(self, num_iters: int = 3, use_fast_sampling: bool = False, method: str = "butterworth", order: int = 4,
                         spatial_stop_frequency: float = 0.25, temporal_stop_frequency: float = 0.25):
        """diffusers' FreeInitMixin.enable_free_init: `num_iters` sampling passes, each after the first restarting from
        the low frequencies of the previous result (filter `method`: butterworth, gaussian or ideal, see
        `free_init_filter`) and the high frequencies of fresh noise.  With `use_fast_sampling` (coarse-to-fine), pass i
        of n runs max(1, int(num_inference_steps / n * (i + 1))) steps.  An unknown `method` raises NotImplementedError
        here; diffusers raises it at the second pass."""
        if method not in FREE_INIT_METHODS:
            raise NotImplementedError("`filter_type` must be one of gaussian, butterworth or ideal")
        self.free_init_enabled, self._free_init_num_iters = True, num_iters
        self._free_init_use_fast_sampling, self._free_init_method = bool(use_fast_sampling), method
        self._fi = (order, spatial_stop_frequency, temporal_stop_frequency)

    def disable_free_init(self):
        self.free_init_enabled = False

    def enable_vae_slicing(self):
        pass

    # -------------------------------------------------------------------------------------------- conditioning encoders
    # The CLIP text / image towers and the VAE are the reference's own third-party modules (transformers CLIPTextModel /
    # CLIPVisionModelWithProjection, diffusers AutoencoderKL): they are injected, not re-implemented -- transformers is a
    # library here exactly as it is in the reference.  Callables are accepted too (round-1 behaviour).
    def encode_prompt(self, prompt, device=None, num_images_per_prompt: int = 1, do_classifier_free_guidance: bool = True,
                      negative_prompt=None, prompt_embeds=None, negative_prompt_embeds=None, lora_scale=None, clip_skip=None):
        """pipeline.py:345-512 without the LoRA / textual-inversion branches: tokenize (max_length, truncation), text encoder
        (optionally the clip_skip hidden state through final_layer_norm), repeat per view, same for the negative prompt."""
        device = device or self.device
        if prompt_embeds is None:
            if self.text_encoder is None:
                raise ValueError("pass prompt_embeds or construct the pipeline with tokenizer + text_encoder")
            if self.tokenizer is None:                                     # plain callable: (prompt, n) -> embeddings
                return self.text_encoder(prompt, num_images_per_prompt), self.text_encoder(negative_prompt or "", num_images_per_prompt)
            prompt_embeds = self._encode_text([prompt] if isinstance(prompt, str) else list(prompt), device, clip_skip)
        bs, seq, _ = prompt_embeds.shape
        prompt_embeds = prompt_embeds.repeat(1, num_images_per_prompt, 1).view(bs * num_images_per_prompt, seq, -1)
        if do_classifier_free_guidance and negative_prompt_embeds is None:
            neg = [""] * bs if negative_prompt is None else ([negative_prompt] * bs if isinstance(negative_prompt, str) else list(negative_prompt))
            if len(neg) != bs:
                raise ValueError(f"`negative_prompt` has batch size {len(neg)}, but `prompt` has batch size {bs}")
            negative_prompt_embeds = self._encode_text(neg, device, None)
        if do_classifier_free_guidance:
            negative_prompt_embeds = negative_prompt_embeds.to(prompt_embeds.dtype).repeat(1, num_images_per_prompt, 1).view(
                bs * num_images_per_prompt, seq, -1)
        return prompt_embeds, negative_prompt_embeds

    def _encode_text(self, texts, device, clip_skip):
        tok = self.tokenizer(texts, padding="max_length", max_length=self.tokenizer.model_max_length, truncation=True, return_tensors="pt")
        ids = tok.input_ids.to(device)
        if clip_skip is None:
            return self.text_encoder(ids)[0]
        out = self.text_encoder(ids, output_hidden_states=True)
        return self.text_encoder.text_model.final_layer_norm(out[-1][-(clip_skip + 1)])

    def encode_image(self, image, device=None):
        """pipeline.py:514-526: CLIP image embeds of the condition view(s) + their all-zero unconditional twin."""
        device = device or self.device
        if self.image_encoder is None:
            raise ValueError("construct the pipeline with image_encoder (+ feature_extractor) or pass ip_adapter_image_embeds")
        if not hasattr(self.image_encoder, "parameters"):                 # plain callable
            emb = self.image_encoder(image)
            return emb, torch.zeros_like(emb)
        dtype = next(self.image_encoder.parameters()).dtype
        if not isinstance(image, torch.Tensor):
            image = self.feature_extractor(image, return_tensors="pt").pixel_values
        emb = self.image_encoder(image.to(device=device, dtype=dtype)).image_embeds
        return emb, torch.zeros_like(emb)

    def encode_latents(self, image_size, image_list):
        """pipeline.py:528-551: PIL condition images -> VAE latents * scaling_factor (resize to image_size[0], normalise to [-1,1])."""
        import numpy as np
        if self.vae is None:
            raise ValueError("construct the pipeline with a VAE or pass first_frame_latents")
        x = torch.stack([torch.from_numpy(np.array(im)) for im in image_list], 0).float() / 255
        x = x.permute(0, 3, 1, 2)
        x = torch.nn.functional.interpolate(x, size=(image_size[0], image_size[0] * x.shape[3] // x.shape[2]) if x.shape[2] <= x.shape[3]
                                            else (image_size[0] * x.shape[2] // x.shape[3], image_size[0]), mode="bilinear",
                                            antialias=True, align_corners=False)
        x = (x - 0.5) / 0.5
        with torch.no_grad():
            lat = self.vae.encode(x.to(self.device)).latent_dist.sample()
        return lat * self.vae.config.scaling_factor

    def decode_latents(self, latents: torch.Tensor) -> torch.Tensor:
        """pipeline.py:554-567: [B, 4, F, h, w] -> video [B, 3, F, 8h, 8w] in [-1, 1] (fp32)."""
        if self.vae is None:
            raise ValueError("construct the pipeline with a VAE to decode latents")
        latents = latents / self.vae.config.scaling_factor
        b, c, f, h, w = latents.shape
        image = self.vae.decode(latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)).sample
        return image[None].reshape((b, f, -1) + image.shape[2:]).permute(0, 2, 1, 3, 4).float()

    # -------------------------------------------------------------------------------------------- one denoise step
    def denoise_step(self, latents: torch.Tensor, t: int, prompt_embeds: torch.Tensor, camera: torch.Tensor,
                     image_embeds: torch.Tensor, first_frame_latents: torch.Tensor, guidance_scale: float,
                     i2v_cond_time_zero: bool = False, num_views: int = 4, do_classifier_free_guidance: bool = True,
                     eta: float = 0.0, generator: Optional[torch.Generator] = None,
                     variance_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Body of the loop at pipeline.py:1006-1031, in place on `latents` [Nv, 4, F, h, w] (fp32, device).
        With guidance, prompt_embeds / camera / image_embeds carry the (uncond, cond) CFG duplication; without it
        (guidance_scale <= 1 in `__call__`) they are the conditional ones only and the UNet batch is `latents` itself.
        eta > 0 adds std_dev * variance_noise (DDIMScheduler.step); unless given, the noise is drawn with `generator`, one
        draw of the latents' full shape per step, after the UNet call, as diffusers does."""
        if variance_noise is not None and generator is not None:
            raise ValueError("pass either `generator` or `variance_noise`, not both (DDIMScheduler.step)")
        x = torch.cat([latents, latents], 0) if do_classifier_free_guidance else latents
        noise_pred = self.unet(x, t, prompt_embeds, camera=camera, added_cond_kwargs={"image_embeds": image_embeds},
                               num_views=num_views, i2v_cond_time_zero=i2v_cond_time_zero).sample
        bn, c, f, h, w = latents.shape
        if do_classifier_free_guidance and eta == 0:
            # the released sampler: a3d_ddim_cfg_step runs the same kernel as a3d_ddim_step with std_dev 0
            a_t, a_p = self.scheduler.alphas_for(int(t))
            ops.ddim_cfg_step(latents, noise_pred.contiguous(), first_frame_latents.contiguous(), bn, c, f, h * w, guidance_scale,
                              a_t, a_p, uncond_first=True)
            return latents
        a_t, a_p, dir_coef, std_dev = self.scheduler.step_coefficients(int(t), eta)
        if eta > 0 and variance_noise is None:
            variance_noise = randn_tensor(latents.shape, generator, latents.device)
        z = variance_noise.to(latents.device, torch.float32).contiguous() if eta > 0 else None
        ops.ddim_step(latents, noise_pred.contiguous(), first_frame_latents.contiguous(), z, bn, c, f, h * w,
                      1 if do_classifier_free_guidance else 0, guidance_scale, a_t, a_p, dir_coef, std_dev if eta > 0 else 0.0)
        return latents

    def denoise_step_host(self, latents_host: torch.Tensor, t: int, prompt_embeds_host, camera_host, image_embeds_host,
                          first_frame_host, guidance_scale: float, out_host: Optional[torch.Tensor] = None,
                          num_views: int = 4) -> torch.Tensor:
        """Same step through HOST (pinned) buffers: copies the step's inputs to the device, runs it, copies the updated
        latents back -- what an external caller holding numpy/CPU tensors pays (bench.py's e2e leg)."""
        dev = self.device
        lat = latents_host.to(dev, non_blocking=True)
        pe = prompt_embeds_host.to(dev, non_blocking=True)
        cam = camera_host.to(dev, non_blocking=True)
        ie = image_embeds_host.to(dev, non_blocking=True)
        ff = first_frame_host.to(dev, non_blocking=True)
        self.denoise_step(lat, t, pe, cam, ie, ff, guidance_scale, num_views=num_views)
        if out_host is None:
            out_host = torch.empty_like(latents_host).pin_memory()
        out_host.copy_(lat, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return out_host

    def denoise_step_sharded(self, latents_local: torch.Tensor, t: int, prompt_embeds_local: torch.Tensor,
                             camera_local: torch.Tensor, image_embeds_local: torch.Tensor, first_frame_local: torch.Tensor,
                             guidance_scale: float, cfg_group=None, num_views_local: int = 4,
                             i2v_cond_time_zero: bool = False) -> torch.Tensor:
        """One denoise step of ONE prompt spread over ranks (SURVEY 8e): this rank owns `num_views_local` views (all of them,
        or one when `self.unet.view_group` shards the views) and either both CFG branches (cfg_group None: inputs carry the
        (uncond, cond) duplication) or one of them (cfg_group of size 2: rank 0 = uncond, rank 1 = cond).  Collectives: the
        K|V all-gathers inside the UNet (view group) and ONE all-gather of the noise prediction over the CFG group
        (n_local x 4 x F x h x w fp32 = 0.25 MB per view).  The latents stay sharded by view across steps."""
        nloc = latents_local.shape[0]
        if cfg_group is None:
            x = torch.cat([latents_local, latents_local], 0)
        else:
            x = latents_local
        eps = self.unet(x, t, prompt_embeds_local, camera=camera_local, added_cond_kwargs={"image_embeds": image_embeds_local},
                        num_views=num_views_local, i2v_cond_time_zero=i2v_cond_time_zero).sample
        if cfg_group is not None:
            import torch.distributed as dist
            eps2 = self._eps2 if getattr(self, "_eps2", None) is not None and self._eps2.shape[0] == 2 * nloc else None
            if eps2 is None:
                eps2 = self._eps2 = torch.empty(2 * nloc, *eps.shape[1:], device=eps.device, dtype=eps.dtype)
            dist.all_gather_into_tensor(eps2.view(-1), eps.contiguous().view(-1), group=cfg_group)
            eps = eps2
        a_t, a_p = self.scheduler.alphas_for(int(t))
        _, c, f, h, w = latents_local.shape
        ops.ddim_cfg_step(latents_local, eps.contiguous(), first_frame_local.contiguous(), nloc, c, f, h * w, guidance_scale, a_t,
                          a_p, uncond_first=True)
        return latents_local

    # -------------------------------------------------------------------------------------------- full sampler
    def _free_init_steps(self, it: int, num_inference_steps: int) -> int:
        """Steps of FreeInit pass `it`: all of them, or with coarse-to-fine sampling diffusers' share of them."""
        if not self._free_init_use_fast_sampling:
            return num_inference_steps
        return max(1, int(num_inference_steps / self._free_init_num_iters * (it + 1)))

    def _apply_free_init(self, latents, it, num_inference_steps, generator):
        """FreeInitMixin._apply_free_init on frames 1.. (pipeline.py:990-992; SURVEY Appendix B.11): keep the first pass's
        noise, or mix the previous result noised to t = 999 with fresh noise through the low-pass filter; then set this
        pass's schedule, which restarts the scheduler's step counter and history."""
        if it == 0:
            self._free_init_initial_noise = latents.detach().clone()
        else:
            order, ds, dt = self._fi
            if isinstance(self.scheduler, SOLVER_SCHEDULERS):
                # the scheduler's own add_noise at t = 999, on the schedule of the previous iteration
                t_T = torch.full((latents.shape[0],), self.scheduler.num_train_timesteps - 1, dtype=torch.long)
                z_T = self.scheduler.add_noise(latents, self._free_init_initial_noise, t_T)
            else:
                a = float(self.scheduler.alphas_cumprod[self.scheduler.num_train_timesteps - 1])
                z_T = math.sqrt(a) * latents + math.sqrt(1 - a) * self._free_init_initial_noise
            z_rand = randn_tensor(latents.shape, generator, latents.device)
            key = (tuple(latents.shape[-3:]), self._free_init_method, order, ds, dt, latents.device)
            if self._free_init_filter is None or self._free_init_filter[0] != key:
                self._free_init_filter = (key, free_init_filter(latents.shape, self._free_init_method, order, ds, dt,
                                                                latents.device))
            lpf = self._free_init_filter[1]
            dims = (-3, -2, -1)
            zf = torch.fft.fftshift(torch.fft.fftn(z_T, dim=dims), dim=dims)
            rf = torch.fft.fftshift(torch.fft.fftn(z_rand, dim=dims), dim=dims)
            latents = torch.fft.ifftn(torch.fft.ifftshift(zf * lpf + rf * (1 - lpf), dim=dims), dim=dims).real.contiguous()
        self.scheduler.set_timesteps(self._free_init_steps(it, num_inference_steps))
        return latents, self.scheduler.timesteps

    @torch.no_grad()
    def __call__(self, prompt=None, num_frames: int = 16, height: int = 256, width: int = 256, num_inference_steps: int = 50,
                 guidance_scale: float = 7.5, negative_prompt=None, num_videos_per_prompt: int = 1, eta: float = 0.0,
                 generator=None, latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, ip_adapter_image=None,
                 ip_adapter_image_embeds: Optional[torch.Tensor] = None, output_type: str = "pil", return_dict: bool = True,
                 cross_attention_kwargs=None, clip_skip=None, callback_on_step_end: Optional[Callable] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ("latents",), i2v_cond_time_zero: bool = False,
                 i2v_similarity_init=None, first_frame_latents: Optional[torch.Tensor] = None):
        """Argument names follow pipeline.py:760-786.  `num_videos_per_prompt` is the number of views.  Text / image
        encoders are only invoked if they were injected; otherwise prompt_embeds / negative_prompt_embeds [Nv,77,768],
        ip_adapter_image_embeds [Nv,1024] and first_frame_latents [Nv,4,1,h,w] must be given.  `generator` is one
        torch.Generator or a list of one per view, from which every draw of that view comes (`randn_tensor`)."""
        if isinstance(generator, list) and len(generator) != num_videos_per_prompt:     # prepare_latents, 699-703
            raise ValueError(f"generator is a list of {len(generator)} generators, but the call samples "
                             f"{num_videos_per_prompt} views (num_videos_per_prompt): pass one generator per view")
        if i2v_similarity_init is not None and self.free_init_enabled:
            # the reference reads an undefined `strength` on this path (pipeline.py:997): it has no defined meaning
            raise ValueError("i2v_similarity_init cannot be combined with FreeInit: the reference raises NameError there "
                             "(pipeline.py:997); call disable_free_init() or drop i2v_similarity_init")
        dev = self.device
        nv = num_videos_per_prompt
        do_cfg = guidance_scale > 1.0                                                  # pipeline.py:746-748
        if prompt_embeds is None or (do_cfg and negative_prompt_embeds is None):
            prompt_embeds, negative_prompt_embeds = self.encode_prompt(prompt, dev, nv, do_cfg, negative_prompt, prompt_embeds=prompt_embeds,
                                                                       negative_prompt_embeds=negative_prompt_embeds, clip_skip=clip_skip)
        if ip_adapter_image_embeds is None:
            ip_adapter_image_embeds, _ = self.encode_image(ip_adapter_image, dev)
        if first_frame_latents is None:
            first_frame_latents = self.encode_latents((height, width), ip_adapter_image)
        cam = get_camera(nv).to(dev)
        if do_cfg:
            pe = torch.cat([negative_prompt_embeds, prompt_embeds]).to(dev, torch.float32)            # (uncond, cond): line 932
            ie = torch.cat([torch.zeros_like(ip_adapter_image_embeds), ip_adapter_image_embeds]).to(dev, torch.float32)  # 537
            cam = torch.cat([cam, cam])
        else:                                                                          # pipeline.py:929-937, 1008-1018
            pe = prompt_embeds.to(dev, torch.float32)
            ie = ip_adapter_image_embeds.to(dev, torch.float32)
        first = first_frame_latents.to(dev, torch.float32).reshape(nv, -1, 1, height // 8, width // 8).contiguous()
        c = self.unet.config.in_channels
        if isinstance(self.scheduler, SOLVER_SCHEDULERS):
            lat = self._solver_loop(first, latents, num_frames, num_inference_steps, pe, cam, ie, guidance_scale,
                                    i2v_cond_time_zero, nv, do_cfg, generator, i2v_similarity_init, callback_on_step_end)
            return self._output(lat, output_type, return_dict)
        if i2v_similarity_init is not None:                                            # pipeline.py:940-946, 700-733
            timesteps = self.scheduler.get_timesteps(num_inference_steps, i2v_similarity_init["strength"])
            if latents is None:
                latents = similarity_init_latents(first, num_frames - 1, int(timesteps[0]), i2v_similarity_init["origin_prob"],
                                                  self.scheduler, generator)
        if latents is None:
            latents = randn_tensor((nv, c, num_frames - 1, height // 8, width // 8), generator, dev)
        rest = latents.to(dev, torch.float32)
        iters = self._free_init_num_iters if self.free_init_enabled else 1
        lat = torch.cat([first, rest], dim=2).contiguous()
        for it in range(iters):
            if self.free_init_enabled:
                rest, timesteps = self._apply_free_init(lat[:, :, 1:].contiguous(), it, num_inference_steps, generator)
                lat = torch.cat([first, rest], dim=2).contiguous()
            elif i2v_similarity_init is None:
                timesteps = self.scheduler.set_timesteps(num_inference_steps)
            for i, t in enumerate(timesteps):
                self.denoise_step(lat, int(t), pe, cam, ie, first, guidance_scale, i2v_cond_time_zero, nv, do_cfg, eta, generator)
                if callback_on_step_end is not None:
                    res = callback_on_step_end(self, i, int(t), {"latents": lat})
                    lat = res.pop("latents", lat)
        return self._output(lat, output_type, return_dict)

    def _output(self, lat, output_type, return_dict):
        if output_type == "latent":
            video = lat
        else:
            if self.vae is None:
                raise ValueError('output_type "pil" / "np" / "pt" needs a VAE; pass output_type="latent" to get the latents '
                                 "(pipeline.py:1049-1056)")
            video = tensor2vid(self.decode_latents(lat), getattr(self, "image_processor", None), output_type=output_type)
        return AnimateDiffMVI2VPipelineOutput(frames=video) if return_dict else (video,)

    def _solver_loop(self, first, latents, num_frames, num_inference_steps, pe, cam, ie, guidance_scale, i2v_cond_time_zero,
                     nv, do_cfg, generator, similarity, callback_on_step_end):
        """The sampling loop of pipeline.py:939-1047 for DPM-Solver++, the Euler, PNDM and LMS schedulers: scale_model_input
        on the UNet input, each entry of the schedule into the UNet, then one a3d_sampler_step or a3d_multistep_step (CFG
        combine, solver update, frame-0 re-injection).  The Euler schedulers draw one normal sample of the latents' shape
        per step after the UNet call, as diffusers' step does; DPM-Solver++ keeps each step's m0 in one of two device
        buffers that swap roles.  PNDM and LMS keep their past model outputs or derivatives in a ring of four device
        buffers whose slots each step names, and PNDM its saved sample and Runge-Kutta sum in two more; they draw
        nothing."""
        sched, dev = self.scheduler, self.device
        c, h, w = first.shape[1], first.shape[3], first.shape[4]
        if similarity is not None:                                                     # pipeline.py:943-946, 707-729
            timesteps = sched.get_timesteps(num_inference_steps, similarity["strength"])
            if latents is None:
                latents = similarity_init_latents(first, num_frames - 1, timesteps[0], similarity["origin_prob"], sched,
                                                  generator)
            rest = latents.to(dev, torch.float32)
        else:                                                                          # pipeline.py:941, 700-732
            timesteps = sched.set_timesteps(num_inference_steps)
            if latents is None:
                latents = randn_tensor((nv, c, num_frames - 1, h, w), generator, dev)
            rest = latents.to(dev, torch.float32) * sched.init_noise_sigma
        lat = torch.cat([first, rest], dim=2).contiguous()
        dpm = isinstance(sched, DPMSolverMultistepScheduler)
        hist = (torch.empty_like(lat), torch.empty_like(lat)) if dpm else (None, None)
        multistep = isinstance(sched, MULTISTEP_SCHEDULERS)
        ring = [torch.empty_like(lat) for _ in range(RING)] if multistep else None
        pndm = (torch.empty_like(lat), torch.empty_like(lat)) if isinstance(sched, PNDMScheduler) else (None, None)
        for it in range(self._free_init_num_iters if self.free_init_enabled else 1):
            if self.free_init_enabled:
                rest, timesteps = self._apply_free_init(lat[:, :, 1:].contiguous(), it, num_inference_steps, generator)
                lat = torch.cat([first, rest], dim=2).contiguous()
            for i, t in enumerate(timesteps):
                x = torch.cat([lat, lat], 0) if do_cfg else lat
                x = sched.scale_model_input(x, t)
                noise_pred = self.unet(x, float(t), pe, camera=cam, added_cond_kwargs={"image_embeds": ie}, num_views=nv,
                                       i2v_cond_time_zero=i2v_cond_time_zero).sample
                step = sched.next_step(t)
                if multistep:
                    ops.multistep_step(lat, noise_pred.contiguous(), first, nv, c, num_frames, h * w, 1 if do_cfg else 0,
                                       guidance_scale, step, ring, *pndm)
                else:
                    z = None if dpm else randn_tensor(lat.shape, generator, dev)
                    ops.sampler_step(lat, noise_pred.contiguous(), first, nv, c, num_frames, h * w, 1 if do_cfg else 0,
                                     guidance_scale, step, noise=z if step.sigma_up != 0.0 else None,
                                     history_out=hist[i % 2], history_in=hist[(i + 1) % 2] if step.order == 2 else None)
                if callback_on_step_end is not None:
                    res = callback_on_step_end(self, i, t.item(), {"latents": lat})
                    lat = res.pop("latents", lat)
        return lat


AnimationPipeline = AnimateDiffMVI2VPipeline   # name used by BASELINE.json's north_star


def read_yaml(config) -> dict:
    """A parsed config (returned as a plain dict) or the path of a YAML file, read with PyYAML (the inference configs use
    no OmegaConf interpolation)."""
    if isinstance(config, dict):
        return dict(config)
    import yaml
    with open(config) as f:
        return yaml.safe_load(f)


def load_pipeline(config, pretrained_unet_path: Optional[str], device: str = "cuda", num_views: int = 4,
                  num_frames: int = 16) -> AnimateDiffMVI2VPipeline:
    """The sampling pipeline of inference.py:60-245 from the files `config` (configs/inference/inference.yaml, parsed or a
    path) names: DDIMScheduler(**noise_scheduler_kwargs); transformers' CLIPTokenizer and CLIPTextModel from
    `<pretrained_model_path>/tokenizer` and `/text_encoder` (local files only); the engine's VAE from `/vae`, UNet
    (`MVUNetMotionModel.from_pretrained` with the motion adapter, IP-Adapter and `pretrained_unet_path`) and IP-Adapter
    image tower from `<ip_adapter_path>/models/image_encoder` behind a `CLIPImageProcessor`; FreeInit (butterworth, no fast
    sampling) when `freeinit_enabled`.  num_views / num_frames wire the UNet's attention processors, as inference.py's
    --N / --L do."""
    from transformers import CLIPTextModel, CLIPTokenizer

    from . import pretrained as PT
    from .clip import CLIPImageProcessor, CLIPVisionModelWithProjection
    from .vae import AutoencoderKL
    cfg = read_yaml(config)
    base, ip = cfg["pretrained_model_path"], cfg.get("ip_adapter_path")
    scheduler = DDIMScheduler(**(cfg.get("noise_scheduler_kwargs") or {}))
    tokenizer = CLIPTokenizer.from_pretrained(PT.resolve(base, "tokenizer"), local_files_only=True)
    text_encoder = CLIPTextModel.from_pretrained(PT.resolve(base, "text_encoder"), local_files_only=True).to(device).eval()
    vae = AutoencoderKL.from_pretrained(base, subfolder="vae", device=device)
    model_config = {k: cfg[k] for k in ("mvdream_attn_cfg", "motion_module_attn_cfg", "i2v_cond_time_zero") if k in cfg}
    unet = MVUNetMotionModel.from_pretrained(base, cfg.get("motion_adapter_path"), ip, pretrained_unet_path, model_config,
                                             device=device, num_views=num_views, num_frames=num_frames)
    image_encoder = feature_extractor = None
    if ip:
        image_encoder = CLIPVisionModelWithProjection.from_pretrained(PT.resolve(ip, "models/image_encoder"), device=device)
        feature_extractor = CLIPImageProcessor(device=device)
    pipe = AnimateDiffMVI2VPipeline(vae=vae, text_encoder=text_encoder, tokenizer=tokenizer, unet=unet, scheduler=scheduler,
                                    feature_extractor=feature_extractor, image_encoder=image_encoder)
    if cfg.get("freeinit_enabled"):
        pipe.enable_free_init(method="butterworth", num_iters=cfg.get("freeinit_num_iters", 3), use_fast_sampling=False)
    return pipe
