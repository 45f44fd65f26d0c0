"""Drop-in for the reference's threestudio guidance plugin `AnimateMVDiffusionGuidance`
(custom/threestudio-animate3d/guidance/animatemv_guidance.py:54-793, registered "animatemv-diffusion-guidance"):

    guidance = threestudio.find("animatemv-diffusion-guidance")(cfg)
    out = guidance(rgb, prompt_utils, elevation, azimuth, camera_distances, c2w, rgb_as_latents=False, guidance_eval=False)
    out["loss_sds"].backward()                                   # animate3d.py:180-215
    guidance.update_step(epoch, global_step)

Hot path = `compute_mvdream_recon_loss` (391-513): noise frames 1.., ONE classifier-free-guided UNet evaluation with no
grad (422-459; (cond, uncond) order, `text + s*(text - uncond)`), x0 through the DDIM scheduler (466), std-rescale
(468-487), x0-reconstruction MSE (497-501).  The UNet evaluation runs on the sm_90a engine (`MVUNetMotionModel`); the
remaining arithmetic is a handful of elementwise/reduction ops on [B*Nv*F, 4, 32, 32] latents that must stay on the
autograd tape (the loss's gradient flows to `latents` and from there through the VAE encoder to the rasterizer), so they
are torch ops.

Differences from the reference class, all at construction time (there are no Hugging Face checkpoints to load here):
`configure()` accepts the already-built components (`unet`, `vae`, `ip_image_processor`, `scheduler`) as keyword arguments;
with none given it builds the engine UNet from `cfg.model_config` and loads `cfg.pretrained_unet_path` through
`weights.load_unet_checkpoint` (inference.py:213-223 semantics)."""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Any, Optional

import torch
import torch.nn.functional as F

from .capture import capturing
from .registry import BaseObject, C, register
from .scheduler import DDIMScheduler


def normalize_camera(camera_matrix: torch.Tensor) -> torch.Tensor:
    """animatemv_guidance.py:40-52: translation of each 4x4 c2w normalised onto the unit sphere, flattened to 16.
    (The reference normalises IN PLACE on a view of its argument; this returns a copy.)"""
    cam = camera_matrix.clone().reshape(-1, 4, 4)
    t = cam[:, :3, 3]
    cam[:, :3, 3] = t / (torch.norm(t, dim=1, keepdim=True) + 1e-8)
    return cam.reshape(-1, 16)


get_camera_cond = normalize_camera          # round-1 name, kept for callers/tests


class PrecomputedPromptUtils:
    """Minimal stand-in for threestudio's PromptProcessorOutput when text embeddings are computed elsewhere:
    `get_text_embeddings(elevation, azimuth, camera_distances, view_dependent_prompting)` returns
    [2 * B*Nv, 77, 768] in (cond, uncond) order (threestudio/models/prompt_processors/base.py:79-80)."""
    use_perp_neg = False

    def __init__(self, text_embeddings: torch.Tensor, uncond_text_embeddings: torch.Tensor):
        self.text, self.uncond = text_embeddings, uncond_text_embeddings          # [77, 768] each (or [1, 77, 768])

    def get_text_embeddings(self, elevation, azimuth, camera_distances, view_dependent_prompting: bool = False):
        if view_dependent_prompting:
            raise NotImplementedError("view-dependent prompting is off in every shipped config (refine_frame_16.yaml)")
        bs = elevation.shape[0]
        t = self.text.reshape(1, *self.text.shape[-2:]).expand(bs, -1, -1)
        u = self.uncond.reshape(1, *self.uncond.shape[-2:]).expand(bs, -1, -1)
        return torch.cat([t, u], dim=0)


def _resize_bilinear(x: torch.Tensor, size) -> torch.Tensor:
    """F.interpolate(x, size, mode="bilinear", align_corners=False) on the SDS gradient path.  PyTorch's CUDA backward of that
    resize scatters with atomics and raises under torch.use_deterministic_algorithms(True); there the same interpolation
    weights (read off F.interpolate applied to identity matrices) are applied as two matmuls, whose backward is deterministic."""
    if not (torch.are_deterministic_algorithms_enabled() and x.requires_grad):
        return F.interpolate(x, size, mode="bilinear", align_corners=False)
    h, w = x.shape[-2:]
    with torch.no_grad():
        eye = lambda n: torch.eye(n, device=x.device, dtype=x.dtype)[None, None]
        wy = F.interpolate(eye(h), (size[0], h), mode="bilinear", align_corners=False)[0, 0]     # [Ho, h]
        wx = F.interpolate(eye(w), (size[1], w), mode="bilinear", align_corners=False)[0, 0]     # [Wo, w]
    return wy @ x @ wx.t()


@register("animatemv-diffusion-guidance")
class AnimateMVDiffusionGuidance(BaseObject):
    @dataclass
    class Config(BaseObject.Config):
        # field names / defaults of animatemv_guidance.py:56-101
        pretrained_model_name_or_path: str = ""
        motion_adapter_path: Optional[str] = None
        ip_adapter_path: Optional[str] = None
        pretrained_unet_path: Optional[str] = None
        model_config: Optional[dict] = None
        enable_sequential_cpu_offload: bool = False
        enable_channels_last_format: bool = False
        guidance_scale: float = 100.0
        grad_clip: Optional[Any] = None
        half_precision_weights: bool = True
        min_step_percent: Any = 0.02
        max_step_percent: Any = 0.98
        sqrt_anneal: bool = False
        trainer_max_steps: int = 25000
        token_merging: bool = False
        token_merging_params: Optional[dict] = field(default_factory=dict)
        max_items_eval: int = 4
        camera_condition_type: str = "rotation"
        view_dependent_prompting: bool = False
        i2v_cond_time_zero: bool = False
        n_view: int = 4
        n_frame: int = 8
        image_size: int = 256
        recon_loss: bool = True
        recon_std_rescale: float = 0.5
        noise_scheduler_kwargs: Optional[dict] = None

    cfg: Config

    def configure(self, unet=None, vae=None, ip_image_processor=None, scheduler: Optional[DDIMScheduler] = None) -> None:
        cfg = self.cfg
        if cfg.token_merging or cfg.enable_sequential_cpu_offload or cfg.enable_channels_last_format:
            raise NotImplementedError("token merging / cpu offload / channels_last change the attention processors or the "
                                      "layout of the reference model; the engine has one fixed layout")
        if not cfg.recon_loss:
            raise NotImplementedError("only the x0-reconstruction loss path exists in the reference (recon_loss=True)")
        self.weights_dtype = torch.float16 if cfg.half_precision_weights else torch.float32
        if unet is None:
            from .unet import MVUNetMotionModel
            from .unet_config import UNetConfig
            from .weights import load_unet_checkpoint
            mc = dict(cfg.model_config or {})
            unet = MVUNetMotionModel(UNetConfig(num_views=cfg.n_view, num_frames=cfg.n_frame, **mc.get("unet_additional_kwargs", {})))
            if not cfg.pretrained_unet_path or not os.path.exists(cfg.pretrained_unet_path):
                raise FileNotFoundError("pretrained_unet_path is required when no `unet` is injected "
                                        f"(got {cfg.pretrained_unet_path!r})")
            load_unet_checkpoint(unet, cfg.pretrained_unet_path)
        self.unet = unet
        self.vae = vae
        self.ip_image_processor = ip_image_processor
        self.scheduler = scheduler or DDIMScheduler(**(cfg.noise_scheduler_kwargs or {}))
        self.num_train_timesteps = self.scheduler.num_train_timesteps
        self.scheduler.set_timesteps(self.num_train_timesteps)              # animatemv_guidance.py:313 -> prev = t - 1
        dev = getattr(unet, "device", self.device)
        self.device = torch.device(dev)
        self.alphas = torch.from_numpy(self.scheduler.alphas_cumprod).to(self.device)
        self.set_min_max_steps()                                            # defaults (0.02, 0.98) until update_step
        self.grad_clip_val: Optional[float] = None

    # ---------------------------------------------------------------------------------------------- small helpers
    def set_min_max_steps(self, min_step_percent: float = 0.02, max_step_percent: float = 0.98):
        """Also writes [min_step, max_step] into the device tensor `step_bounds` in place, where a captured step's
        `draw_timestep` reads them at every replay."""
        self.min_step = int(self.num_train_timesteps * min_step_percent)
        self.max_step = int(self.num_train_timesteps * max_step_percent)
        if getattr(self, "step_bounds", None) is None:
            self.step_bounds = torch.tensor([self.min_step, self.max_step], dtype=torch.long, device=self.device)
        else:
            self.step_bounds[0].fill_(self.min_step)
            self.step_bounds[1].fill_(self.max_step)

    def draw_timestep(self, batch_size: int) -> torch.Tensor:
        """[batch_size] int64 timesteps drawn uniformly from min_step .. max_step inclusive, on the device and from torch's
        generator of that device, with the bounds read from `step_bounds`: no host read, so a CUDA graph that records the
        draw follows `set_min_max_steps` / `update_step` at every replay."""
        lo, hi = self.step_bounds[0], self.step_bounds[1]
        u = torch.rand(batch_size, dtype=torch.float64, device=self.step_bounds.device)
        return torch.minimum(lo + (u * (hi - lo + 1)).long(), hi)

    def forward_unet(self, latents, t, encoder_hidden_states, camera, i2v_cond_time_zero: bool, added_cond_kwargs=None):
        """animatemv_guidance.py:328-346 (the dtype casts there are the engine's own fp16 entry)."""
        return self.unet(latents, t, encoder_hidden_states, camera=camera, added_cond_kwargs=added_cond_kwargs,
                         num_views=self.cfg.n_view, i2v_cond_time_zero=i2v_cond_time_zero).sample.to(latents.dtype)

    def get_camera_cond(self, camera: torch.Tensor, fovy=None) -> torch.Tensor:
        if self.cfg.camera_condition_type != "rotation":
            raise NotImplementedError(f"Unknown camera_condition_type={self.cfg.camera_condition_type}")
        return normalize_camera(camera)

    def encode_images(self, imgs: torch.Tensor) -> torch.Tensor:
        """[B,3,256,256] in [0,1] -> [B,4,32,32] (365-373); differentiable w.r.t. imgs (the SDS gradient path)."""
        if self.vae is None:
            raise ValueError("no VAE was given to the guidance: pass `vae=` at construction or call with rgb_as_latents=True")
        posterior = self.vae.encode(imgs * 2.0 - 1.0).latent_dist
        return (posterior.sample() * self.vae.config.scaling_factor).to(imgs.dtype)

    def decode_latents(self, latents: torch.Tensor, latent_height: int = 64, latent_width: int = 64) -> torch.Tensor:
        """375-389."""
        if self.vae is None:
            raise ValueError("no VAE was given to the guidance")
        latents = F.interpolate(latents, (latent_height, latent_width), mode="bilinear", align_corners=False)
        image = self.vae.decode(latents / self.vae.config.scaling_factor).sample
        return (image * 0.5 + 0.5).clamp(0, 1).to(latents.dtype)

    def _alpha(self, t: torch.Tensor) -> torch.Tensor:
        return self.alphas[t.to(self.alphas.device)]

    # ---------------------------------------------------------------------------------------------- the loss
    def compute_mvdream_recon_loss(self, latents, t, prompt_utils, elevation, azimuth, camera_distances, camera=None,
                                   image_embeds=None, noise: Optional[torch.Tensor] = None):
        """animatemv_guidance.py:391-513.  latents [(b n f), 4, h, w] with grad; t [b] long; camera [(b n f), 4, 4] c2w;
        image_embeds [b*n, 1024].  `noise` (not in the reference signature) fixes the draw of line 428 for tests."""
        cfg = self.cfg
        n, f = cfg.n_view, cfg.n_frame
        b = elevation.shape[0] // (n * f)
        first_of = lambda x: x.reshape(b, n, f)[..., 0].reshape(-1)
        text_embeddings = prompt_utils.get_text_embeddings(first_of(elevation), first_of(azimuth), first_of(camera_distances),
                                                           cfg.view_dependent_prompting)            # (cond, uncond): 410-412
        loss, aux = self._recon_loss(latents, t, text_embeddings, camera, image_embeds, noise)
        aux.update({"use_perp_neg": getattr(prompt_utils, "use_perp_neg", False), "neg_guidance_weights": None,
                    "text_embeddings": text_embeddings})
        return loss, aux

    def _recon_loss(self, latents, t, text_embeddings, camera, image_embeds, noise=None):
        cfg = self.cfg
        n, f = cfg.n_view, cfg.n_frame
        bnf, c, h, w = latents.shape
        b = bnf // (n * f)
        t = t.to(latents.device)
        lat = latents.reshape(b, n, f, c, h, w).permute(0, 1, 3, 2, 4, 5)          # b n c f h w   (line 414)
        first = lat[:, :, :, 0:1]
        rest = lat[:, :, :, 1:]
        with torch.no_grad():
            if noise is None:
                noise = torch.randn_like(rest)
            a = self._alpha(t).reshape(b, 1, 1, 1, 1, 1).to(latents.dtype)
            rest_noisy = a.sqrt() * rest + (1 - a).sqrt() * noise                   # scheduler.add_noise (line 429)
            noisy = torch.cat([first, rest_noisy], dim=3).reshape(b * n, c, f, h, w)
            cam2 = None
            if camera is not None:
                cam = self.get_camera_cond(camera.reshape(b, n, f, 4, 4)[:, :, 0].reshape(b * n, 4, 4))
                cam2 = torch.cat([cam, cam])
            ts = t[:, None].repeat(1, n).reshape(-1)
            eps2 = self.forward_unet(torch.cat([noisy, noisy]), torch.cat([ts, ts]).float(), text_embeddings, cam2,
                                     cfg.i2v_cond_time_zero,
                                     {"image_embeds": torch.cat([image_embeds, torch.zeros_like(image_embeds)])})
            e_text, e_unc = eps2.chunk(2)                                           # (cond, uncond): line 452
            to_img = lambda x: x.permute(0, 2, 1, 3, 4).reshape(b * n * f, c, h, w)  # "b c f h w -> (b f) c h w"
            e_text, e_unc = to_img(e_text), to_img(e_unc)
            eps = e_text + cfg.guidance_scale * (e_text - e_unc)                    # line 457
            noisy_img = to_img(noisy)
            a_img = self._alpha(t).repeat_interleave(n * f).reshape(-1, 1, 1, 1).to(latents.dtype)
            x0 = (noisy_img - (1 - a_img).sqrt() * eps) / a_img.sqrt()              # pred_original_sample (466)
            if cfg.recon_std_rescale > 0:
                x0_nocfg = (noisy_img - (1 - a_img).sqrt() * e_text) / a_img.sqrt()
                r = lambda x: x.reshape(b, n, f, c, h, w)[:, :, 1:]
                factor = (r(x0_nocfg).std([1, 2, 3, 4, 5], keepdim=True) + 1e-8) / (r(x0).std([1, 2, 3, 4, 5], keepdim=True) + 1e-8)
                adj = x0 * factor.reshape(b, 1, 1, 1).repeat_interleave(n * f, dim=0)
                x0 = cfg.recon_std_rescale * adj + (1 - cfg.recon_std_rescale) * x0
            x0 = x0.reshape(b * n, f, c, h, w)
            x0 = torch.cat([latents.detach().reshape(b * n, f, c, h, w)[:, 0:1], x0[:, 1:]], dim=1).reshape(bnf, c, h, w)
        loss = 0.5 * F.mse_loss(latents, x0, reduction="sum") / latents.shape[0] * f / (f - 1)     # 497-501
        return loss, {"t_orig": t, "latents_noisy": noisy_img, "noise_pred": eps, "latents_recon": x0}

    # ---------------------------------------------------------------------------------------------- plugin entry
    def __call__(self, rgb, prompt_utils, elevation, azimuth, camera_distances, c2w, rgb_as_latents: bool = False,
                 guidance_eval: bool = False, **kwargs):
        """animatemv_guidance.py:515-600.  rgb [B,H,W,3] in [0,1] with grad, B = b * n_view * n_frame.
        Extra keyword hooks (not in the reference): `image_embeds` [b*n_view, 1024] bypasses the CLIP image encoder,
        `timestep` [b] fixes the draw of line 556.

        Inside a CUDA-graph capture the timestep is drawn by `draw_timestep` (eagerly by torch.randint, as the reference
        does); either way `last_timestep` holds the draw.  guidance_eval reads the device from the host and raises there."""
        in_capture = capturing(self.device)
        if guidance_eval and in_capture:
            raise ValueError("guidance_eval reads the device from the host and runs 25 more UNet evaluations: it cannot be "
                             "part of a captured step; call it eagerly")
        cfg = self.cfg
        batch_size = rgb.shape[0] // (cfg.n_view * cfg.n_frame)
        rgb_bchw = rgb.permute(0, 3, 1, 2)
        if rgb_as_latents:
            latents = _resize_bilinear(rgb_bchw, (32, 32))
        else:
            latents = self.encode_images(_resize_bilinear(rgb_bchw, (256, 256)))
        image_embeds = kwargs.get("image_embeds")
        if image_embeds is None:
            if self.ip_image_processor is None:
                raise ValueError("no IP-adapter image processor: pass `ip_image_processor=` at construction or `image_embeds=`")
            with torch.no_grad():      # frame 0 of every view is the condition image (541-550)
                cond = rgb_bchw.reshape(-1, cfg.n_frame, *rgb_bchw.shape[1:])[:, 0]
                image_embeds = self.ip_image_processor.encode_image(cond)
        t = kwargs.get("timestep")
        if t is None:
            if in_capture:
                t = self.draw_timestep(batch_size)
            else:
                t = torch.randint(self.min_step, self.max_step + 1, [batch_size], dtype=torch.long, device=latents.device)
        self.last_timestep = t
        loss, aux = self.compute_mvdream_recon_loss(latents, t, prompt_utils, elevation, azimuth, camera_distances, c2w, image_embeds)
        out = {"loss_sds": loss, "min_step": self.min_step, "max_step": self.max_step}
        if guidance_eval:
            ev = self.guidance_eval(camera=c2w, image_embeds=image_embeds, **aux)
            ev["texts"] = [f"n{nl:.02f}\ne{e.item():.01f}\na{a.item():.01f}\nc{c.item():.02f}"
                           for nl, e, a, c in zip(ev["noise_levels"], elevation, azimuth, camera_distances)]
            out["eval"] = ev
        return out

    @torch.no_grad()
    def get_noise_pred(self, latents_noisy, t, text_embeddings, use_perp_neg=False, neg_guidance_weights=None, camera=None,
                       i2v_cond_time_zero=False, image_embeds=None):
        """602-667 (the perp-neg branch is dead in the reference: it calls forward_unet without camera/image embeds)."""
        if use_perp_neg:
            raise NotImplementedError("perp-neg is not wired to the multi-view UNet in the reference either (614-640)")
        cfg = self.cfg
        n, f = cfg.n_view, cfg.n_frame
        b = latents_noisy.shape[0] // (n * f)
        c, h, w = latents_noisy.shape[1:]
        x = latents_noisy.reshape(b * n, f, c, h, w).permute(0, 2, 1, 3, 4)
        cam = self.get_camera_cond(camera.reshape(b, n, f, 4, 4)[:, :, 0].reshape(b * n, 4, 4))
        tt = torch.as_tensor(t, device=latents_noisy.device).reshape(1).float().repeat(b * n * 2)
        eps2 = self.forward_unet(torch.cat([x, x]), tt, text_embeddings, torch.cat([cam, cam]), i2v_cond_time_zero,
                                 {"image_embeds": torch.cat([image_embeds, torch.zeros_like(image_embeds)])})
        e_text, e_unc = eps2.chunk(2)
        eps = e_text + cfg.guidance_scale * (e_text - e_unc)
        return eps.permute(0, 2, 1, 3, 4).reshape(b * n * f, c, h, w)

    @torch.no_grad()
    def guidance_eval(self, camera, image_embeds, t_orig, text_embeddings, latents_noisy, latents_recon, noise_pred,
                      use_perp_neg=False, neg_guidance_weights=None):
        """670-765: finish the denoising from the sampled noise level with a 25-step DDIM schedule (debug visualisation).
        Returns latents for every stage and, when a VAE is attached, the decoded videos under the reference's keys."""
        cfg = self.cfg
        f = cfg.n_frame
        sched = DDIMScheduler(**(cfg.noise_scheduler_kwargs or {}))
        steps = torch.as_tensor(sched.set_timesteps(25).copy(), device=latents_noisy.device)
        bs = latents_noisy.shape[0]
        t0 = t_orig.reshape(-1)[0]
        larger = steps > t0
        idx = int(torch.min(larger.to(torch.int64), dim=0)[1])         # first schedule entry that is NOT larger than t_orig
        t = int(steps[idx])
        fracs = [t / self.num_train_timesteps] * min(bs, len(t_orig.reshape(-1)) * cfg.n_view * f)

        def keep_first(x):                                             # frame 0 of every view is never denoised
            x = x.reshape(-1, f, *x.shape[1:])
            r = latents_recon.reshape(-1, f, *latents_recon.shape[1:])
            return torch.cat([r[:, 0:1], x[:, 1:]], dim=1).reshape(bs, *latents_recon.shape[1:])

        a_t, a_p = sched.alphas_for(t)
        x0 = (latents_noisy - (1 - a_t) ** 0.5 * noise_pred) / a_t ** 0.5
        lat_1step = keep_first(a_p ** 0.5 * x0 + (1 - a_p) ** 0.5 * noise_pred)
        lat_1orig = keep_first(x0)
        lat = lat_1step
        for tt in steps[idx + 1:].tolist():
            eps = self.get_noise_pred(lat, tt, text_embeddings, use_perp_neg, neg_guidance_weights, camera,
                                      cfg.i2v_cond_time_zero, image_embeds)
            a_t, a_p = sched.alphas_for(int(tt))
            x0 = (lat - (1 - a_t) ** 0.5 * eps) / a_t ** 0.5
            lat = keep_first(a_p ** 0.5 * x0 + (1 - a_p) ** 0.5 * eps)
        out = {"bs": bs, "noise_levels": fracs, "latents_noisy": latents_noisy, "latents_recon": latents_recon,
               "latents_1step": lat_1step, "latents_1orig": lat_1orig, "latents_final": lat}
        if self.vae is not None:
            dec = lambda x: self.decode_latents(x, x.shape[-2], x.shape[-1])
            out.update({"video_noisy": dec(latents_noisy), "video_recon": dec(latents_recon), "video_1step": dec(lat_1step),
                        "video_1orig": dec(lat_1orig), "video_final": dec(lat)})
        return out

    def update_step(self, epoch: int, global_step: int, on_load_weights: bool = False):
        """767-793: gradient-clip schedule and the [min_step, max_step] annealing."""
        cfg = self.cfg
        if cfg.grad_clip is not None:
            self.grad_clip_val = C(cfg.grad_clip, epoch, global_step)
        if cfg.sqrt_anneal:
            percentage = (float(global_step) / cfg.trainer_max_steps) ** 0.5
            mx = cfg.max_step_percent if isinstance(cfg.max_step_percent, (float, int)) else cfg.max_step_percent[1]
            mn = C(cfg.min_step_percent, epoch, global_step)
            cur = (mx - mn) * (1 - percentage) + mn
            self.set_min_max_steps(min_step_percent=cur, max_step_percent=cur)
        else:
            self.set_min_max_steps(min_step_percent=C(cfg.min_step_percent, epoch, global_step),
                                   max_step_percent=C(cfg.max_step_percent, epoch, global_step))
