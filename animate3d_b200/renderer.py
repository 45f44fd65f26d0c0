"""Drop-in for the reference's 4D renderer plugin: `DiffGaussian4D` (custom/threestudio-animate3d/renderer/
diff_gaussian_rasterizer_advanced_4d.py:23-192, registered "diff-gaussian-rasterizer-advanced-4d") with its
`forward(viewpoint_camera, bg_color, scaling_modifier, override_color, timestamps, **kwargs)` and the
`Gaussian4DBatchRenderer.batch_forward(batch)` mix-in (renderer/gaussian_batch_renderer_4d.py:11-111).

The reference loops over the `bs` cameras of a batch in Python (line 27): per camera 2 x torch.inverse, a k-planes lookup +
3 MLPs, ~8 rasterizer kernels, 2 CUB calls and a blocking D2H read.  Here `batch_forward` does: camera matrices for all
cameras at once (threestudio/utils/ops.py:305-359), ONE deformation launch for the distinct timestamps, ONE launch per
rasterizer stage for all cameras, one host sync per batch.  `forward` (single camera) is the same path with bs = 1.

Per-camera semantics kept from `forward` (lines 65-192):
  * training-time background inversion with probability 1 - invert_bg_prob, drawn per camera (65-70)
  * static gaussians for the condition frame (timestamp -1) unless `first_frame_trainable` (77-83)
  * `do_guidance=False` (reconstruction stage): scales are NOT deformed (132-135) and only a random ~10 % of the gaussians of
    each camera receive gradient through means / scales / rotations: x*mask + x.detach()*(1-mask) (147-154)
  * `do_reconstruction=False`: means3D detached at the rasterizer input (161)
  * SH features = cat(features_dc, features_rest) (pc.get_features, line 141) at `active_sh_degree`
  * outputs: render (clamped), depth, mask, viewspace_points (per-camera tensors whose .grad holds the screen-space
    gradient), visibility_filter, radii, means3D / scales / rotations BEFORE the gradient mask, opacities."""
from __future__ import annotations

import math
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch

from .gaussian4d import Gaussian4DModel
from .rasterizer import _RasterizeBatch
from .registry import BaseObject, register


def get_cam_info_gaussian(c2w: torch.Tensor, fovx, fovy, znear: float = 0.1, zfar: float = 100.0):
    """threestudio/utils/ops.py:344-359, batched over a leading camera dimension (fovx / fovy: floats or [bs] tensors):
    returns (world_view_transform, full_proj_transform, camera_center, tan(fovx/2), tan(fovy/2)) in the row-vector
    convention of the rasterizer."""
    c2w = c2w.float().reshape(-1, 4, 4)
    bs, dev = c2w.shape[0], c2w.device
    flip = torch.eye(4, device=dev)
    flip[1, 1] = -1
    flip[2, 2] = -1
    wv = torch.linalg.inv(c2w @ flip).transpose(1, 2).contiguous()
    tx = torch.tan(torch.as_tensor(fovx, dtype=torch.float32, device=dev).reshape(-1) * 0.5).expand(bs)
    ty = torch.tan(torch.as_tensor(fovy, dtype=torch.float32, device=dev).reshape(-1) * 0.5).expand(bs)
    P = torch.zeros(bs, 4, 4, device=dev)
    P[:, 0, 0] = 1.0 / tx
    P[:, 1, 1] = 1.0 / ty
    P[:, 3, 2] = 1.0
    P[:, 2, 2] = zfar / (zfar - znear)
    P[:, 2, 3] = -(zfar * znear) / (zfar - znear)
    full = wv @ P.transpose(1, 2)
    cam = torch.linalg.inv(wv)[:, 3, :3]
    return wv, full, cam, tx, ty


class Gaussian4DBatchRenderer:
    """Mix-in of gaussian_batch_renderer_4d.py.  Expects `self.geometry`, `self.background_tensor`, `self.cfg` (with
    invert_bg_prob / first_frame_trainable) and `self.training`."""

    def _render_cameras(self, wv, full, cam, tx, ty, H: int, W: int, ts: Optional[torch.Tensor], bg_color: torch.Tensor,
                        scaling_modifier: float, override_color, do_guidance: bool, do_reconstruction: bool) -> Dict[str, Any]:
        pc: Gaussian4DModel = self.geometry
        bs = wv.shape[0]
        dev = pc._xyz.device
        P = pc._xyz.shape[0]
        # ---- deformation: one evaluation per DISTINCT timestamp (the views of a frame share it)
        if ts is None:
            means = pc._xyz[None].expand(bs, P, 3)
            scales = torch.exp(pc._scaling)[None].expand(bs, P, 3)
            rots = torch.nn.functional.normalize(pc._rotation, dim=-1)[None].expand(bs, P, 4)
        else:
            uniq, inverse = torch.unique(ts.reshape(bs).float(), return_inverse=True)
            # 132-137; static gaussians for the condition frame unless first_frame_trainable (77-83: hidden_feats stays None)
            means_t, scales_t, rots_t = pc.deform_frames(uniq, deform_scale=bool(do_guidance),
                                                         first_frame_trainable=self.cfg.first_frame_trainable)
            means, scales, rots = means_t[inverse], scales_t[inverse], rots_t[inverse]
        # per-camera tensors that are ON the autograd path (callers read / retain_grad `out["means3D"][i]` like the reference's
        # per-camera `means3D`): unbind first, render from the re-stacked batch
        means_l, scales_l, rots_l = list(means.unbind(0)), list(scales.unbind(0)), list(rots.unbind(0))
        means, scales, rots = torch.stack(means_l), torch.stack(scales_l), torch.stack(rots_l)
        # ---- reconstruction-stage gradient gating (147-154): ~10 % of the gaussians of every camera keep their gradient
        if not do_guidance:
            mask = (torch.rand(bs, P, 1, device=dev) < 0.1).float()
            gate = lambda x: x * mask + x.detach() * (1 - mask)
            means_in, scales_in, rots_in = gate(means), gate(scales), gate(rots)
        else:
            means_in, scales_in, rots_in = means, scales, rots
        if not do_reconstruction:
            means_in = means_in.detach()                                                          # 161
        # ---- screen-space points: one tensor per camera, like the reference's list of `screenspace_points`
        vsp = [v.requires_grad_() for v in torch.zeros(bs, P, 3, device=dev).unbind(0)]      # leaves: .grad is populated
        m2 = torch.stack(vsp, 0)
        opacity = pc.get_opacity
        shs = colors = None
        if override_color is None:
            shs = pc.get_features                                                                 # [P, (deg+1)^2, 3]
        else:
            colors = override_color
        cams_t = torch.cat([wv.reshape(bs, 16), full.reshape(bs, 16), cam, tx[:, None], ty[:, None]], dim=1).contiguous()
        # ---- background: inverted per camera with probability 1 - invert_bg_prob while training (65-70)
        if self.training:
            inv = np.random.rand(bs) > self.cfg.invert_bg_prob
        else:
            inv = np.zeros(bs, dtype=bool)
        bg = bg_color.detach().float().reshape(3)
        groups = [(np.nonzero(~inv)[0], bg), (np.nonzero(inv)[0], 1.0 - bg)]
        color = depth = alpha = radii = None
        for idx, bgc in groups:
            if len(idx) == 0:
                continue
            sel = torch.as_tensor(idx, device=dev)
            whole = len(idx) == bs
            pick = (lambda x: x) if whole else (lambda x: x[sel])
            meta = (H, W, int(pc.active_sh_degree), True, float(scaling_modifier), [float(x) for x in bgc.tolist()])
            c_, r_, d_, a_ = _RasterizeBatch.apply(pick(means_in), pick(m2), pick(scales_in), pick(rots_in), opacity, shs, colors,
                                                   pick(cams_t), meta)
            if whole:
                color, radii, depth, alpha = c_, r_, d_, a_
            else:
                if color is None:
                    color = torch.empty(bs, *c_.shape[1:], device=dev); depth = torch.empty(bs, *d_.shape[1:], device=dev)
                    alpha = torch.empty(bs, *a_.shape[1:], device=dev); radii = torch.empty(bs, P, dtype=r_.dtype, device=dev)
                color = color.index_copy(0, sel, c_); depth = depth.index_copy(0, sel, d_)
                alpha = alpha.index_copy(0, sel, a_); radii = radii.index_copy(0, sel, r_)
        return {"render": color.clamp(0, 1), "depth": depth, "mask": alpha, "viewspace_points": vsp, "radii": radii,
                "means3D": means_l, "scales": scales_l, "rotations": rots_l, "opacities": opacity}

    def batch_forward(self, batch: Dict) -> Dict:
        """batch: c2w [bs,4,4], fovy [bs], width, height, timestamps [bs] (optional), do_guidance, do_reconstruction
        (gaussian_batch_renderer_4d.py:11-50).  Returns the reference's output dict (72-109)."""
        c2w, fovy = batch["c2w"], batch["fovy"]
        bs = c2w.shape[0]
        H, W = int(batch["height"]), int(batch["width"])
        wv, full, cam, tx, ty = get_cam_info_gaussian(c2w, fovy, fovy, znear=0.1, zfar=100)
        r = self._render_cameras(wv, full, cam, tx, ty, H, W, batch.get("timestamps"), self.background_tensor,
                                 batch.get("scaling_modifier", 1.0), batch.get("override_color"),
                                 bool(batch.get("do_guidance", True)), bool(batch.get("do_reconstruction", True)))
        return {"comp_rgb": r["render"].permute(0, 2, 3, 1), "comp_depth": r["depth"].permute(0, 2, 3, 1),
                "comp_mask": r["mask"].permute(0, 2, 3, 1), "viewspace_points": r["viewspace_points"],
                "visibility_filter": list((r["radii"] > 0).unbind(0)), "radii": list(r["radii"].unbind(0)),
                "means3D": list(r["means3D"]), "scales": list(r["scales"]), "rotations": list(r["rotations"]),
                "opacities": [r["opacities"]] * bs}


@register("diff-gaussian-rasterizer-advanced-4d")
class DiffGaussian4D(BaseObject, Gaussian4DBatchRenderer):
    """threestudio `Rasterizer` plugin of the reference.  `configure(geometry, material, background)` as in
    threestudio/models/renderers/base.py (material / background are unused by gaussian splatting: line 39-41)."""

    @dataclass
    class Config(BaseObject.Config):
        radius: float = 1.0                                   # Renderer.Config (threestudio/models/renderers/base.py)
        invert_bg_prob: float = 1.0
        back_ground_color: Tuple[float, float, float] = (1, 1, 1)
        first_frame_trainable: bool = False

    cfg: Config

    def configure(self, geometry: Gaussian4DModel = None, material=None, background=None) -> None:
        if geometry is None:
            raise ValueError("DiffGaussian4D needs the 4D gaussian geometry")
        self.geometry, self.material, self.background = geometry, material, background
        self.background_tensor = torch.tensor(self.cfg.back_ground_color, dtype=torch.float32, device=geometry._xyz.device)
        self.training = False

    def train(self, mode: bool = True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    def forward(self, viewpoint_camera, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None, timestamps=None,
                **kwargs) -> Dict[str, Any]:
        """Single camera (lines 50-192).  viewpoint_camera: FoVx, FoVy, image_width, image_height, world_view_transform,
        full_proj_transform, camera_center (threestudio-3dgs `Camera`).  kwargs: batch_idx, do_guidance, do_reconstruction."""
        dev = self.geometry._xyz.device
        ts = None
        if timestamps is not None:
            ts = timestamps[kwargs["batch_idx"]].reshape(1)
        f32 = lambda t: torch.as_tensor(t, dtype=torch.float32, device=dev)
        tx = f32(math.tan(float(viewpoint_camera.FoVx) * 0.5)).reshape(1)
        ty = f32(math.tan(float(viewpoint_camera.FoVy) * 0.5)).reshape(1)
        r = self._render_cameras(f32(viewpoint_camera.world_view_transform).reshape(1, 4, 4),
                                 f32(viewpoint_camera.full_proj_transform).reshape(1, 4, 4),
                                 f32(viewpoint_camera.camera_center).reshape(1, 3), tx, ty, int(viewpoint_camera.image_height),
                                 int(viewpoint_camera.image_width), ts, bg_color, scaling_modifier, override_color,
                                 bool(kwargs.get("do_guidance", True)), bool(kwargs.get("do_reconstruction", True)))
        return {"render": r["render"][0], "depth": r["depth"][0], "mask": r["mask"][0], "viewspace_points": r["viewspace_points"][0],
                "visibility_filter": r["radii"][0] > 0, "radii": r["radii"][0], "means3D": r["means3D"][0],
                "scales": r["scales"][0], "rotations": r["rotations"][0], "opacities": r["opacities"]}

    __call__ = forward


def make_renderer(geometry: Gaussian4DModel, back_ground_color=(0.5, 0.5, 0.5), first_frame_trainable: bool = False,
                  invert_bg_prob: float = 1.0) -> DiffGaussian4D:
    """Convenience constructor (tests, bench): DiffGaussian4D with the refine_frame_16.yaml:96-100 renderer settings."""
    return DiffGaussian4D({"back_ground_color": tuple(back_ground_color), "first_frame_trainable": first_frame_trainable,
                           "invert_bg_prob": invert_bg_prob}, geometry=geometry)
