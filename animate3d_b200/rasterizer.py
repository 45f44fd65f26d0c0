"""Drop-in for the `diff_gaussian_rasterization` Python API the reference imports at
custom/threestudio-animate3d/renderer/diff_gaussian_rasterizer_advanced_4d.py:8-11 and calls at 102-117, 161-170:

    settings = GaussianRasterizationSettings(image_height, image_width, tanfovx, tanfovy, bg, scale_modifier, viewmatrix,
                                             projmatrix, sh_degree, campos, prefiltered, debug)
    color, radii, depth, alpha = GaussianRasterizer(settings)(means3D, means2D, opacities, shs, colors_precomp, scales,
                                                               rotations, cov3D_precomp)

plus `rasterize_batch`, which renders ALL cameras of a batch (the reference's Python loop over cameras,
gaussian_batch_renderer_4d.py:27) through one launch per stage.  Forward and backward run in liba3d.so; torch provides
memory, the stream and the autograd tape.  Under torch.use_deterministic_algorithms(True) the backward sums every gradient
in a fixed order (bit-reproducible), at the cost of 40 B of scratch per (tile, gaussian) pair."""
from __future__ import annotations

import ctypes as C
from typing import List, NamedTuple, Optional, Sequence

import torch

from . import _lib as L


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


_cap_hint = {}
last_num_rendered = 0      # (tile, gaussian) pairs of the most recent forward (diagnostics / bench roofline)
last_backward_scratch_bytes = 0   # deterministic-backward scratch of the most recent backward (0 with the flag off)


def _pack_cams(settings: Sequence[GaussianRasterizationSettings], device) -> torch.Tensor:
    """[num_cams, 37] float32 rows laid out like a3d_raster_cam (viewmatrix 16, projmatrix 16, campos 3, tanfovx, tanfovy)."""
    rows = []
    for s in settings:
        rows.append(torch.cat([s.viewmatrix.reshape(16).float().to(device), s.projmatrix.reshape(16).float().to(device),
                               s.campos.reshape(3).float().to(device),
                               torch.tensor([s.tanfovx, s.tanfovy], dtype=torch.float32, device=device)]))
    return torch.stack(rows).contiguous()


def _make_args(P, H, W, cams_t, means3D, scales, rotations, opacities, shs, colors, sh_degree, per_cam, scale_modifier, bg):
    a = L.RasterArgs()
    a.P, a.H, a.W, a.num_cams = P, H, W, cams_t.shape[0]
    a.cams = cams_t.data_ptr()
    a.means3D, a.scales, a.rotations, a.opacities = means3D.data_ptr(), scales.data_ptr(), rotations.data_ptr(), opacities.data_ptr()
    a.shs = L.ptr(shs)
    a.colors_precomp = L.ptr(colors)
    a.sh_degree = sh_degree
    a.sh_coeffs = shs.shape[1] if shs is not None else 0
    a.per_cam_geometry = int(per_cam)
    a.scale_modifier = scale_modifier
    for i in range(3):
        a.bg[i] = float(bg[i])
    return a


class _RasterizeBatch(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, scales, rotations, opacities, shs, colors_precomp, cams_t, meta):
        lib = L.load()
        H, W, sh_degree, per_cam, scale_modifier, bg = meta
        f = lambda t: None if t is None else t.detach().contiguous().float()
        means3D, scales, rotations, opacities, shs, colors_precomp = map(f, (means3D, scales, rotations, opacities, shs, colors_precomp))
        dev = means3D.device
        ncam = cams_t.shape[0]
        P = means3D.shape[-2]
        color = torch.empty(ncam, 3, H, W, device=dev)
        depth = torch.empty(ncam, 1, H, W, device=dev)
        alpha = torch.empty(ncam, 1, H, W, device=dev)
        radii = torch.empty(ncam, P, dtype=torch.int32, device=dev)
        key = (P, H, W, ncam)
        cap = _cap_hint.get(key, max(1 << 16, 4 * P * ncam))
        counts = torch.empty(ncam + 2, dtype=torch.int64).pin_memory()
        while True:
            nbytes = lib.a3d_raster_workspace_bytes(P, H, W, ncam, C.c_int64(cap))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            args = _make_args(P, H, W, cams_t, means3D, scales, rotations, opacities, shs, colors_precomp, sh_degree, per_cam,
                              scale_modifier, bg)
            L.check(lib.a3d_raster_forward(C.byref(args), C.c_void_p(color.data_ptr()), C.c_void_p(depth.data_ptr()),
                                           C.c_void_p(alpha.data_ptr()), C.c_void_p(radii.data_ptr()), C.c_void_p(ws.data_ptr()),
                                           C.c_size_t(nbytes), C.c_int64(cap), C.c_void_p(counts.data_ptr()), L.stream_ptr()))
            torch.cuda.current_stream().synchronize()      # one sync per BATCH (the reference syncs per camera)
            total = int(counts[ncam])
            if int(counts[ncam + 1]) == 0:
                break
            cap = int(total * 1.25) + 1024                 # overflowed: grow and redo
        global last_num_rendered
        last_num_rendered = total
        _cap_hint[key] = max(int(total * 1.08) + 1024, 1 << 16)   # the radix sort runs over the capacity: keep the slack small
        ctx.save_for_backward(means3D, scales, rotations, opacities, shs, colors_precomp, cams_t, radii, ws)
        ctx.meta = (meta, cap, nbytes, P, ncam)
        ctx.m2_shape = None if means2D is None else tuple(means2D.shape)
        ctx.num_rendered = counts[:ncam].clone()
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, g_color, g_radii, g_depth, g_alpha):
        lib = L.load()
        means3D, scales, rotations, opacities, shs, colors_precomp, cams_t, radii, ws = ctx.saved_tensors
        (H, W, sh_degree, per_cam, scale_modifier, bg), cap, nbytes, P, ncam = ctx.meta
        dev = means3D.device
        g_color = g_color.contiguous().float()
        g_depth = None if g_depth is None else g_depth.contiguous().float()
        g_alpha = None if g_alpha is None else g_alpha.contiguous().float()
        dm = torch.zeros_like(means3D); ds = torch.zeros_like(scales); dr = torch.zeros_like(rotations)
        do = torch.zeros_like(opacities)
        dc = torch.zeros_like(colors_precomp) if colors_precomp is not None else None
        dsh = torch.zeros_like(shs) if shs is not None else None
        dm2 = torch.zeros(ncam, P, 3, device=dev)
        args = _make_args(P, H, W, cams_t, means3D, scales, rotations, opacities, shs, colors_precomp, sh_degree, per_cam,
                          scale_modifier, bg)
        args.deterministic = L.deterministic()
        sbytes = lib.a3d_raster_backward_scratch_bytes(C.byref(args), C.c_int64(cap))
        scratch = L.scratch(sbytes, dev)
        global last_backward_scratch_bytes
        last_backward_scratch_bytes = sbytes
        L.check(lib.a3d_raster_backward(C.byref(args), C.c_void_p(g_color.data_ptr()), C.c_void_p(L.ptr(g_depth)),
                                        C.c_void_p(L.ptr(g_alpha)), C.c_void_p(radii.data_ptr()), C.c_void_p(ws.data_ptr()),
                                        C.c_size_t(nbytes), C.c_int64(cap), C.c_void_p(dm.data_ptr()), C.c_void_p(ds.data_ptr()),
                                        C.c_void_p(dr.data_ptr()), C.c_void_p(do.data_ptr()), C.c_void_p(L.ptr(dc)),
                                        C.c_void_p(L.ptr(dsh)), C.c_void_p(dm2.data_ptr()), C.c_void_p(L.ptr(scratch)),
                                        C.c_size_t(sbytes), L.stream_ptr()))
        g_m2 = None if ctx.m2_shape is None else dm2.reshape(ctx.m2_shape)   # `viewspace_points` gradient, NDC units
        return dm, g_m2, ds, dr, do, dsh, dc, None, None


def rasterize_batch(means3D, scales, rotations, opacities, shs, colors_precomp, settings: Sequence[GaussianRasterizationSettings],
                    per_cam_geometry: bool = False, means2D: Optional[torch.Tensor] = None):
    """Render every camera in `settings` at once.  means3D/scales/rotations are [P,*] (shared) or [num_cams,P,*] when
    per_cam_geometry (one deformed gaussian set per camera, as in the 4D renderer).  Returns color [cams,3,H,W],
    radii [cams,P], depth [cams,1,H,W], alpha [cams,1,H,W]."""
    s0 = settings[0]
    dev = means3D.device
    for s in settings:
        if (s.image_height, s.image_width, s.sh_degree, s.scale_modifier) != (s0.image_height, s0.image_width, s0.sh_degree, s0.scale_modifier):
            raise ValueError("all cameras of a batch must share resolution / sh_degree / scale_modifier")
    cams_t = _pack_cams(settings, dev)
    meta = (int(s0.image_height), int(s0.image_width), int(s0.sh_degree), bool(per_cam_geometry), float(s0.scale_modifier),
            [float(x) for x in s0.bg.reshape(3).tolist()])
    return _RasterizeBatch.apply(means3D, means2D, scales, rotations, opacities, shs, colors_precomp, cams_t, meta)


class GaussianRasterizer(torch.nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        if (shs is None) == (colors_precomp is None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        if cov3D_precomp is not None or scales is None or rotations is None:
            raise NotImplementedError("cov3D_precomp is never passed by the reference (diff_gaussian_rasterizer_advanced_4d.py:139)")
        m2 = means2D[None] if means2D is not None else None
        color, radii, depth, alpha = rasterize_batch(means3D, scales, rotations, opacities, shs, colors_precomp,
                                                     [self.raster_settings], means2D=m2)
        return color[0], radii[0], depth[0], alpha[0]
