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

import contextlib
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

# ---- CUDA-graph capture.  An eager forward reads the pair count back and retries with a larger capacity on overflow; a
# captured one cannot.  It runs at a fixed capacity (the eager hint of its (P, H, W, cams) key times CAPTURE_SLACK) and
# leaves its counters on the device, where the caller checks the overflow flag after each replay.
CAPTURE_SLACK = 1.2
_pair_log: Optional[list] = None


def capture_capacity(hint: int) -> int:
    """Pair capacity of a captured forward whose eager hint is `hint`."""
    return int(hint * CAPTURE_SLACK)


def grow_hint(key, needed: int) -> int:
    """After a replay whose forward of `key` needed `needed` pairs and overflowed: the hint the eager path would have set."""
    _cap_hint[key] = max(_cap_hint.get(key, 0), int(needed * 1.08) + 1024, 1 << 16)
    return _cap_hint[key]


@contextlib.contextmanager
def collect_pair_counts():
    """Forwards captured inside this context append (key, counts) to the yielded list: counts is a device int64
    [total pairs, overflow flag] that every replay rewrites.  A captured forward outside it raises, since nobody would check
    whether its render was complete."""
    global _pair_log
    prev, _pair_log = _pair_log, []
    try:
        yield _pair_log
    finally:
        _pair_log = prev


def _captured_forward(lib, key, args, outs, dev):
    if _pair_log is None:
        raise L.A3DError("a rasterizer forward captured into a CUDA graph must run inside rasterizer.collect_pair_counts(), "
                         "whose owner checks the overflow flag after every replay")
    if key not in _cap_hint:
        raise L.A3DError(f"no eager forward of (P, H, W, cams) = {key} yet: the captured capacity is sized from one")
    P, H, W, ncam = key
    cap = capture_capacity(_cap_hint[key])
    nbytes = lib.a3d_raster_workspace_bytes(P, H, W, ncam, C.c_int64(cap))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    L.check(lib.a3d_raster_forward(C.byref(args), *[C.c_void_p(t.data_ptr()) for t in outs], C.c_void_p(ws.data_ptr()),
                                   C.c_size_t(nbytes), C.c_int64(cap), None, L.stream_ptr()))
    off = lib.a3d_raster_counters_offset(P, H, W, ncam, C.c_int64(cap))
    counters = ws[off:off + 8 * (ncam + 2)].view(torch.int64)
    _pair_log.append((key, counters[ncam:].clone()))     # a copy: the workspace is reused once the backward has run
    return cap, nbytes, ws, counters[:ncam]


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
        if torch.cuda.is_current_stream_capturing():
            args = _make_args(P, H, W, cams_t, means3D, scales, rotations, opacities, shs, colors_precomp, sh_degree, per_cam,
                              scale_modifier, bg)
            cap, nbytes, ws, ctx.num_rendered = _captured_forward(lib, key, args, (color, depth, alpha, radii), dev)
            ctx.save_for_backward(means3D, scales, rotations, opacities, shs, colors_precomp, cams_t, radii, ws)
            ctx.meta = (meta, cap, nbytes, P, ncam)
            ctx.m2_shape = None if means2D is None else tuple(means2D.shape)
            ctx.mark_non_differentiable(radii)
            return color, radii, depth, alpha
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


class PairBudgetExceeded(L.A3DError):
    """A multi-camera RGBA8 render needs more (tile, gaussian) pairs than its budget: render fewer cameras per call."""


class RGBA8Renderer:
    """Forward-only renders straight to RGBA8 (a3d_raster_forward_rgba8): no autograd, no float planes, no backward state.
    One workspace is reused across calls and grown when a call needs more.  The pair capacity of a call comes from the pairs
    per camera of the previous one; on overflow the call grows it and renders again, like the eager training forward."""

    def __init__(self, max_pairs: int = 1 << 27):
        self.max_pairs = max_pairs
        self.ws: Optional[torch.Tensor] = None
        self.pairs_per_cam = 0.0
        self.overflows = 0          # re-renders after an overflow, over the renderer's lifetime
        self.last_total = 0         # pairs of the last call
        self._counts: Optional[torch.Tensor] = None

    def render(self, cams_t, H: int, W: int, means3D, scales, rotations, opacities, shs, colors, sh_degree: int, per_cam: bool,
               bg, scale_modifier: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """rgba [cams, H, W, 4] uint8 (into `out` when given, which must be contiguous).  Arguments as `_make_args`;
        means3D / scales / rotations are [cams, P, *] with per_cam, else [P, *].  Synchronises the stream once per render."""
        lib = L.load()
        ncam, P, dev = cams_t.shape[0], means3D.shape[-2], means3D.device
        if out is None:
            out = torch.empty(ncam, H, W, 4, dtype=torch.uint8, device=dev)
        if out.shape != (ncam, H, W, 4) or out.dtype != torch.uint8 or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous uint8 [{ncam}, {H}, {W}, 4] tensor")
        if self._counts is None or self._counts.numel() < ncam + 2:
            self._counts = torch.empty(ncam + 2, dtype=torch.int64).pin_memory()
        counts = self._counts
        args = _make_args(P, H, W, cams_t, means3D, scales, rotations, opacities, shs, colors, sh_degree, per_cam, scale_modifier, bg)
        cap = max(int(self.pairs_per_cam * ncam * 1.08) + 1024, 1 << 16) if self.pairs_per_cam else max(1 << 16, 4 * P * ncam)
        cap = min(cap, self.max_pairs if ncam > 1 else 0x7FFFFFFF)
        while True:
            nbytes = lib.a3d_raster_forward_rgba8_workspace_bytes(P, H, W, ncam, C.c_int64(cap))
            if self.ws is None or self.ws.numel() < nbytes:
                self.ws = None                              # free the old one first
                self.ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            L.check(lib.a3d_raster_forward_rgba8(C.byref(args), C.c_void_p(out.data_ptr()), None, C.c_void_p(self.ws.data_ptr()),
                                                 C.c_size_t(self.ws.numel()), C.c_int64(cap), C.c_void_p(counts.data_ptr()),
                                                 L.stream_ptr()))
            torch.cuda.current_stream().synchronize()
            total = int(counts[ncam])
            if int(counts[ncam + 1]) == 0:
                break
            self.overflows += 1
            cap = int(total * 1.25) + 1024
            if cap > self.max_pairs and ncam > 1:
                raise PairBudgetExceeded(f"{ncam} cameras need {total} pairs, over the budget of {self.max_pairs}")
        self.last_total = total
        self.pairs_per_cam = total / ncam
        return out


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
