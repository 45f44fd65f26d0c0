"""Host-side mirror of the reference's 4D gaussian geometry for the hot path: `Gaussian4DModel.interpolate_ms_features`,
`get_xyz`, `get_scaling`, `get_rotation` (custom/threestudio-animate3d/geometry/gaussian_4d.py:450-548) evaluated for ALL
frames of a batch in one CUDA launch (forward and backward in liba3d.so), de-duplicated across the views of a frame.

State (same tensors the reference keeps): static `_xyz [P,3]`, `_scaling [P,3]` (log), `_rotation [P,4]`, `_opacity`,
`_features_dc`; learnable k-planes `grids[scale][plane] : [1, 16, H, W]` (gaussian_4d.py:101-117, 151-174) and the three
bias-free MLPs delta_xyz / delta_rot / delta_scaling (119-147; VanillaMLP, threestudio/models/networks.py:214-251).
The global rotation/translation branch (`use_global_trans`, 129-142, 499-511, 525-539; on in refine_frame_16.yaml:56) runs as
(1) a3d_deform_featmean: per-frame mean k-planes feature, (2) the two 32-wide global MLPs + Euler matrix on [T, 32] in
torch (autograd), (3) the fused deformation launch with the rotated base quaternions; see `deform_all`.
The mean feature is always summed in a fixed order; the backward follows torch.use_deterministic_algorithms (fixed-order
reductions and a plane-gradient gather instead of float atomics, with 768 B of scratch per (frame, gaussian))."""
from __future__ import annotations

import ctypes as C
import itertools
import math
from typing import List, Optional, Sequence

import torch

from . import _lib as L


class DeformArgs(C.Structure):
    _fields_ = [("P", C.c_int), ("T", C.c_int), ("xyz", C.c_void_p), ("scaling", C.c_void_p), ("rotation", C.c_void_p),
                ("times", C.c_void_p), ("num_scales", C.c_int), ("channels", C.c_int), ("hidden", C.c_int),
                ("planes", C.c_void_p * 12), ("plane_h", C.c_int * 12), ("plane_w", C.c_int * 12),
                ("w1", C.c_void_p * 3), ("w2", C.c_void_p * 3), ("deform_scale", C.c_int),
                ("grad_planes", C.c_void_p * 12), ("grad_w1", C.c_void_p * 3), ("grad_w2", C.c_void_p * 3),
                ("rot_base", C.c_void_p), ("grad_rot_base", C.c_void_p), ("grad_featmean", C.c_void_p), ("deterministic", C.c_int)]


def _args(xyz, scaling, rotation, times, planes, w1s, w2s, deform_scale, gplanes=None, gw1=None, gw2=None):
    a = DeformArgs()
    a.P, a.T = xyz.shape[0], times.shape[0]
    a.xyz, a.scaling, a.rotation, a.times = xyz.data_ptr(), scaling.data_ptr(), rotation.data_ptr(), times.data_ptr()
    a.num_scales, a.channels, a.hidden = len(planes) // 6, planes[0].shape[-3], w1s[0].shape[0]
    for i, pl in enumerate(planes):
        a.planes[i] = pl.data_ptr()
        a.plane_h[i], a.plane_w[i] = pl.shape[-2], pl.shape[-1]
        if gplanes is not None:
            a.grad_planes[i] = gplanes[i].data_ptr()
    for m in range(3):
        a.w1[m], a.w2[m] = w1s[m].data_ptr(), w2s[m].data_ptr()
        if gw1 is not None:
            a.grad_w1[m], a.grad_w2[m] = gw1[m].data_ptr(), gw2[m].data_ptr()
    a.deform_scale = int(deform_scale)
    return a


def _plane_grad_scratch(plane: torch.Tensor) -> torch.Tensor:
    """Channel-last accumulation buffer [H, W, C] for the gradient of a [1, C, H, W] plane (a3d_deform_backward writes the C
    channels of a texel as contiguous vector reductions)."""
    _, c, h, w = plane.shape
    return torch.zeros(h, w, c, device=plane.device, dtype=torch.float32)


def _plane_grad_out(scratch: torch.Tensor, plane: torch.Tensor) -> torch.Tensor:
    return scratch.permute(2, 0, 1).reshape(plane.shape).contiguous()


def _backward(lib, a, g_means, g_scales, g_rots, device):
    """a3d_deform_backward; with torch's deterministic flag set, the fixed-order path and its scratch."""
    a.deterministic = L.deterministic()
    nbytes = lib.a3d_deform_backward_scratch_bytes(C.byref(a))
    scratch = L.scratch(nbytes, device)
    L.check(lib.a3d_deform_backward(C.byref(a), C.c_void_p(L.ptr(g_means)), C.c_void_p(L.ptr(g_scales)), C.c_void_p(L.ptr(g_rots)),
                                    C.c_void_p(L.ptr(scratch)), C.c_size_t(nbytes), L.stream_ptr()))


class _FeatMean(torch.autograd.Function):
    """hidden_feats.mean(0) of every frame: [T, 32]; backward folds d/d mean into the plane gradients."""

    @staticmethod
    def forward(ctx, xyz, scaling, rotation, times, n_planes, *params):
        lib = L.load()
        planes = [p.detach().contiguous().float() for p in params[:n_planes]]
        w1s = [p.detach().contiguous().float() for p in params[n_planes:n_planes + 3]]
        w2s = [p.detach().contiguous().float() for p in params[n_planes + 3:n_planes + 6]]
        xyz, scaling, rotation, times = [t.detach().contiguous().float() for t in (xyz, scaling, rotation, times)]
        a = _args(xyz, scaling, rotation, times, planes, w1s, w2s, True)
        out = torch.empty(times.shape[0], a.num_scales * a.channels, device=xyz.device)
        L.check(lib.a3d_deform_featmean(C.byref(a), C.c_void_p(out.data_ptr()), L.stream_ptr()))
        ctx.save_for_backward(xyz, scaling, rotation, times, *planes, *w1s, *w2s)
        ctx.n_planes = n_planes
        return out

    @staticmethod
    def backward(ctx, g_mean):
        lib = L.load()
        n_planes = ctx.n_planes
        xyz, scaling, rotation, times, *rest = ctx.saved_tensors
        planes, w1s, w2s = rest[:n_planes], rest[n_planes:n_planes + 3], rest[n_planes + 3:]
        gp = [_plane_grad_scratch(p) for p in planes]
        g1 = [torch.zeros_like(w) for w in w1s]
        g2 = [torch.zeros_like(w) for w in w2s]
        g_mean = g_mean.contiguous().float()
        a = _args(xyz, scaling, rotation, times, planes, w1s, w2s, True, gp, g1, g2)
        a.grad_featmean = g_mean.data_ptr()
        _backward(lib, a, None, None, None, xyz.device)
        return (None, None, None, None, None, *[_plane_grad_out(g, p) for g, p in zip(gp, planes)], None, None, None, None, None, None)


class _Deform(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, scaling, rotation, times, deform_scale, n_planes, rot_base, *params):
        lib = L.load()
        planes = [p.detach().contiguous().float() for p in params[:n_planes]]
        w1s = [p.detach().contiguous().float() for p in params[n_planes:n_planes + 3]]
        w2s = [p.detach().contiguous().float() for p in params[n_planes + 3:n_planes + 6]]
        xyz, scaling, rotation, times = [t.detach().contiguous().float() for t in (xyz, scaling, rotation, times)]
        P, T = xyz.shape[0], times.shape[0]
        means = torch.empty(T, P, 3, device=xyz.device)
        scales = torch.empty(T, P, 3, device=xyz.device)
        rots = torch.empty(T, P, 4, device=xyz.device)
        a = _args(xyz, scaling, rotation, times, planes, w1s, w2s, deform_scale)
        rb = None
        if rot_base is not None:
            rb = rot_base.detach().contiguous().float()
            assert rb.shape == (T, P, 4)
            a.rot_base = rb.data_ptr()
        L.check(lib.a3d_deform_forward(C.byref(a), C.c_void_p(means.data_ptr()), C.c_void_p(scales.data_ptr()),
                                       C.c_void_p(rots.data_ptr()), L.stream_ptr()))
        ctx.save_for_backward(xyz, scaling, rotation, times, *planes, *w1s, *w2s)
        ctx.rot_base = rb
        ctx.meta = (deform_scale, n_planes)
        return means, scales, rots

    @staticmethod
    def backward(ctx, g_means, g_scales, g_rots):
        lib = L.load()
        deform_scale, n_planes = ctx.meta
        xyz, scaling, rotation, times, *rest = ctx.saved_tensors
        planes, w1s, w2s = rest[:n_planes], rest[n_planes:n_planes + 3], rest[n_planes + 3:]
        gp = [_plane_grad_scratch(p) for p in planes]
        g1 = [torch.zeros_like(w) for w in w1s]
        g2 = [torch.zeros_like(w) for w in w2s]
        f = lambda t: None if t is None else t.contiguous().float()
        g_means, g_scales, g_rots = f(g_means), f(g_scales), f(g_rots)
        a = _args(xyz, scaling, rotation, times, planes, w1s, w2s, deform_scale, gp, g1, g2)
        g_rb = None
        if ctx.rot_base is not None:
            a.rot_base = ctx.rot_base.data_ptr()
            g_rb = torch.zeros_like(ctx.rot_base)
            a.grad_rot_base = g_rb.data_ptr()
        _backward(lib, a, g_means, g_scales, g_rots, xyz.device)
        return (None, None, None, None, None, None, g_rb, *[_plane_grad_out(g, p) for g, p in zip(gp, planes)], *g1, *g2)


def quat_to_matrix(q: torch.Tensor) -> torch.Tensor:
    """build_rotation (geometry/utils.py:33-62): [..., 4] (r,x,y,z), normalised first -> [..., 3, 3]."""
    q = q / q.norm(dim=-1, keepdim=True)
    r, x, y, z = q.unbind(-1)
    m = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1)
    return m.reshape(*q.shape[:-1], 3, 3)


def matrix_to_quat(m: torch.Tensor) -> torch.Tensor:
    """extract_rotation_torch (geometry/utils.py:73-133): same branch order and strict comparisons, batched over any
    leading dims; unselected branches get a harmless square-root argument so that no NaN reaches autograd."""
    d0, d1, d2 = m[..., 0, 0], m[..., 1, 1], m[..., 2, 2]
    tr = d0 + d1 + d2
    c1 = tr > 0
    c2 = (~c1) & (d0 > d1) & (d0 > d2)
    c3 = (~c1) & (~c2) & (d1 > d2)
    c4 = ~(c1 | c2 | c3)
    one = torch.ones_like(tr)
    t = [torch.sqrt(torch.where(c, a, one)) * 2 for c, a in
         ((c1, tr + 1.0), (c2, 1.0 + d0 - d1 - d2), (c3, 1.0 + d1 - d0 - d2), (c4, 1.0 + d2 - d0 - d1))]
    a21, a02, a10 = m[..., 2, 1] - m[..., 1, 2], m[..., 0, 2] - m[..., 2, 0], m[..., 1, 0] - m[..., 0, 1]
    s01, s02, s12 = m[..., 0, 1] + m[..., 1, 0], m[..., 0, 2] + m[..., 2, 0], m[..., 1, 2] + m[..., 2, 1]
    cand = ((0.25 * t[0], a21 / t[0], a02 / t[0], a10 / t[0]),
            (a21 / t[1], 0.25 * t[1], s01 / t[1], s02 / t[1]),
            (a02 / t[2], s01 / t[2], 0.25 * t[2], s12 / t[2]),
            (a10 / t[3], s02 / t[3], s12 / t[3], 0.25 * t[3]))
    comps = [torch.where(c1, cand[0][k], torch.where(c2, cand[1][k], torch.where(c3, cand[2][k], cand[3][k]))) for k in range(4)]
    q = torch.stack(comps, dim=-1)
    return q / q.norm(p=2, dim=-1, keepdim=True)


def euler_to_matrix(angles: torch.Tensor) -> torch.Tensor:
    """euler_angles_to_rotation_matrix (geometry/utils.py:135-167), batched: [..., 3] (roll, pitch, yaw) -> Rz Ry Rx."""
    cr, sr = torch.cos(angles[..., 0]), torch.sin(angles[..., 0])
    cp, sp = torch.cos(angles[..., 1]), torch.sin(angles[..., 1])
    cy, sy = torch.cos(angles[..., 2]), torch.sin(angles[..., 2])
    z, o = torch.zeros_like(cr), torch.ones_like(cr)
    shp = (*angles.shape[:-1], 3, 3)
    rx = torch.stack([o, z, z, z, cr, -sr, z, sr, cr], dim=-1).reshape(shp)
    ry = torch.stack([cp, z, sp, z, o, z, -sp, z, cp], dim=-1).reshape(shp)
    rz = torch.stack([cy, -sy, z, sy, cy, z, z, z, o], dim=-1).reshape(shp)
    return rz @ (ry @ rx)


class Gaussian4DModel(torch.nn.Module):
    """Registered in the reference as "gaussian-splatting-4d" (gaussian_4d.py:67)."""

    def __init__(self, xyz, scaling, rotation, opacity, features_dc, grid_size=((50, 50, 50, 8), (100, 100, 100, 16)),
                 n_grid_dims: int = 16, n_neurons: int = 32, seed: int = 0, device="cuda", use_global_trans: bool = False,
                 features_rest: Optional[torch.Tensor] = None, sh_degree: int = 0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        features_dc = features_dc.reshape(features_dc.shape[0], 1, 3)
        if features_rest is None:
            features_rest = torch.zeros(features_dc.shape[0], 0, 3)
        if features_rest.shape[1] != (sh_degree + 1) ** 2 - 1:
            raise ValueError(f"features_rest holds {features_rest.shape[1]} coefficients, sh_degree {sh_degree} needs "
                             f"{(sh_degree + 1) ** 2 - 1}")
        for name, t in (("_xyz", xyz), ("_scaling", scaling), ("_rotation", rotation), ("_opacity", opacity),
                        ("_features_dc", features_dc), ("_features_rest", features_rest)):
            self.register_buffer(name, t.float().to(device))      # frozen after load_ply (gaussian_4d.py:262-297)
        self.max_sh_degree = sh_degree
        self.grids = torch.nn.ModuleList()
        for reso in grid_size:
            planes = torch.nn.ParameterList()
            for comb in itertools.combinations(range(4), 2):
                shape = [1, n_grid_dims] + [reso[cc] for cc in comb[::-1]]
                init = torch.ones(shape) if 3 in comb else torch.rand(shape, generator=g) * 0.4 + 0.1     # 168-171
                planes.append(torch.nn.Parameter(init.to(device)))
            self.grids.append(planes)
        feat = n_grid_dims * len(grid_size)

        def mlp(out):   # VanillaMLP: Linear(no bias) - ReLU - Linear(no bias); last layer zero-init (145-147)
            w1 = torch.nn.Parameter((torch.rand(n_neurons, feat, generator=g) * 2 - 1).div_(feat ** 0.5).to(device))
            w2 = torch.nn.Parameter(torch.zeros(out, n_neurons, device=device))
            return torch.nn.ParameterList([w1, w2])
        self.delta_xyz_network, self.delta_rot_network, self.delta_scaling_network = mlp(3), mlp(4), mlp(3)
        self.use_global_trans = use_global_trans
        if use_global_trans:   # gaussian_4d.py:129-142, zero-init last layers -> identity rotation / zero translation at start
            self.global_rot_network, self.global_trans_network = mlp(3), mlp(3)
        self.active_sh_degree = sh_degree      # load_ply sets active_sh_degree = max_sh_degree (gaussian_4d.py:306)

    @classmethod
    def from_ply(cls, path: str, rot_x_degree: float = 0.0, rot_z_degree: float = 0.0, scale_factor: float = 1.0,
                 sh_degree: int = 0, **kw):
        """`load_ply` (gaussian_4d.py:177-306): static gaussians from a 3DGS PLY with the load-time rotate / scale."""
        from .io import load_gaussian_ply
        g = load_gaussian_ply(path, rot_x_degree, rot_z_degree, scale_factor, max_sh_degree=sh_degree)
        t = lambda k: torch.from_numpy(g[k])
        return cls(t("_xyz"), t("_scaling"), t("_rotation"), t("_opacity"), t("_features_dc"), features_rest=t("_features_rest"),
                   sh_degree=sh_degree, **kw)

    @property
    def get_features(self):
        """GaussianBaseModel.get_features: cat(features_dc, features_rest) -> [P, (deg+1)^2, 3]."""
        return torch.cat([self._features_dc, self._features_rest], dim=1)

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    def deform_all(self, timestamps: torch.Tensor, deform_scale: bool = True):
        """(means3D [T,P,3], scales [T,P,3], rotations [T,P,4]) for every timestamp in one launch.  Frames with
        timestamp == -1 keep the static gaussians when `first_frame_trainable` is off in the caller."""
        planes = [p for pl in self.grids for p in pl]
        nets = (self.delta_xyz_network, self.delta_rot_network, self.delta_scaling_network)
        params = planes + [n[0] for n in nets] + [n[1] for n in nets]
        times = timestamps.float().to(self._xyz.device)
        if not self.use_global_trans:
            return _Deform.apply(self._xyz, self._scaling, self._rotation, times, deform_scale, len(planes), None, *params)
        # use_global_trans (gaussian_4d.py:499-511, 525-539): per-frame rigid motion predicted from the mean feature
        hg = _FeatMean.apply(self._xyz, self._scaling, self._rotation, times, len(planes), *params)            # [T, 32]
        mlp = lambda net, x: torch.nn.functional.linear(torch.relu(torch.nn.functional.linear(x, net[0])), net[1])
        ang = torch.sigmoid(mlp(self.global_rot_network, hg)) * (2 * math.pi) - math.pi                          # [T, 3]
        trans = torch.sigmoid(mlp(self.global_trans_network, hg)) * 2 - 1                                        # [T, 3]
        rmat = euler_to_matrix(ang)                                                                              # [T, 3, 3]
        rot_base = matrix_to_quat(rmat[:, None] @ quat_to_matrix(self._rotation)[None])                          # [T, P, 4]
        means, scales, rots = _Deform.apply(self._xyz, self._scaling, self._rotation, times, deform_scale, len(planes), rot_base,
                                            *params)
        # means = R xyz + trans + delta = (xyz + delta) + (R xyz - xyz) + trans
        means = means + (torch.einsum("tij,pj->tpi", rmat, self._xyz) - self._xyz[None]) + trans[:, None]
        return means, scales, rots

    def deform_frames(self, timestamps: torch.Tensor, deform_scale: bool = True, first_frame_trainable: bool = False):
        """`deform_all` with the condition-frame rule of the reference renderer (diff_gaussian_rasterizer_advanced_4d.py:77-83):
        unless `first_frame_trainable`, frames with timestamp == -1 are the static gaussians (`_xyz`, exp(`_scaling`),
        normalised `_rotation`).  The renderer and the trajectory export both go through here."""
        means, scales, rots = self.deform_all(timestamps, deform_scale=deform_scale)
        if not first_frame_trainable:
            first = timestamps.reshape(-1).float().to(self._xyz.device) == -1
            if bool(first.any()):
                keep = first[:, None, None]
                means = torch.where(keep, self._xyz[None], means)
                scales = torch.where(keep, torch.exp(self._scaling)[None], scales)
                rots = torch.where(keep, torch.nn.functional.normalize(self._rotation, dim=-1)[None], rots)
        return means, scales, rots
