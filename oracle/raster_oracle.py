"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the differentiable 3D-Gaussian rasterizer the
reference calls at custom/threestudio-animate3d/renderer/diff_gaussian_rasterizer_advanced_4d.py:161-170.

The arithmetic lives in a third-party package that is NOT in /root/reference and is installed unpinned
(`ashawkey/diff-gaussian-rasterization` @ HEAD, docs/install.md:18-20).  This file restates the published algorithm of
graphdeco-inria/diff-gaussian-rasterization + ashawkey's depth/alpha fork as recorded in SURVEY.md Appendix C
(preprocess C.1, binning C.2, render C.3; backward = torch autograd through this restatement).  PARITY UNPINNED: no
reference test, golden vector or buildable source exists for it; where upstream is ambiguous (floating-point operation
order inside preprocess) the order written here IS the contract the CUDA kernels are tested against bit-for-bit.

Everything is fp32 torch on CPU with one IEEE operation per python operation (eager mode never fuses a*b+c), which is what
makes radii / tile rectangles / sort keys reproducible bit-for-bit by CUDA code written with __fmul_rn/__fadd_rn.
Camera conventions follow threestudio/utils/ops.py:305-359 (row-vector matrices: p_view = [x y z 1] @ viewmatrix).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

BLOCK = 16
SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


# ------------------------------------------------------------------------------------------------ cameras
def get_projection_matrix(znear: float, zfar: float, fovx: float, fovy: float) -> torch.Tensor:
    """threestudio/utils/ops.py:314-334 get_projection_matrix_gaussian."""
    ty, tx = math.tan(fovy / 2), math.tan(fovx / 2)
    top, right = ty * znear, tx * znear
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def get_cam_info_gaussian(c2w: torch.Tensor, fovx: float, fovy: float, znear: float = 0.1, zfar: float = 100.0):
    """threestudio/utils/ops.py:344-359 -> (world_view_transform, full_proj_transform, camera_center), row-vector form."""
    flip = torch.eye(4)
    flip[1, 1] = -1
    flip[2, 2] = -1
    c2w = c2w.float() @ flip
    wv = torch.inverse(c2w).transpose(0, 1).float()
    proj = get_projection_matrix(znear, zfar, fovx, fovy).transpose(0, 1)
    full = wv @ proj
    cam = wv.inverse()[3, :3]
    return wv.contiguous(), full.contiguous(), cam.contiguous()


# ------------------------------------------------------------------------------------------------ preprocess (C.1)
@dataclass
class Preprocessed:
    depth: torch.Tensor        # [P]
    radii: torch.Tensor        # [P] int32
    xy: torch.Tensor           # [P,2] pixel centre
    conic_opacity: torch.Tensor  # [P,4]
    rgb: torch.Tensor          # [P,3]
    rect_min: torch.Tensor     # [P,2] int32 (x,y)
    rect_max: torch.Tensor     # [P,2] int32
    tiles_touched: torch.Tensor  # [P] int32


def quat_to_rot(q: torch.Tensor) -> torch.Tensor:
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([
        1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - r * z), 2.0 * (x * z + r * y),
        2.0 * (x * y + r * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - r * x),
        2.0 * (x * z - r * y), 2.0 * (y * z + r * x), 1.0 - 2.0 * (x * x + y * y)], dim=-1)
    return R.reshape(-1, 3, 3)


def cov3d_from_scale_rot(scales: torch.Tensor, rotations: torch.Tensor, mod: float) -> torch.Tensor:
    """Sigma = R diag(s^2) R^T, returned as the 6 upper-triangular entries (xx, xy, xz, yy, yz, zz).
    The quaternion is NOT renormalised (the Python side does it: gaussian_4d.py:517)."""
    R = quat_to_rot(rotations)
    s = scales * mod
    M = R * s[:, None, :]                       # M[i][k] = R[i][k] * s[k]
    def dot(i, j):
        return (M[:, i, 0] * M[:, j, 0] + M[:, i, 1] * M[:, j, 1]) + M[:, i, 2] * M[:, j, 2]
    return torch.stack([dot(0, 0), dot(0, 1), dot(0, 2), dot(1, 1), dot(1, 2), dot(2, 2)], dim=-1)


def eval_sh(deg: int, sh: torch.Tensor, dirs: torch.Tensor) -> torch.Tensor:
    """SH (degree <= 3) -> RGB before the +0.5 / clamp; sh [P, K, 3], dirs [P,3] normalised."""
    res = SH_C0 * sh[:, 0]
    if deg > 0:
        x, y, z = dirs[:, 0:1], dirs[:, 1:2], dirs[:, 2:3]
        res = res - SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            res = (res + SH_C2[0] * xy * sh[:, 4] + SH_C2[1] * yz * sh[:, 5] + SH_C2[2] * (2.0 * zz - xx - yy) * sh[:, 6]
                   + SH_C2[3] * xz * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8])
            if deg > 2:
                res = (res + SH_C3[0] * y * (3.0 * xx - yy) * sh[:, 9] + SH_C3[1] * xy * z * sh[:, 10]
                       + SH_C3[2] * y * (4.0 * zz - xx - yy) * sh[:, 11]
                       + SH_C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy) * sh[:, 12]
                       + SH_C3[4] * x * (4.0 * zz - xx - yy) * sh[:, 13] + SH_C3[5] * z * (xx - yy) * sh[:, 14]
                       + SH_C3[6] * x * (xx - 3.0 * yy) * sh[:, 15])
    return res


def preprocess(means3D, scales, rotations, opacities, shs, colors_precomp, sh_degree, viewmatrix, projmatrix, campos,
               tanfovx, tanfovy, H, W, scale_modifier=1.0) -> Preprocessed:
    f32 = torch.float32
    vm = viewmatrix.reshape(16).to(f32)
    pm = projmatrix.reshape(16).to(f32)
    px, py, pz = means3D[:, 0], means3D[:, 1], means3D[:, 2]

    def tp(m, col):   # ((m[c]*x + m[4+c]*y) + m[8+c]*z) + m[12+c]
        return ((m[col] * px + m[4 + col] * py) + m[8 + col] * pz) + m[12 + col]
    tx, ty, tz = tp(vm, 0), tp(vm, 1), tp(vm, 2)
    hx, hy, hw = tp(pm, 0), tp(pm, 1), tp(pm, 3)
    in_front = tz > 0.2
    p_w = 1.0 / (hw + 1e-7)
    projx, projy = hx * p_w, hy * p_w

    cov3 = cov3d_from_scale_rot(scales, rotations, scale_modifier)
    # the C ABI carries tanfov as float32; all derived constants are float32 operations
    tfx = torch.tensor(float(tanfovx), dtype=f32)
    tfy = torch.tensor(float(tanfovy), dtype=f32)
    focal_x = W / (2.0 * tfx)
    focal_y = H / (2.0 * tfy)
    limx, limy = 1.3 * tfx, 1.3 * tfy
    tzs = torch.where(in_front, tz, torch.ones_like(tz))     # keep culled lanes finite
    txc = torch.minimum(limx, torch.maximum(-limx, tx / tzs)) * tzs
    tyc = torch.minimum(limy, torch.maximum(-limy, ty / tzs)) * tzs
    j00 = focal_x / tzs
    j02 = -(focal_x * txc) / (tzs * tzs)
    j11 = focal_y / tzs
    j12 = -(focal_y * tyc) / (tzs * tzs)
    # M = J * R_view   (rows 0,1 only), R_view[i][k] = vm[4*k + i]
    def rv(i, k):
        return vm[4 * k + i]
    m0 = [j00 * rv(0, k) + j02 * rv(2, k) for k in range(3)]
    m1 = [j11 * rv(1, k) + j12 * rv(2, k) for k in range(3)]
    c = cov3
    S = [[c[:, 0], c[:, 1], c[:, 2]], [c[:, 1], c[:, 3], c[:, 4]], [c[:, 2], c[:, 4], c[:, 5]]]
    def sm(row, k):   # (Sigma * row^T)[k]
        return (S[k][0] * row[0] + S[k][1] * row[1]) + S[k][2] * row[2]
    v0 = [sm(m0, k) for k in range(3)]
    v1 = [sm(m1, k) for k in range(3)]
    a = ((m0[0] * v0[0] + m0[1] * v0[1]) + m0[2] * v0[2]) + 0.3
    b = (m0[0] * v1[0] + m0[1] * v1[1]) + m0[2] * v1[2]
    cc = ((m1[0] * v1[0] + m1[1] * v1[1]) + m1[2] * v1[2]) + 0.3
    det = a * cc - b * b
    ok = in_front & (det != 0)
    det_s = torch.where(det != 0, det, torch.ones_like(det))
    det_inv = 1.0 / det_s
    conic = torch.stack([cc * det_inv, -b * det_inv, a * det_inv], dim=-1)
    mid = 0.5 * (a + cc)
    disc = torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
    lam = torch.maximum(mid + disc, mid - disc)
    radius = torch.ceil(3.0 * torch.sqrt(lam))
    pix_x = ((projx + 1.0) * W - 1.0) * 0.5
    pix_y = ((projy + 1.0) * H - 1.0) * 0.5
    gx, gy = (W + BLOCK - 1) // BLOCK, (H + BLOCK - 1) // BLOCK

    def rect(p, r, g):
        lo = ((p - r) / BLOCK).detach().to(torch.float32)
        hi = ((p + r + (BLOCK - 1)) / BLOCK).detach().to(torch.float32)
        lo = torch.clamp(torch.trunc(torch.nan_to_num(lo, nan=0.0, posinf=1e9, neginf=-1e9)), 0, g).to(torch.int32)
        hi = torch.clamp(torch.trunc(torch.nan_to_num(hi, nan=0.0, posinf=1e9, neginf=-1e9)), 0, g).to(torch.int32)
        return lo, hi
    rx0, rx1 = rect(pix_x, radius, gx)
    ry0, ry1 = rect(pix_y, radius, gy)
    area = (rx1 - rx0) * (ry1 - ry0)
    ok = ok & (area > 0)
    if colors_precomp is not None:
        rgb = colors_precomp
    else:
        d = means3D - campos[None]
        d = d / torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])[:, None]
        rgb = torch.clamp(eval_sh(sh_degree, shs, d) + 0.5, min=0.0)
    z32 = torch.zeros_like(area)
    return Preprocessed(depth=tz, radii=torch.where(ok, radius.detach().to(torch.int32), z32),
                        xy=torch.stack([pix_x, pix_y], -1),
                        conic_opacity=torch.cat([conic, opacities.reshape(-1, 1)], -1), rgb=rgb,
                        rect_min=torch.stack([rx0, ry0], -1), rect_max=torch.stack([rx1, ry1], -1),
                        tiles_touched=torch.where(ok, area, z32))


# ------------------------------------------------------------------------------------------------ binning (C.2)
def binning(pre: Preprocessed, H: int, W: int):
    """-> (sorted keys uint64 [R], point_list int64 [R], ranges int64 [tiles,2]).
    key = (tile_id << 32) | float_as_uint(depth); duplicates emitted in ascending gaussian index and row-major tile
    order; the sort is stable, so equal keys keep ascending index (what makes point_list well defined)."""
    gx, gy = (W + BLOCK - 1) // BLOCK, (H + BLOCK - 1) // BLOCK
    tt = pre.tiles_touched.numpy().astype(np.int64)
    idx = np.nonzero(tt)[0]
    depth_bits = pre.depth.detach().numpy().astype(np.float32).view(np.uint32).astype(np.uint64)
    rmin, rmax = pre.rect_min.numpy(), pre.rect_max.numpy()
    keys, vals = [], []
    for i in idx:
        ys = np.arange(rmin[i, 1], rmax[i, 1], dtype=np.uint64)
        xs = np.arange(rmin[i, 0], rmax[i, 0], dtype=np.uint64)
        t = (ys[:, None] * np.uint64(gx) + xs[None, :]).reshape(-1)
        keys.append((t << np.uint64(32)) | depth_bits[i])
        vals.append(np.full(t.shape, i, dtype=np.int64))
    if keys:
        keys = np.concatenate(keys)
        vals = np.concatenate(vals)
    else:
        keys, vals = np.zeros(0, np.uint64), np.zeros(0, np.int64)
    order = np.argsort(keys, kind="stable")
    keys, vals = keys[order], vals[order]
    ranges = np.zeros((gx * gy, 2), dtype=np.int64)
    if len(keys):
        tile = (keys >> np.uint64(32)).astype(np.int64)
        starts = np.nonzero(np.diff(tile, prepend=-1))[0]
        ends = np.append(starts[1:], len(keys))
        ranges[tile[starts], 0] = starts
        ranges[tile[starts], 1] = ends
    return keys, vals, ranges


# ------------------------------------------------------------------------------------------------ render (C.3)
def render(pre: Preprocessed, point_list: np.ndarray, ranges: np.ndarray, H: int, W: int, bg: torch.Tensor,
           stats: Optional[dict] = None):
    """Front-to-back alpha blending per 16x16 tile; differentiable w.r.t. xy / conic / opacity / rgb / depth.
    Returns color [3,H,W], depth [1,H,W], alpha [1,H,W], n_contrib [H,W] (int64), final_T [H,W].

    With a `stats` dict, also counts which branches the blend took: "alpha_clamped" (contributions whose opacity * G was
    clamped to 0.99), "stopped" (pixels ended by the T < 1e-4 test), and collects in "near_threshold" (a set) every gaussian
    with a pixel where its alpha lies within 1e-6 relative of 1/255 or the T after it within 1e-6 relative of 1e-4: there
    the last bit of exp() decides the branch, so another fp32 implementation may blend that pixel differently."""
    if stats is not None:
        stats.setdefault("alpha_clamped", 0)
        stats.setdefault("stopped", 0)
        stats.setdefault("near_threshold", set())
    gx, gy = (W + BLOCK - 1) // BLOCK, (H + BLOCK - 1) // BLOCK
    color = torch.zeros(3, H, W) + bg.reshape(3, 1, 1)
    depth = torch.zeros(1, H, W)
    alpha = torch.zeros(1, H, W)
    ncon = torch.zeros(H, W, dtype=torch.int64)
    finalT = torch.ones(H, W)
    pl = torch.from_numpy(point_list)
    for t in range(gx * gy):
        s, e = int(ranges[t, 0]), int(ranges[t, 1])
        y0, x0 = (t // gx) * BLOCK, (t % gx) * BLOCK
        y1, x1 = min(y0 + BLOCK, H), min(x0 + BLOCK, W)
        if e <= s:
            continue
        ids = pl[s:e]
        ys, xs = torch.meshgrid(torch.arange(y0, y1), torch.arange(x0, x1), indexing="ij")
        pxf = xs.reshape(1, -1).float()
        pyf = ys.reshape(1, -1).float()
        xy = pre.xy[ids]
        co = pre.conic_opacity[ids]
        dx = xy[:, 0:1] - pxf
        dy = xy[:, 1:2] - pyf
        power = -0.5 * (co[:, 0:1] * dx * dx + co[:, 2:3] * dy * dy) - co[:, 1:2] * dx * dy
        a_raw = co[:, 3:4] * torch.exp(power)
        # min(0.99, .) with a pass-through gradient: upstream's backward ignores the clamp
        a = a_raw + (torch.clamp(a_raw, max=0.99) - a_raw).detach()
        live = (power <= 0) & (a >= 1.0 / 255.0)
        a = torch.where(live, a, torch.zeros_like(a))
        T_after = torch.cumprod(1.0 - a, dim=0)
        T_before = torch.cat([torch.ones_like(T_after[:1]), T_after[:-1]], dim=0)
        # a contributor whose T_after would drop below 1e-4 stops the pixel WITHOUT contributing (only live ones test)
        stop = live & (T_after < 1e-4)
        alive = torch.cumsum(stop.to(torch.int64), dim=0) == 0
        w = torch.where(alive, a * T_before, torch.zeros_like(a))
        Tfin = torch.where(alive, T_after, torch.zeros_like(T_after))
        # final T = T after the last alive entry (or 1)
        last_alive = alive.to(torch.int64).sum(0)                      # number of processed-and-kept list entries
        Tf = torch.where(last_alive > 0, torch.gather(Tfin, 0, (last_alive - 1).clamp(min=0)[None])[0], torch.ones(pxf.shape[1]))
        contrib_idx = torch.where(live & alive, torch.arange(1, len(ids) + 1)[:, None], torch.zeros(1, 1, dtype=torch.int64))
        n_last = contrib_idx.max(0).values
        if stats is not None:
            evaluated = (torch.cumsum(stop.to(torch.int64), dim=0) - stop.to(torch.int64)) == 0   # up to the first stop
            ad, Td = a_raw.detach(), T_after.detach()
            on_edge = evaluated & (power <= 0) & ((ad - 1.0 / 255.0).abs() <= 1e-6 / 255.0)
            on_edge |= evaluated & live & ((Td - 1e-4).abs() <= 1e-4 * 1e-6)
            hit = on_edge.any(1)
            if bool(hit.any()):
                stats["near_threshold"].update(ids[hit].tolist())
            stats["alpha_clamped"] += int((live & alive & (ad > 0.99)).sum())
            stats["stopped"] += int(stop.any(0).sum())
        rgb = pre.rgb[ids]
        dep = pre.depth[ids]
        C = (w[:, None, :] * rgb[:, :, None]).sum(0) + Tf[None] * bg.reshape(3, 1)
        D = (w * dep[:, None]).sum(0)
        A = w.sum(0)
        hh, ww = y1 - y0, x1 - x0
        color[:, y0:y1, x0:x1] = C.reshape(3, hh, ww)
        depth[0, y0:y1, x0:x1] = D.reshape(hh, ww)
        alpha[0, y0:y1, x0:x1] = A.reshape(hh, ww)
        ncon[y0:y1, x0:x1] = n_last.reshape(hh, ww)
        finalT[y0:y1, x0:x1] = Tf.detach().reshape(hh, ww)
    return color, depth, alpha, ncon, finalT


def rasterize(means3D, scales, rotations, opacities, shs, colors_precomp, sh_degree, viewmatrix, projmatrix, campos,
              tanfovx, tanfovy, H, W, bg, scale_modifier=1.0):
    """GaussianRasterizer(raster_settings)(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, None)
    -> (color, radii, depth, alpha) plus the binning tables for index parity."""
    pre = preprocess(means3D, scales, rotations, opacities, shs, colors_precomp, sh_degree, viewmatrix, projmatrix, campos,
                     tanfovx, tanfovy, H, W, scale_modifier)
    keys, pl, ranges = binning(pre, H, W)
    color, depth, alpha, ncon, finalT = render(pre, pl, ranges, H, W, bg)
    return dict(color=color, radii=pre.radii, depth=depth, alpha=alpha, keys=keys, point_list=pl, ranges=ranges,
                n_contrib=ncon, final_T=finalT, pre=pre)


# ------------------------------------------------------------------------------------------------ synthetic scene
def synthetic_scene(P: int, seed: int = 0, sh_degree: int = 0):
    """SURVEY 8(d) config 3 distributions."""
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(P, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    r = 0.5 * torch.rand(P, 1, generator=g) ** (1.0 / 3.0)
    xyz = d * r
    log_s = math.log(0.004) + (math.log(0.02) - math.log(0.004)) * torch.rand(P, 3, generator=g)
    q = torch.randn(P, 4, generator=g)
    q = q / q.norm(dim=-1, keepdim=True)
    opacity = torch.sigmoid(2.0 + torch.randn(P, 1, generator=g))
    K = (sh_degree + 1) ** 2
    shs = torch.rand(P, K, 3, generator=g) * 2 - 1
    if K > 1:
        shs[:, 1:] *= 0.2
    return xyz, torch.exp(log_s), q, opacity, shs


def random_cameras(n_views: int, seed: int = 0):
    """uncond_hybrid.py:188-259 sampler: shared elevation/fovy/distance, azimuths 90 deg apart. -> list of (c2w, fovy)."""
    g = torch.Generator().manual_seed(seed)
    elev = math.radians(30.0 * torch.rand(1, generator=g).item())
    az0 = -180.0 + 90.0 * torch.rand(1, generator=g).item()
    fovy = math.radians(15.0 + 45.0 * torch.rand(1, generator=g).item())
    dist = (0.8 + 0.2 * torch.rand(1, generator=g).item()) / math.tan(fovy / 2)
    cams = []
    for v in range(n_views):
        az = math.radians(az0 + 360.0 / n_views * v)
        pos = torch.tensor([dist * math.cos(elev) * math.cos(az), dist * math.cos(elev) * math.sin(az), dist * math.sin(elev)])
        look = -pos / pos.norm()
        up = torch.tensor([0.0, 0.0, 1.0])
        right = torch.linalg.cross(look, up)
        right = right / right.norm()
        up = torch.linalg.cross(right, look)
        c2w = torch.eye(4)
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, up, -look, pos
        cams.append((c2w, fovy))
    return cams
