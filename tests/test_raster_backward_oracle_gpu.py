"""Rasterizer backward against autograd through the fp32 oracle (oracle/raster_oracle.py), gaussian by gaussian.

Every case renders through `rasterize_batch` twice, with torch.use_deterministic_algorithms off (float atomics) and on
(fixed-order sums), and compares every gradient tensor -- means3D, scales, rotations, opacity, colours or SH, and the
screen-space `means2D` -- with the per-gaussian metric of `per_gaussian_err`: for every gaussian i, or every (camera,
gaussian) pair for per-camera geometry and means2D,

    e_i = |g_i - r_i| / (|r_i| + 1e-3 * max_j |r_j|),   max_i e_i <= TAU.

A wrong gradient on one small gaussian cannot hide behind a large one, as it can under a global max-error / max-reference
ratio.  Gaussians with radius 0 in every camera must get exactly zero gradient.  A contribution that sits on a blending
threshold (alpha at 1/255, T at 1e-4) may take the other branch in the kernel with the last bit of exp(); gaussians of such
pixels are found through the oracle and excluded, and there must be few of them.

Each case asserts through the oracle that the branch it is about was reached: SH degrees 1-3 with the view-direction term
of the colour, means2D on a non-square image, image sizes that are not a multiple of the 16-pixel tile (index tables
bit-exact), scale_modifier != 1, the frustum clamp of the projection Jacobian, the near plane, the colour clamp at 0, the
0.99 alpha clamp with the T < 1e-4 stop, and one mixed case of ~9.4k gaussians x 4 cameras."""
import math
import time

import numpy as np
import pytest
import torch

TAU = 1e-3              # max per-gaussian error of every gradient tensor.  Measured on an H100 80GB HBM3: worst 1.8e-4
                        # (opacity, SH degree 3, per-camera geometry); every other tensor <= 8e-5.  The smallest signal of
                        # the negative controls in test_raster_cpu.py is 0.136 (SH direction detached), so TAU must stay
                        # below 1.3e-2.
FLOOR = 1e-3            # e_i's denominator floor, relative to the largest reference gradient of the tensor
MAX_EXCLUDED = 0.005    # threshold-excluded gaussians, as a share of the visible ones


def per_gaussian_err(mine, ref, item_dims=1, exclude=None):
    """e_i = |mine_i - ref_i| / (|ref_i| + FLOOR * max_j |ref_j|) for every row i of the tensors: a row is one index of
    all but the last `item_dims` dimensions (a gaussian, or a (camera, gaussian) pair).  `exclude` is a bool mask over
    gaussians (the last row dimension); excluded rows score 0.  Computed in float64 on the CPU."""
    m = mine.detach().to("cpu", torch.float64)
    r = ref.detach().to("cpu", torch.float64)
    assert m.shape == r.shape, (m.shape, r.shape)
    rows = r.shape[:r.dim() - item_dims]
    m, r = m.reshape(*rows, -1), r.reshape(*rows, -1)
    rn = r.norm(dim=-1)
    e = (m - r).norm(dim=-1) / (rn + FLOOR * rn.max() + torch.finfo(torch.float64).tiny)
    if exclude is not None:
        e = torch.where(exclude.to(torch.bool), torch.zeros_like(e), e)
    return e


# ------------------------------------------------------------------------------------------------ scenes
def _cams(n, seed):
    from oracle import raster_oracle as R
    cams = R.random_cameras(4, seed) + R.random_cameras(4, seed + 1)
    out = []
    for c2w, fovy in cams[:n]:
        wv, full, cp = R.get_cam_info_gaussian(c2w, fovy, fovy)
        out.append((wv, full, cp, math.tan(fovy / 2)))
    return out


def _to_world(pc, wv):
    """camera-space points [N,3] -> world (row-vector convention: p_view = [x y z 1] @ wv)"""
    h = torch.cat([pc, torch.ones(pc.shape[0], 1)], 1) @ torch.inverse(wv.double()).float()
    return h[:, :3].contiguous()


def _unit_q(n, g):
    q = torch.randn(n, 4, generator=g)
    return q / q.norm(dim=-1, keepdim=True)


def _sh(n, deg, g):
    sh = torch.rand(n, (deg + 1) ** 2, 3, generator=g) * 2 - 1
    sh[:, 1:] *= 0.2
    return sh


def random_part(P, seed, deg):
    from oracle import raster_oracle as R
    xyz, s, q, o, sh = R.synthetic_scene(P, seed, deg)
    return [xyz, s * 3.0, q, o, sh]


def frustum_part(n, cam, deg, g):
    """Large gaussians whose centres lie 1.32-1.6 tanfov off the optical axis in x (first half) or y (second half), just
    outside the frustum clamp of the projection Jacobian, but whose splats reach into the image."""
    wv, _, _, tf = cam
    tz = 1.5 + 1.5 * torch.rand(n, generator=g)
    out = (1.32 + 0.28 * torch.rand(n, generator=g)) * torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    side = (torch.rand(n, generator=g) * 1.6 - 0.8)
    half = torch.arange(n) < n // 2
    rx, ry = torch.where(half, out, side) * tf, torch.where(half, side, out) * tf
    xyz = _to_world(torch.stack([rx * tz, ry * tz, tz], -1), wv)
    s = (0.2 + 0.15 * torch.rand(n, 3, generator=g)) * (tf * tz)[:, None]
    o = 0.6 + 0.35 * torch.rand(n, 1, generator=g)
    return [xyz, s, _unit_q(n, g), o, _sh(n, deg, g)]


def near_part(n, cam, deg, g):
    """Two thirds of the gaussians at depth (0.2, 0.35] in front of the camera, one third at (0.02, 0.2]: culled."""
    wv, _, _, tf = cam
    nn = 2 * n // 3
    tz = torch.cat([0.2 + 0.15 * (1 - torch.rand(nn, generator=g)), 0.02 + 0.18 * torch.rand(n - nn, generator=g)])
    rx, ry = [(torch.rand(n, generator=g) * 1.6 - 0.8) * tf for _ in range(2)]
    xyz = _to_world(torch.stack([rx * tz, ry * tz, tz], -1), wv)
    s = 0.002 + 0.004 * torch.rand(n, 3, generator=g)
    o = 0.3 + 0.6 * torch.rand(n, 1, generator=g)
    return [xyz, s, _unit_q(n, g), o, _sh(n, deg, g)]


def stack_part(nx, ny, layers, cam, deg, g):
    """An nx x ny grid of stacks of `layers` co-located gaussians of opacity 0.9-0.999 one behind another, the front one at
    0.999: alpha reaches the 0.99 clamp within ~0.13 sigma of the centres, and the pixels stop on T < 1e-4."""
    wv, _, _, tf = cam
    k = nx * ny
    gx, gy = torch.meshgrid(torch.linspace(-0.75, 0.75, nx), torch.linspace(-0.7, 0.7, ny), indexing="ij")
    rx, ry = (gx.reshape(-1) + 0.05 * torch.randn(k, generator=g)) * tf, (gy.reshape(-1) + 0.05 * torch.randn(k, generator=g)) * tf
    tz0 = 1.0 + 0.5 * torch.rand(k, generator=g)
    tz = (tz0[:, None] + 0.01 * torch.arange(layers)[None]).reshape(-1)
    jit = 1e-3 * torch.randn(k * layers, 2, generator=g)
    pc = torch.stack([rx.repeat_interleave(layers) * tz + jit[:, 0] * tz, ry.repeat_interleave(layers) * tz + jit[:, 1] * tz, tz], -1)
    xyz = _to_world(pc, wv)
    s = (0.1 * tf * tz)[:, None] * (1 + 0.3 * torch.rand(k * layers, 3, generator=g))    # sigma ~ W / 20 pixels
    o = torch.where(torch.rand(k * layers, 1, generator=g) < 0.6, 0.999, 0.9 + 0.09 * torch.rand(k * layers, 1, generator=g))
    o[::layers] = 0.999
    return [xyz, s, _unit_q(k * layers, g), o, _sh(k * layers, deg, g)]


def clamp_dc(sh, frac, g):
    """Put the DC term of a random `frac` of (gaussian, channel) pairs where C0 * dc + 0.5 is within +-0.04 of 0 and raise
    the higher-order terms to +-0.3, so the colour goes below 0 (and is clamped) for some view directions only."""
    from oracle import raster_oracle as R
    sh = sh.clone()
    pick = torch.rand(sh.shape[0], 3, generator=g) < frac
    dc = (-0.5 + 0.08 * (torch.rand(sh.shape[0], 3, generator=g) - 0.5)) / R.SH_C0
    sh[:, 0] = torch.where(pick, dc, sh[:, 0])
    if sh.shape[1] > 1:
        hi = (torch.rand(sh.shape[0], sh.shape[1] - 1, 3, generator=g) * 2 - 1) * 0.3
        sh[:, 1:] = torch.where(pick[:, None, :], hi, sh[:, 1:])
    return sh


def concat(*parts):
    return [torch.cat([p[k] for p in parts]).contiguous() for k in range(5)]


def per_camera(xyz, s, q, ncam, g):
    """one slightly deformed copy of the geometry per camera, as the 4D renderer produces"""
    off = torch.randn(ncam, xyz.shape[0], 3, generator=g) * 0.01
    return (torch.stack([xyz + off[c] for c in range(ncam)]), torch.stack([s * (1 + 0.05 * c) for c in range(ncam)]),
            torch.stack([torch.nn.functional.normalize(q + 0.02 * c, dim=-1) for c in range(ncam)]))


# ------------------------------------------------------------------------------------------------ oracle side
def oracle_run(geo, o, sh, col, deg, per_cam, cams, H, W, bg, mod, grads, means2D_scale=None):
    """Autograd through the oracle over all cameras with loss sum_c <color_c, dC_c> + <depth_c, dD_c> + <alpha_c, dA_c>.
    means2D enters as a zero [cams, P, 3] leaf added to the pixel centres as xy += m2[:, :2] * (W/2, H/2), the NDC
    convention of the rasterizer's `viewspace_points` gradient (`means2D_scale` overrides the factor).
    -> dict of gradients, per-camera images, radii [cams, P], the binning tables, branch statistics, SH clamp counts."""
    from oracle import raster_oracle as R
    ncam, P = len(cams), o.shape[0]
    leaves = {k: t.clone().requires_grad_(True) for k, t in zip(("means3D", "scales", "rotations"), geo)}
    leaves["opacity"] = o.clone().requires_grad_(True)
    if sh is not None:
        leaves["shs"] = sh.clone().requires_grad_(True)
    else:
        leaves["colors"] = col.clone().requires_grad_(True)
    leaves["means2D"] = torch.zeros(ncam, P, 3, requires_grad=True)
    m2s = torch.tensor([W / 2, H / 2]) if means2D_scale is None else torch.tensor(means2D_scale)
    stats, out, clamp = {}, {"color": [], "depth": [], "alpha": [], "radii": [], "tables": []}, []
    dC, dD, dA = grads
    loss = 0
    for c, (wv, full, cp, tf) in enumerate(cams):
        m, s, q = [leaves[k][c] if per_cam else leaves[k] for k in ("means3D", "scales", "rotations")]
        pre = R.preprocess(m, s, q, leaves["opacity"], leaves.get("shs"), leaves.get("colors"), deg, wv, full, cp, tf, tf,
                           H, W, mod)
        pre.xy = pre.xy + leaves["means2D"][c, :, :2] * m2s
        keys, pl, ranges = R.binning(pre, H, W)
        color, depth, alpha, _, _ = R.render(pre, pl, ranges, H, W, bg, stats)
        loss = loss + (color * dC[c]).sum() + (depth * dD[c]).sum() + (alpha * dA[c]).sum()
        for k, v in (("color", color), ("depth", depth), ("alpha", alpha), ("radii", pre.radii), ("tables", (keys, pl, ranges))):
            out[k].append(v.detach() if torch.is_tensor(v) else v)
        if sh is not None:
            with torch.no_grad():
                d = m.detach() - cp[None]
                d = d / d.norm(dim=-1, keepdim=True)
                clamp.append(R.eval_sh(deg, sh, d) + 0.5 < 0)
    loss.backward()
    out["grads"] = {k: t.grad for k, t in leaves.items()}
    out["radii"] = torch.stack(out["radii"])
    out["stats"] = stats
    out["clamp"] = torch.stack(clamp) if clamp else None
    return out


# ------------------------------------------------------------------------------------------------ CUDA side
def _settings(cams, H, W, bg, deg, mod):
    from animate3d_b200.rasterizer import GaussianRasterizationSettings
    return [GaussianRasterizationSettings(H, W, tf, tf, bg.cuda(), mod, wv.cuda(), full.cuda(), deg, cp.cuda(), False, False)
            for wv, full, cp, tf in cams]


def cuda_run(geo, o, sh, col, deg, per_cam, cams, H, W, bg, mod, grads, deterministic):
    from animate3d_b200 import rasterizer as RZ
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        leaves = {k: t.cuda().requires_grad_(True) for k, t in zip(("means3D", "scales", "rotations"), geo)}
        leaves["opacity"] = o.cuda().requires_grad_(True)
        if sh is not None:
            leaves["shs"] = sh.cuda().requires_grad_(True)
        else:
            leaves["colors"] = col.cuda().requires_grad_(True)
        leaves["means2D"] = torch.zeros(len(cams), o.shape[0], 3, device="cuda", requires_grad=True)
        settings = _settings(cams, H, W, bg, deg, mod)
        color, radii, depth, alpha = RZ.rasterize_batch(leaves["means3D"], leaves["scales"], leaves["rotations"], leaves["opacity"],
                                                        leaves.get("shs"), leaves.get("colors"), settings,
                                                        per_cam_geometry=per_cam, means2D=leaves["means2D"])
        # the forward, element by element, from the workspace the backward is about to read
        from test_raster_forward_oracle_gpu import check_saved
        node = color.grad_fn
        forward = check_saved(node.saved_tensors[-1], node.meta[1],
                              [leaves[k] if k in leaves else None for k in ("means3D", "scales", "rotations", "opacity", "shs", "colors")],
                              deg, per_cam, settings, dict(color=color.detach(), depth=depth.detach(), alpha=alpha.detach()), radii,
                              mod, name=f"deterministic={int(deterministic)}")
        dC, dD, dA = grads
        ((color * dC.cuda()).sum() + (depth * dD.cuda()).sum() + (alpha * dA.cuda()).sum()).backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    return dict(grads={k: t.grad.cpu() for k, t in leaves.items()}, radii=radii.cpu(), color=color.detach().cpu(),
                depth=depth.detach().cpu(), alpha=alpha.detach().cpu(), forward=forward)


# ------------------------------------------------------------------------------------------------ comparison
_ITEM_DIMS = {"shs": 2}
_PER_CAMERA = ("means3D", "scales", "rotations")


def excluded_mask(ora, P):
    ex = torch.zeros(P, dtype=torch.bool)
    near = sorted(ora["stats"]["near_threshold"])
    if near:
        ex[torch.tensor(near)] = True
    return ex


def compare_grads(name, mine, ora, per_cam, tau=TAU):
    """per-gaussian metric on every gradient tensor + exact zeros for culled gaussians; returns {tensor: worst e}"""
    P = ora["radii"].shape[1]
    visible = (ora["radii"] > 0).any(0)
    ex = excluded_mask(ora, P)
    n_ex = int((ex & visible).sum())
    print(f"[{name}] visible {int(visible.sum())} / {P}, threshold-excluded {n_ex}")
    assert n_ex <= MAX_EXCLUDED * int(visible.sum()), f"{name}: {n_ex} gaussians excluded at blending thresholds"
    worst = {}
    for k, ref in ora["grads"].items():
        got = mine["grads"][k]
        e = per_gaussian_err(got, ref, _ITEM_DIMS.get(k, 1), ex)
        worst[k] = float(e.max())
        i = np.unravel_index(int(e.argmax()), tuple(e.shape))
        print(f"[{name}] {k:9s} worst e = {worst[k]:.3e} at {i}")
        assert worst[k] <= tau, f"{name}: grad {k} per-gaussian error {worst[k]:.3e} at {i} > {tau:g}"
        # culled: zero gradient, bit for bit
        if k == "means2D" or (per_cam and k in _PER_CAMERA):
            dead = ora["radii"] == 0                                 # per (camera, gaussian)
        else:
            dead = ~visible
        assert torch.count_nonzero(got[dead]) == 0, f"{name}: grad {k} non-zero on a gaussian with radius 0"
    assert torch.count_nonzero(mine["grads"]["means2D"][..., 2]) == 0, f"{name}: means2D z gradient must be exactly 0"
    return worst


def compare_images(name, mine, ora):
    """radii equal to the fp32 oracle's; the images were checked element by element in cuda_run (check_saved)"""
    assert torch.equal(mine["radii"], ora["radii"]), f"{name}: radii"
    assert mine["forward"]["color"] <= 1.0 and mine["forward"]["n_contrib"] == 0.0


def loss_grads(ncam, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(ncam, 3, H, W, generator=g), torch.randn(ncam, 1, H, W, generator=g) * 0.3,
            torch.randn(ncam, 1, H, W, generator=g))


def run_case(name, scene, deg, cams, H, W, per_cam=False, mod=1.0, sh_colours=True, seed=0, check=None):
    """Oracle once, then the CUDA rasterizer in both summation orders against it."""
    t0 = time.time()
    xyz, s, q, o, sh = scene
    g = torch.Generator().manual_seed(seed + 1000)
    geo = per_camera(xyz, s, q, len(cams), g) if per_cam else (xyz, s, q)
    col = None if sh_colours else torch.clamp(0.28209479177387814 * sh[:, 0] + 0.5, min=0)
    sh = sh if sh_colours else None
    bg = torch.tensor([0.5, 0.3, 0.7])
    grads = loss_grads(len(cams), H, W, seed)
    ora = oracle_run(geo, o, sh, col, deg, per_cam, cams, H, W, bg, mod, grads)
    t1 = time.time()
    if check is not None:
        check(ora, geo)
    for det in (False, True):
        mine = cuda_run(geo, o, sh, col, deg, per_cam, cams, H, W, bg, mod, grads, det)
        compare_images(f"{name} det={int(det)}", mine, ora)
        compare_grads(f"{name} det={int(det)}", mine, ora, per_cam)
    print(f"[{name}] oracle {t1 - t0:.1f} s, total {time.time() - t0:.1f} s")
    return ora


# ------------------------------------------------------------------------------------------------ cases
gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("per_cam", [False, True])
@pytest.mark.parametrize("deg", [1, 2, 3])
def test_sh_colour_and_view_direction(deg, per_cam):
    """dshs, and dmeans3D including the dependence of the colour on the mean through the view direction."""
    cams = _cams(4, 40 + deg)
    run_case(f"sh{deg}{'_percam' if per_cam else ''}", random_part(1500, 40 + deg, deg), deg, cams, 56, 88, per_cam=per_cam,
             seed=deg)


@gpu
def test_means2D_non_square():
    """dL/dmeans2D (NDC units) against the oracle on a 72 x 120 image: a swapped W / H would be off by 5/3."""
    cams = _cams(2, 50)
    run_case("means2D", random_part(2000, 50, 0), 0, cams, 72, 120, sh_colours=False, seed=50)


@gpu
@pytest.mark.parametrize("H,W,P", [(37, 53, 1200), (129, 200, 4000), (17, 100, 800)])
def test_ragged_image_sizes(H, W, P):
    """Image sizes that are not a multiple of the tile: the partial tiles' out-of-image lanes.  Index tables bit-exact."""
    from animate3d_b200 import rasterizer as RZ
    from test_raster_gpu import _binning_tables
    cams = _cams(2, 60)
    ora = run_case(f"ragged{H}x{W}", random_part(P, 60, 1), 1, cams, H, W, seed=60)
    xyz, s, q, o, sh = random_part(P, 60, 1)
    bg = torch.tensor([0.5, 0.3, 0.7])

    class Ctx:
        def save_for_backward(self, *a): self.saved = a
        def mark_non_differentiable(self, *a): pass
    ctx = Ctx()
    settings = _settings(cams, H, W, bg, 1, 1.0)
    RZ._RasterizeBatch.forward(ctx, xyz.cuda(), None, s.cuda(), q.cuda(), o.cuda(), sh.cuda(), None, RZ._pack_cams(settings, "cuda"),
                               (H, W, 1, False, 1.0, bg.tolist()))
    tables = _binning_tables(P, H, W, len(cams), ctx.num_rendered, ctx.saved[-1], ctx.meta[1])
    for c, (k, pl, rg) in enumerate(tables):
        keys, pl_o, rg_o = ora["tables"][c]
        assert np.array_equal(k, keys) and np.array_equal(pl, pl_o) and np.array_equal(rg, rg_o), f"cam {c}: index tables differ"


@gpu
@pytest.mark.parametrize("mod", [0.6, 1.7])
def test_scale_modifier(mod):
    cams = _cams(2, 70)
    run_case(f"mod{mod}", random_part(1500, 70, 0), 0, cams, 64, 80, mod=mod, sh_colours=False, seed=70)


def _check_frustum(min_count):
    def check(ora, geo):
        n = 0
        for c, (wv, _, _, tf) in enumerate(ora["cams"]):
            m = geo[0][c] if geo[0].dim() == 3 else geo[0]
            t = torch.cat([m, torch.ones(m.shape[0], 1)], 1) @ wv
            r = torch.maximum((t[:, 0] / t[:, 2]).abs(), (t[:, 1] / t[:, 2]).abs())
            n += int(((r > 1.3 * tf) & (ora["radii"][c] > 0)).sum())
        print(f"visible (camera, gaussian) pairs beyond the frustum clamp: {n}")
        assert n >= min_count
    return check


@gpu
def test_frustum_clamp():
    """Gaussians just outside +-1.3 tanfov whose splats reach into the image: the clamped branch of the Jacobian."""
    cams = _cams(2, 80)
    g = torch.Generator().manual_seed(80)
    scene = concat(random_part(400, 80, 1), frustum_part(400, cams[0], 1, g))
    run_case("frustum", scene, 1, cams, 64, 96, seed=80, check=_with_cams(cams, _check_frustum(100)))


def _check_near(lo, min_near, min_culled):
    def check(ora, geo):
        wv = ora["cams"][0][0]
        m = geo[0][0] if geo[0].dim() == 3 else geo[0]
        tz = (torch.cat([m, torch.ones(m.shape[0], 1)], 1) @ wv)[lo:, 2]
        r = ora["radii"][0, lo:]
        near, culled = (tz > 0.2) & (tz <= 0.35) & (r > 0), (tz <= 0.2) & (tz > 0)
        print(f"near-plane gaussians visible: {int(near.sum())}, behind z = 0.2: {int(culled.sum())}")
        assert int(near.sum()) >= min_near and int(culled.sum()) >= min_culled
        assert int(r[culled].abs().sum()) == 0, "a gaussian behind the near plane has a radius"
    return check


def _with_cams(cams, check):
    def wrapped(ora, geo):
        ora["cams"] = cams
        check(ora, geo)
    return wrapped


@gpu
def test_near_plane():
    """Gaussians at depth (0.2, 0.35] and behind 0.2: culled ones get radius 0 and exactly zero gradient."""
    cams = _cams(2, 90)
    g = torch.Generator().manual_seed(90)
    scene = concat(random_part(600, 90, 0), near_part(300, cams[0], 0, g))
    run_case("near", scene, 0, cams, 64, 80, seed=90, check=_with_cams(cams, _check_near(600, 60, 60)))


def _check_clamp(min_pairs, min_partial):
    def check(ora, geo):
        cl = ora["clamp"].any(-1) & (ora["radii"] > 0)           # [cams, P]: a channel clamped in a visible pair
        partial = cl.any(0) & ~cl.all(0) & (ora["radii"] > 0).all(0)
        print(f"visible pairs with a clamped channel: {int(cl.sum())}, gaussians clamped in some cameras only: {int(partial.sum())}")
        assert int(cl.sum()) >= min_pairs and int(partial.sum()) >= min_partial
    return check


@gpu
def test_colour_clamp():
    """SH degree 3 with DC terms near -0.5 / C0: channels clamped at 0 for some cameras only."""
    cams = _cams(4, 100)
    g = torch.Generator().manual_seed(100)
    xyz, s, q, o, sh = random_part(1500, 100, 3)
    run_case("clamp", [xyz, s, q, o, clamp_dc(sh, 0.4, g)], 3, cams, 64, 80, seed=100, check=_check_clamp(300, 100))


def _check_stack(min_clamped, min_stopped):
    def check(ora, geo):
        st = ora["stats"]
        print(f"alpha-clamped contributions {st['alpha_clamped']}, pixels stopped on T {st['stopped']}")
        assert st["alpha_clamped"] >= min_clamped and st["stopped"] >= min_stopped
    return check


@gpu
def test_opaque_stack():
    """Co-located layers of opacity up to 0.999: the 0.99 alpha clamp (pass-through gradient) and the T < 1e-4 stop."""
    cams = _cams(2, 110)
    g = torch.Generator().manual_seed(110)
    scene = concat(random_part(500, 110, 0), stack_part(5, 4, 8, cams[0], 0, g))
    run_case("stack", scene, 0, cams, 64, 80, seed=110, check=_check_stack(15, 300))


def mixed_scene(cams, seed, deg):
    g = torch.Generator().manual_seed(seed)
    scene = concat(random_part(8000, seed, deg), frustum_part(600, cams[0], deg, g), near_part(600, cams[1], deg, g),
                   stack_part(5, 4, 8, cams[2], deg, g))
    scene[4] = clamp_dc(scene[4], 0.3, g)
    return scene


@gpu
def test_mixed_large():
    """~9.4k gaussians x 4 cameras at 128 x 160, SH degree 3, per-camera geometry: every branch above at once, at a size
    where the atomics of the backward collide."""
    cams = _cams(4, 120)
    scene = mixed_scene(cams, 120, 3)

    def check(ora, geo):
        _check_stack(15, 100)(ora, geo)
        _check_clamp(300, 100)(ora, geo)
        _check_frustum(30)(ora, geo)
    run_case("mixed", scene, 3, cams, 128, 160, per_cam=True, seed=120, check=_with_cams(cams, check))
