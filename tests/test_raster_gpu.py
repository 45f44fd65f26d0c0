"""Rasterizer parity on an H100 against oracle/raster_oracle.py: sorted (tile|depth) keys, point_list and tile ranges
bit-exact per camera; every record and every pixel of colour / depth / alpha / n_contrib / final_T within the per-element
bound of oracle/raster_abi_oracle.py; every gradient tensor within fp32 tolerance; batched cameras with per-camera
geometry; SH colour path; the diff_gaussian_rasterization-style single-camera API."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _scene(P, seed, scale_mul=3.0, sh_degree=0):
    from oracle import raster_oracle as R
    xyz, s, q, o, sh = R.synthetic_scene(P, seed, sh_degree)
    return xyz, s * scale_mul, q, o, sh


def _settings(cams, H, W, bg, sh_degree=0):
    from animate3d_b200.rasterizer import GaussianRasterizationSettings
    from oracle import raster_oracle as R
    out, raw = [], []
    for c2w, fovy in cams:
        wv, full, cp = R.get_cam_info_gaussian(c2w, fovy, fovy)
        tf = math.tan(fovy / 2)
        out.append(GaussianRasterizationSettings(H, W, tf, tf, bg.cuda(), 1.0, wv.cuda(), full.cuda(), sh_degree, cp.cuda(), False, False))
        raw.append((wv, full, cp, tf))
    return out, raw


def _binning_tables(P, H, W, ncam, num_rendered, ws, cap):
    """Slice the global sorted tables of the last forward into per-camera (keys, point_list, ranges)."""
    from animate3d_b200 import _lib as L
    lib = L.load()
    gx, gy = (W + 15) // 16, (H + 15) // 16
    keys = torch.empty(cap, dtype=torch.int64, device="cuda")
    vals = torch.empty(cap, dtype=torch.int32, device="cuda")
    ranges = torch.empty(ncam * gx * gy, 2, dtype=torch.int32, device="cuda")
    L.check(lib.a3d_raster_binning_tap(C.c_void_p(ws.data_ptr()), P, H, W, ncam, C.c_int64(cap), 0, C.c_void_p(keys.data_ptr()),
                                       C.c_void_p(vals.data_ptr()), C.c_void_p(ranges.data_ptr()), L.stream_ptr()))
    torch.cuda.synchronize()
    keys = keys.cpu().numpy().view(np.uint64)
    vals = vals.cpu().numpy().view(np.uint32)
    ranges = ranges.cpu().numpy().view(np.uint32).astype(np.int64)
    out = []
    start = 0
    T = gx * gy
    for c in range(ncam):
        n = int(num_rendered[c])
        k = keys[start:start + n]
        local = ((k >> np.uint64(32)) - np.uint64(c * T)) << np.uint64(32) | (k & np.uint64(0xFFFFFFFF))
        r = ranges[c * T:(c + 1) * T].copy()
        nz = r[:, 1] > r[:, 0]
        r[nz] -= start
        out.append((local, vals[start:start + n].astype(np.int64), r))
        start += n
    return out


@pytest.mark.parametrize("P,H,W,ncam,seed", [(2000, 64, 64, 1, 0), (5000, 128, 96, 4, 1), (20000, 256, 256, 2, 2)])
def test_forward_indices_bit_exact_and_images(P, H, W, ncam, seed):
    from animate3d_b200 import rasterizer as RZ
    from oracle import raster_oracle as R
    xyz, s, q, o, sh = _scene(P, seed)
    bg = torch.tensor([0.5, 0.3, 0.7])
    cams = R.random_cameras(4, seed)[:ncam]
    settings, raw = _settings(cams, H, W, bg)
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    fn = RZ._RasterizeBatch
    cams_t = RZ._pack_cams(settings, "cuda")
    meta = (H, W, 0, False, 1.0, bg.tolist())

    class Ctx:   # minimal stand-in to reach the saved workspace
        def save_for_backward(self, *a): self.saved = a
        def mark_non_differentiable(self, *a): pass
    ctx = Ctx()
    color, radii, depth, alpha = fn.forward(ctx, xyz.cuda(), None, s.cuda(), q.cuda(), o.cuda(), None, col.cuda(), cams_t, meta)
    ws = ctx.saved[-1]
    cap = ctx.meta[1]
    tables = _binning_tables(P, H, W, ncam, ctx.num_rendered, ws, cap)
    for c, (wv, full, cp, tf) in enumerate(raw):
        ora = R.rasterize(xyz, s, q, o, None, col, 0, wv, full, cp, tf, tf, H, W, bg)
        assert torch.equal(radii[c].cpu(), ora["radii"]), f"cam {c}: radii"
        k, pl, rg = tables[c]
        assert np.array_equal(k, ora["keys"]), f"cam {c}: sorted keys differ"
        assert np.array_equal(pl, ora["point_list"]), f"cam {c}: point_list differs"
        assert np.array_equal(rg, ora["ranges"]), f"cam {c}: tile ranges differ"
    # every record and every pixel of every plane within the float64 oracle's bound
    from test_raster_forward_oracle_gpu import check_saved
    check_saved(ws, cap, (xyz, s, q, o, None, col), 0, False, settings, dict(color=color, depth=depth, alpha=alpha), radii,
                name=f"P{P} {H}x{W}")


@pytest.mark.parametrize("per_cam", [False, True])
def test_backward_matches_autograd_through_oracle(per_cam):
    from animate3d_b200 import rasterizer as RZ
    from oracle import raster_oracle as R
    P, H, W, ncam, seed = 1500, 64, 80, 3, 5
    xyz, s, q, o, sh = _scene(P, seed)
    bg = torch.tensor([0.5, 0.5, 0.5])
    cams = R.random_cameras(4, seed)[:ncam]
    settings, raw = _settings(cams, H, W, bg)
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    g = torch.Generator().manual_seed(seed)
    dC = torch.randn(ncam, 3, H, W, generator=g); dD = torch.randn(ncam, 1, H, W, generator=g) * 0.3
    dA = torch.randn(ncam, 1, H, W, generator=g)
    if per_cam:   # every camera sees its own (slightly deformed) gaussians
        off = torch.randn(ncam, P, 3, generator=g) * 0.01
        geo = [(xyz + off[c], s * (1 + 0.05 * c), torch.nn.functional.normalize(q + 0.02 * c, dim=-1)) for c in range(ncam)]
    else:
        geo = [(xyz, s, q)] * ncam
    # oracle: autograd over all cameras
    leaves = {"o": o.clone().requires_grad_(True), "col": col.clone().requires_grad_(True)}
    gl = [[t.clone().requires_grad_(True) for t in geo[c]] for c in range(ncam)] if per_cam else \
        [[t.clone().requires_grad_(True) for t in geo[0]]] * ncam
    loss = 0
    for c, (wv, full, cp, tf) in enumerate(raw):
        ora = R.rasterize(gl[c][0], gl[c][1], gl[c][2], leaves["o"], None, leaves["col"], 0, wv, full, cp, tf, tf, H, W, bg)
        loss = loss + (ora["color"] * dC[c]).sum() + (ora["depth"] * dD[c]).sum() + (ora["alpha"] * dA[c]).sum()
    loss.backward()
    # CUDA
    if per_cam:
        m = torch.stack([g_[0] for g_ in geo]).cuda().requires_grad_(True)
        sc = torch.stack([g_[1] for g_ in geo]).cuda().requires_grad_(True)
        rt = torch.stack([g_[2] for g_ in geo]).cuda().requires_grad_(True)
    else:
        m, sc, rt = [t.cuda().requires_grad_(True) for t in geo[0]]
    oc = o.cuda().requires_grad_(True)
    cc = col.cuda().requires_grad_(True)
    color, radii, depth, alpha = RZ.rasterize_batch(m, sc, rt, oc, None, cc, settings, per_cam_geometry=per_cam)
    ((color * dC.cuda()).sum() + (depth * dD.cuda()).sum() + (alpha * dA.cuda()).sum()).backward()

    def cmp(name, mine, ref):
        ref = ref.numpy(); mine = mine.cpu().numpy()
        err = np.abs(mine - ref).max() / (np.abs(ref).max() + 1e-12)
        assert err < 3e-3, f"grad {name}: {err:.3e}"
    if per_cam:
        cmp("means3D", m.grad, torch.stack([gl[c][0].grad for c in range(ncam)]))
        cmp("scales", sc.grad, torch.stack([gl[c][1].grad for c in range(ncam)]))
        cmp("rotations", rt.grad, torch.stack([gl[c][2].grad for c in range(ncam)]))
    else:
        cmp("means3D", m.grad, gl[0][0].grad); cmp("scales", sc.grad, gl[0][1].grad); cmp("rotations", rt.grad, gl[0][2].grad)
    cmp("opacity", oc.grad, leaves["o"].grad)
    cmp("colors", cc.grad, leaves["col"].grad)


def test_reference_style_api_and_sh_colour():
    """GaussianRasterizer(settings)(means3D, means2D, opacities, shs, ...) -> (color, radii, depth, alpha), SH degree 2."""
    from animate3d_b200.rasterizer import GaussianRasterizer
    from oracle import raster_oracle as R
    P, H, W = 3000, 96, 96
    xyz, s, q, o, sh = _scene(P, 7, sh_degree=2)
    bg = torch.tensor([0.1, 0.2, 0.3])
    cams = R.random_cameras(4, 7)[:1]
    settings, raw = _settings(cams, H, W, bg, sh_degree=2)
    wv, full, cp, tf = raw[0]
    ora = R.rasterize(xyz, s, q, o, sh, None, 2, wv, full, cp, tf, tf, H, W, bg)
    m2 = torch.zeros(P, 3, device="cuda", requires_grad=True)
    shc = sh.cuda().requires_grad_(True)
    color, radii, depth, alpha = GaussianRasterizer(settings[0])(xyz.cuda(), m2, o.cuda(), shs=shc, scales=s.cuda(), rotations=q.cuda())
    assert color.shape == (3, H, W) and radii.shape == (P,) and depth.shape == (1, H, W) and alpha.shape == (1, H, W)
    torch.testing.assert_close(color.cpu(), ora["color"], rtol=1e-4, atol=5e-5)
    color.sum().backward()
    # dshs and the screen-space (NDC) means2D gradient per gaussian against autograd through the oracle
    from test_raster_backward_oracle_gpu import TAU, oracle_run, per_gaussian_err
    ref = oracle_run((xyz, s, q), o, sh, None, 2, False, raw, H, W, bg, 1.0,
                     (torch.ones(1, 3, H, W), torch.zeros(1, 1, H, W), torch.zeros(1, 1, H, W)))
    ex = torch.zeros(P, dtype=torch.bool)
    ex[list(ref["stats"]["near_threshold"])] = True
    assert int(ex.sum()) <= 0.005 * P
    assert float(per_gaussian_err(shc.grad, ref["grads"]["shs"], 2, ex).max()) <= TAU
    assert float(per_gaussian_err(m2.grad, ref["grads"]["means2D"][0], 1, ex).max()) <= TAU
    assert m2.grad.abs().sum() > 0 and shc.grad.abs().sum() > 0
    with pytest.raises(Exception):
        GaussianRasterizer(settings[0])(xyz.cuda(), m2, o.cuda(), scales=s.cuda(), rotations=q.cuda())


def test_config3_size_indices_bit_exact_and_overflow_retry():
    """BASELINE config 3 geometry: 50 000 gaussians at 512x512 (1024 tiles per camera), 8 cameras in one batch.  Sorted
    keys / point_list / ranges / radii bit-exact for EVERY camera (the global sort key is (camera*1024+tile) << 32 | depth:
    45 significant bits), images checked on one camera.  The first attempt runs with a deliberately tiny pair capacity, so
    the overflow -> grow -> redo path of `_RasterizeBatch.forward` (rasterizer.py) is the one that produces the result."""
    from animate3d_b200 import rasterizer as RZ
    from oracle import raster_oracle as R
    P, H, W, ncam, seed = 50000, 512, 512, 8, 11
    xyz, s, q, o, sh = _scene(P, seed, scale_mul=1.0)          # config-3 scales (SURVEY 8d), not the enlarged test scenes
    bg = torch.tensor([0.5, 0.5, 0.5])
    cams = R.random_cameras(4, seed) + R.random_cameras(4, seed + 1)
    settings, raw = _settings(cams, H, W, bg)
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    cams_t = RZ._pack_cams(settings, "cuda")
    meta = (H, W, 0, False, 1.0, bg.tolist())

    class Ctx:
        def save_for_backward(self, *a): self.saved = a
        def mark_non_differentiable(self, *a): pass

    def forward():
        ctx = Ctx()
        out = RZ._RasterizeBatch.forward(ctx, xyz.cuda(), None, s.cuda(), q.cuda(), o.cuda(), None, col.cuda(), cams_t, meta)
        return ctx, out

    key = (P, H, W, ncam)
    RZ._cap_hint[key] = 1 << 12                                 # far below the ~1e6 pairs of this scene: must overflow
    ctx, (color, radii, depth, alpha) = forward()
    total = int(ctx.num_rendered.sum())
    assert total > (1 << 12), "scene too small to overflow the forced capacity"
    assert ctx.meta[1] >= total, "retry must have grown the capacity to hold every pair"
    ctx2, (color2, radii2, depth2, alpha2) = forward()          # second call: capacity hint from the first, no retry
    assert torch.equal(color, color2) and torch.equal(depth, depth2) and torch.equal(alpha, alpha2) and torch.equal(radii, radii2)
    tables = _binning_tables(P, H, W, ncam, ctx.num_rendered, ctx.saved[-1], ctx.meta[1])
    for c, (wv, full, cp, tf) in enumerate(raw):
        pre = R.preprocess(xyz, s, q, o, None, col, 0, wv, full, cp, tf, tf, H, W, 1.0)
        keys, pl, ranges = R.binning(pre, H, W)
        assert int(ctx.num_rendered[c]) == len(keys), f"cam {c}: pair count {int(ctx.num_rendered[c])} != {len(keys)}"
        assert torch.equal(radii[c].cpu(), pre.radii), f"cam {c}: radii"
        k, p_, rg = tables[c]
        assert np.array_equal(k, keys), f"cam {c}: sorted keys differ"
        assert np.array_equal(p_, pl), f"cam {c}: point_list differs"
        assert np.array_equal(rg, ranges), f"cam {c}: tile ranges differ"
    from test_raster_forward_oracle_gpu import check_saved
    check_saved(ctx.saved[-1], ctx.meta[1], (xyz, s, q, o, None, col), 0, False, settings,
                dict(color=color, depth=depth, alpha=alpha), radii, name="config3 overflow retry")
