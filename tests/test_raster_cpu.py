"""The rasterizer arithmetic shared by the CUDA kernels (animate3d_b200/csrc/a3d_raster_math.h), driven serially on the
CPU through tests/cpu_harness/raster_cpu.cpp, against the oracle (oracle/raster_oracle.py): tile/bin indices bit-exact,
images and all gradients (torch autograd through the oracle) within fp32 tolerance.  CPU-only."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import test_raster_backward_oracle_gpu as BW   # the per-gaussian metric and the scene / oracle drivers of the GPU backward tests
from oracle import raster_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("h") / "raster_cpu.so")
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(ROOT, "tests", "cpu_harness", "raster_cpu.cpp"), "-o", out])
    lib = C.CDLL(out)
    lib.raster_cpu_forward.restype = C.c_long
    return lib


def fp(a):
    return a.ctypes.data_as(C.c_void_p)


def run_harness(lib, xyz, s, q, o, col, wv, full, tf, H, W, bg, grads=None, sh=None, deg=0, campos=None, mod=1.0):
    """col: precomputed colours [P,3], or None for SH colours from sh [P,K,3] at degree deg seen from campos."""
    P = xyz.shape[0]
    f = lambda t: np.ascontiguousarray(t.detach().numpy().astype(np.float32))
    xyz_, s_, q_, o_, wv_, full_ = f(xyz), f(s), f(q), f(o), f(wv), f(full)
    col_ = None if col is None else f(col)
    sh_ = None if sh is None else f(sh)
    cp_ = None if campos is None else f(campos)
    K = 0 if sh is None else sh.shape[1]
    bg_ = f(bg)
    opt = lambda a: None if a is None else fp(a)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    color = np.zeros((3, H, W), np.float32); depth = np.zeros((H, W), np.float32); alpha = np.zeros((H, W), np.float32)
    radii = np.zeros(P, np.int32); ncon = np.zeros((H, W), np.int32); fT = np.zeros((H, W), np.float32)
    cap = P * gx * gy
    keys = np.zeros(cap, np.uint64); vals = np.zeros(cap, np.uint32); ranges = np.zeros((gx * gy, 2), np.int64)
    pre = np.zeros((P, 8), np.float32)
    rgb = np.zeros((P, 3), np.float32); clamped = np.zeros(P, np.uint8); rgba = np.zeros((H, W, 4), np.uint8)
    n = lib.raster_cpu_forward(P, fp(xyz_), fp(s_), fp(q_), fp(o_), opt(col_), opt(sh_), deg, K, opt(cp_), fp(wv_), fp(full_),
                               C.c_float(tf), C.c_float(tf), H, W, fp(bg_), C.c_float(mod), fp(color), fp(depth), fp(alpha), fp(radii), fp(ncon), fp(fT), fp(keys),
                               fp(vals), C.c_long(cap), fp(ranges), fp(pre), fp(rgb), fp(clamped), fp(rgba))
    res = dict(color=color, depth=depth, alpha=alpha, radii=radii, ncon=ncon, fT=fT, keys=keys[:n], vals=vals[:n], ranges=ranges, pre=pre,
               rgba=rgba)
    t = torch.from_numpy
    # the records the render reads, laid out as a3d_raster_state_tap returns them (one camera)
    res["rec"] = dict(xy=t(pre[None, :, 1:3].copy()), conic_opac=t(np.concatenate([pre[:, 3:6], o_.reshape(P, 1)], 1)[None]),
                      rgb_depth=t(np.concatenate([rgb, pre[:, 0:1]], 1)[None]), clamped=t(clamped[None]))
    if grads is not None:
        dC, dD, dA = [np.ascontiguousarray(g.numpy().astype(np.float32)) for g in grads]
        gm = np.zeros((P, 3), np.float32); gs = np.zeros((P, 3), np.float32); gr = np.zeros((P, 4), np.float32)
        go = np.zeros(P, np.float32); gc = np.zeros((P, 3), np.float32); gsh = np.zeros((P, max(K, 1), 3), np.float32)
        lib.raster_cpu_backward(P, fp(xyz_), fp(s_), fp(q_), fp(o_), opt(col_), opt(sh_), deg, K, opt(cp_), fp(wv_), fp(full_),
                                C.c_float(tf), C.c_float(tf), H, W, fp(bg_), C.c_float(mod), fp(vals), fp(ranges), fp(ncon), fp(fT),
                                fp(dC), fp(dD), fp(dA), fp(gm), fp(gs), fp(gr), fp(go), fp(gc), fp(gsh))
        res.update(gm=gm, gs=gs, gr=gr, go=go, gc=gc, gsh=gsh)
    return res


@pytest.mark.parametrize("P,H,W,seed", [(300, 48, 64, 0), (1500, 64, 64, 1), (800, 40, 72, 2)])
def test_forward_indices_bit_exact_and_image_close(harness, P, H, W, seed):
    xyz, s, q, o, sh = R.synthetic_scene(P, seed)
    s = s * 3.0                                   # larger splats -> several tiles per gaussian
    (c2w, fovy) = R.random_cameras(4, seed)[seed % 4]
    wv, full, cp = R.get_cam_info_gaussian(c2w, fovy, fovy)
    tf = math.tan(fovy / 2)
    bg = torch.tensor([0.5, 0.2, 0.8])
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    ora = R.rasterize(xyz, s, q, o, None, col, 0, wv, full, cp, tf, tf, H, W, bg)
    got = run_harness(harness, xyz, s, q, o, col, wv, full, tf, H, W, bg)
    assert np.array_equal(got["radii"], ora["radii"].numpy())
    assert np.array_equal(got["keys"], ora["keys"]), "sorted (tile | depth) keys must be bit-exact"
    assert np.array_equal(got["vals"].astype(np.int64), ora["point_list"])
    assert np.array_equal(got["ranges"], ora["ranges"])
    assert len(got["keys"]) > P // 2
    assert np.array_equal(got["ncon"], ora["n_contrib"].numpy().astype(np.int32))
    # every record, plane and byte within the float64 oracle's per-element bound
    check_harness(got, (xyz, s, q, o, None, col, 0), (wv, full, cp, tf), H, W, bg)


def check_harness(got, scene, cam, H, W, bg, mod=1.0, max_excluded=None):
    """The harness's records, planes, n_contrib, final_T and bytes against oracle/raster_abi_oracle.py."""
    from oracle import raster_abi_oracle as RA
    xyz, s, q, o, sh, col, deg = scene
    wv, full, cp, tf = cam
    spec = [RA.CamSpec(wv, full, cp, RA.f32c(tf), RA.f32c(tf))]
    rep = RA.check_records(xyz, s, q, o, sh, col, deg, False, spec, H, W, mod, got["rec"], torch.from_numpy(got["radii"])[None])
    ora = RA.render(got["rec"], got["vals"], got["ranges"], H, W, bg)
    planes = dict(color=torch.from_numpy(got["color"])[None], depth=torch.from_numpy(got["depth"])[None],
                  alpha=torch.from_numpy(got["alpha"])[None], n_contrib=torch.from_numpy(got["ncon"])[None],
                  final_T=torch.from_numpy(got["fT"])[None])
    rep.update(RA.compare_forward(planes, ora, RA.MAX_EXCLUDED if max_excluded is None else max_excluded, "harness",
                                  rgba=torch.from_numpy(got["rgba"])[None]))
    rep.update(ora["stats"])
    return rep


@pytest.mark.parametrize("P,H,W,seed", [(200, 32, 48, 3), (600, 48, 48, 4)])
def test_backward_matches_autograd_through_oracle(harness, P, H, W, seed):
    xyz, s, q, o, sh = R.synthetic_scene(P, seed)
    s = s * 3.0
    (c2w, fovy) = R.random_cameras(4, seed)[1]
    wv, full, cp = R.get_cam_info_gaussian(c2w, fovy, fovy)
    tf = math.tan(fovy / 2)
    bg = torch.tensor([0.5, 0.5, 0.5])
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    leaves = [t.clone().requires_grad_(True) for t in (xyz, s, q, o, col)]
    ora = R.rasterize(leaves[0], leaves[1], leaves[2], leaves[3], None, leaves[4], 0, wv, full, cp, tf, tf, H, W, bg)
    g = torch.Generator().manual_seed(seed)
    dC = torch.randn(3, H, W, generator=g); dD = torch.randn(H, W, generator=g) * 0.3; dA = torch.randn(H, W, generator=g)
    loss = (ora["color"] * dC).sum() + (ora["depth"][0] * dD).sum() + (ora["alpha"][0] * dA).sum()
    loss.backward()
    got = run_harness(harness, xyz, s, q, o, col, wv, full, tf, H, W, bg, grads=(dC, dD, dA))
    for name, ref, mine in (("means3D", leaves[0].grad, got["gm"]), ("scales", leaves[1].grad, got["gs"]),
                            ("rotations", leaves[2].grad, got["gr"]), ("opacity", leaves[3].grad[:, 0], got["go"]),
                            ("colors", leaves[4].grad, got["gc"])):
        ref = ref.numpy()
        scale = np.abs(ref).max() + 1e-12
        err = np.abs(mine - ref).max() / scale
        assert err < 2e-3, f"grad {name}: max err / max ref = {err:.3e}"


def test_cam_info_matches_reference_source(golden_dir):
    """Camera -> (world_view, full_proj, centre) of threestudio/utils/ops.py:305-359: the oracle and the product's batched
    version against outputs of the reference functions themselves."""
    import os

    import torch

    from animate3d_b200.renderer import get_cam_info_gaussian as batched
    from oracle import raster_oracle as R
    cams = torch.load(os.path.join(golden_dir, "ref_cam_info.pt"), weights_only=False)
    for c in cams:
        wv, full, centre = R.get_cam_info_gaussian(c["c2w"], c["fovx"], c["fovy"], 0.1, 100.0)
        torch.testing.assert_close(wv, c["wv"], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(full, c["full"], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(centre, c["center"], rtol=1e-5, atol=1e-6)
    c2w = torch.stack([c["c2w"] for c in cams])
    wv, full, centre, tx, ty = batched(c2w, torch.tensor([c["fovx"] for c in cams]), torch.tensor([c["fovy"] for c in cams]))
    torch.testing.assert_close(wv, torch.stack([c["wv"] for c in cams]), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(full, torch.stack([c["full"] for c in cams]), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(centre, torch.stack([c["center"] for c in cams]), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(tx, torch.tan(torch.tensor([c["fovx"] for c in cams]) * 0.5))


# ------------------------------------------------------------------------------------------------ SH colour backward


@pytest.mark.parametrize("deg,H,W,mod,seed", [(1, 37, 53, 1.0, 5), (2, 40, 72, 0.8, 6), (3, 45, 30, 1.3, 7)])
def test_sh_backward_matches_oracle_per_gaussian(harness, deg, H, W, mod, seed):
    """SH colours at degree 1-3 on non-square images with partial tiles: dmeans3D (with the view-direction term of the
    colour), dshs, dscales, drotations and dopacity per gaussian against autograd through the oracle.  A third of the
    (gaussian, channel) colours sit near 0, so the clamp mask is exercised too."""
    g = torch.Generator().manual_seed(seed)
    xyz, s, q, o, sh = BW.random_part(500, seed, deg)
    sh = BW.clamp_dc(sh, 0.3, g)
    cam = BW._cams(1, seed)
    wv, full, cp, tf = cam[0]
    bg = torch.tensor([0.5, 0.3, 0.7])
    grads = BW.loss_grads(1, H, W, seed)
    ora = BW.oracle_run((xyz, s, q), o, sh, None, deg, False, cam, H, W, bg, mod, grads)
    assert int(ora["clamp"].any(-1)[0][ora["radii"][0] > 0].sum()) >= 20, "the colour clamp was not reached"
    got = run_harness(harness, xyz, s, q, o, None, wv, full, tf, H, W, bg, grads=[t[0] for t in grads], sh=sh, deg=deg,
                      campos=cp, mod=mod)
    assert np.array_equal(got["radii"], ora["radii"][0].numpy())
    ex = BW.excluded_mask(ora, xyz.shape[0])
    visible = torch.from_numpy(got["radii"] > 0)
    assert int((ex & visible).sum()) <= BW.MAX_EXCLUDED * int(visible.sum())
    for name, mine, item in (("means3D", got["gm"], 1), ("shs", got["gsh"], 2), ("scales", got["gs"], 1),
                             ("rotations", got["gr"], 1), ("opacity", got["go"][:, None], 1)):
        e = BW.per_gaussian_err(torch.from_numpy(mine), ora["grads"][name], item, ex)
        assert float(e.max()) <= BW.TAU, f"grad {name}: per-gaussian error {float(e.max()):.3e} at {int(e.argmax())}"
        assert not np.any(mine[~visible.numpy()]), f"grad {name}: non-zero on a culled gaussian"


# ------------------------------------------------------------------------------------------------ negative controls
# The per-gaussian metric must flag each of these mutations of the oracle's own gradients by at least 10x its tolerance.
def _controls_scene(deg, seed, n=400):
    xyz, s, q, o, sh = BW.random_part(n, seed, deg)
    return xyz, s, q, o, sh


def test_metric_flags_detached_sh_direction():
    deg, H, W = 1, 40, 56
    xyz, s, q, o, sh = _controls_scene(deg, 11)
    cams = BW._cams(1, 11)
    grads = BW.loss_grads(1, H, W, 11)
    bg = torch.zeros(3)
    ref = BW.oracle_run((xyz, s, q), o, sh, None, deg, False, cams, H, W, bg, 1.0, grads)
    # the same colours with the view direction detached: the mean gradient misses the colour's direction term
    cp = cams[0][2]
    m = xyz.clone().requires_grad_(True)
    d = (m - cp[None]).detach()
    col = torch.clamp(R.eval_sh(deg, sh, d / d.norm(dim=-1, keepdim=True)) + 0.5, min=0)
    mut = BW.oracle_run((xyz, s, q), o, None, col, deg, False, cams, H, W, bg, 1.0, grads)
    e = BW.per_gaussian_err(mut["grads"]["means3D"], ref["grads"]["means3D"])
    assert float(e.max()) >= 10 * BW.TAU, float(e.max())


def test_metric_flags_swapped_means2D_scale():
    H, W = 40, 72
    xyz, s, q, o, sh = _controls_scene(0, 12)
    cams = BW._cams(1, 12)
    grads = BW.loss_grads(1, H, W, 12)
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    ref = BW.oracle_run((xyz, s, q), o, None, col, 0, False, cams, H, W, torch.zeros(3), 1.0, grads)
    mut = BW.oracle_run((xyz, s, q), o, None, col, 0, False, cams, H, W, torch.zeros(3), 1.0, grads, means2D_scale=(H / 2, W / 2))
    e = BW.per_gaussian_err(mut["grads"]["means2D"], ref["grads"]["means2D"])
    assert float(e.max()) >= 10 * BW.TAU, float(e.max())


def test_metric_flags_ignored_colour_clamp():
    deg, H, W = 1, 40, 56
    g = torch.Generator().manual_seed(13)
    xyz, s, q, o, sh = _controls_scene(deg, 13)
    sh = BW.clamp_dc(sh, 0.4, g)
    cams = BW._cams(1, 13)
    grads = BW.loss_grads(1, H, W, 13)
    bg = torch.zeros(3)
    ref = BW.oracle_run((xyz, s, q), o, sh, None, deg, False, cams, H, W, bg, 1.0, grads)
    # the forward keeps the clamp; the backward lets the gradient through clamped channels
    shl = sh.clone().requires_grad_(True)
    m = xyz.clone().requires_grad_(True)
    d = m - cams[0][2][None]
    raw = R.eval_sh(deg, shl, d / torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])[:, None]) + 0.5
    col = raw + (torch.clamp(raw, min=0) - raw).detach()
    mut = BW.oracle_run((xyz, s, q), o, None, col.detach(), deg, False, cams, H, W, bg, 1.0, grads)
    col.backward(mut["grads"]["colors"])
    e = BW.per_gaussian_err(shl.grad, ref["grads"]["shs"], 2)
    assert float(e.max()) >= 10 * BW.TAU, float(e.max())


def test_metric_flags_one_dropped_camera_contribution():
    H, W = 40, 56
    xyz, s, q, o, sh = _controls_scene(0, 14)
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    cams = BW._cams(3, 14)
    grads = BW.loss_grads(3, H, W, 14)
    bg = torch.zeros(3)
    ref = BW.oracle_run((xyz, s, q), o, None, col, 0, False, cams, H, W, bg, 1.0, grads)
    cam0 = BW.oracle_run((xyz, s, q), o, None, col, 0, False, cams[:1], H, W, bg, 1.0, [t[:1] for t in grads])
    # drop camera 0's part of the mean gradient of one gaussian seen by every camera (the median one by gradient size)
    seen = torch.nonzero((ref["radii"] > 0).all(0)).reshape(-1)
    i = int(seen[ref["grads"]["means3D"][seen].norm(dim=-1).argsort()[len(seen) // 2]])
    mut = ref["grads"]["means3D"].clone()
    mut[i] -= cam0["grads"]["means3D"][i]
    e = BW.per_gaussian_err(mut, ref["grads"]["means3D"])
    assert float(e.max()) >= 10 * BW.TAU, float(e.max())


def test_metric_flags_scale_modifier_applied_twice():
    H, W, mod = 40, 56, 0.6
    xyz, s, q, o, sh = _controls_scene(0, 15)
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    cams = BW._cams(1, 15)
    ref = BW.oracle_run((xyz, s, q), o, None, col, 0, False, cams, H, W, torch.zeros(3), mod, BW.loss_grads(1, H, W, 15))
    e = BW.per_gaussian_err(ref["grads"]["scales"] * mod, ref["grads"]["scales"])
    assert float(e.max()) >= 10 * BW.TAU, float(e.max())
