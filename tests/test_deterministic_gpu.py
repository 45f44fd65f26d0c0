"""torch.use_deterministic_algorithms(True) on the 4D path: every engine op (mean feature, deformation field, rasterizer,
ARAP) gives bit-identical outputs and gradients for identical inputs, the results still pass the existing oracle tests, and
they agree with the default (float-atomic) kernels; one motion-reconstruction step and one 4D-SDS step through the engine
repeat bit for bit.

Each case runs in a fresh interpreter: PyTorch needs CUBLAS_WORKSPACE_CONFIG set before CUDA initialises for its own
deterministic cuBLAS calls (the host MLPs of the global motion branch, the UNet's fp32 embeddings)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))


def _run(case, *args):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), case, *map(str, args)], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=1800)
    assert r.returncode == 0 and f"CASE {case} OK" in r.stdout, (r.stdout[-3000:], r.stderr[-6000:])
    print(r.stdout[-2000:])


# ---------------------------------------------------------------------------------------------------------------- helpers
def _rel(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-12))


def _same(name, a, b):
    import torch
    if a is None or b is None:
        assert a is None and b is None, name
        return
    assert torch.equal(a, b), f"{name}: differs between two identical calls (max |diff| {float((a - b).abs().max()):.3e})"


def _close(name, det, ref, tol=3e-3):
    if det is None or ref is None:
        assert det is None and ref is None, name
        return
    err = _rel(det, ref)
    assert err < tol, f"{name}: deterministic vs default kernels {err:.3e}"


def _flag(on):
    import torch
    torch.use_deterministic_algorithms(on)


def _spy_scratch():
    """Records the byte counts the wrappers ask for: > 0 only on the deterministic entry points."""
    from animate3d_b200 import _lib as L
    seen = []
    orig = L.scratch

    def spy(nbytes, device):
        seen.append(nbytes)
        return orig(nbytes, device)
    L.scratch = spy
    return seen


def _deform_model(P, seed, use_global_trans, device="cuda"):
    import torch
    from animate3d_b200.gaussian4d import Gaussian4DModel
    from oracle import raster_oracle as R
    xyz, s, q, o, sh = R.synthetic_scene(P, seed)
    model = Gaussian4DModel(xyz, torch.log(s), q, o, sh[:, 0], grid_size=((20, 18, 22, 6), (40, 36, 44, 12)), seed=3,
                            use_global_trans=use_global_trans, device=device)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name in ("delta_xyz_network", "delta_rot_network", "delta_scaling_network", "global_rot_network", "global_trans_network"):
            if hasattr(model, name):
                net = getattr(model, name)
                net[1].copy_((torch.randn(net[1].shape, generator=g) * 0.08).to(device))
        for pl in model.grids:
            for p in pl:
                p.copy_((torch.rand(p.shape, generator=g) * 0.8 + 0.3).to(device))
    return model


# ---------------------------------------------------------------------------------------------------------------- cases
def case_featmean():
    """Mean k-planes feature: fixed order with the flag on AND off; matches the oracle's mean."""
    import torch
    from animate3d_b200.gaussian4d import _FeatMean
    from oracle import gaussian4d_oracle as G
    P, T = 50000, 16
    model = _deform_model(P, 21, True)
    planes = [p for pl in model.grids for p in pl]
    nets = (model.delta_xyz_network, model.delta_rot_network, model.delta_scaling_network)
    params = planes + [n[0] for n in nets] + [n[1] for n in nets]
    times = torch.linspace(-1, 1, T, device="cuda")
    outs = {}
    for on in (False, True):
        _flag(on)
        with torch.no_grad():
            a = _FeatMean.apply(model._xyz, model._scaling, model._rotation, times, len(planes), *params)
            b = _FeatMean.apply(model._xyz, model._scaling, model._rotation, times, len(planes), *params)
        _same(f"featmean (flag {on})", a, b)
        outs[on] = a
    _same("featmean flag on vs off", outs[True], outs[False])
    grids = [[p.detach().cpu().double() for p in pl] for pl in model.grids]
    xyz = model._xyz.cpu().double()
    for t in (0, 7, T - 1):
        pts = torch.cat([xyz, torch.full((P, 1), float(times[t]), dtype=torch.float64)], 1)
        ref = G.interpolate_ms_features(pts, grids).mean(0)
        torch.testing.assert_close(outs[True][t].cpu().double(), ref, rtol=1e-4, atol=1e-6)


def case_deform():
    """Deformation forward + backward with the global motion branch (rot_base, grad_featmean) and deform_scale."""
    import torch
    P, T = 20000, 16
    model = _deform_model(P, 23, True)
    times = torch.linspace(-1, 1, T, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(2)
    gm, gs, gr = (torch.randn(T, P, k, device="cuda", generator=g) for k in (3, 3, 4))
    params = [p for p in model.parameters() if p.requires_grad]

    def run():
        for p in params:
            p.grad = None
        m, s, r = model.deform_all(times, True)
        ((m * gm).sum() + (s * gs).sum() + (r * gr).sum()).backward()
        return [m.detach(), s.detach(), r.detach()] + [p.grad.clone() for p in params]

    seen = _spy_scratch()
    _flag(True)
    a, b = run(), run()
    assert seen and all(n > 0 for n in seen), seen
    for i, (x, y) in enumerate(zip(a, b)):
        _same(f"deform output/grad {i}", x, y)
    _flag(False)
    ref = run()
    for i, (x, y) in enumerate(zip(a, ref)):
        _close(f"deform output/grad {i}", x, y)


def _raster_inputs(per_cam, sh_degree, ncam=64, P=50000, H=512, W=512, seed=11):
    import math
    import torch
    from animate3d_b200.rasterizer import GaussianRasterizationSettings
    from oracle import raster_oracle as R
    xyz, s, q, o, sh = R.synthetic_scene(P, seed, sh_degree)
    cams = [c for k in range(ncam // 4) for c in R.random_cameras(4, seed + k)]
    bg = torch.tensor([0.5, 0.5, 0.5])
    settings = []
    for c2w, fovy in cams:
        wv, full, cp = R.get_cam_info_gaussian(c2w, fovy, fovy)
        tf = math.tan(fovy / 2)
        settings.append(GaussianRasterizationSettings(H, W, tf, tf, bg.cuda(), 1.0, wv.cuda(), full.cuda(), sh_degree, cp.cuda(),
                                                      False, False))
    g = torch.Generator().manual_seed(seed)
    if per_cam:
        m = xyz[None] + torch.randn(ncam, P, 3, generator=g) * 0.01
        sc, rt = s[None].expand(ncam, P, 3) * 1.02, q[None].expand(ncam, P, 4)
    else:
        m, sc, rt = xyz, s, q
    col = None if sh_degree else torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    shs = sh if sh_degree else None
    dC = torch.randn(ncam, 3, H, W, generator=g)
    dD = torch.randn(ncam, 1, H, W, generator=g) * 0.3
    dA = torch.randn(ncam, 1, H, W, generator=g)
    cu = lambda t: None if t is None else t.contiguous().cuda()
    return [cu(t) for t in (m, sc, rt, o, shs, col)], settings, [cu(t) for t in (dC, dD, dA)]


def case_raster(per_cam, sh_degree):
    """Config-3 size: 50 000 gaussians, 64 cameras at 512^2."""
    import torch
    from animate3d_b200 import rasterizer as RZ
    per_cam, sh_degree = bool(int(per_cam)), int(sh_degree)
    leaves, settings, (dC, dD, dA) = _raster_inputs(per_cam, sh_degree)
    ncam, P = len(settings), leaves[0].shape[-2]

    def run():
        xs = [None if t is None else t.clone().requires_grad_(True) for t in leaves]
        m2 = torch.zeros(ncam, P, 3, device="cuda", requires_grad=True)
        color, radii, depth, alpha = RZ.rasterize_batch(xs[0], xs[1], xs[2], xs[3], xs[4], xs[5], settings, per_cam_geometry=per_cam,
                                                        means2D=m2)
        ((color * dC).sum() + (depth * dD).sum() + (alpha * dA).sum()).backward()
        return [color.detach(), radii, depth.detach(), alpha.detach(), m2.grad] + [None if x is None else x.grad for x in xs]

    _flag(True)
    a = run()
    scratch = RZ.last_backward_scratch_bytes
    b = run()
    names = ["color", "radii", "depth", "alpha", "means2D", "means3D", "scales", "rotations", "opacity", "shs", "colors"]
    for n, x, y in zip(names, a, b):
        _same(n, x, y)
    _flag(False)
    ref = run()
    assert RZ.last_backward_scratch_bytes == 0
    for n, x, y in zip(names, a, ref):
        if n in ("color", "radii", "depth", "alpha"):
            _same(n + " (forward, flag on vs off)", x, y)
        else:
            _close(n, x, y)
    print(f"RASTER per_cam={per_cam} sh_degree={sh_degree}: {RZ.last_num_rendered} pairs, deterministic scratch {scratch} bytes")


def case_arap():
    """Repeated samples (np.random.choice draws with replacement) on a 3000-node, 5-frame problem."""
    import numpy as np
    import torch
    from animate3d_b200 import arap as AP
    from oracle import arap_oracle as A
    g = torch.Generator().manual_seed(4)
    base = torch.rand(3000, 3, generator=g)
    seq = torch.stack([base + 0.02 * t * torch.randn(3000, 3, generator=g) for t in range(5)])
    ii, jj, nn, _ = AP.cal_connectivity_from_points(seq[:1].cuda(), radius=0.01, K=3)
    idx = torch.from_numpy(np.random.default_rng(0).choice(3000, 512))
    idx[:16] = idx[16:32]                                   # make sure repeats are present
    assert len(torch.unique(idx)) < len(idx)

    def run():
        x = seq.cuda().requires_grad_(True)
        e = AP.cal_arap_error(x, ii, jj, nn, K=3, sample_idx=idx)
        e.backward()
        return e.detach(), x.grad

    seen = _spy_scratch()
    _flag(True)
    (ea, ga), (eb, gb) = run(), run()
    assert seen and all(n > 0 for n in seen), seen
    _same("arap energy", ea, eb)
    _same("arap grad", ga, gb)
    xo = seq.clone().requires_grad_(True)
    eo = A.arap_error(xo, ii.cpu(), jj.cpu(), nn.cpu(), 3, sample_idx=idx)
    eo.backward()
    assert abs(float(ea) - float(eo)) <= 5e-4 * abs(float(eo)), (float(ea), float(eo))
    assert (ga.cpu() - xo.grad).abs().max() <= 5e-3 * xo.grad.abs().max()
    _flag(False)
    er, gr = run()
    assert abs(float(ea) - float(er)) <= 5e-4 * abs(float(er))
    _close("arap grad", ga, gr, 5e-3)


def case_oracles():
    """The existing oracle tests of the rasterizer, the deformation field and ARAP, run with the flag on."""
    import torch
    sys.path.insert(0, HERE)
    import test_arap_gpu
    import test_deform
    import test_raster_gpu
    seen = _spy_scratch()
    _flag(True)
    for per_cam in (False, True):
        test_raster_gpu.test_backward_matches_autograd_through_oracle(per_cam)
    test_raster_gpu.test_reference_style_api_and_sh_colour()
    test_deform.test_deform_global_trans_matches_oracle()
    for ds in (True, False):
        test_deform.test_deform_forward_backward_match_oracle(ds)
    n_before = len(seen)
    exec(compile(test_arap_gpu.SCRIPT, "arap_script", "exec"), {"__name__": "arap_script"})
    assert len(seen) > n_before and all(n > 0 for n in seen), seen
    assert torch.are_deterministic_algorithms_enabled()


def _seed(s):
    import numpy as np
    import torch
    torch.manual_seed(s)
    np.random.seed(s)


def _grads(model):
    return [(n, p.grad.clone()) for n, p in model.named_parameters() if p.grad is not None]


def case_recon_step():
    """Motion reconstruction: do_guidance=False (10 % gradient mask), L2 to a target, ARAP on the deformed means."""
    import torch
    from animate3d_b200 import arap as AP
    from animate3d_b200.renderer import make_renderer
    from tools.splat_bench import cameras
    _flag(True)
    model = _deform_model(50000, 31, True)
    rend = make_renderer(model).train()
    c2w, fovy, ts = cameras(n_views=4, n_frames=8)
    batch = {"c2w": c2w, "fovy": fovy, "width": 256, "height": 256, "timestamps": ts, "do_guidance": False, "do_reconstruction": True}
    target = torch.rand(c2w.shape[0], 256, 256, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    uniq = torch.unique(ts)
    with torch.no_grad():
        rest = model.deform_all(uniq)[0]
    ii, jj, nn, _ = AP.cal_connectivity_from_points(rest[:1], radius=0.05, K=3)

    def step():
        _seed(5)
        model.zero_grad(set_to_none=True)
        out = rend.batch_forward(batch)
        loss = ((out["comp_rgb"] - target) ** 2).mean()
        means = model.deform_all(uniq)[0]
        loss = loss + 0.1 * AP.cal_arap_error(means, ii, jj, nn, K=3, sample_num=512)
        loss.backward()
        return loss.detach(), _grads(model)

    (la, ga), (lb, gb) = step(), step()
    _same("recon loss", la, lb)
    assert len(ga) >= 12 + 6, [n for n, _ in ga]
    for (n, x), (_, y) in zip(ga, gb):
        _same(f"recon grad {n}", x, y)
    print(f"RECON loss {float(la):.6f}, {len(ga)} parameter gradients bit-identical")


def case_sds_step():
    """4D-SDS through the engine: render -> VAE encoder with grad -> CFG UNet (1 view x 4 frames) -> loss -> backward -> ARAP."""
    import torch
    from animate3d_b200 import arap as AP
    from animate3d_b200.guidance import AnimateMVDiffusionGuidance, PrecomputedPromptUtils
    from animate3d_b200.renderer import make_renderer
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from animate3d_b200.vae import AutoencoderKL
    from oracle import unet_oracle as O
    from oracle import vae_oracle as VO
    from tools.splat_bench import cameras
    _flag(True)
    nv, nf = 1, 4
    unet = MVUNetMotionModel(UNetConfig(num_views=nv, num_frames=nf))
    unet.load_state_dict(O.make_state_dict(O.UNetConfig(num_views=nv, num_frames=nf), 3))
    unet.use_cuda_graph = False
    vae = AutoencoderKL()
    vae.load_state_dict(VO.make_state_dict(VO.VAEConfig(), 0))
    model = _deform_model(20000, 37, True)
    rend = make_renderer(model).train()
    c2w, fovy, ts = cameras(n_views=nv, n_frames=nf)
    batch = {"c2w": c2w, "fovy": fovy, "width": 256, "height": 256, "timestamps": ts, "do_guidance": True, "do_reconstruction": True}
    guide = AnimateMVDiffusionGuidance({"n_view": nv, "n_frame": nf, "guidance_scale": 5.0, "recon_std_rescale": 0.5,
                                        "min_step_percent": 0.02, "max_step_percent": 0.5}, unet=unet, vae=vae)
    guide.update_step(0, 0)
    g = torch.Generator(device="cuda").manual_seed(7)
    pu = PrecomputedPromptUtils(torch.randn(77, 768, device="cuda", generator=g), torch.randn(77, 768, device="cuda", generator=g))
    img = torch.randn(nv, 1024, device="cuda", generator=g)
    z = torch.zeros(nv * nf, device="cuda")
    uniq = torch.unique(ts)
    with torch.no_grad():
        rest = model.deform_all(uniq)[0]
    ii, jj, nn, _ = AP.cal_connectivity_from_points(rest[:1], radius=0.05, K=3)

    def step():
        _seed(9)
        model.zero_grad(set_to_none=True)
        out = rend.batch_forward(batch)
        go = guide(out["comp_rgb"], pu, z, z, z, c2w, image_embeds=img)
        loss = go["loss_sds"] + 0.1 * AP.cal_arap_error(model.deform_all(uniq)[0], ii, jj, nn, K=3, sample_num=512)
        loss.backward()
        return loss.detach(), _grads(model)

    (la, ga), (lb, gb) = step(), step()
    assert torch.isfinite(la)
    _same("sds loss", la, lb)
    assert len(ga) >= 12 + 6 + 4, [n for n, _ in ga]
    assert sum(float(x.abs().sum()) for _, x in ga) > 0
    for (n, x), (_, y) in zip(ga, gb):
        _same(f"sds grad {n}", x, y)
    print(f"SDS loss {float(la):.6f}, {len(ga)} parameter gradients bit-identical")


CASES = {"featmean": case_featmean, "deform": case_deform, "raster": case_raster, "arap": case_arap, "oracles": case_oracles,
         "recon_step": case_recon_step, "sds_step": case_sds_step}


# ---------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.gpu
def test_featmean_fixed_order():
    _run("featmean")


@pytest.mark.gpu
def test_deform_bit_identical():
    _run("deform")


@pytest.mark.gpu
@pytest.mark.parametrize("per_cam,sh_degree", [(0, 0), (1, 0), (0, 3), (1, 3)])
def test_raster_config3_bit_identical(per_cam, sh_degree):
    _run("raster", per_cam, sh_degree)


@pytest.mark.gpu
def test_arap_repeated_samples_bit_identical():
    _run("arap")


@pytest.mark.gpu
def test_existing_oracles_pass_with_flag():
    _run("oracles")


@pytest.mark.gpu
def test_motion_reconstruction_step_bit_identical():
    _run("recon_step")


@pytest.mark.gpu
def test_sds_step_bit_identical():
    _run("sds_step")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    CASES[sys.argv[1]](*sys.argv[2:])
    print(f"CASE {sys.argv[1]} OK", flush=True)
