"""The float64 deformation-field oracle (oracle/deform_abi_oracle.py) on the CPU: its float32 cells against grid_sample, its
values against the reference-pinned gaussian4d_oracle in float64, its bounds against an honest float32 implementation, and
negative controls that each bound must reject by at least 10x."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import deform_abi_oracle as D
from oracle import gaussian4d_oracle as G

GRID2 = ((9, 8, 11, 6), (17, 15, 21, 16))
GRID1 = ((13, 11, 7, 16),)


def _coords(n, g, lo=-1.5, hi=1.5):
    return torch.rand(n, generator=g) * (hi - lo) + lo


def _scene(P, T, grid, seed, spread=1.5):
    """Gaussians uniform in [-spread, spread]^3, a block of them exactly on +-1 and on the texel centres of every scale, planes
    that are not all ones (time planes included) and non-zero last MLP layers; times linspace(-1, 1, T)."""
    g = torch.Generator().manual_seed(seed)
    xyz = torch.stack([_coords(P, g, -spread, spread) for _ in range(3)], 1)
    k = min(P // 4, 64)
    xyz[:k] = torch.tensor([-1.0, 1.0])[torch.randint(0, 2, (k, 3), generator=g)]
    for ax in range(3):   # texel centres of each scale on this axis
        cen = torch.cat([torch.linspace(-1, 1, r[ax]) for r in grid])
        xyz[k:2 * k, ax] = cen[torch.randint(0, len(cen), (k,), generator=g)]
    scaling = torch.log(torch.rand(P, 3, generator=g) * 0.05 + 0.01)
    rotation = torch.randn(P, 4, generator=g)
    times = torch.linspace(-1, 1, T)
    planes = []
    for reso in grid:
        for a, b in D.PLANE_AXES:
            planes.append(torch.rand(1, 16, reso[b], reso[a], generator=g) * 0.8 + 0.3)
    nfeat = 16 * len(grid)
    w1s = [(torch.rand(32, nfeat, generator=g) * 2 - 1) / math.sqrt(nfeat) for _ in range(3)]
    w2s = [torch.randn(o, 32, generator=g) * 0.08 for o in D.OUT_DIMS]
    return xyz, scaling, rotation, times, planes, w1s, w2s


def _rot_base(T, P, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(T, P, 4, generator=g)
    return q / q.norm(dim=-1, keepdim=True)


def _upstream(T, P, seed, nfeat):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(T, P, 3, generator=g), torch.randn(T, P, 3, generator=g), torch.randn(T, P, 4, generator=g),
            torch.randn(T, nfeat, generator=g))


def ref_deform(xyz, scaling, rotation, times, planes, w1s, w2s, deform_scale, rot_base=None):
    """gaussian4d_oracle's deformation of every frame, with the base quaternions optionally given per frame (what the product
    passes to the ABI as rot_base), in the dtype of the planes.  Returns means, scales, rotations [T, P, *] and featmean [T, nfeat]."""
    S = len(planes) // 6
    grids = [planes[s * 6:(s + 1) * 6] for s in range(S)]
    dt = planes[0].dtype
    means, scales, rots, fm = [], [], [], []
    for ti, t in enumerate(times.tolist()):
        pts = torch.cat([xyz, torch.full_like(xyz[:, :1], t)], 1).to(dt)
        h = G.interpolate_ms_features(pts, grids)
        fm.append(h.mean(0))
        base = rotation.to(dt) if rot_base is None else rot_base[ti].to(dt)
        means.append(xyz.to(dt) + G.mlp(h, w1s[0], w2s[0]))
        sc = scaling.to(dt) + (G.mlp(h, w1s[2], w2s[2]) if deform_scale else 0.0)
        scales.append(torch.exp(sc))
        rots.append(F.normalize(base + G.mlp(h, w1s[1], w2s[1]), dim=-1))
    return torch.stack(means), torch.stack(scales), torch.stack(rots), torch.stack(fm)


def _ref_with_grads(scene, dtype, deform_scale, rot_base, ups):
    """ref_deform in `dtype` with autograd: outputs and the gradients of sum(out * upstream) (+ featmean . g_featmean)."""
    xyz, scaling, rotation, times, planes, w1s, w2s = scene
    leaf = lambda t: t.detach().to(dtype).clone().requires_grad_(True)
    pl, w1, w2 = [leaf(p) for p in planes], [leaf(w) for w in w1s], [leaf(w) for w in w2s]
    rb = None if rot_base is None else leaf(rot_base)
    m, s, r, fm = ref_deform(xyz, scaling, rotation, times, pl, w1, w2, deform_scale, rb)
    gm, gs, gr, gf = [u.to(dtype) for u in ups]
    ((m * gm).sum() + (s * gs).sum() + (r * gr).sum() + (fm * gf).sum()).backward()
    return (m, s, r, fm), pl, w1, w2, rb


def _oracle(scene, deform_scale, rot_base, ups, cells=torch.float32, sm_count=132, init_seed=None):
    xyz, scaling, rotation, times, planes, w1s, w2s = scene
    fld = D.Field(xyz, scaling, rotation, times, planes, w1s, w2s, deform_scale, rot_base, cells=cells)
    gi = torch.Generator().manual_seed(init_seed) if init_seed is not None else None
    mk = (lambda shape: torch.randn(shape, generator=gi) * 0.01) if gi is not None else torch.zeros
    gp = [mk((p.shape[-2], p.shape[-1], 16)) for p in planes]
    g1 = [mk(w.shape) for w in w1s]
    g2 = [mk(w.shape) for w in w2s]
    grb = mk((times.shape[0], xyz.shape[0], 4)) if rot_base is not None else None
    gm, gs, gr, gf = ups
    refs, amb = fld.backward(gm, gs, gr, gf, sm_count=sm_count, grad_planes=gp, grad_w1=g1, grad_w2=g2, grad_rot_base=grb)
    return fld, refs, amb, (gp, g1, g2, grb)


def _plane_grad_cl(grad):
    """[1, 16, H, W] parameter gradient -> channel-last [H, W, 16] (the ABI's scratch layout)."""
    return grad.reshape(grad.shape[-3:]).permute(1, 2, 0)


# ------------------------------------------------------------------------------------------------ cells
def test_float32_cells_match_grid_sample_within_coordinate_rounding():
    """The kernel's float32 cells against float64 grid_sample, within the coordinate Lipschitz term, on points outside +-1,
    exactly on +-1, on texel centres and at the 16-frame timestamps -- six of which land one rounding below a texel."""
    g = torch.Generator().manual_seed(0)
    for H, W in ((16, 16), (8, 50), (1, 7), (5, 1)):
        plane = torch.rand(16, H, W, generator=g, dtype=torch.float64) * 2 - 1
        gx = torch.cat([_coords(500, g), torch.tensor([-1.0, 1.0, -1.0, 1.0]), torch.linspace(-1, 1, W), torch.linspace(-1, 1, 16),
                        torch.tensor([-1.5, 2.0, -3.0])]).float()
        gy = torch.cat([_coords(500, g), torch.tensor([1.0, -1.0, -1.0, 1.0]), torch.linspace(-1, 1, W).flip(0),
                        torch.linspace(-1, 1, 16), torch.tensor([0.3, 1.0000001, -1.25])]).float()
        n = min(len(gx), len(gy))
        gx, gy = gx[:n], gy[:n]
        mine = D.sample(plane, gx, gy)
        ref = F.grid_sample(plane[None], torch.stack([gx, gy], -1).double().reshape(1, 1, -1, 2), align_corners=True,
                            padding_mode="border").reshape(16, -1).t()
        f32 = lambda c, k: (((c + 1) * 0.5) * (k - 1)).clamp(0, k - 1).double()
        f64 = lambda c, k: (((c.double() + 1) * 0.5) * (k - 1)).clamp(0, k - 1)
        lx = (plane[:, :, 1:] - plane[:, :, :-1]).abs().max() if W > 1 else torch.tensor(0.0, dtype=torch.float64)
        ly = (plane[:, 1:] - plane[:, :-1]).abs().max() if H > 1 else torch.tensor(0.0, dtype=torch.float64)
        lip = (f32(gx, W) - f64(gx, W)).abs() * lx + (f32(gy, H) - f64(gy, H)).abs() * ly
        err = (mine - ref).abs()
        assert bool((err <= lip[:, None] + 1e-14).all()), float((err - lip[:, None]).max())
    # the 16-frame timestamps on a 16-texel time axis: frames 1, 2, 8, 9, 10, 12 sit one float32 rounding below a texel
    t = torch.linspace(-1, 1, 16)
    i0, _, _, w = D.cell_axis(t, 16)
    below = [k for k in range(16) if w[k] > 1 - 1e-5]
    assert below == [1, 2, 8, 9, 10, 12], below
    assert [int(i0[k]) for k in below] == [k - 1 for k in below]
    # and float64 cells of the same float32 timestamps pick a different texel than the kernel for frame 11
    i64 = D.cell_axis(t, 16, torch.float64)[0]
    assert (i0 != i64).nonzero().flatten().tolist() == [11]


# ------------------------------------------------------------------------------------------------ pinned to the reference
@pytest.mark.parametrize("grid", [GRID2, GRID1], ids=["2scales", "1scale"])
def test_float64_restatement_matches_reference_oracle(grid):
    """With float64 cells the restatement is gaussian4d_oracle (pinned to the reference source) run in float64: forward,
    featmean and every backward output, including d/d rot_base and the featmean fold, to about 1e-12."""
    P, T = 200, 5
    scene = _scene(P, T, grid, 1)
    nfeat = 16 * len(grid)
    ups = _upstream(T, P, 2, nfeat)
    # without rot_base the helper is gaussian4d_oracle.deform itself
    xyz, scaling, rotation, times, planes, w1s, w2s = scene
    grids = [[p.double() for p in planes[s * 6:(s + 1) * 6]] for s in range(len(grid))]
    mlps = {"xyz": [w1s[0].double(), w2s[0].double()], "rot": [w1s[1].double(), w2s[1].double()],
            "scale": [w1s[2].double(), w2s[2].double()]}
    m0, s0, r0 = G.deform(xyz.double(), scaling.double(), rotation.double(), float(times[2]), grids, mlps, True)
    m1, s1, r1, _ = ref_deform(xyz.double(), scaling.double(), rotation.double(), times, [p.double() for p in planes],
                               [w.double() for w in w1s], [w.double() for w in w2s], True)
    for a, b in ((m0, m1[2]), (s0, s1[2]), (r0, r1[2])):
        torch.testing.assert_close(a, b, rtol=1e-14, atol=1e-14)
    close = lambda got, want, what: torch.testing.assert_close(got, want.reshape(-1), rtol=1e-12, atol=1e-12, msg=what)
    for deform_scale, rot_base in ((True, None), (False, _rot_base(T, P, 3)), (True, _rot_base(T, P, 4))):
        (m, s, r, fm), pl, w1, w2, rb = _ref_with_grads(scene, torch.float64, deform_scale, rot_base, ups)
        fld, refs, _, _ = _oracle(scene, deform_scale, rot_base, ups, cells=torch.float64)
        fw = fld.forward()
        close(fw["means"].value, m.detach(), "means")
        close(fw["scales"].value, s.detach(), "scales")
        close(fw["rotations"].value, r.detach(), "rotations")
        close(fld.featmean().value, fm.detach(), "featmean")
        for i, p in enumerate(pl):
            close(refs[f"grad_planes[{i}]"].value, _plane_grad_cl(p.grad), f"grad_planes[{i}]")
        for k in range(3):
            want_w1 = w1[k].grad if (k != 2 or deform_scale) else torch.zeros_like(w1[k])
            want_w2 = w2[k].grad if (k != 2 or deform_scale) else torch.zeros_like(w2[k])
            close(refs[f"grad_w1[{k}]"].value, want_w1, f"grad_w1[{k}]")
            close(refs[f"grad_w2[{k}]"].value, want_w2, f"grad_w2[{k}]")
        if rot_base is not None:
            close(refs["grad_rot_base"].value, rb.grad, "grad_rot_base")


# ------------------------------------------------------------------------------------------------ bounds admit fp32
@pytest.mark.parametrize("grid,P,T", [(GRID2, 1000, 4), (GRID1, 1500, 3), (GRID2, 37, 3)], ids=["2scales", "1scale", "tiny"])
def test_bounds_admit_float32_reference(grid, P, T):
    """gaussian4d_oracle run in float32 on the CPU (its own summation orders, float32 grid_sample, autograd) is an honest fp32
    implementation of the same field: it must pass every per-element bound, with border and texel-centre points and
    accumulation into non-zero initial buffers."""
    scene = _scene(P, T, grid, 5)
    nfeat = 16 * len(grid)
    ups = _upstream(T, P, 6, nfeat)
    rot_base = _rot_base(T, P, 7)
    for deform_scale in (True, False):
        (m, s, r, fm), pl, w1, w2, rb = _ref_with_grads(scene, torch.float32, deform_scale, rot_base, ups)
        fld, refs, amb, (gp, g1, g2, grb) = _oracle(scene, deform_scale, rot_base, ups, init_seed=8)
        fw = fld.forward()
        D.assert_within(m.detach(), fw["means"], "means")
        D.assert_within(s.detach(), fw["scales"], "scales")
        D.assert_within(r.detach(), fw["rotations"], "rotations")
        D.assert_within(fm.detach(), fld.featmean(), "featmean")
        for i, p in enumerate(pl):
            D.assert_within(gp[i] + _plane_grad_cl(p.grad), refs[f"grad_planes[{i}]"], f"grad_planes[{i}]")
        for k in range(3):
            zero = k == 2 and not deform_scale
            D.assert_within(g1[k] + (0 if zero else w1[k].grad), refs[f"grad_w1[{k}]"], f"grad_w1[{k}]")
            D.assert_within(g2[k] + (0 if zero else w2[k].grad), refs[f"grad_w2[{k}]"], f"grad_w2[{k}]")
        D.assert_within(rb.grad, refs["grad_rot_base"], "grad_rot_base")


def test_unwritten_outputs_carry_zero_bound():
    """A null upstream rotation gradient leaves d/d rot_base untouched, and with deform_scale off the scale MLP's gradients
    keep their initial value exactly: any change is an infinite ratio."""
    P, T = 50, 2
    scene = _scene(P, T, GRID2, 9)
    gm, gs, _, _ = _upstream(T, P, 10, 32)
    xyz, scaling, rotation, times, planes, w1s, w2s = scene
    fld = D.Field(xyz, scaling, rotation, times, planes, w1s, w2s, False, _rot_base(T, P, 11))
    init = torch.randn(T, P, 4)
    g1 = [torch.randn(w.shape) for w in w1s]
    refs, _ = fld.backward(gm, gs, None, None, sm_count=132, grad_w1=g1, grad_w2=[torch.zeros(w.shape) for w in w2s],
                           grad_rot_base=init)
    assert D.check(init, refs["grad_rot_base"]).ratio == 0
    assert D.check(init + 1e-7, refs["grad_rot_base"]).ratio == math.inf
    assert D.check(torch.zeros(w2s[2].shape), refs["grad_w2[2]"]).ratio == 0
    assert D.check(torch.full(w2s[2].shape, 1e-30), refs["grad_w2[2]"]).ratio == math.inf


# ------------------------------------------------------------------------------------------------ negative controls
def _zeros_padding_axis(g, n, cells=torch.float32):
    f = ((g.to(cells) + 1) * 0.5) * (n - 1)
    i0 = torch.floor(f)
    w = (f - i0).to(D.F64)
    i0 = i0.long()
    i1 = i0 + 1
    w0 = torch.where((i0 >= 0) & (i0 <= n - 1), 1 - w, torch.zeros_like(w))
    w1 = torch.where((i1 >= 0) & (i1 <= n - 1), w, torch.zeros_like(w))
    return i0.clamp(0, n - 1), i1.clamp(0, n - 1), w0, w1


def _dropped_x1_axis(g, n, cells=torch.float32):
    """Cells anchored at min(floor, n - 2) (so x1 = x0 + 1 is always in range) with the x1 corner dropped where the
    coordinate was clamped: at the upper border all the weight sits on x1 and is lost."""
    raw = ((g.to(cells) + 1) * 0.5) * (n - 1)
    f = raw.clamp(0, n - 1)
    i0 = torch.clamp(torch.floor(f), max=max(n - 2, 0))
    w = (f - i0).to(D.F64)
    i0 = i0.long()
    clamped = (raw < 0) | (raw > n - 1)
    return i0, torch.clamp(i0 + 1, max=n - 1), 1 - w, torch.where(clamped, torch.zeros_like(w), w)


NEG_P, NEG_T, NEG_SM = 1500, 4, 2     # 6000 items; 2 "SMs" make a 512-item sweep, so the backward runs 12 sweeps


@pytest.fixture(scope="module")
def neg_base():
    scene = _scene(NEG_P, NEG_T, GRID2, 12)
    ups = _upstream(NEG_T, NEG_P, 13, 32)
    rot_base = _rot_base(NEG_T, NEG_P, 14)
    fld, refs, amb, inits = _oracle(scene, True, rot_base, ups, sm_count=NEG_SM)
    return scene, ups, rot_base, fld, refs, inits


def _worst(values, refs):
    return max(D.check(v, ref).ratio for v, ref in zip(values, refs))


def _forward_ratio(fld_bad, fld):
    a, b = fld_bad.forward(), fld.forward()
    return _worst([a[k].value for k in b], [b[k] for k in b])


def _neg(name, ratio):
    print(f"negative control {name}: worst |err| / bound = {ratio:.3g}")
    assert ratio >= 10, f"{name}: the bound admits this perturbation (worst ratio {ratio:.3g})"


def test_negative_control_first_sweep_only(neg_base):
    """Weight gradients summed over the first persistent sweep only (the carry of s_acc across chunks lost)."""
    scene, ups, rot_base, fld, refs, _ = neg_base
    sweep = 2 * NEG_SM * D.BWD_THREADS
    keep = (torch.arange(NEG_T * NEG_P) < sweep).reshape(NEG_T, NEG_P, 1)
    gm, gs, gr, gf = ups
    bad, _ = fld.backward(gm * keep, gs * keep, gr * keep, gf, sm_count=NEG_SM, grad_w1=[torch.zeros(w.shape) for w in scene[5]],
                          grad_w2=[torch.zeros(w.shape) for w in scene[6]])
    names = [f"grad_w{j}[{m}]" for j in (1, 2) for m in range(3)]
    _neg("first sweep only", _worst([bad[k].value for k in names], [refs[k] for k in names]))


def test_negative_control_zeros_padding(neg_base, monkeypatch):
    scene, ups, rot_base, fld, refs, _ = neg_base
    monkeypatch.setattr(D, "cell_axis", _zeros_padding_axis)
    _neg("zeros padding", _forward_ratio(D.Field(*scene, True, rot_base), fld))


def test_negative_control_swapped_plane_axes(neg_base, monkeypatch):
    scene, ups, rot_base, fld, refs, _ = neg_base
    monkeypatch.setattr(D, "PLANE_AXES", ((0, 1), (2, 0)) + D.PLANE_AXES[2:])
    _neg("axis pair of plane 1 swapped", _forward_ratio(D.Field(*scene, True, rot_base), fld))


def test_negative_control_featmean_fold_without_mean(neg_base, monkeypatch):
    scene, ups, rot_base, fld, refs, inits = neg_base
    monkeypatch.setattr(D, "_featmean_fold", lambda g, P: g)
    gp = inits[0]
    bad, _ = fld.backward(*ups, sm_count=NEG_SM, grad_planes=gp)
    names = [f"grad_planes[{i}]" for i in range(12)]
    _neg("featmean fold without 1/P", _worst([bad[k].value for k in names], [refs[k] for k in names]))


def test_negative_control_dropped_border_corner(neg_base, monkeypatch):
    scene, ups, rot_base, fld, refs, _ = neg_base
    monkeypatch.setattr(D, "cell_axis", _dropped_x1_axis)
    _neg("x1 corner dropped at a clamped border", _forward_ratio(D.Field(*scene, True, rot_base), fld))


def test_negative_control_neighbouring_timestamp(neg_base):
    """The time-plane factor of frame 1 taken from frame 2's timestamp (the only use of t is the time planes)."""
    scene, ups, rot_base, fld, refs, _ = neg_base
    xyz, scaling, rotation, times, planes, w1s, w2s = scene
    t2 = times.clone()
    t2[1] = times[2]
    _neg("time factor from the neighbouring frame", _forward_ratio(D.Field(xyz, scaling, rotation, t2, planes, w1s, w2s, True, rot_base), fld))
