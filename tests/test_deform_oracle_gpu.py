"""The deformation-field kernels against the float64 oracle (oracle/deform_abi_oracle.py), element by element: forward,
mean feature and backward through the C ABI (so that null gradient pointers are reachable), each backward case with the
atomic and with the fixed-order path, and the autograd wrapper once.  Every output is checked as a whole span against a
per-element bound; on failure the message names the tensor, the texel or entry and the item count behind it."""
import ctypes as C
import os
import sys

import pytest
import torch

from oracle import deform_abi_oracle as D

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_deform_oracle_cpu as S  # noqa: E402

pytestmark = pytest.mark.gpu

REFINE = ((50, 50, 50, 8), (100, 100, 100, 16))
SMALL = ((20, 18, 22, 6), (40, 36, 44, 12))


def _lib():
    from animate3d_b200 import _lib as L
    return L, L.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cuda_scene(P, T, grid, seed, spread=1.5):
    return [t.cuda() if torch.is_tensor(t) else [u.cuda() for u in t] for t in S._scene(P, T, grid, seed, spread)]


def _args(scene, deform_scale, *, gp=None, g1=None, g2=None):
    from animate3d_b200.gaussian4d import DeformArgs
    xyz, scaling, rotation, times, planes, w1s, w2s = scene
    a = DeformArgs()
    a.P, a.T = xyz.shape[0], times.shape[0]
    a.xyz, a.scaling, a.rotation, a.times = xyz.data_ptr(), scaling.data_ptr(), rotation.data_ptr(), times.data_ptr()
    a.num_scales, a.channels, a.hidden = len(planes) // 6, 16, 32
    for i, pl in enumerate(planes):
        a.planes[i] = pl.data_ptr()
        a.plane_h[i], a.plane_w[i] = pl.shape[-2], pl.shape[-1]
        a.grad_planes[i] = None if gp is None or gp[i] is None else gp[i].data_ptr()
    for m in range(3):
        a.w1[m], a.w2[m] = w1s[m].data_ptr(), w2s[m].data_ptr()
        a.grad_w1[m] = None if g1 is None or g1[m] is None else g1[m].data_ptr()
        a.grad_w2[m] = None if g2 is None or g2[m] is None else g2[m].data_ptr()
    a.deform_scale = int(deform_scale)
    return a


def _ptr(t):
    return C.c_void_p(None if t is None else t.data_ptr())


def _forward(scene, deform_scale, rot_base, det):
    L, lib = _lib()
    P, T = scene[0].shape[0], scene[3].shape[0]
    outs = [torch.full((T, P, k), float("nan"), device="cuda") for k in (3, 3, 4)]
    a = _args(scene, deform_scale)
    a.rot_base = None if rot_base is None else rot_base.data_ptr()
    a.deterministic = det
    L.check(lib.a3d_deform_forward(C.byref(a), *[_ptr(o) for o in outs], L.stream_ptr()))
    return outs


def _backward(scene, deform_scale, rot_base, ups, inits, det):
    """a3d_deform_backward into copies of the initial buffers (None entries stay null pointers)."""
    L, lib = _lib()
    gm, gs, gr, gf = ups
    gp, g1, g2, grb = [None if x is None else [None if t is None else t.clone() for t in x] for x in inits[:3]] + \
        [None if inits[3] is None else inits[3].clone()]
    a = _args(scene, deform_scale, gp=gp, g1=g1, g2=g2)
    a.rot_base = None if rot_base is None else rot_base.data_ptr()
    a.grad_rot_base = None if grb is None else grb.data_ptr()
    a.grad_featmean = None if gf is None else gf.data_ptr()
    a.deterministic = det
    nbytes = lib.a3d_deform_backward_scratch_bytes(C.byref(a))
    assert (nbytes > 0) == bool(det)
    scratch = L.scratch(nbytes, "cuda")
    L.check(lib.a3d_deform_backward(C.byref(a), _ptr(gm), _ptr(gs), _ptr(gr), _ptr(scratch), C.c_size_t(nbytes), L.stream_ptr()))
    torch.cuda.synchronize()
    return gp, g1, g2, grb


def _report(case, path, name, v, worst):
    key = (path, name.split("[")[0])
    worst[key] = max(worst.get(key, 0.0), v.ratio)


def _run_case(case, scene, *, deform_scale=True, rot_base=None, g_means=True, g_scales=True, g_rots=True, g_featmean=True,
              null_scale=None, null_w1=(), null_w2=(), item_mask=None, seed=0):
    """Forward (both flag settings, bit-identical) and backward (atomic and fixed-order) of one case against the oracle.
    `item_mask` [T * P] zeroes the upstream gradients of the items it leaves out."""
    xyz, scaling, rotation, times, planes, w1s, w2s = scene
    P, T = xyz.shape[0], times.shape[0]
    nfeat = 16 * (len(planes) // 6)
    gm, gs, gr, gf = [u.cuda() for u in S._upstream(T, P, seed + 1, nfeat)]
    if item_mask is not None:
        k = item_mask.reshape(T, P, 1)
        gm, gs, gr, gf = gm * k, gs * k, gr * k, None
    ups = (gm if g_means else None, gs if g_scales else None, gr if g_rots else None, gf if g_featmean else None)
    g = torch.Generator(device="cuda").manual_seed(seed + 2)
    rnd = lambda shape: torch.randn(shape, generator=g, device="cuda") * 0.01
    gp = [None if null_scale is not None and i // 6 == null_scale else rnd((p.shape[-2], p.shape[-1], 16)) for i, p in enumerate(planes)]
    g1 = [None if m in null_w1 else rnd(w.shape) for m, w in enumerate(w1s)]
    g2 = [None if m in null_w2 else rnd(w.shape) for m, w in enumerate(w2s)]
    grb = rnd((T, P, 4)) if rot_base is not None else None
    inits = (gp, g1, g2, grb)
    fld = D.Field(xyz, scaling, rotation, times, planes, w1s, w2s, deform_scale, rot_base)
    fw = fld.forward()
    refs, amb = fld.backward(*ups, sm_count=_sms(), grad_planes=gp, grad_w1=g1, grad_w2=g2, grad_rot_base=grb)
    worst = {}
    fwd = {}
    for det in (0, 1):
        path = "fixed-order" if det else "atomic"
        outs = _forward(scene, deform_scale, rot_base, det)
        fwd[det] = outs
        for name, o in zip(("means", "scales", "rotations"), outs):
            _report(case, path, name, D.assert_within(o, fw[name], f"{case} [{path}] {name}"), worst)
        bp, b1, b2, brb = _backward(scene, deform_scale, rot_base, ups, inits, det)
        got = {f"grad_planes[{i}]": t for i, t in enumerate(bp) if t is not None}
        got.update({f"grad_w1[{m}]": t for m, t in enumerate(b1) if t is not None})
        got.update({f"grad_w2[{m}]": t for m, t in enumerate(b2) if t is not None})
        if brb is not None:
            got["grad_rot_base"] = brb
        assert sorted(got) == sorted(refs), (sorted(got), sorted(refs))
        for name, t in got.items():
            _report(case, path, name, D.assert_within(t, refs[name], f"{case} [{path}] {name}"), worst)
        if not deform_scale or not g_scales:   # no gradient reaches the scale MLP: its buffers keep their contents bit for bit
            for cur, ini in ((b1[2], g1[2]), (b2[2], g2[2])):
                if ini is not None:
                    assert torch.equal(cur, ini), f"{case} [{path}]: scale-MLP gradient changed with no upstream scale gradient"
    for a, b in zip(fwd[0], fwd[1]):
        assert torch.equal(a, b)
    print(f"\n{case}: P={P} T={T}, {amb} ambiguous ReLUs; worst |err|/bound: " +
          ", ".join(f"{p}/{n} {r:.3g}" for (p, n), r in sorted(worst.items())))
    return worst, amb


# ------------------------------------------------------------------------------------------------ cases
def test_refine_config_full_size():
    """The refine config: 50k gaussians x 16 frames (linspace(-1, 1, 16)) on the (50, 50, 50, 8) / (100, 100, 100, 16) grids,
    with rot_base, the featmean fold and deform_scale: about 24 persistent sweeps per backward CTA."""
    P, T = 50000, 16
    assert P * T > 2 * _sms() * D.BWD_THREADS, "the case must run more than one sweep per CTA"
    scene = _cuda_scene(P, T, REFINE, 21, spread=1.0)
    _run_case("refine", scene, rot_base=S._rot_base(T, P, 22).cuda(), seed=23)


@pytest.mark.parametrize("delta", [0, 1, -1])
def test_sweep_edges(delta):
    """T * P exactly one persistent sweep (2 CTAs per SM x 128 items), one more and one fewer item."""
    sweep = 2 * _sms() * D.BWD_THREADS
    P, T = ((sweep // 2, 2) if delta == 0 else (sweep + delta, 1))
    scene = _cuda_scene(P, T, SMALL, 31 + delta)
    _run_case(f"sweep{delta:+d}", scene, rot_base=S._rot_base(T, P, 34).cuda(), seed=35)


def test_chunk_carry():
    """Upstream gradients on the items of CTA 0 only (chunks 0, C, 2C, 3C of a 3-sweep launch), so the weight-gradient bound
    covers a few hundred terms: an owned entry that is not carried from one chunk to the next is far outside it."""
    sweep = 2 * _sms() * D.BWD_THREADS
    P, T = (3 * sweep + 5 + 1) // 2, 2
    n = P * T
    chunks = -(-n // D.BWD_THREADS)
    keep = torch.zeros(n, dtype=torch.bool, device="cuda")
    for c in range(0, chunks, 2 * _sms()):
        keep[c * D.BWD_THREADS:(c + 1) * D.BWD_THREADS] = True
    assert int(keep.sum()) > 3 * D.BWD_THREADS
    scene = _cuda_scene(P, T, SMALL, 111)
    _run_case("carry", scene, rot_base=S._rot_base(T, P, 112).cuda(), item_mask=keep, seed=113)


@pytest.mark.parametrize("P,T", [(37, 3), (1, 1)])
def test_fewer_items_than_a_chunk(P, T):
    scene = _cuda_scene(P, T, SMALL, 41)
    _run_case(f"P{P}T{T}", scene, rot_base=S._rot_base(T, P, 42).cuda(), seed=43)


def test_border_and_texel_centres():
    """xyz uniform in [-1.5, 1.5]^3 (the clamp on every spatial axis), a block exactly on +-1 and a block on the texel centres of
    both scales, against the 16-frame timestamps on the refine grids."""
    P, T = 20000, 16
    scene = _cuda_scene(P, T, REFINE, 51)
    _run_case("border", scene, rot_base=S._rot_base(T, P, 52).cuda(), seed=53)


def test_one_scale():
    """num_scales = 1: nfeat = 16 and W1 is [32, 16]."""
    P, T = 5000, 4
    _run_case("one-scale", _cuda_scene(P, T, ((20, 18, 22, 16),), 61), seed=62)


def test_one_wide_planes():
    """Planes with W = 1 (scale 0's x axis) and H = 1 (scale 1's time axis)."""
    P, T = 5000, 3
    _run_case("one-wide", _cuda_scene(P, T, ((1, 18, 22, 6), (40, 36, 44, 1)), 71), seed=72)


@pytest.mark.parametrize("which", ["g_means_only", "g_rots_only", "null_scale_planes", "null_mlp_grads", "deform_scale_0"])
def test_partial_gradients(which):
    P, T = 6000, 4
    scene = _cuda_scene(P, T, SMALL, 81)
    rb = S._rot_base(T, P, 82).cuda()
    kw = {
        "g_means_only": dict(g_scales=False, g_rots=False, g_featmean=False),
        "g_rots_only": dict(rot_base=rb, g_means=False, g_scales=False, g_featmean=False),
        "null_scale_planes": dict(rot_base=rb, null_scale=1),
        "null_mlp_grads": dict(rot_base=rb, null_w1=(1,), null_w2=(0,)),
        "deform_scale_0": dict(rot_base=rb, deform_scale=False),
    }[which]
    _run_case(which, scene, seed=83, **kw)


@pytest.mark.parametrize("T", [1, 16])
@pytest.mark.parametrize("P", [1, 2047, 2048, 2049, 50000])
def test_featmean(P, T):
    """The mean feature of every frame with P below, at and just above one cluster's 2048 threads."""
    L, lib = _lib()
    scene = _cuda_scene(P, T, REFINE, 91 + P % 7)
    out = torch.full((T, 32), float("nan"), device="cuda")
    a = _args(scene, True)
    L.check(lib.a3d_deform_featmean(C.byref(a), _ptr(out), L.stream_ptr()))
    torch.cuda.synchronize()
    v = D.assert_within(out, D.Field(*scene, True).featmean(), f"featmean P={P} T={T}")
    print(f"\nfeatmean P={P} T={T}: worst |err|/bound {v.ratio:.3g}")


@pytest.mark.parametrize("det", [False, True])
def test_autograd_wrapper(det):
    """Gaussian4DModel.deform_all and its backward, once, against the same oracle: the wrapper's transposes of the
    channel-last plane scratch and its zero-initialised weight gradients."""
    from animate3d_b200.gaussian4d import Gaussian4DModel
    P, T = 4000, 5
    xyz, scaling, rotation, times, planes, w1s, w2s = S._scene(P, T, SMALL, 101)
    model = Gaussian4DModel(xyz, scaling, rotation, torch.zeros(P, 1), torch.zeros(P, 3), grid_size=SMALL, seed=3)
    nets = (model.delta_xyz_network, model.delta_rot_network, model.delta_scaling_network)
    with torch.no_grad():
        for p, src in zip([p for pl in model.grids for p in pl], planes):
            p.copy_(src)
        for net, w1, w2 in zip(nets, w1s, w2s):
            net[0].copy_(w1)
            net[1].copy_(w2)
    gm, gs, gr, _ = [u.cuda() for u in S._upstream(T, P, 102, 32)]
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        means, scales, rots = model.deform_all(times.cuda(), True)
        ((means * gm).sum() + (scales * gs).sum() + (rots * gr).sum()).backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    scene = [t.cuda() if torch.is_tensor(t) else [u.cuda() for u in t] for t in (xyz, scaling, rotation, times, planes, w1s, w2s)]
    fld = D.Field(*scene, True)
    fw = fld.forward()
    for name, o in zip(("means", "scales", "rotations"), (means, scales, rots)):
        D.assert_within(o.detach(), fw[name], name)
    zeros = lambda ts: [torch.zeros(t.shape[-2], t.shape[-1], 16, device="cuda") if t.dim() == 4 else torch.zeros_like(t) for t in ts]
    refs, _ = fld.backward(gm, gs, gr, None, sm_count=_sms(), grad_planes=zeros(scene[4]), grad_w1=zeros(scene[5]),
                           grad_w2=zeros(scene[6]))
    for i, p in enumerate(p for pl in model.grids for p in pl):
        D.assert_within(S._plane_grad_cl(p.grad), refs[f"grad_planes[{i}]"], f"grid {i}")
    for m, net in enumerate(nets):
        D.assert_within(net[0].grad, refs[f"grad_w1[{m}]"], f"mlp{m}.w1")
        D.assert_within(net[1].grad, refs[f"grad_w2[{m}]"], f"mlp{m}.w2")
