"""Rasterizer forward on an H100 against the float64 oracle (oracle/raster_abi_oracle.py), element by element.

Every case calls a3d_raster_forward through the C ABI into NaN-filled colour / depth / alpha buffers with a guard tail and
a 0xFF-filled workspace, taps the records and the per-pixel state (a3d_raster_state_tap) and the tables
(a3d_raster_binning_tap), and checks: every visible record against the float64 preprocess, every pixel of every plane,
n_contrib and final_T against the float64 blend of the kernel's own records, and the guards bit for bit.  The same call
through a3d_raster_forward_rgba8, twice (output prefilled with 0x00 and with 0xFF, which must agree, so every byte was
written), gives bytes within the oracle's RGBA8 bound, and its records equal the float forward's.  Each case asserts
through the oracle or the tap that it reached its edge.

Measured on an H100 80GB HBM3 (700 W limit): the file runs in 37 s; worst |err| / bound over all cases: colour 0.18,
depth 0.19, alpha 0.19, final_T 0.16, RGBA8 0.05 (the distance of 255 v from the byte's level), conic 0.13, SH colour
0.49; n_contrib, xy, depth records and opacity exact.  One pixel of 24 576 is excluded (the 1/255-threshold case, two
ambiguous decisions), none in any other case.  DESIGN.md section 4 has the per-case coverage."""
import ctypes as C
import math
import time

import pytest
import torch

import test_raster_backward_oracle_gpu as BW
import test_raster_forward_oracle_cpu as FC
from oracle import raster_abi_oracle as RA
from oracle import raster_oracle as R

pytestmark = pytest.mark.gpu

GUARD = 4096                 # elements after every output span
MAX_EXCLUDED = RA.MAX_EXCLUDED
WORST = {}                   # worst |err| / bound per plane over the file, printed at the end


def _settings(cams, H, W, bg, deg, mod=1.0):
    return BW._settings(cams, H, W, bg, deg, mod)


def run_forward(scene, cams, H, W, bg, deg=0, per_cam=False, colours=None, mod=1.0, max_excluded=MAX_EXCLUDED, name=""):
    """One scene through both entry points, checked against the oracle.  scene: [xyz, s, q, o, sh] (geometry [cams,P,*]
    with per_cam); colours: precomputed [P,3] (then sh is ignored).  -> (report dict, oracle output, tapped state)."""
    from animate3d_b200 import _lib as L
    from animate3d_b200 import rasterizer as RZ
    t0 = time.time()
    lib = L.load()
    xyz, s, q, o, sh = [t.cuda().contiguous() for t in scene]
    col = None if colours is None else colours.cuda().contiguous()
    shs = None if col is not None else sh
    settings = _settings(cams, H, W, bg, deg, mod)
    cams_t = RZ._pack_cams(settings, "cuda")
    ncam, P = len(cams), o.shape[0]
    args = RZ._make_args(P, H, W, cams_t, xyz, s, q, o, shs, col, deg, per_cam, mod, bg.tolist())
    hw = H * W
    nan = float("nan")
    color = torch.full((ncam * 3 * hw + GUARD,), nan, device="cuda")
    depth = torch.full((ncam * hw + GUARD,), nan, device="cuda")
    alpha = torch.full((ncam * hw + GUARD,), nan, device="cuda")
    radii = torch.full((ncam * P,), -7, dtype=torch.int32, device="cuda")
    counts = torch.empty(ncam + 2, dtype=torch.int64).pin_memory()
    cap = max(1 << 16, 8 * P * ncam)
    while True:
        nbytes = lib.a3d_raster_workspace_bytes(P, H, W, ncam, C.c_int64(cap))
        ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
        L.check(lib.a3d_raster_forward(C.byref(args), C.c_void_p(color.data_ptr()), C.c_void_p(depth.data_ptr()),
                                       C.c_void_p(alpha.data_ptr()), C.c_void_p(radii.data_ptr()), C.c_void_p(ws.data_ptr()),
                                       C.c_size_t(nbytes), C.c_int64(cap), C.c_void_p(counts.data_ptr()), L.stream_ptr()))
        torch.cuda.synchronize()
        if int(counts[ncam + 1]) == 0:
            break
        cap = int(counts[ncam]) + 1024
    st = RA.tap_state(ws, P, H, W, ncam, cap)
    for buf, n in ((color, ncam * 3 * hw), (depth, ncam * hw), (alpha, ncam * hw)):
        assert bool(torch.isnan(buf[n:]).all()), f"{name}: a store past the output span"
        assert torch.equal(buf[n:].view(torch.int32), torch.full((GUARD,), nan, device="cuda").view(torch.int32))
    specs = RA.cam_specs(settings)
    rr = radii.view(ncam, P)
    rep = RA.check_records(xyz, s, q, o, shs, col, deg, per_cam, specs, H, W, mod, st, rr)
    ora = RA.render(st, st["vals"], st["ranges"], H, W, bg.tolist())
    got = dict(color=color[:ncam * 3 * hw].view(ncam, 3, H, W), depth=depth[:ncam * hw].view(ncam, H, W),
               alpha=alpha[:ncam * hw].view(ncam, H, W), n_contrib=st["n_contrib"], final_T=st["final_T"])
    rep.update(RA.compare_forward(got, ora, max_excluded, f"{name} float"))
    # the RGBA8 entry point: same records, every byte written, bytes within the bound, guard untouched
    rb = lib.a3d_raster_forward_rgba8_workspace_bytes(P, H, W, ncam, C.c_int64(cap))
    outs = []
    for fill in (0x00, 0xFF):
        out = torch.full((ncam * hw * 4 + GUARD,), fill, dtype=torch.uint8, device="cuda")
        ws8 = torch.full((rb,), fill, dtype=torch.uint8, device="cuda")
        L.check(lib.a3d_raster_forward_rgba8(C.byref(args), C.c_void_p(out.data_ptr()), None, C.c_void_p(ws8.data_ptr()),
                                             C.c_size_t(rb), C.c_int64(cap), None, L.stream_ptr()))
        torch.cuda.synchronize()
        assert bool((out[ncam * hw * 4:] == fill).all()), f"{name}: RGBA8 store past the output span"
        st8 = RA.tap_state(ws8, P, H, W, ncam, cap, per_pixel=False)
        vis = (rr > 0)
        for k in ("xy", "conic_opac", "rgb_depth", "clamped"):
            assert torch.equal(st8[k][vis], st[k][vis]), f"{name}: RGBA8 workspace record {k} differs from the forward's"
        assert torch.equal(st8["ranges"], st["ranges"])
        outs.append(out[:ncam * hw * 4].view(ncam, H, W, 4))
    assert torch.equal(outs[0], outs[1]), f"{name}: {int((outs[0] != outs[1]).sum())} RGBA8 bytes depend on the prefill (unwritten)"
    rep.update({"rgba8": RA.compare_forward({}, ora, max_excluded, f"{name} rgba8", rgba=outs[0])["rgba8"]})
    rep["pairs"] = int(counts[ncam])
    rep["seconds"] = time.time() - t0
    for k in ("rec_conic", "rec_rgb", "color", "depth", "alpha", "final_T", "rgba8"):
        WORST[k] = max(WORST.get(k, 0.0), rep.get(k, 0.0))
    print(f"[{name}] " + ", ".join(f"{k} {v:.3g}" if isinstance(v, float) else f"{k} {v}" for k, v in {**rep, **ora["stats"]}.items()))
    print(f"[worst so far] " + ", ".join(f"{k} {v:.3g}" for k, v in WORST.items()))
    return rep, ora, st


def check_saved(ws, cap, scene, deg, per_cam, settings, planes, radii, mod=1.0, max_excluded=MAX_EXCLUDED, name=""):
    """The forward behind a saved workspace (the autograd wrapper's): records, planes (color [cams,3,H,W], depth, alpha),
    n_contrib and final_T against the oracle.  scene: (means3D, scales, rotations, opacities, shs, colors) as passed."""
    xyz, s, q, o, shs, col = [None if t is None else t.detach().cuda().float() for t in scene]
    s0 = settings[0]
    H, W, ncam, P = s0.image_height, s0.image_width, len(settings), o.shape[0]
    st = RA.tap_state(ws, P, H, W, ncam, cap)
    rep = RA.check_records(xyz, s, q, o, shs, col, deg, per_cam, RA.cam_specs(settings), H, W, mod, st, radii.view(ncam, P))
    ora = RA.render(st, st["vals"], st["ranges"], H, W, s0.bg.reshape(3).tolist())
    got = dict(planes, n_contrib=st["n_contrib"], final_T=st["final_T"])
    rep.update(RA.compare_forward(got, ora, max_excluded, name))
    print(f"[{name}] forward: " + ", ".join(f"{k} {v:.3g}" if isinstance(v, float) else f"{k} {v}" for k, v in rep.items()))
    return rep


def list_len(st, ncam_tiles_index):
    r = st["ranges"][ncam_tiles_index]
    return int(r[1] - r[0])


# ------------------------------------------------------------------------------------------------ shipped size
@pytest.mark.parametrize("deg,per_cam", [(0, False), (0, True), (3, False), (3, True)])
def test_config3(deg, per_cam):
    """50 k gaussians x 512^2 x 8 cameras (config 3 scales), precomputed colours (deg 0) or SH degree 3."""
    P, H, W, ncam, seed = 50000, 512, 512, 8, 11
    xyz, s, q, o, sh = R.synthetic_scene(P, seed, deg)
    cams = BW._cams(ncam, seed)
    g = torch.Generator().manual_seed(seed)
    if per_cam:
        xyz, s, q = BW.per_camera(xyz, s, q, ncam, g)
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0) if deg == 0 else None
    rep, ora, st = run_forward([xyz, s, q, o, sh], cams, H, W, torch.tensor([0.5, 0.5, 0.5]), deg=deg, per_cam=per_cam,
                               colours=col, name=f"config3 deg{deg}{' percam' if per_cam else ''}")
    assert rep["pairs"] > 500000 and ora["stats"]["max_list"] > 256 and ora["stats"]["stopped"] > 0


# ------------------------------------------------------------------------------------------------ staging rounds
@pytest.mark.parametrize("n", [255, 256, 257, 512, 513])
def test_staging_rounds(n):
    """One tile whose list holds exactly n faint gaussians at distinct depths: no pixel stops."""
    H, W = 32, 32
    cams = BW._cams(1, 200 + n)
    rep, ora, st = run_forward(FC.faint_tile_stack(n, cams[0], H, W, (1, 1)), cams, H, W, torch.tensor([0.2, 0.4, 0.6]),
                               colours=torch.rand(n, 3, generator=torch.Generator().manual_seed(n)), name=f"rounds{n}")
    assert list_len(st, 3) == n and ora["stats"]["max_list"] == n, "the stack must make exactly one tile of n entries"
    assert ora["stats"]["stopped"] == 0
    assert int(st["n_contrib"][0, 16:32, 16:32].max()) == n, "the deepest entry must contribute at the centre"


# ------------------------------------------------------------------------------------------------ early exit
def test_early_exit_whole_tile_in_round0():
    """An opaque front of 6 large gaussians over a 700-entry list: every pixel of tile (1, 1) stops within the first 8
    entries, so the CTA leaves through the __syncthreads_count break before round 1."""
    H, W = 48, 48
    cams = BW._cams(1, 300)
    g = torch.Generator().manual_seed(300)
    scene = BW.concat(FC.opaque_front(cams[0], H, W, (1, 1), g=g), FC.faint_tile_stack(700, cams[0], H, W, (1, 1), tz0=2.0, g=g))
    rep, ora, st = run_forward(scene, cams, H, W, torch.tensor([0.1, 0.1, 0.1]), colours=torch.rand(706, 3, generator=g), name="exit0")
    tile = st["final_T"][0, 16:32, 16:32]
    assert list_len(st, 4) > 600
    assert bool((st["n_contrib"][0, 16:32, 16:32] <= 6).all()) and float(tile.max()) < 1e-2


def test_early_exit_one_pixel_left():
    """Opaque per-pixel stacks on 255 pixels of tile (1, 1) and one pixel (8, 8) uncovered: the CTA keeps looping for it
    through all rounds of a 1065-entry list, while its neighbours stopped on their own stacks."""
    H, W = 48, 48
    cams = BW._cams(1, 310)
    g = torch.Generator().manual_seed(310)
    stacks = FC.pixel_stacks(cams[0], H, W, (1, 1), skip=(8, 8), g=g)
    scene = BW.concat(stacks, FC.faint_tile_stack(300, cams[0], H, W, (1, 1), tz0=2.0, g=g))
    P = scene[3].shape[0]
    rep, ora, st = run_forward(scene, cams, H, W, torch.tensor([0.1, 0.7, 0.3]), colours=torch.rand(P, 3, generator=g), name="exit1")
    n = list_len(st, 4)
    nc = st["n_contrib"][0, 16:32, 16:32].clone()
    lone = int(nc[8, 8])
    assert n > 1000 and lone > n - 300 and lone > 3 * 256, (n, lone)
    assert float(st["final_T"][0, 16 + 8, 16 + 8]) > 1e-4
    assert int(ora["stats"]["stopped"]) >= 255


def test_ragged_edge_tile():
    """A 40 x 40 image: the opaque front on the last (partial) tile, whose out-of-image threads start as done."""
    H, W = 40, 40
    cams = BW._cams(1, 320)
    g = torch.Generator().manual_seed(320)
    scene = BW.concat(FC.opaque_front(cams[0], H, W, (2, 2), g=g), FC.faint_tile_stack(400, cams[0], H, W, (2, 2), tz0=2.0, g=g))
    rep, ora, st = run_forward(scene, cams, H, W, torch.tensor([0.9, 0.1, 0.1]), colours=torch.rand(406, 3, generator=g), name="ragged")
    assert list_len(st, 8) > 400 and bool((st["n_contrib"][0, 32:, 32:] <= 6).all()), "every inside pixel stops on the front"


# ------------------------------------------------------------------------------------------------ image sizes
@pytest.mark.parametrize("H,W", [(15, 15), (16, 16), (17, 100), (37, 53), (1, 64), (64, 1)])
def test_image_sizes(H, W):
    cams = BW._cams(2, 400 + H)
    rep, ora, st = run_forward(BW.random_part(1500, 400 + H, 1), cams, H, W, torch.tensor([0.5, 0.3, 0.7]), deg=1,
                               name=f"size{H}x{W}")
    assert rep["pairs"] > 0 and rep["visible"] > 0


# ------------------------------------------------------------------------------------------------ empty cameras / tiles
def test_empty_camera_and_tiles():
    """Camera 1 looks away (no pair at all) in the same launch as camera 0, which sees thousands; camera 0 has empty
    tiles between full ones.  Empty pixels: bg, zero depth / alpha, n_contrib 0, final_T 1, exactly."""
    H, W = 64, 96
    cams = BW._cams(2, 500)
    wv, full, cp, tf = cams[0]
    away = torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0]))
    cams[1] = (wv @ away, wv @ away @ torch.inverse(wv) @ full, cp, tf)     # looks the opposite way: every gaussian behind it
    g = torch.Generator().manual_seed(500)
    scene = BW.concat(*[FC.faint_tile_stack(400, cams[0], H, W, t, g=g) for t in ((0, 0), (2, 0), (4, 2), (5, 3))])
    P = scene[3].shape[0]
    bg = torch.tensor([0.25, 0.5, 0.75])
    rep, ora, st = run_forward(scene, cams, H, W, bg, colours=torch.rand(P, 3, generator=g), name="empty")
    T = ((W + 15) // 16) * ((H + 15) // 16)
    r = st["ranges"]
    n0 = (r[:T, 1] - r[:T, 0]).clamp_min(0)
    assert int(n0.sum()) > 1000 and int((n0 == 0).sum()) > 0 and int(n0[1]) == 0, "camera 0: empty tile 1 between full tiles 0 and 2"
    assert int((r[T:, 1] - r[T:, 0]).clamp_min(0).sum()) == 0, "camera 1 must see nothing"
    assert bool((st["n_contrib"][1] == 0).all()) and bool((st["final_T"][1] == 1).all())
    assert bool((st["n_contrib"][0, :16, 16:32] == 0).all())


# ------------------------------------------------------------------------------------------------ thresholds
def test_clamp_and_stop_thresholds():
    cams = BW._cams(2, 600)
    g = torch.Generator().manual_seed(600)
    scene = BW.concat(BW.random_part(500, 600, 0), BW.stack_part(5, 4, 8, cams[0], 0, g))
    rep, ora, st = run_forward(scene, cams, 64, 80, torch.tensor([0.5, 0.3, 0.7]), colours=None, name="stack")
    assert ora["stats"]["clamped"] >= 15 and ora["stats"]["stopped"] >= 300


def test_alpha_threshold_replay():
    """Faint gaussians with opacity just above 1/255: decisions within their bound of 1/255, replayed both ways."""
    H, W = 96, 128
    cams = BW._cams(2, 700)
    g = torch.Generator().manual_seed(700)
    scene = BW.concat(FC.faint_threshold_part(4000, cams[0], H, W, g), BW.random_part(500, 700, 0))
    rep, ora, st = run_forward(scene, cams, H, W, torch.tensor([0.5, 0.3, 0.7]), name="alpha_threshold")
    print(f"[alpha_threshold] pixels that took the ambiguity replay: {ora['stats']['replayed']}, "
          f"on the flipped branch: {rep['took_alt']}, excluded: {ora['stats']['excluded']}")
    assert ora["stats"]["replayed"] >= 100 and rep["took_alt"] > 0


@pytest.mark.parametrize("bgv", [0.0, 1.0])
def test_rgba8_clamp(bgv):
    """Precomputed colours in [-0.5, 1.5] and bg 0 / 1: the clamp of C + T bg at both ends before the byte."""
    cams = BW._cams(2, 800)
    g = torch.Generator().manual_seed(800)
    scene = BW.random_part(3000, 800, 0)
    col = FC.precomp_colours(scene[4], g)
    rep, ora, st = run_forward(scene, cams, 64, 80, torch.full((3,), bgv), colours=col, name=f"rgba8 bg{bgv}")
    c = ora["nom"]["color"]
    assert int((c < 0).sum()) > 100 and int((c > 1).sum()) > 100


# ------------------------------------------------------------------------------------------------ flag
def test_forward_ignores_deterministic_flag():
    from animate3d_b200 import rasterizer as RZ
    cams = BW._cams(4, 900)
    xyz, s, q, o, sh = [t.cuda() for t in BW.random_part(5000, 900, 2)]
    settings = _settings(cams, 96, 128, torch.tensor([0.5, 0.3, 0.7]), 2)
    outs = []
    for det in (False, True):
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            with torch.no_grad():
                outs.append(RZ.rasterize_batch(xyz, s, q, o, sh, None, settings))
        finally:
            torch.use_deterministic_algorithms(prev)
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    print(f"[worst over the file] " + ", ".join(f"{k} {v:.3g}" for k, v in WORST.items()))
