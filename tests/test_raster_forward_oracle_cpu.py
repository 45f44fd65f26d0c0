"""The rasterizer forward's float64 oracle (oracle/raster_abi_oracle.py) without a GPU: agreement with
oracle/raster_oracle.py in float64, the serial harness of a3d_raster_math.h against every bound at SH degree 1-3 and on the
edge scenes of the GPU tests, and negative controls -- mutated float32 replays of the tile render's loop, each rejected by at
least 10x its bound, each with an unmutated twin that passes.  The scene builders here are shared with
tests/test_raster_forward_oracle_gpu.py."""
import math

import numpy as np
import pytest
import torch

import test_raster_backward_oracle_gpu as BW
from oracle import raster_abi_oracle as RA
from oracle import raster_oracle as R
from test_raster_cpu import check_harness, harness, run_harness  # noqa: F401  (harness is a fixture)

TILE = 16


# ------------------------------------------------------------------------------------------------ scenes (shared with the GPU tests)
def pix_to_cam(cx, cy, tz, H, W, tf):
    """camera-space points [N,3] whose splat centres land on pixel (cx, cy) at depth tz (tanfovx = tanfovy = tf)"""
    rx = ((2.0 * cx + 1.0) / W - 1.0) * tf
    ry = ((2.0 * cy + 1.0) / H - 1.0) * tf
    return torch.stack([rx * tz, ry * tz, tz], -1)


def point_stack(cx, cy, n, cam, H, W, sigma_px, opacity, tz0=1.0, dz=1e-3, g=None, deg=0):
    """n isotropic gaussians of `sigma_px` pixels centred on pixel (cx, cy) (scalars or [n] tensors) at distinct depths
    tz0 + k dz, opacity a float or [n] tensor."""
    wv, _, _, tf = cam
    g = g or torch.Generator().manual_seed(0)
    tz = tz0 + dz * torch.arange(n, dtype=torch.float64)
    cx = torch.as_tensor(cx, dtype=torch.float64).expand(n)
    cy = torch.as_tensor(cy, dtype=torch.float64).expand(n)
    xyz = BW._to_world(pix_to_cam(cx, cy, tz, H, W, tf).float(), wv)
    s = (sigma_px * 2.0 * tf * tz / W).float()[:, None].expand(n, 3).contiguous()
    o = torch.as_tensor(opacity, dtype=torch.float32).expand(n).reshape(n, 1).contiguous()
    return [xyz, s, BW._unit_q(n, g), o, BW._sh(n, deg, g)]


def tile_centre(tx, ty):
    return tx * TILE + 7.5, ty * TILE + 7.5


def faint_tile_stack(n, cam, H, W, tile=(0, 0), tz0=1.0, deg=0, g=None):
    """n faint gaussians (sigma 1.5 px: radius 5, so exactly one tile) stacked on the centre of `tile` at distinct depths,
    opacity 0.012: no pixel stops even at n = 513 (0.988^513 = 2e-3)."""
    cx, cy = tile_centre(*tile)
    return point_stack(cx, cy, n, cam, H, W, 1.5, 0.012, tz0=tz0, g=g, deg=deg)


def opaque_front(cam, H, W, tile, layers=6, tz0=0.5, deg=0, g=None):
    """`layers` large (sigma 24 px) gaussians of opacity 0.999 on the centre of `tile`: every pixel of it stops on them."""
    cx, cy = tile_centre(*tile)
    return point_stack(cx, cy, layers, cam, H, W, 24.0, 0.999, tz0=tz0, g=g, deg=deg)


def pixel_stacks(cam, H, W, tile, skip=None, layers=3, tz0=0.5, deg=0, g=None):
    """3 tiny (sigma 0.05 px, so the 0.3 low-pass dominates) gaussians of opacity 0.98 on every pixel centre of `tile`
    except `skip` (a (dx, dy) inside the tile), pixel-major in depth: every covered pixel stops on its own stack, the skipped
    one sees only its neighbours' flanks (T ~ 0.05) and walks the whole list."""
    cs = [(tile[0] * TILE + i, tile[1] * TILE + j) for j in range(TILE) for i in range(TILE)
          if skip is None or (i, j) != tuple(skip)]
    cx = torch.tensor([c[0] for c in cs], dtype=torch.float64).repeat_interleave(layers)
    cy = torch.tensor([c[1] for c in cs], dtype=torch.float64).repeat_interleave(layers)
    return point_stack(cx, cy, len(cs) * layers, cam, H, W, 0.05, 0.98, tz0=tz0, dz=1e-5, g=g, deg=deg)


def faint_threshold_part(n, cam, H, W, g, deg=0):
    """n small gaussians scattered over the image with opacity in (1/255, 1.02/255]: alpha crosses 1/255 close to every
    centre.  An eighth sit on pixel centres with opacity within 1e-6 relative of 1/255, so at that pixel the decision lies
    within its bound of the threshold about half the time and the ambiguity replay runs (two of them on one pixel make it
    excluded)."""
    wv, _, _, tf = cam
    cx = torch.rand(n, generator=g, dtype=torch.float64) * W
    cy = torch.rand(n, generator=g, dtype=torch.float64) * H
    cx[: n // 8] = torch.randint(0, W, (n // 8,), generator=g).double()
    cy[: n // 8] = torch.randint(0, H, (n // 8,), generator=g).double()
    tz = 1.0 + torch.rand(n, generator=g, dtype=torch.float64)
    xyz = BW._to_world(pix_to_cam(cx, cy, tz, H, W, tf).float(), wv)
    s = ((0.3 + 2.0 * torch.rand(n, generator=g, dtype=torch.float64)) * 2.0 * tf * tz / W).float()[:, None].expand(n, 3).contiguous()
    o = (RA.ALPHA_MIN * (1.0 + 0.02 * torch.rand(n, 1, generator=g))).float()
    o[: n // 8] = RA.ALPHA_MIN * (1.0 + 1e-6 * torch.rand(n // 8, 1, generator=g))   # alpha at the centre within ~1e-6 of 1/255
    return [xyz, s, BW._unit_q(n, g), o, BW._sh(n, deg, g)]


def precomp_colours(sh, g, lo=-0.5, hi=1.5):
    """precomputed colours spread over [lo, hi]: the RGBA8 clamp at both ends"""
    return (lo + (hi - lo) * torch.rand(sh.shape[0], 3, generator=g)).contiguous()


# ------------------------------------------------------------------------------------------------ float32 replay of the tile render
MUTATIONS = ("skip_round_last", "centre_half", "stop_after_contrib", "bg_prev_T", "count_contributors", "depth_alpha",
             "no_clamp", "round_q", "neighbour_cam", "eight_pixels")


def replay(rec, vals, ranges, H, W, bg, mut=None, mut_tile=(1, 0)):
    """raster_render_forward_kernel restated in float32 torch (one rounding per operation), every tile of every camera at
    once, the list walked in 256-entry rounds.  `mut` names one of MUTATIONS.  -> planes, n_contrib, final_T and bytes."""
    f32 = torch.float32
    ncam, P = rec["xy"].shape[:2]
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    T_ = gx * gy
    vals = torch.as_tensor(np.asarray(vals).astype(np.int64))
    ranges = torch.as_tensor(np.asarray(ranges).astype(np.int64)).reshape(ncam * T_, 2)
    n = (ranges[:, 1] - ranges[:, 0]).clamp_min(0)
    L = int(n.max()) if n.numel() else 0
    t = torch.arange(ncam * T_)
    cam, tl = t // T_, t % T_
    lid = torch.arange(TILE * TILE)
    px = ((tl % gx)[:, None] * TILE + lid % TILE).to(f32)
    py = ((tl // gx)[:, None] * TILE + lid // TILE).to(f32)
    inside = (px < W) & (py < H)
    if mut == "centre_half":
        px, py = px + 0.5, py + 0.5
    src_cam = cam.clone()
    if mut == "neighbour_cam":
        src_cam[1 * T_ + mut_tile[1] * gx + mut_tile[0]] = 0
    B, N = ncam * T_, TILE * TILE
    Tt = torch.ones(B, N, dtype=f32)
    Cc = torch.zeros(B, 3, N, dtype=f32)
    D = torch.zeros(B, N, dtype=f32)
    A = torch.zeros(B, N, dtype=f32)
    Tprev = torch.ones(B, N, dtype=f32)
    done = ~inside
    contributor = torch.zeros(B, N, dtype=torch.int64)
    last = torch.zeros(B, N, dtype=torch.int64)
    count = torch.zeros(B, N, dtype=torch.int64)
    amax, amin, tmin = torch.tensor(0.99, dtype=f32), torch.tensor(RA.ALPHA_MIN, dtype=f32), torch.tensor(1e-4, dtype=f32)
    for j in range(L):
        valid = (j < n)[:, None]
        if mut == "skip_round_last" and j % 256 == 255:
            continue
        act = valid & ~done
        contributor = contributor + act
        gid = vals[(ranges[:, 0] + j).clamp(max=max(vals.numel() - 1, 0))] * (j < n)
        flat = src_cam * P + gid
        xy = rec["xy"].reshape(-1, 2)[flat].to(f32)
        co = rec["conic_opac"].reshape(-1, 4)[flat].to(f32)
        cd = rec["rgb_depth"].reshape(-1, 4)[flat].to(f32)
        dx = xy[:, 0:1] - px
        dy = xy[:, 1:2] - py
        power = -0.5 * (co[:, 0:1] * dx * dx + co[:, 2:3] * dy * dy) - co[:, 1:2] * dx * dy
        araw = co[:, 3:4] * torch.exp(power)
        alpha = araw if mut == "no_clamp" else torch.minimum(amax, araw)
        alpha = torch.where((power > 0) | (alpha < amin), torch.zeros_like(alpha), alpha)
        ok = act & (alpha != 0)
        test_T = Tt * (1.0 - alpha)
        stop = ok & (test_T < tmin)
        done = done | stop
        contrib = ok & ~stop if mut != "stop_after_contrib" else ok
        w = alpha * Tt
        for ch in range(3):
            Cc[:, ch] = torch.where(contrib, Cc[:, ch] + cd[:, ch:ch + 1] * w, Cc[:, ch])
        D = torch.where(contrib, D + cd[:, 3:4] * (alpha if mut == "depth_alpha" else w), D)
        A = torch.where(contrib, A + w, A)
        Tprev = torch.where(contrib, Tt, Tprev)
        Tt = torch.where(contrib, test_T, Tt)
        count = count + contrib
        last = torch.where(contrib, contributor, last)
    bgt = torch.tensor([float(b) for b in bg], dtype=f32)
    Tb = Tprev if mut == "bg_prev_T" else Tt
    col = Cc + Tb[:, None, :] * bgt[None, :, None]
    ncon = count if mut == "count_contributors" else last
    clamp01 = lambda v: v.clamp(0.0, 1.0)
    if mut == "round_q":
        q = lambda v: torch.round(v * 255.0).to(torch.int32).to(torch.uint8)
    else:
        q = lambda v: (v * 255.0).to(torch.int32).to(torch.uint8)
    bytes_ = torch.cat([q(clamp01(col)), q(A)[:, None]], 1)                  # [B, 4, N]

    def to_img(x, ch=None):
        v = x.reshape(ncam, gy, gx, *(((ch,) if ch else ())), TILE, TILE)
        v = v.permute(0, 3, 1, 4, 2, 5) if ch else v.permute(0, 1, 3, 2, 4)
        v = v.reshape(ncam, ch, gy * TILE, gx * TILE) if ch else v.reshape(ncam, gy * TILE, gx * TILE)
        return v[..., :H, :W].contiguous()
    out = dict(color=to_img(col, 3), depth=to_img(D), alpha=to_img(A), n_contrib=to_img(ncon), final_T=to_img(Tt))
    out["rgba8"] = to_img(bytes_, 4).permute(0, 2, 3, 1).contiguous()
    if mut == "eight_pixels":
        c = out["color"]
        for k in range(8):
            c[0, 0, (3 * k) % H, (5 * k) % W] += 4e-3
    return out


def _ratio_of(fn):
    """worst |err| / bound an AssertionError from the comparator reports (inf for an exact mismatch), 0 when it passes"""
    try:
        fn()
    except AssertionError as e:
        msg = str(e)
        if "|err|/bound = " in msg:
            return float(msg.split("|err|/bound = ")[1].split(" ")[0])
        return math.inf
    return 0.0


def compare_replay(out, ora, planes=("color", "depth", "alpha", "n_contrib", "final_T"), rgba=True):
    got = {k: out[k] for k in planes}
    return RA.compare_forward(got, ora, RA.MAX_EXCLUDED, "replay", rgba=out["rgba8"] if rgba else None)


# ------------------------------------------------------------------------------------------------ tests
def _harness_scene(scene, deg, H, W, cam, bg, lib, mod=1.0, colours=None):
    xyz, s, q, o, sh = scene
    wv, full, cp, tf = cam
    col = colours if deg < 0 else None
    d = max(deg, 0)
    got = run_harness(lib, xyz, s, q, o, col, wv, full, tf, H, W, bg, sh=None if col is not None else sh, deg=d, campos=cp, mod=mod)
    rep = check_harness(got, (xyz, s, q, o, None if col is not None else sh, col, d), cam, H, W, bg, mod)
    return got, rep


def test_render_oracle_equals_raster_oracle_in_float64():
    """With float64 records the oracle's nominal branch is raster_oracle.render in float64 (cumprod form) to round-off."""
    P, H, W, seed = 1500, 48, 64, 3
    xyz, s, q, o, sh = R.synthetic_scene(P, seed)
    s, o = s * 3.0, o.clamp(max=0.98)                  # no 0.99 clamp: the float64 form would clamp at 0.99, the kernel at 0.99f
    (c2w, fovy) = R.random_cameras(4, seed)[0]
    wv, full, cp = R.get_cam_info_gaussian(c2w, fovy, fovy)
    tf = math.tan(fovy / 2)
    bg = torch.tensor([0.5, 0.2, 0.8], dtype=torch.float64)
    col = torch.clamp(R.SH_C0 * sh[:, 0] + 0.5, min=0)
    pre = R.preprocess(xyz, s, q, o, None, col, 0, wv, full, cp, tf, tf, H, W)
    keys, pl, ranges = R.binning(pre, H, W)
    for k in ("xy", "conic_opacity", "rgb", "depth"):
        setattr(pre, k, getattr(pre, k).double())
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        color, depth, alpha, ncon, fT = R.render(pre, pl, ranges, H, W, bg)
    finally:
        torch.set_default_dtype(prev)
    rec = dict(xy=pre.xy[None], conic_opac=pre.conic_opacity[None], rgb_depth=torch.cat([pre.rgb, pre.depth[:, None]], 1)[None])
    ora = RA.render(rec, pl, ranges, H, W, bg.tolist())
    ok = ora["namb"] == 0
    assert int(ok.sum()) >= 0.99 * H * W, int((~ok).sum())
    for name, mine, ref in (("color", ora["nom"]["color"][0], color), ("depth", ora["nom"]["depth"][0], depth[0]),
                            ("alpha", ora["nom"]["alpha"][0], alpha[0]), ("final_T", ora["nom"]["final_T"][0], fT)):
        m = ok[0][None] if mine.dim() == 3 else ok[0]
        err = ((mine - ref).abs() / (1.0 + ref.abs()))[m.expand_as(mine)].max()
        assert float(err) <= 1e-12, (name, float(err))
    assert torch.equal(ora["nom"]["n_contrib"][0][ok[0]], ncon[ok[0]])
    assert ora["stats"]["stopped"] > 0 and len(keys) > P


@pytest.mark.parametrize("deg,H,W,mod,seed", [(1, 37, 53, 1.0, 5), (2, 40, 72, 0.8, 6), (3, 45, 30, 1.3, 7)])
def test_harness_sh_within_every_bound(harness, deg, H, W, mod, seed):
    """SH degree 1-3 with a third of the colours near the clamp at 0: records (conic, SH colour, clamp bits), planes and
    bytes of the serial harness within the oracle's bounds."""
    g = torch.Generator().manual_seed(seed)
    xyz, s, q, o, sh = BW.random_part(500, seed, deg)
    sh = BW.clamp_dc(sh, 0.3, g)
    cam = BW._cams(1, seed)[0]
    _, rep = _harness_scene([xyz, s, q, o, sh], deg, H, W, cam, torch.tensor([0.5, 0.3, 0.7]), harness, mod)
    print(rep)
    assert rep["clamped_bits"] >= 20 and rep["rec_rgb"] > 0


def test_harness_edge_scenes_within_every_bound(harness):
    """A 300-entry faint stack (two staging rounds), an opaque front over a long list, the 0.99 clamp and the T stop, and
    faint gaussians at the 1/255 threshold, through the serial harness."""
    H, W = 48, 64
    cam = BW._cams(1, 21)[0]
    g = torch.Generator().manual_seed(21)
    scene = BW.concat(faint_tile_stack(300, cam, H, W, (0, 0), g=g), opaque_front(cam, H, W, (2, 1), g=g),
                      faint_tile_stack(200, cam, H, W, (2, 1), tz0=2.0, g=g), BW.stack_part(3, 2, 6, cam, 0, g),
                      faint_threshold_part(400, cam, H, W, g))
    col = precomp_colours(scene[4], g)
    got, rep = _harness_scene(scene, -1, H, W, cam, torch.tensor([0.0, 1.0, 0.5]), harness, colours=col)
    print(rep)
    assert rep["max_list"] >= 300 and rep["stopped"] > 0 and rep["clamped"] > 0


@pytest.fixture(scope="module")
def control_scene():
    """Two cameras at 48 x 64: a 300-entry faint stack on tile (1, 0) (entry 255 contributes), an opaque stack reaching
    the 0.99 clamp and the T stop, and a random part; precomputed colours."""
    H, W = 48, 64
    cams = BW._cams(2, 31)
    g = torch.Generator().manual_seed(31)
    scene = BW.concat(faint_tile_stack(300, cams[0], H, W, (1, 0), g=g), BW.stack_part(3, 2, 6, cams[0], 0, g),
                      BW.random_part(600, 31, 0))
    col = torch.clamp(R.SH_C0 * scene[4][:, 0] + 0.5, min=0) * 1.3 - 0.1
    bg = torch.tensor([0.3, 0.6, 0.9])
    recs, vals, ranges = {"xy": [], "conic_opac": [], "rgb_depth": []}, [], []
    start = 0
    gx, gy = (W + 15) // 16, (H + 15) // 16
    for c, (wv, full, cp, tf) in enumerate(cams):
        pre = R.preprocess(scene[0], scene[1], scene[2], scene[3], None, col, 0, wv, full, cp, tf, tf, H, W)
        keys, pl, rg = R.binning(pre, H, W)
        recs["xy"].append(pre.xy)
        recs["conic_opac"].append(pre.conic_opacity)
        recs["rgb_depth"].append(torch.cat([pre.rgb, pre.depth[:, None]], 1))
        nz = rg[:, 1] > rg[:, 0]
        rg = rg.copy()
        rg[nz] += start
        vals.append(pl)
        ranges.append(rg)
        start += len(pl)
    rec = {k: torch.stack(v) for k, v in recs.items()}
    vals, ranges = np.concatenate(vals), np.concatenate(ranges)
    ora = RA.render(rec, vals, ranges, H, W, bg.tolist())
    assert int(ranges[1, 1] - ranges[1, 0]) >= 300, "tile (1, 0) of camera 0 must hold two staging rounds"
    assert ora["stats"]["stopped"] > 0 and ora["stats"]["clamped"] > 0
    return rec, vals, ranges, H, W, bg, ora


def test_replay_unmutated_passes(control_scene):
    rec, vals, ranges, H, W, bg, ora = control_scene
    rep = compare_replay(replay(rec, vals, ranges, H, W, bg), ora)
    print(rep)


@pytest.mark.parametrize("mut", MUTATIONS)
def test_negative_control_rejected(control_scene, mut):
    """Each mutation of the float32 replay fails the comparator by at least 10x its bound (inf: an exact mismatch of
    n_contrib, or a bound of 0), while the unmutated replay passes (test_replay_unmutated_passes)."""
    rec, vals, ranges, H, W, bg, ora = control_scene
    out = replay(rec, vals, ranges, H, W, bg, mut=mut)
    if mut == "round_q":
        r = _ratio_of(lambda: compare_replay(out, ora, planes=()))
    elif mut == "count_contributors":
        r = _ratio_of(lambda: compare_replay(out, ora, planes=("n_contrib",), rgba=False))
    else:
        r = _ratio_of(lambda: compare_replay(out, ora, rgba=False))
    print(f"{mut}: worst |err| / bound {r:.3g}")
    assert r >= 10.0, (mut, r)
    if mut == "eight_pixels":      # the rule this comparator replaces lets it through
        base = replay(rec, vals, ranges, H, W, bg)
        assert RA.loose_rule_accepts(out["color"][0], base["color"][0])
