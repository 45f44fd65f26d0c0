"""float64 restatement of the rasterizer forward's C ABI (a3d_raster_forward, a3d_raster_forward_rgba8 in include/a3d.h):
the per-(camera, gaussian) records the tile render consumes, and every output element of the render, each with a
per-element bound in the terms of oracle/abi_oracle.py (same Ref / check / assert_within; u32 = 2^-24, every bound
multiplied by SLACK = 2).

Records (`check_records`, from the float32 inputs).  xy and depth are pinned bit for bit to oracle/raster_oracle.py's float32
preprocess (the kernel's translation unit is built with --fmad=false and keeps its operation order; the sorted keys and tile
rectangles, which are built from them, are already bit-exact).  The conic and the SH colour are restated in float64 with a
running error bound (`E`): every float32 operation of the kernel, in the kernel's order, adds u32 |result| to the bound it
inherits from its operands (first order: a + b -> e_a + e_b; a b -> |a| e_b + |b| e_a; a / b -> (e_a + |a / b| e_b) / |b|;
sqrt a -> e_a / (2 sqrt a)).  This is a magnitude pass times counted u32 steps, with the magnitudes taken where cancellation
happens instead of at the inputs.
  conic      (c, -b, a) / det of the 2D covariance (a, b, c) incl. the +0.3 low-pass, det = a c - b^2: the bound carries
             (|a| e_c + |c| e_a + 2 |b| e_b) / |det| relative to the conic, i.e. the u32 steps of the covariance times the
             conditioning (|a c| + b^2) / |det|.
  colour     SH degree 0-3 with the view direction d / |d| (d = mean - campos), the basis polynomials and the sequential sum
             over the coefficients, + 0.5, max(., 0).  A `clamped` bit is exact unless the float64 channel lies within its
             bound of 0 (then either bit passes; the value check is unaffected, max(., 0) being 1-Lipschitz).
  opacity    an exact copy; depth in rgb_depth.w equals depth bit for bit; precomputed colours are exact copies.
Records of gaussians with radius 0 are never written and are not compared.

Render (`render`, from the kernel's own float32 records, point_list and ranges, so only the render's arithmetic is left):
one pixel walks its tile's list front to back (raster_render_forward_kernel, splat_alpha in a3d_raster_math.h).  a3d_raster.cu
is built without fast math, with FMA contraction allowed; a fused operation rounds once where the bound charges two.
  power      p = -0.5 (A dx^2 + C dy^2) - B dx dy, dx = fl(x - px): dx's rounding twice, two products, one sum and the
             final difference on the longest chain: |dp| <= 6 u32 p~, p~ = 0.5 (|A| dx^2 + |C| dy^2) + |B| |dx dy|.
  G          expf is accurate to 2 ulp = 4 u32 relative: |dG| <= G (expm1(|dp|) + 4 u32 e^|dp|).
  alpha      min(0.99f, o G): |da| <= o |dG| + u32 |o G| (the clamp is 1-Lipschitz).
  T          T_j = prod_{i <= j, live} fl(1 - a_i): relative error sum_i ((|da_i| + u32 (1 - a_i)) / (1 - a_i) + u32).
  w          a T_before: |dw| <= |da| T + a |dT| + u32 w.
  sums       C = sum_j c_j w_j in list order (sequential fp32): sum |c_j| |dw_j| + u32 sum |c_j w_j| + u32 sum_k |S_k|~, the
             last being the running sums of magnitudes at every add.  Depth (c = depth) and alpha (c = 1) the same.
  outputs    colour C + T bg (+ |bg| |dT| + 2 rounding steps), depth D, alpha A, final_T; n_contrib exact.
Empty tiles give bg, 0, 0, n_contrib 0 and final_T 1 exactly (bound 0).

Decisions.  power > 0 (skip), alpha < 1/255 (skip) and T_after < 1e-4 (stop) use the kernel's float32 thresholds.  One is
ambiguous when its float64 value lies within its own bound of the threshold; the 0.99 clamp is continuous and only counted.
A pixel with exactly one ambiguous decision is replayed with that decision flipped and passes if it matches either branch
in every plane (n_contrib exactly that branch's); a pixel with two or more (counting those met on the flipped branch) is
excluded and counted, and the caller caps the count.

RGBA8.  The bytes are q(clamp01(C + T bg)) and q(A), q(v) = trunc(fl(255 v)).  A byte passes when [255 (v - b), 255 (v + b)],
widened by the multiply's rounding u32 255 |v|, meets [byte, byte + 1): one level either way only where 255 v lies within
255 b of an integer.  `byte_got` turns a byte into the point of its level nearest 255 v, so `check` reports the distance."""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, NamedTuple, Optional

import numpy as np
import torch

from oracle import raster_oracle as R
from oracle.abi_oracle import F64, SLACK, U32, Ref, Verdict, assert_within, check  # noqa: F401  (re-exported for the tests)

TILE = 16
NPIX = TILE * TILE
ALPHA_MIN = float(np.float32(1.0) / np.float32(255.0))     # 1.0f / 255.0f
T_MIN = float(np.float32(1e-4))                              # 0.0001f
ALPHA_MAX = float(np.float32(0.99))                          # 0.99f
N_POW = 6                                                    # u32 steps of the power on its longest chain
EXP_ULP = 4 * U32                                            # 2 ulp of expf, relative
MAX_EXCLUDED = 2e-4     # pixels with two or more ambiguous decisions, as a share of a call's pixels.  Measured on an H100:
                        # 1 of 24 576 (4.1e-5) in the 1/255-threshold scene of the forward tests, none anywhere else


def f32c(x: float) -> float:
    """the float32 constant a literal `x`f of the kernel holds"""
    return float(np.float32(x))


# ------------------------------------------------------------------------------------------------ running error bounds
class E:
    """float64 value of a float32 expression and a first-order bound on |float32 result - value|."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    @staticmethod
    def of(x) -> "E":
        return x if isinstance(x, E) else E(torch.as_tensor(x, dtype=F64))

    def _r(self, v, e) -> "E":
        return E(v, e + U32 * (v.abs() + e))

    def __add__(a, b):
        b = E.of(b)
        return a._r(a.v + b.v, a.e + b.e)

    __radd__ = __add__

    def __sub__(a, b):
        b = E.of(b)
        return a._r(a.v - b.v, a.e + b.e)

    def __rsub__(a, b):
        return E.of(b) - a

    def __mul__(a, b):
        b = E.of(b)
        return a._r(a.v * b.v, a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e)

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = E.of(b)
        q = a.v / b.v
        return a._r(q, (a.e + q.abs() * b.e) / (b.v.abs() - b.e).clamp_min(1e-300))

    def __rtruediv__(a, b):
        return E.of(b) / a

    def __neg__(a):
        return E(-a.v, a.e)

    def sqrt(a):
        s = torch.sqrt(a.v.clamp_min(0))
        lo = torch.sqrt((a.v - a.e).clamp_min(0))
        return a._r(s, a.e / (s + lo).clamp_min(1e-300))

    def clamp(a, lo, hi):
        """min(hi, max(lo, a)) with constant-error bounds lo / hi (E)"""
        v = torch.minimum(hi.v, torch.maximum(lo.v, a.v))
        return E(v, torch.maximum(a.e, torch.maximum(lo.e, hi.e)))


def _quat_rot(q):
    r, x, y, z = q
    one = f32c(1.0)
    return [one - 2.0 * (y * y + z * z), 2.0 * (x * y - r * z), 2.0 * (x * z + r * y),
            2.0 * (x * y + r * z), one - 2.0 * (x * x + z * z), 2.0 * (y * z - r * x),
            2.0 * (x * z - r * y), 2.0 * (y * z + r * x), one - 2.0 * (x * x + y * y)]


def conic64(means, scales, rots, mod, wv, tanfovx, tanfovy, H, W):
    """(conA, conB, conC) as E, from float32 inputs [P,3], [P,3], [P,4] and one camera (preprocess_gaussian's order)."""
    d = lambda t: E(t.to(F64))
    px, py, pz = d(means[:, 0]), d(means[:, 1]), d(means[:, 2])
    vm = [float(v) for v in wv.reshape(16).float()]
    tp = lambda c: ((vm[c] * px + vm[4 + c] * py) + vm[8 + c] * pz) + vm[12 + c]
    tx, ty, tz = tp(0), tp(1), tp(2)
    tfx, tfy = E.of(f32c(tanfovx)), E.of(f32c(tanfovy))
    focal_x, focal_y = float(W) / (2.0 * tfx), float(H) / (2.0 * tfy)
    limx, limy = f32c(1.3) * tfx, f32c(1.3) * tfy
    txc = (tx / tz).clamp(-limx, limx) * tz
    tyc = (ty / tz).clamp(-limy, limy) * tz
    j00, j02 = focal_x / tz, -(focal_x * txc) / (tz * tz)
    j11, j12 = focal_y / tz, -(focal_y * tyc) / (tz * tz)
    m0 = [j00 * vm[4 * k] + j02 * vm[4 * k + 2] for k in range(3)]
    m1 = [j11 * vm[4 * k + 1] + j12 * vm[4 * k + 2] for k in range(3)]
    Rm = _quat_rot([d(rots[:, k]) for k in range(4)])
    s = [d(scales[:, k]) * f32c(mod) for k in range(3)]
    M = [Rm[i * 3 + k] * s[k] for i in range(3) for k in range(3)]
    dot = lambda i, j: (M[i * 3] * M[j * 3] + M[i * 3 + 1] * M[j * 3 + 1]) + M[i * 3 + 2] * M[j * 3 + 2]
    c = [dot(0, 0), dot(0, 1), dot(0, 2), dot(1, 1), dot(1, 2), dot(2, 2)]
    S = [[c[0], c[1], c[2]], [c[1], c[3], c[4]], [c[2], c[4], c[5]]]
    v0 = [(S[k][0] * m0[0] + S[k][1] * m0[1]) + S[k][2] * m0[2] for k in range(3)]
    v1 = [(S[k][0] * m1[0] + S[k][1] * m1[1]) + S[k][2] * m1[2] for k in range(3)]
    a = ((m0[0] * v0[0] + m0[1] * v0[1]) + m0[2] * v0[2]) + f32c(0.3)
    b = (m0[0] * v1[0] + m0[1] * v1[1]) + m0[2] * v1[2]
    cc = ((m1[0] * v1[0] + m1[1] * v1[1]) + m1[2] * v1[2]) + f32c(0.3)
    det_inv = 1.0 / (a * cc - b * b)
    return cc * det_inv, -b * det_inv, a * det_inv


_SH_C = [f32c(x) for x in (R.SH_C0, R.SH_C1) + R.SH_C2 + R.SH_C3]


def sh_colour64(deg, means, campos, sh):
    """rgb (E, 3 channels, before the clamp) of sh_colour: means [P,3], campos [3], sh [P,K,3] float32."""
    cp = [float(v) for v in campos.reshape(3).float()]
    dx, dy, dz = [E(means[:, k].to(F64)) - cp[k] for k in range(3)]
    n = ((dx * dx + dy * dy) + dz * dz).sqrt()
    x, y, z = dx / n, dy / n, dz / n
    c0, c1 = _SH_C[0], _SH_C[1]
    c2, c3 = _SH_C[2:7], _SH_C[7:14]
    b = [E.of(torch.full_like(x.v, c0))]
    if deg > 0:
        b += [-c1 * y, c1 * z, -c1 * x]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            b += [c2[0] * xy, c2[1] * yz, c2[2] * ((2.0 * zz - xx) - yy), c2[3] * xz, c2[4] * (xx - yy)]
            if deg > 2:
                b += [c3[0] * y * ((3.0 * xx) - yy), c3[1] * xy * z, c3[2] * y * ((4.0 * zz - xx) - yy),
                      c3[3] * z * ((2.0 * zz - 3.0 * xx) - 3.0 * yy), c3[4] * x * ((4.0 * zz - xx) - yy),
                      c3[5] * z * (xx - yy), c3[6] * x * (xx - 3.0 * yy)]
    out = []
    for ch in range(3):
        v = E.of(torch.zeros_like(x.v))
        for k in range(len(b)):
            v = v + b[k] * E(sh[:, k, ch].to(F64))
        out.append(v + f32c(0.5))
    return out


# ------------------------------------------------------------------------------------------------ records
class CamSpec(NamedTuple):
    viewmatrix: torch.Tensor     # [4,4] float32, row-vector convention
    projmatrix: torch.Tensor
    campos: torch.Tensor         # [3]
    tanfovx: float
    tanfovy: float


def check_records(means3D, scales, rotations, opacities, shs, colors, deg, per_cam, cams, H, W, mod, rec, radii):
    """Every visible (camera, gaussian) record against the float64 preprocess.  rec: dict of xy [cams,P,2], conic_opac
    [cams,P,4], rgb_depth [cams,P,4], clamped [cams,P] uint8 (any device); radii [cams,P] of the same forward.
    -> dict: worst |err| / bound per field, and counts of visible pairs, clamped bits and ambiguous clamp bits."""
    dev = means3D.device
    out = {"rec_conic": 0.0, "rec_rgb": 0.0, "visible": 0, "clamped_bits": 0, "ambiguous_bits": 0}
    for c, cam in enumerate(cams):
        g = (lambda t: t[c]) if per_cam else (lambda t: t)
        m, s, q = g(means3D), g(scales), g(rotations)
        vis = radii[c].to(dev) > 0
        out["visible"] += int(vis.sum())
        if not bool(vis.any()):
            continue
        mc, sc, qc = m.cpu().float(), s.cpu().float(), q.cpu().float()
        ref = R.preprocess(mc, sc, qc, opacities.cpu().float(), None if shs is None else shs.cpu().float(),
                           None if colors is None else colors.cpu().float(), deg, cam.viewmatrix.cpu(), cam.projmatrix.cpu(),
                           cam.campos.cpu(), cam.tanfovx, cam.tanfovy, H, W, mod)
        assert torch.equal(ref.radii, radii[c].cpu().to(torch.int32)), f"cam {c}: radii differ from the float32 preprocess"
        vc = vis.cpu()
        xy, co, cd = rec["xy"][c].cpu(), rec["conic_opac"][c].cpu(), rec["rgb_depth"][c].cpu()
        bad = (xy[vc] != ref.xy[vc]).any(-1)
        assert not bool(bad.any()), f"cam {c}: xy not bit-exact at gaussian {int(torch.nonzero(vc)[0][int(bad.nonzero()[0])])}"
        assert torch.equal(cd[vc, 3], ref.depth[vc]), f"cam {c}: depth not bit-exact"
        assert torch.equal(co[vc, 3], opacities.reshape(-1).cpu().float()[vc]), f"cam {c}: opacity is not an exact copy"
        cA, cB, cC = conic64(m.float(), s.float(), q.float(), mod, cam.viewmatrix.to(dev), cam.tanfovx, cam.tanfovy, H, W)
        where = lambda i, c=c, k=None: f"cam {c} gaussian {int(torch.nonzero(vc)[i // 3][0])} component {i % 3}"
        got = co[vc, :3].to(dev)
        val = torch.stack([cA.v, cB.v, cC.v], -1)[vis]
        bnd = SLACK * torch.stack([cA.e, cB.e, cC.e], -1)[vis]
        v = assert_within(got, Ref(val.reshape(-1), bnd.reshape(-1), where), f"cam {c} conic")
        out["rec_conic"] = max(out["rec_conic"], v.ratio)
        if colors is not None:
            assert torch.equal(cd[vc, :3], colors.cpu().float()[vc]), f"cam {c}: precomputed colours are not exact copies"
            assert int(rec["clamped"][c].cpu()[vc].count_nonzero()) == 0, f"cam {c}: clamp bits with precomputed colours"
            continue
        rgb = sh_colour64(deg, m.float(), cam.campos.to(dev), shs.float())
        raw = torch.stack([ch.v for ch in rgb], -1)[vis]
        bnd = SLACK * torch.stack([ch.e for ch in rgb], -1)[vis]
        v = assert_within(cd[vc, :3].to(dev), Ref(raw.clamp_min(0).reshape(-1), bnd.reshape(-1), where), f"cam {c} SH colour")
        out["rec_rgb"] = max(out["rec_rgb"], v.ratio)
        bits = rec["clamped"][c].to(dev)[vis].to(torch.int64)
        got_bits = torch.stack([(bits >> ch) & 1 for ch in range(3)], -1).bool()
        amb = raw.abs() <= bnd
        wrong = (got_bits != (raw < 0)) & ~amb
        assert not bool(wrong.any()), f"cam {c}: {int(wrong.sum())} clamp bits wrong"
        out["clamped_bits"] += int(got_bits.sum())
        out["ambiguous_bits"] += int(amb.sum())
    return out


# ------------------------------------------------------------------------------------------------ render
def _blend(g, px, py, bg, flip=None):
    """Front-to-back blend of B tiles' padded lists over their 256 pixels, in float64.  g: dict of [B, L] tensors (x, y, A,
    Bc, Cc, op, r, gr, b, d; valid bool); px, py [B, N].  flip: (P, A, T) bool [B, L, N] decisions to invert.
    -> dict of per-pixel [B, N] (or [B, 3, N]) values, raw bounds, n_contrib and counts."""
    u = U32
    dx = g["x"][..., None] - px[:, None, :]
    dy = g["y"][..., None] - py[:, None, :]
    A, Bc, Cc, op = (g[k][..., None] for k in ("A", "Bc", "Cc", "op"))
    valid = g["valid"][..., None].expand_as(dx)
    power = -0.5 * (A * dx * dx + Cc * dy * dy) - Bc * dx * dy
    e_p = N_POW * u * (0.5 * (A.abs() * dx * dx + Cc.abs() * dy * dy) + Bc.abs() * (dx * dy).abs())
    del dx, dy
    skipP = power > 0
    ambP = (power.abs() <= SLACK * e_p) & (e_p > 0)     # a bound of 0 is an exact result (dx = dy = 0): no ambiguity
    if flip is not None:
        skipP = skipP ^ flip[0]
    G = torch.exp(power.clamp(max=80.0))
    Ghi = torch.exp((power + e_p).clamp(max=80.0))      # G e^|dp| without 0 * inf where G underflows
    e_G = (Ghi - G) + EXP_ULP * Ghi
    del power, e_p
    araw = op * G
    e_al = op * e_G + u * araw
    del G, e_G
    clampA = araw > ALPHA_MAX
    alpha = araw.clamp(max=ALPHA_MAX)
    del araw
    skipA = alpha < ALPHA_MIN
    ambA = (alpha - ALPHA_MIN).abs() <= SLACK * e_al
    if flip is not None:
        skipA = skipA ^ flip[1]
    live = valid & ~skipP & ~skipA
    om = 1.0 - alpha
    rstep = torch.where(live, (e_al + u * om) / om + u, torch.zeros_like(om))
    T_after = torch.cumprod(torch.where(live, om, torch.ones_like(om)), dim=1)
    del om
    rel = torch.cumsum(rstep, dim=1)
    e_Ta = T_after * rel
    one = torch.ones_like(T_after[:, :1])
    T_before = torch.cat([one, T_after[:, :-1]], 1)
    e_Tb = T_before * (rel - rstep)
    del rel, rstep
    stop = live & (T_after < T_MIN)
    ambT = live & ((T_after - T_MIN).abs() <= SLACK * e_Ta)
    if flip is not None:
        stop = stop ^ (flip[2] & live)
    nstop = torch.cumsum(stop.to(torch.int32), dim=1)
    alive = nstop == 0
    evaluated = valid & ((nstop - stop.to(torch.int32)) == 0)
    del nstop
    contrib = live & alive
    kinds = (evaluated & ambP, evaluated & ~skipP & ambA, evaluated & ambT)
    namb = sum(k.sum(1) for k in kinds)
    cf = contrib.to(F64)
    w = alpha * T_before * cf
    e_w = (e_al * T_before + alpha * e_Tb + u * w) * cf
    del T_before, e_Tb
    pos = torch.arange(1, w.shape[1] + 1, device=w.device)[None, :, None]
    n_contrib = (pos * contrib).amax(1)
    last = (n_contrib - 1).clamp_min(0)[:, None, :]
    has = n_contrib > 0
    Tf = torch.where(has, torch.gather(T_after, 1, last)[:, 0], torch.ones_like(T_after[:, 0]))
    e_Tf = torch.where(has, torch.gather(e_Ta, 1, last)[:, 0], torch.zeros_like(T_after[:, 0]))

    def sum_of(c):
        t = c[..., None] * w if c is not None else w
        ta = t.abs()
        e = ((c[..., None].abs() * e_w) if c is not None else e_w).sum(1) + u * ta.sum(1) + u * (torch.cumsum(ta, 1) * cf).sum(1)
        return t.sum(1), e

    cols, ecols = [], []
    for ch, k in enumerate(("r", "gr", "b")):
        S, e = sum_of(g[k])
        out = S + Tf * bg[ch]
        cols.append(out)
        ecols.append(e + abs(bg[ch]) * e_Tf + u * (Tf * abs(bg[ch])) + u * (out.abs() + e))
    D, eD = sum_of(g["d"])
    Aa, eA = sum_of(None)
    return dict(color=torch.stack(cols, 1), e_color=torch.stack(ecols, 1), depth=D, e_depth=eD, alpha=Aa, e_alpha=eA,
                final_T=Tf, e_final_T=e_Tf, n_contrib=n_contrib, namb=namb, kinds=kinds,
                clamped=(clampA & contrib).sum(1), stopped=stop.any(1), evaluated=evaluated.sum(1))


PLANES = ("color", "depth", "alpha", "final_T")


def render(rec, vals, ranges, H, W, bg, chunk: Optional[int] = None):
    """Expected render of every camera from the kernel's records (rec: xy [cams,P,2], conic_opac [cams,P,4], rgb_depth
    [cams,P,4]), point_list `vals` (global, uint32 or int) and `ranges` [cams * tiles, 2] (global, as the binning tap returns
    them).  Runs on rec's device.  -> dict with, per branch ("nom", "alt"), values and SLACK-scaled bounds of every plane
    ([cams,3,H,W], [cams,H,W] ...) and n_contrib; per pixel `namb` (ambiguous decisions; the alt branch is meaningful where it
    is 1) and `excluded`; and counts: list lengths, clamped contributions, stopped pixels, replayed and excluded pixels."""
    dev = rec["xy"].device
    ncam, P = rec["xy"].shape[:2]
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    T = gx * gy
    vals = torch.as_tensor(np.asarray(vals).astype(np.int64) if not torch.is_tensor(vals) else vals).to(dev).long()
    ranges = torch.as_tensor(np.asarray(ranges).astype(np.int64) if not torch.is_tensor(ranges) else ranges).to(dev).long()
    ranges = ranges.reshape(ncam * T, 2)
    bgl = [float(b) for b in bg]
    npix = ncam * H * W
    res = {}
    for br in ("nom", "alt"):
        res[br] = {"color": torch.tensor(bgl, dtype=F64, device=dev)[None, :, None, None].expand(ncam, 3, H, W).clone(),
                   "depth": torch.zeros(ncam, H, W, dtype=F64, device=dev), "alpha": torch.zeros(ncam, H, W, dtype=F64, device=dev),
                   "final_T": torch.ones(ncam, H, W, dtype=F64, device=dev),
                   "n_contrib": torch.zeros(ncam, H, W, dtype=torch.int64, device=dev)}
        for k in PLANES:
            res[br]["b_" + k] = torch.zeros_like(res[br][k])
    namb_map = torch.zeros(ncam, H, W, dtype=torch.int64, device=dev)
    stats = dict(tiles=ncam * T, empty_tiles=0, max_list=0, clamped=0, stopped=0, replayed=0, excluded=0, pixels=npix,
                 evaluations=0)
    n = (ranges[:, 1] - ranges[:, 0]).clamp_min(0)
    stats["empty_tiles"] = int((n == 0).sum())
    stats["max_list"] = int(n.max()) if n.numel() else 0
    lid = torch.arange(NPIX, device=dev)
    chunk = chunk or (1 << 23 if dev.type == "cuda" else 1 << 20)
    nz = torch.nonzero(n > 0).reshape(-1)
    if nz.numel() == 0:
        return _finish(res, namb_map, stats)
    Lb = torch.clamp(2 ** torch.ceil(torch.log2(n[nz].to(F64))), min=16).long()
    for L in torch.unique(Lb).tolist():
        tiles = nz[Lb == L]
        per = max(1, chunk // (L * NPIX))
        for t0 in range(0, tiles.numel(), per):
            t = tiles[t0:t0 + per]
            B = t.numel()
            cam, tl = t // T, t % T
            j = torch.arange(L, device=dev)[None, :]
            idx = ranges[t, 0][:, None] + j
            valid = j < n[t][:, None]
            gid = vals[idx.clamp(max=vals.numel() - 1)] * valid
            flat = cam[:, None] * P + gid
            # padding entries read gaussian 0, whose record may be unwritten (culled): zero them, so no NaN enters a 0 * x
            pad = lambda t: torch.where(valid[..., None], t.to(F64), torch.zeros((), dtype=F64, device=dev))
            xy = pad(rec["xy"].reshape(-1, 2)[flat])
            co = pad(rec["conic_opac"].reshape(-1, 4)[flat])
            cd = pad(rec["rgb_depth"].reshape(-1, 4)[flat])
            g = dict(x=xy[..., 0], y=xy[..., 1], A=co[..., 0], Bc=co[..., 1], Cc=co[..., 2], op=co[..., 3],
                     r=cd[..., 0], gr=cd[..., 1], b=cd[..., 2], d=cd[..., 3], valid=valid)
            pxi = (tl % gx)[:, None] * TILE + lid[None, :] % TILE
            pyi = (tl // gx)[:, None] * TILE + lid[None, :] // TILE
            inside = (pxi < W) & (pyi < H)
            nom = _blend(g, pxi.to(F64), pyi.to(F64), bgl)
            one = (nom["namb"] == 1) & inside
            alt = nom
            if bool(one.any()):   # exactly one ambiguous decision in the pixel: its mask marks it
                flips = tuple(k & one[:, None, :] for k in nom["kinds"])
                alt = _blend(g, pxi.to(F64), pyi.to(F64), bgl, flip=flips)
            ci = cam[:, None].expand_as(pxi)[inside]
            yi, xi = pyi[inside], pxi[inside]
            for br, o in (("nom", nom), ("alt", alt)):
                d = res[br]
                d["color"][ci, :, yi, xi] = o["color"].permute(0, 2, 1)[inside]
                d["b_color"][ci, :, yi, xi] = SLACK * o["e_color"].permute(0, 2, 1)[inside]
                for k in ("depth", "alpha", "final_T"):
                    d[k][ci, yi, xi] = o[k][inside]
                    d["b_" + k][ci, yi, xi] = SLACK * o["e_" + k][inside]
                d["n_contrib"][ci, yi, xi] = o["n_contrib"][inside]
            na = nom["namb"].clone()
            na = torch.where(one & (alt["namb"] > 1), alt["namb"], na)
            namb_map[ci, yi, xi] = na[inside]
            stats["clamped"] += int(nom["clamped"][inside].sum())
            stats["stopped"] += int(nom["stopped"][inside].sum())
            stats["evaluations"] += int(nom["evaluated"][inside].sum())
    return _finish(res, namb_map, stats)


def _finish(res, namb_map, stats):
    res["namb"] = namb_map
    res["excluded"] = namb_map >= 2
    stats["replayed"] = int((namb_map == 1).sum())
    stats["excluded"] = int(res["excluded"].sum())
    res["stats"] = stats
    return res


# ------------------------------------------------------------------------------------------------ comparison
def _pixel_where(shape):
    def where(i):
        idx = np.unravel_index(int(i), shape)
        return "[cam, ...] index " + str(tuple(int(v) for v in idx))
    return where


def byte_got(got_bytes: torch.Tensor, value255: torch.Tensor) -> torch.Tensor:
    """the point of each byte's level [byte, byte + 1] nearest 255 v: check() then measures the distance from the level"""
    g = got_bytes.to(F64)
    return torch.minimum(torch.maximum(value255, g), g + 1.0)


def _ratio(x, v, b):
    """|x - v| / b per element: 0 where equal, inf where the bound is 0 or x is NaN"""
    r = ((x - v).abs() / b).nan_to_num(nan=math.inf, posinf=math.inf)
    return torch.where(x == v, torch.zeros_like(r), r)


def _branch_ratio(got, o, planes):
    """per pixel max over planes of |err| / bound"""
    r = None
    for k in planes:
        rr = _ratio(got[k].to(F64), o[k], o["b_" + k])
        rr = rr.amax(1) if k == "color" else rr
        r = rr if r is None else torch.maximum(r, rr)
    return r


def compare_forward(got: Dict[str, torch.Tensor], ora, max_excluded: float, what="", rgba: Optional[torch.Tensor] = None):
    """Every plane of a forward (got: color [cams,3,H,W], depth, alpha [cams,(1,)H,W]; n_contrib, final_T [cams,H,W]; any of
    them may be missing) and/or the RGBA8 bytes [cams,H,W,4] against `render`'s branches.  A pixel passes on the nominal
    branch, or, with exactly one ambiguous decision, on the flipped one; pixels with more are excluded (at most
    max_excluded of the pixels).  -> dict: worst |err| / bound per plane, and the counts."""
    dev = ora["nom"]["depth"].device
    ncam, H, W = ora["nom"]["depth"].shape
    g = {k: (v.to(dev).reshape(ncam, 3, H, W) if k == "color" else v.to(dev).reshape(ncam, H, W)) for k, v in got.items()}
    planes = [k for k in PLANES if k in g]
    exc = ora["excluded"]
    n_ex = int(exc.sum())
    assert n_ex <= max_excluded * exc.numel(), f"{what}: {n_ex} pixels excluded with two or more ambiguous decisions"
    nom, alt = ora["nom"], ora["alt"]
    single = ora["namb"] == 1
    # the branch the kernel took: nominal unless only the flipped one matches
    if planes or "n_contrib" in g:
        def ok(o):
            r = _branch_ratio(g, o, planes) if planes else torch.zeros(ncam, H, W, dtype=F64, device=dev)
            nc = (g["n_contrib"].long() == o["n_contrib"]) if "n_contrib" in g else torch.ones_like(r, dtype=torch.bool)
            return (r <= 1.0) & nc
        use_alt = single & ~ok(nom) & ok(alt)
    else:
        use_alt = torch.zeros(ncam, H, W, dtype=torch.bool, device=dev)
    if rgba is not None:
        rg = rgba.to(dev)
        rb = _byte_ratio(rg, nom)
        ra = _byte_ratio(rg, alt)
        use_alt = use_alt | (single & (rb > 1.0) & (ra <= 1.0))
    out = {"excluded": n_ex, "replayed": int(single.sum()), "took_alt": int(use_alt.sum())}
    sel = lambda k, x: torch.where(use_alt[:, None] if x.dim() == 4 else use_alt, alt[k], nom[k])
    for k in planes:
        v, b = sel(k, nom[k]), sel("b_" + k, nom[k])
        x = g[k].to(F64)
        e = exc[:, None].expand_as(v) if v.dim() == 4 else exc
        v = torch.where(e, x, v)
        b = torch.where(e, torch.zeros_like(b), b)
        out[k] = assert_within(x, Ref(v.reshape(-1), b.reshape(-1), _pixel_where(tuple(v.shape))), f"{what} {k}").ratio
    if "n_contrib" in g:
        want = torch.where(exc, g["n_contrib"].long(), sel("n_contrib", nom["n_contrib"]))
        bad = want != g["n_contrib"].long()
        if bool(bad.any()):
            i = int(torch.nonzero(bad.reshape(-1))[0])
            raise AssertionError(f"{what} n_contrib: {int(bad.sum())} pixels differ, first at "
                                 f"{_pixel_where(tuple(want.shape))(i)}: got {int(g['n_contrib'].reshape(-1)[i])}, "
                                 f"want {int(want.reshape(-1)[i])}")
        out["n_contrib"] = 0.0
    if rgba is not None:
        v255, b255 = _byte_ref(nom)
        va, ba = _byte_ref(alt)
        m = use_alt[..., None]
        v255, b255 = torch.where(m, va, v255), torch.where(m, ba, b255)
        x = rgba.to(dev)
        gb = byte_got(x, v255)
        gb = torch.where(exc[..., None], v255, gb)
        out["rgba8"] = assert_within(gb, Ref(v255.reshape(-1), b255.reshape(-1), _pixel_where(tuple(v255.shape))),
                                     f"{what} rgba8").ratio
    return out


def _byte_ref(o):
    """255 v and its bound for the 4 bytes of every pixel: [cams, H, W, 4]"""
    col = o["color"].clamp(0.0, 1.0)
    v = torch.cat([col, o["alpha"][:, None]], 1).permute(0, 2, 3, 1) * 255.0
    b = torch.cat([o["b_color"], o["b_alpha"][:, None]], 1).permute(0, 2, 3, 1) * 255.0
    return v, b + SLACK * U32 * v + 1e-300


def _byte_ratio(rgba, o):
    v, b = _byte_ref(o)
    d = (byte_got(rgba, v) - v).abs()
    return (d / b).amax(-1)


def loose_rule_accepts(got, ref, n_pixels=8, atol=5e-3):
    """The image check this module replaces: at most n_pixels off by more than 3e-5 + 1e-4 |ref|, none by atol or more."""
    bad = (got - ref).abs() > 3e-5 + 1e-4 * ref.abs()
    return int(bad.sum()) <= n_pixels and float((got - ref).abs().max()) < atol


# ------------------------------------------------------------------------------------------------ device taps
def tap_state(ws, P, H, W, ncam, cap, per_pixel=True):
    """Records of every camera (xy, conic_opac, rgb_depth, clamped, stacked over cameras), with per_pixel the n_contrib /
    final_T planes, and the global point_list / ranges of a forward's workspace `ws` (a3d_raster_state_tap,
    a3d_raster_binning_tap)."""
    from animate3d_b200 import _lib as L
    lib = L.load()
    dev = ws.device
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    out = {"xy": torch.empty(ncam, P, 2, device=dev), "conic_opac": torch.empty(ncam, P, 4, device=dev),
           "rgb_depth": torch.empty(ncam, P, 4, device=dev), "clamped": torch.empty(ncam, P, dtype=torch.uint8, device=dev)}
    if per_pixel:
        out["n_contrib"] = torch.empty(ncam, H, W, dtype=torch.int32, device=dev)
        out["final_T"] = torch.empty(ncam, H, W, device=dev)
    p = lambda k, c: C.c_void_p(out[k][c].data_ptr()) if k in out else None
    for c in range(ncam):
        L.check(lib.a3d_raster_state_tap(C.c_void_p(ws.data_ptr()), P, H, W, ncam, C.c_int64(cap), c, p("xy", c),
                                         p("conic_opac", c), p("rgb_depth", c), p("clamped", c), p("n_contrib", c),
                                         p("final_T", c), L.stream_ptr()))
    vals = torch.empty(cap, dtype=torch.int32, device=dev)
    ranges = torch.empty(ncam * gx * gy, 2, dtype=torch.int32, device=dev)
    L.check(lib.a3d_raster_binning_tap(C.c_void_p(ws.data_ptr()), P, H, W, ncam, C.c_int64(cap), 0, None,
                                       C.c_void_p(vals.data_ptr()), C.c_void_p(ranges.data_ptr()), L.stream_ptr()))
    torch.cuda.synchronize()
    out["vals"] = vals.long() & 0xFFFFFFFF
    out["ranges"] = ranges.long() & 0xFFFFFFFF
    return out


def cam_specs(settings):
    """CamSpec of each GaussianRasterizationSettings, as the C ABI sees it (float32)"""
    return [CamSpec(s.viewmatrix.float(), s.projmatrix.float(), s.campos.float(), f32c(s.tanfovx), f32c(s.tanfovy)) for s in settings]
