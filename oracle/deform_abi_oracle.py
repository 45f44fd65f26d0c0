"""float64 restatement of the deformation-field C ABI (a3d_deform_forward, a3d_deform_featmean, a3d_deform_backward in
include/a3d.h), with a per-element error bound for every output, in the terms of oracle/abi_oracle.py (same Ref / check /
assert_within; u32 = 2^-24, every bound multiplied by SLACK = 2).

Cells.  The kernel turns a normalised coordinate g into a texel position with float32 arithmetic,
fx = fl(fl(fl(g + 1) * 0.5) * (W - 1)), clamps it to [0, W - 1], takes x0 = floor(fx), x1 = min(x0 + 1, W - 1) and
wx = fx - x0 (exact).  `cell_axis` restates exactly that; everything after it runs in float64.  Restating the cell in float64
instead would put a coordinate-rounding term of about u32 W |texel step| on every sample, and near a texel boundary the two
pick different cells: linspace(-1, 1, 16) puts 6 of 16 frames one rounding below a texel of a 16-texel axis.  With the
kernel's own cells the only rounding left is in the arithmetic counted below.  `cells=torch.float64` gives the exact
grid_sample(align_corners=True, padding_mode="border") cells of the reference, to pin this module to it.

Bounds (first order; a "magnitude pass" is the same computation on |texels|, |W1|, |W2| and |upstream gradients|, written
S~, F~, H~, O~, D~ below):

  sample     s = (t00 (1 - wx) + t01 wx)(1 - wy) + (t10 (1 - wx) + t11 wx) wy: a term passes 2 weight roundings, 2 products
             and 2 sums: |ds| <= 6 u32 S~.
  feature    f = prod of the 6 plane samples of a scale (5 roundings): |df| <= (6 * 6 + 6) u32 F~, F~ = prod S~.
  MLP        a = W1 f, 32-term fused sums: |da| <= 32 u32 H~ + |W1| |df|, H~ = |W1| F~; the ReLU is 1-Lipschitz;
             o = W2 relu(a): |do| <= 32 u32 O~ + |W2| |da|, O~ = |W2| H~.
  outputs    means = xyz + o0 (+ u32 |.|); scales = expf(scaling + o2): |exp| (|d arg|) + 4 u32 |exp| (expf is within 2 ulp,
             the library builds without fast-math); rotations y = q / |q|, q = base + o1: |dy_k| <= |dq_k| / |q| + |y_k| d|q| / |q|
             + u32 |y_k|, d|q| <= sum |y_j| |dq_j| + 4 u32 |q|.
  featmean   (1 / P) sum_i f_i: per thread ceil(P / 2048) items, then 256 threads and 8 CTAs in a fixed order, then / P:
             (ceil(P / 2048) + 264) u32 mean F~ + mean |df| + u32 |mean|.
  backward   dout: g_means exactly; g_scales exp(.) with the scale bound above; (g - y (y.g)) / |q| with the errors of y and |q|
             carried through (u32 per operation).  dh = [a > 0] W2^T dout (4 fused terms): |W2|^T |ddout| + 4 u32 |W2|^T D~.
             A ReLU whose pre-activation lies within SLACK |da| of 0 may take either branch: it is charged the whole
             |W2|^T D~ + its own bound and reported (`ambiguous`).  dfeat = sum_m W1_m^T dh_m (32 fused terms per MLP, 3 sums):
             |W1|^T (|ddh| + 35 u32 |dh|~).  The featmean fold adds g_featmean / P (3 roundings).  The factor of plane p is
             d * prod_{q != p} s_q: (|dd| + 36 u32 D~) prod_{q != p} S~.  A corner's term w * factor adds 4 u32 (the float32
             corner weight and the product).
  sums       a texel of the plane-gradient scratch is init + the terms of the n (item, corner) pairs that touch it; in any
             order (atomics, or the fixed-order gather) that sum is within n u32 (sum |terms| + |init|) of the exact one.
             A weight-gradient entry is summed per CTA over its items in a fixed chain (at most L = 128 * ceil(chunks / CTAs)
             fused steps), then over the C = min(chunks, 2 * SM) CTAs (atomics, or the CTA-ordered reduce) into init:
             (L + C) u32 (sum |terms| + |init|).  The per-term errors (|ddh| F~ + |dh|~ |df| for W1, |ddout| H~ + D~ |da| for
             W2, the factor's bound for planes) add on top.

A bound is a worst case, not a statistic: elements the call must not write carry bound 0 and their pre-call contents, and a
weight-gradient MLP whose upstream gradient is zero must keep its initial value exactly."""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import torch

from oracle.abi_oracle import F64, SLACK, U32, Ref, assert_within, check  # noqa: F401  (re-exported for the tests)

PLANE_AXES = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))   # (coordinate indexing W, coordinate indexing H) of each plane
CHANNELS = 16
HIDDEN = 32
OUT_DIMS = (3, 4, 3)            # xyz, rotation, scale MLPs
BWD_THREADS = 128               # items per chunk of the backward kernel
FM_THREADS, FM_CTAS = 256, 8    # featmean: threads per CTA, CTAs per frame

C_SAMPLE = 6                    # u32 steps of one bilinear sample
C_FEAT = 6 * C_SAMPLE + 6       # the 6-plane product


def cell_axis(g: torch.Tensor, n: int, cells=torch.float32):
    """One axis of grid_sample(align_corners=True, padding_mode="border") on an axis of n texels: (i0, i1, w0, w1) with the
    two texel indices and their float64 weights, the position computed in `cells` arithmetic."""
    f = ((g.to(cells) + 1) * 0.5) * (n - 1)
    f = f.clamp(0, n - 1)
    i0 = torch.floor(f)
    w = (f - i0).to(F64)
    i0 = i0.long()
    return i0, torch.clamp(i0 + 1, max=n - 1), 1 - w, w


def _featmean_fold(g_featmean: torch.Tensor, P: int) -> torch.Tensor:
    """d loss / d feature of every gaussian of a frame from d loss / d (mean feature of the frame)."""
    return g_featmean / P


def _bilerp(tex: torch.Tensor, W: int, ay, ax) -> torch.Tensor:
    iy0, iy1, vy0, vy1 = ay
    ix0, ix1, vx0, vx1 = ax
    t = lambda iy, ix: tex[iy * W + ix]
    return ((t(iy0, ix0) * vx0[:, None] + t(iy0, ix1) * vx1[:, None]) * vy0[:, None]
            + (t(iy1, ix0) * vx0[:, None] + t(iy1, ix1) * vx1[:, None]) * vy1[:, None])


def sample(plane: torch.Tensor, gx: torch.Tensor, gy: torch.Tensor, cells=torch.float32) -> torch.Tensor:
    """Bilinear border-clamped sample of plane [C, H, W] (any leading 1s) at normalised (gx -> W, gy -> H): [n, C] float64."""
    C, H, W = plane.shape[-3:]
    tex = plane.reshape(C, H * W).t().to(F64)
    return _bilerp(tex, W, cell_axis(gy, H, cells), cell_axis(gx, W, cells))


def _rep_items(x: torch.Tensor, T: int) -> torch.Tensor:
    """Per-gaussian rows [P, k] -> per-item rows [T P, k] (item t P + i)."""
    return x.reshape(x.shape[0], -1).to(F64).repeat(T, 1)


class Field:
    """The deformation field of T frames x P gaussians as a3d_deform_* sees it: `planes` is the flat list of
    6 * num_scales [1, 16, H, W] (or [16, H, W]) grids in the ABI's order, `w1s` / `w2s` the [32, nfeat] / [out, 32] weights of
    the xyz, rotation and scale MLPs, `rot_base` the optional [T, P, 4] base quaternions.  Tensors may live on any device;
    the restatement runs on xyz's device."""

    def __init__(self, xyz, scaling, rotation, times, planes: Sequence[torch.Tensor], w1s, w2s, deform_scale, rot_base=None,
                 cells=torch.float32):
        self.P, self.T = xyz.shape[0], times.shape[0]
        self.n = self.P * self.T
        self.S = len(planes) // 6
        self.nfeat = self.S * CHANNELS
        self.deform_scale = bool(deform_scale)
        dev = xyz.device
        P, T = self.P, self.T
        self.pts = torch.cat([xyz.float().repeat(T, 1), times.float().to(dev).repeat_interleave(P)[:, None]], 1)   # [n, 4]
        self.hw = []                  # [s][p] (H, W)
        self.cells = []               # [s][p] (ay, ax)
        self.smp, self.sabs = [], []  # [s][p] [n, 16]
        feat, fabs = [], []
        for s in range(self.S):
            hw, cl, sm, sa = [], [], [], []
            f = torch.ones(self.n, CHANNELS, dtype=F64, device=dev)
            fa = torch.ones_like(f)
            for p, (a, b) in enumerate(PLANE_AXES):
                pl = planes[s * 6 + p]
                H, W = pl.shape[-2:]
                tex = pl.reshape(CHANNELS, H * W).t().to(F64).to(dev)
                ay, ax = cell_axis(self.pts[:, b], H, cells), cell_axis(self.pts[:, a], W, cells)
                v, va = _bilerp(tex, W, ay, ax), _bilerp(tex.abs(), W, ay, ax)
                hw.append((H, W)); cl.append((ay, ax)); sm.append(v); sa.append(va)
                f, fa = f * v, fa * va
            self.hw.append(hw); self.cells.append(cl); self.smp.append(sm); self.sabs.append(sa)
            feat.append(f); fabs.append(fa)
        self.feat, self.fabs = torch.cat(feat, 1), torch.cat(fabs, 1)
        self.ef = C_FEAT * U32 * self.fabs
        self.w1 = [w.to(F64).to(dev) for w in w1s]
        self.w2 = [w.to(F64).to(dev) for w in w2s]
        self.a, self.ea, self.habs, self.hid, self.out, self.eo, self.oabs = [], [], [], [], [], [], []
        for m in range(3):
            w1a, w2a = self.w1[m].abs(), self.w2[m].abs()
            a = self.feat @ self.w1[m].t()
            habs = self.fabs @ w1a.t()
            ea = HIDDEN * U32 * habs + self.ef @ w1a.t()
            hid = a.clamp_min(0)
            o = hid @ self.w2[m].t()
            oabs = habs @ w2a.t()
            self.a.append(a); self.ea.append(ea); self.habs.append(habs); self.hid.append(hid); self.out.append(o)
            self.oabs.append(oabs); self.eo.append(HIDDEN * U32 * oabs + ea @ w2a.t())
        # outputs
        self.means = self.pts[:, :3].to(F64) + self.out[0]
        self.e_means = self.eo[0] + U32 * (self.pts[:, :3].to(F64).abs() + self.oabs[0])
        sc = _rep_items(scaling.to(dev), T)
        arg, earg = sc, torch.zeros_like(sc)
        if self.deform_scale:
            arg = sc + self.out[2]
            earg = self.eo[2] + U32 * (sc.abs() + self.oabs[2])
        self.scales = torch.exp(arg)
        self.e_scales = self.scales * earg * (1 + 2 * earg) + 4 * U32 * self.scales
        qb = rot_base.reshape(-1, 4).to(F64).to(dev) if rot_base is not None else _rep_items(rotation.to(dev), T)
        q = qb + self.out[1]
        eq = self.eo[1] + U32 * (qb.abs() + self.oabs[1])
        self.qn = q.norm(dim=1, keepdim=True).clamp_min(1e-12)
        self.y = q / self.qn
        self.eqn = (self.y.abs() * eq).sum(1, keepdim=True) + 4 * U32 * self.qn
        self.e_y = eq / self.qn + self.y.abs() * self.eqn / self.qn + U32 * self.y.abs()

    def _item_where(self, k: int, name: str):
        return lambda i: f"{name}: frame {i // k // self.P}, gaussian {(i // k) % self.P}, component {i % k}"

    # ------------------------------------------------------------------------------------------ forward
    def forward(self) -> Dict[str, Ref]:
        """a3d_deform_forward: means / scales [T, P, 3], rotations [T, P, 4]."""
        out = {}
        for name, v, e, k in (("means", self.means, self.e_means, 3), ("scales", self.scales, self.e_scales, 3),
                              ("rotations", self.y, self.e_y, 4)):
            out[name] = Ref(v.reshape(-1), (SLACK * e).reshape(-1), self._item_where(k, name))
        return out

    def featmean(self) -> Ref:
        """a3d_deform_featmean: [T, nfeat], the mean feature of every frame."""
        T, P, nf = self.T, self.P, self.nfeat
        v = self.feat.view(T, P, nf).mean(1)
        steps = math.ceil(P / (FM_THREADS * FM_CTAS)) + FM_THREADS + FM_CTAS
        e = self.ef.view(T, P, nf).mean(1) + steps * U32 * self.fabs.view(T, P, nf).mean(1) + U32 * v.abs()
        return Ref(v.reshape(-1), (SLACK * e).reshape(-1), lambda i: f"featmean: frame {i // nf}, channel {i % nf} ({P} gaussians)")

    # ------------------------------------------------------------------------------------------ backward
    def backward(self, g_means=None, g_scales=None, g_rots=None, g_featmean=None, *, sm_count: int,
                 grad_planes: Optional[Sequence[Optional[torch.Tensor]]] = None,
                 grad_w1: Optional[Sequence[Optional[torch.Tensor]]] = None,
                 grad_w2: Optional[Sequence[Optional[torch.Tensor]]] = None,
                 grad_rot_base: Optional[torch.Tensor] = None):
        """a3d_deform_backward.  The grad_* arguments are the output buffers' contents BEFORE the call (None: the pointer is
        null): plane-gradient scratch [H, W, 16] channel-last, weight gradients [32, nfeat] / [out, 32], d/d rot_base
        [T, P, 4].  Returns (dict name -> Ref, number of ambiguous ReLUs)."""
        n, P, T, nf = self.n, self.P, self.T, self.nfeat
        dev = self.feat.device
        z = lambda k: torch.zeros(n, k, dtype=F64, device=dev)
        dout, ed, dabs = [z(3), z(4), z(3)], [z(3), z(4), z(3)], [z(3), z(4), z(3)]
        if g_means is not None:
            dout[0] = g_means.reshape(n, 3).to(F64).to(dev)
            dabs[0] = dout[0].abs()
        if self.deform_scale and g_scales is not None:
            g = g_scales.reshape(n, 3).to(F64).to(dev)
            dout[2] = g * self.scales
            ed[2] = g.abs() * self.e_scales + U32 * dout[2].abs()
            dabs[2] = dout[2].abs()
        if g_rots is not None:
            g = g_rots.reshape(n, 4).to(F64).to(dev)
            y, ey, qn, eqn = self.y, self.e_y, self.qn, self.eqn
            dot = (y * g).sum(1, keepdim=True)
            edot = (ey * g.abs()).sum(1, keepdim=True) + 4 * U32 * (y * g).abs().sum(1, keepdim=True)
            num = g - y * dot
            enum = ey * dot.abs() + y.abs() * edot + 2 * U32 * (g.abs() + y.abs() * dot.abs())
            dout[1] = num / qn
            ed[1] = enum / qn + num.abs() / qn * eqn / qn + U32 * dout[1].abs()
            dabs[1] = (g.abs() + y.abs() * (y * g).abs().sum(1, keepdim=True)) / qn
        ambiguous = 0
        dh, edh, dhabs = [], [], []
        for m in range(3):
            w2a = self.w2[m].abs()
            pre = dout[m] @ self.w2[m]
            epre = ed[m] @ w2a + 4 * U32 * (dabs[m] @ w2a)
            pabs = dabs[m] @ w2a
            on = self.a[m] > 0
            amb = (self.a[m].abs() <= SLACK * self.ea[m]) & (pabs > 0)
            ambiguous += int(amb.sum())
            dh.append(torch.where(on, pre, torch.zeros_like(pre)))
            edh.append(torch.where(amb, pabs + epre, torch.where(on, epre, torch.zeros_like(epre))))
            dhabs.append(torch.where(on | amb, pabs, torch.zeros_like(pabs)))
        dfeat = sum(dh[m] @ self.w1[m] for m in range(3))
        dfabs = sum(dhabs[m] @ self.w1[m].abs() for m in range(3))
        edf = sum((edh[m] + 35 * U32 * dhabs[m]) @ self.w1[m].abs() for m in range(3))
        d, dd, dda = dfeat, edf, dfabs
        if g_featmean is not None:
            fold = _featmean_fold(g_featmean.reshape(T, nf).to(F64).to(dev), P).repeat_interleave(P, 0)
            d = dfeat + fold
            dd = edf + U32 * (dfabs + fold.abs()) + 2 * U32 * fold.abs()
            dda = dfabs + fold.abs()
        refs: Dict[str, Ref] = {}
        # ---- plane gradients
        for s in range(self.S):
            for p in range(6):
                H, W = self.hw[s][p]
                init = None if grad_planes is None else grad_planes[s * 6 + p]
                if init is None:
                    continue
                cs = slice(s * CHANNELS, (s + 1) * CHANNELS)
                others = torch.ones_like(d[:, cs])
                oabs = torch.ones_like(d[:, cs])
                for q in range(6):
                    if q != p:
                        others, oabs = others * self.smp[s][q], oabs * self.sabs[s][q]
                fac = d[:, cs] * others
                efac = (dd[:, cs] + 36 * U32 * dda[:, cs]) * oabs
                fabs = dda[:, cs] * oabs
                val = init.reshape(H * W, CHANNELS).to(F64).to(dev).clone()
                esum = torch.zeros_like(val)
                asum = torch.zeros_like(val)
                cnt = torch.zeros(H * W, dtype=F64, device=dev)
                (iy0, iy1, vy0, vy1), (ix0, ix1, vx0, vx1) = self.cells[s][p]
                for iy, vy in ((iy0, vy0), (iy1, vy1)):
                    for ix, vx in ((ix0, vx0), (ix1, vx1)):
                        w = (vy * vx)[:, None]
                        key = iy * W + ix
                        val.index_add_(0, key, fac * w)
                        esum.index_add_(0, key, w * (efac + 4 * U32 * fabs))
                        asum.index_add_(0, key, w * fabs)
                        cnt.index_add_(0, key, torch.ones_like(w[:, 0]))
                init64 = init.reshape(H * W, CHANNELS).to(F64).to(dev)
                bound = SLACK * (esum + cnt[:, None] * U32 * (asum + init64.abs()))
                counts = cnt.cpu()

                def where(i, s=s, p=p, W=W, counts=counts):
                    texel, c = divmod(int(i), CHANNELS)
                    return (f"grad_planes[{s * 6 + p}] (scale {s}, plane {p}): texel (y {texel // W}, x {texel % W}), channel {c}, "
                            f"{int(counts[texel])} (item, corner) terms")
                refs[f"grad_planes[{s * 6 + p}]"] = Ref(val.reshape(-1), bound.reshape(-1), where)
        # ---- weight gradients: per-CTA chains of at most `chain` items, then `ctas` partial sums
        chunks = -(-n // BWD_THREADS)
        ctas = min(chunks, 2 * sm_count)
        chain = BWD_THREADS * -(-chunks // ctas)
        steps = chain + ctas
        for m in range(3):
            for kind, init in (("grad_w1", None if grad_w1 is None else grad_w1[m]),
                               ("grad_w2", None if grad_w2 is None else grad_w2[m])):
                if init is None:
                    continue
                i64 = init.to(F64).to(dev)
                if kind == "grad_w1":
                    v = i64 + dh[m].t() @ self.feat
                    e = edh[m].t() @ self.fabs + dhabs[m].t() @ self.ef
                    a = dhabs[m].t() @ self.fabs
                else:
                    v = i64 + dout[m].t() @ self.hid[m]
                    e = ed[m].t() @ self.habs[m] + dabs[m].t() @ self.ea[m]
                    a = dabs[m].t() @ self.habs[m]
                bound = SLACK * (e + steps * U32 * (a + i64.abs()))
                cols = v.shape[1]

                def where(i, kind=kind, m=m, cols=cols):
                    return (f"{kind}[{m}] entry (row {int(i) // cols}, col {int(i) % cols}): {n} items in {ctas} CTAs of at most "
                            f"{chain} items each")
                refs[f"{kind}[{m}]"] = Ref(v.reshape(-1), bound.reshape(-1), where)
        if grad_rot_base is not None:
            if g_rots is not None:
                refs["grad_rot_base"] = Ref(dout[1].reshape(-1), (SLACK * ed[1]).reshape(-1), self._item_where(4, "grad_rot_base"))
            else:
                v = grad_rot_base.reshape(-1).to(F64).to(dev)
                refs["grad_rot_base"] = Ref(v, torch.zeros_like(v), self._item_where(4, "grad_rot_base (must stay untouched)"))
        return refs, ambiguous
