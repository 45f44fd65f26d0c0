"""float64 restatement of the ARAP C ABI (a3d_knn_graph and a3d_arap in include/a3d.h), with a per-element error bound for
every output, in the terms of oracle/abi_oracle.py (same Ref / check / assert_within; u32 = 2^-24, every bound multiplied by
SLACK = 2).  Built on oracle/arap_oracle.py (pinned to the reference's systems/util.py) without changing it.

Discrete decisions are replayed exactly.  The edges e = x_i - x_j are computed in the dtype of `nodes`: for float32 nodes
that is one correctly rounded IEEE subtraction, the same bits the kernel's edge gather (a3d_arap_math.h:arap_gather)
produces, so edge rounding contributes nothing to the bounds below; float64 nodes give the float64 edges of
arap_oracle.arap_error.  Slot validity (-1 or >= Nv is absent, j == i is a zero edge), sample entries outside [0, Nv) (they
contribute nothing) and the same-axis rule (util.py:152-153: an axis whose K edge components are all unchanged sets S = 0,
R = I) are decided on those exact edges.  Everything after runs in float64.

ARAP, per (frame t >= 1, sample entry) with edges s_n (frame 0), t_n (frame t) and weights w_n:
  S = sum_n w_n s_n t_n^T; R = the reference's SVD rotation with the reflection fix (arap_oracle.estimate_rotation);
  energy sum_n w_n |t_n - R s_n|^2, g_t[n] = 2 w_n (t_n - R s_n), g_0[n] = -R^T g_t[n] = -2 w_n (R^T t_n - s_n).
  The scatter is the ABI's: frame t gets +g_t at i and -g_t at j, frame 0 gets +-g_0 of every frame; repeated samples add
  once per occurrence.

Bounds (first order; S~ = sum_n |w_n s_n t_n^T| is the magnitude pass of S, |x|_1 / |x|_2 vector norms):

  S          the kernel's fp32 S: K fused or unfused multiply-adds of 3-factor products: |dS| <= (K + 2) u32 S~.
  rotation   the kernel takes the quaternion of Horn's symmetric 4x4 N(S) (|N|_F = 2 |S|_F) from a cyclic Jacobi of 8 sweeps
             x 6 plane rotations.  Forming N adds 2 roundings per entry.  One fp32 plane rotation is an exact orthogonal
             similarity of a matrix perturbed by at most 24 u32 |N|_F (two one-sided updates of 3 u32 each, and the
             non-orthogonality of the computed (c, s), 2 x 9 u32), so the 48 of them are exact for N + E,
             |E| <= eN = 2 (K + 2) u32 |S~|_F + 2 u32 |N+(S~)|_F + 1152 u32 |N|_F, with N+ the map N with every sign +.
             By Davis-Kahan the computed quaternion lies within sin(a) <= eN / (gap - eN) of the eigenvector, gap = lambda1 -
             lambda2 of the float64 N of the exact S; the accumulated V drifts by 48 x 12 u32 more.  Quaternions an angle a
             apart give rotations with |R - R'|_2 = 2 sin(a), so dR = min(2, 2 (eN / (gap - eN) + 576 u32)) (2 when gap <=
             eN: any two rotations).  Normalising q and forming R adds 24 u32 per entry (|q| = 1).
  rank 1     when the top eigenvalue is (nearly) double -- a rank-1 S: collinear frame-0 edges, K = 1, one valid slot -- the
             maximiser is a one-parameter family q(psi) = cos psi q1 + sin psi q2 of the top-2 eigenvectors, and the kernel
             returns some member.  Then dR uses gap2 = lambda2 - lambda3 (the distance to the top-2 subspace), and since R is
             quadratic in q, R(psi) = A + B cos 2 psi + C sin 2 psi with A = (R(q1) + R(q2)) / 2, B = (R(q1) - R(q2)) / 2,
             C = R((q1 + q2) / sqrt 2) - A.  Every output is linear in R s_n, R^T t_n and t_n . R s_n, so it is bounded about
             its value at A by the family's spread sqrt((B x)^2 + (C x)^2).  When every t_n is parallel to the common image
             of the s_n, as for one edge or collinear edges that stay collinear, B s_n, C s_n, B^T t_n and C^T t_n vanish and
             the bound is as tight as a full-rank fit: it bounds R s_n, not R.  The mode with the smaller dR + relative
             spread is used per (frame, sample).  S = 0 (same-axis rule or no weighted edge) gives the kernel's exact R = I.
             When collinear frame-0 edges are no longer parallel at frame t, g_0 = -2 w (R^T t_n - s_n) genuinely depends on
             the member (the reference's SVD picks one arbitrarily too): the spread is then of the size of g_0 itself, and
             the tightness check below reports the bound as vacuous instead of passing it.
  R s        a = R s: dR |s|_2 + (24 + 3) u32 |s|_1 (the R entries, and 3 roundings of a 3-term dot) [+ spread];
             d = t - a: ed = ea + u32 (|t| + |s|_1).
  g_t        fl(2 w d): 2 |w| (ed + spread + u32 (|d| + ed)).
  g_0        -2 w fl(R^T d): 2 |w| (dR |d|_2 + (24 + 4) u32 |d|_1 + |ed|_2 + spread of R^T t + u32 |g_0 / 2w|).
  energy     w |d|^2 per slot (|d|^2 - |d*|^2 <= sum 2 |d| ed + ed^2, exact in ed, which matters for rigid motion where
             d is itself a rounding residual) + 4 u32 |w| (|d| + ed)^2 for the squares, sum and weight; the K slots of a
             node add in order (K u32 of their magnitudes).  The (Nt - 1) Ns node energies are summed: the atomic kernel by
             warp shuffles (5), a 4-warp sum (3) and one float atomic per CTA of 128 (arbitrary order):
             8 + ceil(M / 128) steps; the fixed-order path per thread of 1024 then a 10-level tree: ceil(M / 1024) + 10.
  gradient   an element reached by m (entry, slot, frame) contributions, in any order (atomics, or the fixed-order gather):
             sum of their bounds + m u32 sum (|g| + bound).

Tightness: every Ref comes with a magnitude pass (`mag`, the same sums over |w| (|t| + |s|)^2 and 2 |w| (|t| + |s|_2)).
An element whose bound reaches its magnitude would accept any value of that size, including 0 or the negated result: such
a bound is vacuous, and `tightness` reports it so that the tests fail on it.

KNN (a3d_knn_graph).  The kernel's squared distance of a pair is fp32 dx^2 + dy^2 + dz^2 of fp32 differences (fused or
not): relative to the float64 distance of the fp32 points, |d32 - d64| <= 5 u32 d64 + 3 * 2^-150 (a rounding on each
difference, the squares and the sums; all terms are >= 0; the subnormal half-spacing), and d32 == d64 == 0 for coincident
points.  Integer points with |x| <= 2^10 have every intermediate exact: bound 0.  The kernel keeps the K + 1 first in
(d32, index) order and drops the first of them, which is the lowest-index point coincident with i -- i itself unless a
lower-index point shares its position.  `knn_check` accepts a result when dist2 is within its bound and ascending, the
indices are distinct and in range and omit the dropped point, every point not returned is no nearer than the K-th returned
one up to the two bounds, and every rank whose float64 distance is separated from its neighbours' by more than their bounds
(or tied exactly with exact distances) holds the (distance, index)-order index."""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import torch

from oracle.abi_oracle import F64, SLACK, U32, Ref, assert_within, check  # noqa: F401  (re-exported for the tests)

C_JACOBI = 24 * 48          # u32 steps of |E| / |N|_F over 8 sweeps x 6 plane rotations
C_VDRIFT = 12 * 48          # u32 drift of the accumulated eigenvector
C_QUAT = 24                 # u32 per R entry from the normalised quaternion
KNN_EPS = 5 * U32           # relative bound of the fp32 squared distance
SUBNORMAL = 3 * 2.0 ** -150
ARAP_THREADS = 128          # atomic kernel: CTA size
SUM_THREADS = 1024          # fixed-order energy sum: one CTA
LINALG_BATCH = 1 << 16      # matrices per batched eigh / svd call, run on the CPU


class Out(NamedTuple):
    ref: Ref
    mag: torch.Tensor           # magnitude pass, float64, same shape as ref.value


class Tightness(NamedTuple):
    median_rel: float           # median bound / |value| over the non-zero values
    worst_rel: float            # worst bound / |value| over the non-zero values
    worst_mag: float            # worst bound / magnitude (>= 1: vacuous)
    vacuous: int                # elements whose bound reaches their magnitude


def tightness(out: Out) -> Tightness:
    v, b, m = out.ref.value.abs(), out.ref.bound, out.mag.to(out.ref.bound.device)
    nz = v > 0
    rel = b[nz] / v[nz]
    pos = m > 0
    bm = b[pos] / m[pos]
    return Tightness(float(rel.median()) if rel.numel() else 0.0, float(rel.max()) if rel.numel() else 0.0,
                     float(bm.max()) if bm.numel() else 0.0, int((bm >= 1).sum()) + int(((b > 0) & ~pos).sum()))


# ------------------------------------------------------------------------------------------------ rotations
def horn_n(S: torch.Tensor, absolute: bool = False) -> torch.Tensor:
    """Horn's symmetric 4x4 N(S) for S [..., 3, 3] (S[a][b] = sum w s_a t_b), as a3d_arap_math.h forms it; `absolute` puts
    a + on every term (the magnitude pass)."""
    s = S.abs() if absolute else S
    g = (lambda x: x.abs()) if absolute else (lambda x: x)       # a signed term of N, or its magnitude
    n = S.new_zeros(S.shape[:-2] + (4, 4))
    n[..., 0, 0] = s[..., 0, 0] + s[..., 1, 1] + s[..., 2, 2]
    n[..., 0, 1] = s[..., 1, 2] + g(-s[..., 2, 1])
    n[..., 0, 2] = s[..., 2, 0] + g(-s[..., 0, 2])
    n[..., 0, 3] = s[..., 0, 1] + g(-s[..., 1, 0])
    n[..., 1, 1] = s[..., 0, 0] + g(-s[..., 1, 1]) + g(-s[..., 2, 2])
    n[..., 1, 2] = s[..., 0, 1] + s[..., 1, 0]
    n[..., 1, 3] = s[..., 2, 0] + s[..., 0, 2]
    n[..., 2, 2] = g(-s[..., 0, 0]) + s[..., 1, 1] + g(-s[..., 2, 2])
    n[..., 2, 3] = s[..., 1, 2] + s[..., 2, 1]
    n[..., 3, 3] = g(-s[..., 0, 0]) + g(-s[..., 1, 1]) + s[..., 2, 2]
    for a in range(4):
        for b in range(a):
            n[..., a, b] = n[..., b, a]
    return n


def quat_rotation(q: torch.Tensor) -> torch.Tensor:
    """Row-major R [..., 3, 3] of the quaternion (w, x, y, z) = q [..., 4], normalised (a3d_arap_math.h's formula)."""
    q = q / q.norm(dim=-1, keepdim=True)
    w, x, y, z = q.unbind(-1)
    r = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)
    return r.reshape(q.shape[:-1] + (3, 3))


def horn_rotation(S: torch.Tensor) -> torch.Tensor:
    """float64 Horn: the rotation of the top eigenvector of N(S)."""
    _, v = torch.linalg.eigh(horn_n(S.to(F64)))
    return quat_rotation(v[..., :, 3])


def svd_rotation(S: torch.Tensor) -> torch.Tensor:
    """The reference's estimate_rotation on given covariances (util.py:160-173): R = V U^T of S = U diag(sig) V^T, with the
    column of U of the smallest singular value flipped when det(R) <= 0."""
    u, sig, vh = torch.linalg.svd(S.to(F64))
    v = vh.transpose(-1, -2)
    r = v @ u.transpose(-1, -2)
    flip = torch.det(r) <= 0
    if bool(flip.any()):
        um = u.clone()
        col = torch.argmin(sig, dim=-1)
        rows = torch.nonzero(flip).flatten()
        um[rows, :, col[rows]] *= -1
        r = torch.where(flip[:, None, None], v @ um.transpose(-1, -2), r)
    return r


# ------------------------------------------------------------------------------------------------ ARAP
def _batched(fn, x):
    """fn (eigh) over a batch of small matrices, on the CPU in chunks: the device solvers cap the batch size."""
    parts = [fn(c.cpu()) for c in x.split(LINALG_BATCH)] if x.shape[0] else [fn(x.cpu())]
    return torch.cat([p[0] for p in parts]).to(x.device), torch.cat([p[1] for p in parts]).to(x.device)


class Arap:
    """a3d_arap on nodes [Nt, Nv, 3] (float32: the kernel's input; float64: arap_oracle's arithmetic), nbr [Nv, K] int,
    weight [Nv, K] or None, sample [Ns] or None (all nodes).  Tensors may live on any device; the restatement runs on
    nodes' device."""

    def __init__(self, nodes: torch.Tensor, nbr: torch.Tensor, weight: Optional[torch.Tensor] = None,
                 sample: Optional[torch.Tensor] = None):
        dev = nodes.device
        self.Nt, self.Nv, _ = nodes.shape
        self.K = K = nbr.shape[1]
        Nt, Nv = self.Nt, self.Nv
        idx = torch.arange(Nv, device=dev) if sample is None else sample.to(dev).long()
        self.Ns = Ns = idx.numel()
        node_ok = (idx >= 0) & (idx < Nv)
        i = idx.clamp(0, Nv - 1)
        j = nbr.to(dev).long()[i]                                                    # [Ns, K]
        valid = node_ok[:, None] & (j >= 0) & (j < Nv)
        jc = j.clamp(0, Nv - 1)
        if weight is None:
            w = valid.to(F64)
        else:
            w = weight.to(dev).to(F64)[i]
        w = torch.where(valid, w, torch.zeros_like(w))          # absent slots have zero edges: their weight never counts
        self.i, self.j, self.valid, self.w = i, jc, valid, w
        M = (Nt - 1) * Ns
        self.M = M
        e = nodes[:, i, None, :] - nodes[:, jc, :]                                   # [Nt, Ns, K, 3] in nodes' dtype
        e = torch.where(valid[None, :, :, None], e, torch.zeros_like(e)).to(F64)
        s = e[0][None].expand(Nt - 1, Ns, K, 3).reshape(M, K, 3)
        t = e[1:].reshape(M, K, 3)
        wm = w[None].expand(Nt - 1, Ns, K).reshape(M, K)
        self.s, self.t, self.wm = s, t, wm
        same_axis = (s == t).all(dim=1).any(dim=-1)                                  # [M]
        S = torch.einsum("mk,mka,mkb->mab", wm, s, t)
        Sabs = torch.einsum("mk,mka,mkb->mab", wm.abs(), s.abs(), t.abs())
        zero = same_axis | (Sabs == 0).flatten(1).all(1)
        S = torch.where(zero[:, None, None], torch.zeros_like(S), S)
        Sabs = torch.where(zero[:, None, None], torch.zeros_like(Sabs), Sabs)
        self.S, self.zero, self.same_axis = S, zero, same_axis
        # ---- rotation and its error
        N = horn_n(S)
        lam, V = _batched(torch.linalg.eigh, N)
        eN = (2 * (K + 2) * U32 * Sabs.flatten(1).norm(dim=1) + 2 * U32 * horn_n(Sabs, absolute=True).flatten(1).norm(dim=1)
              + C_JACOBI * U32 * N.flatten(1).norm(dim=1))

        def drot(gap):
            a = torch.where(gap > eN, eN / (gap - eN).clamp_min(1e-300), torch.full_like(gap, math.inf)) + C_VDRIFT * U32
            return (2 * a).clamp(max=2.0)

        dR1, dR2 = drot(lam[:, 3] - lam[:, 2]), drot(lam[:, 2] - lam[:, 1])
        R1 = torch.cat([svd_rotation(x.cpu()) for x in S.split(LINALG_BATCH)]).to(dev) if M else S.new_zeros(0, 3, 3)
        q1, q2 = V[:, :, 3], V[:, :, 2]
        Ra, Rb, Rc = quat_rotation(q1), quat_rotation(q2), quat_rotation((q1 + q2) / math.sqrt(2))
        A, B = (Ra + Rb) / 2, (Ra - Rb) / 2
        C = Rc - A
        mv = lambda R, x: torch.einsum("mab,mkb->mka", R, x)
        mtv = lambda R, x: torch.einsum("mba,mkb->mka", R, x)
        hyp = lambda x, y: torch.sqrt(x * x + y * y)
        s2, s1, t2 = s.norm(dim=-1), s.abs().sum(-1), t.norm(dim=-1)
        # mode 2 (rank-1 family about A)
        a2, b2 = mv(A, s), mtv(A, t)
        sa2, sb2 = hyp(mv(B, s), mv(C, s)), hyp(mtv(B, t), mtv(C, t))
        sc2 = hyp((t * mv(B, s)).sum(-1), (t * mv(C, s)).sum(-1))
        rel = lambda sp, nrm: torch.where(nrm > 0, sp.amax(-1) / nrm.clamp_min(1e-300), torch.zeros_like(nrm)).amax(-1)
        score2 = dR2 + torch.maximum(rel(sa2, s2), rel(sb2, t2))
        mode2 = (score2 < dR1) & ~zero
        self.mode2 = mode2
        eye = torch.eye(3, dtype=F64, device=dev).expand_as(R1) if M else R1
        R = torch.where(zero[:, None, None], eye, R1)
        a1, b1 = mv(R, s), mtv(R, t)
        m2 = mode2[:, None, None]
        a = torch.where(m2, a2, a1)
        b = torch.where(m2, b2, b1)
        sa = torch.where(m2, sa2, torch.zeros_like(sa2))
        sb = torch.where(m2, sb2, torch.zeros_like(sb2))
        sc = torch.where(mode2[:, None], sc2, torch.zeros_like(sc2))
        dR = torch.where(zero, torch.zeros_like(dR1), torch.where(mode2, dR2, dR1))[:, None]
        cq = torch.where(zero, torch.zeros_like(dR1), torch.full_like(dR1, C_QUAT * U32))[:, None]
        self.dR, self.R = dR[:, 0], R
        # ---- per slot
        d = t - a
        ea = (dR * s2 + cq * s1 + 3 * U32 * s1)[..., None].expand_as(d)
        dabs = d.abs() + sa
        ed = ea + U32 * (t.abs() + s1[..., None])
        w2 = 2 * wm[..., None]
        self.gt = w2 * d
        self.gt_b = w2.abs() * (ed + sa + U32 * (dabs + ed))
        self.gt_m = w2.abs() * (t.abs() + s2[..., None])
        g0h = b - s
        self.g0 = -w2 * g0h
        eb = (dR * dabs.norm(dim=-1) + cq * dabs.sum(-1) + 4 * U32 * dabs.sum(-1) + ed.norm(dim=-1))[..., None] + sb
        self.g0_b = w2.abs() * (eb + U32 * (g0h.abs() + eb))
        self.g0_m = (w2.abs() * (t2 + s2)[..., None]).expand_as(g0h)
        en1 = wm * (d * d).sum(-1)
        en2 = wm * ((t * t).sum(-1) + (s * s).sum(-1) - 2 * (t * a2).sum(-1))
        en = torch.where(mode2[:, None], en2, en1)
        en_b = wm.abs() * ((2 * dabs * ed + ed * ed).sum(-1) + 2 * sc + 4 * U32 * ((dabs + ed) ** 2).sum(-1))
        self.node_e = en.sum(1)
        self.node_b = en_b.sum(1) + K * U32 * (en.abs() + en_b).sum(1)
        self.node_m = (wm.abs() * (t2 + s2) ** 2).sum(1)

    def err(self, deterministic: bool) -> Out:
        M = self.M
        steps = (math.ceil(M / SUM_THREADS) + 10) if deterministic else (8 + math.ceil(M / ARAP_THREADS))
        v = self.node_e.sum()
        b = self.node_b.sum() + steps * U32 * (self.node_e.abs() + self.node_b).sum()
        where = lambda i: f"err: sum of {M} (frame, sample) energies ({'fixed order' if deterministic else 'atomics'})"
        return Out(Ref(v.reshape(1), (SLACK * b).reshape(1), where), self.node_m.sum().reshape(1))

    def grad(self) -> Out:
        Nt, Nv, Ns, K, M = self.Nt, self.Nv, self.Ns, self.K, self.M
        dev = self.s.device
        n = Nt * Nv * 3
        val = torch.zeros(n, dtype=F64, device=dev)
        bnd, mag, absb, cnt = torch.zeros_like(val), torch.zeros_like(val), torch.zeros_like(val), torch.zeros_like(val)
        if M:
            frame = torch.arange(1, Nt, device=dev).repeat_interleave(Ns)[:, None].expand(M, K)
            ii = self.i[None].expand(Nt - 1, Ns).reshape(M)[:, None].expand(M, K)
            jj = self.j[None].expand(Nt - 1, Ns, K).reshape(M, K)
            ok = self.valid[None].expand(Nt - 1, Ns, K).reshape(M, K)
            sel = ok.reshape(-1)
            for f, g, gb, gm in ((frame, self.gt, self.gt_b, self.gt_m), (torch.zeros_like(frame), self.g0, self.g0_b, self.g0_m)):
                for node, sign in ((ii, 1.0), (jj, -1.0)):
                    key = ((f * Nv + node).reshape(-1)[sel] * 3)[:, None] + torch.arange(3, device=dev)
                    key = key.reshape(-1)
                    gv, gbv, gmv = (x.reshape(-1, 3)[sel].reshape(-1) for x in (g, gb, gm))
                    val.index_add_(0, key, sign * gv)
                    bnd.index_add_(0, key, gbv)
                    absb.index_add_(0, key, gv.abs() + gbv)
                    mag.index_add_(0, key, gmv)
                    cnt.index_add_(0, key, torch.ones_like(gv))
        bound = SLACK * (bnd + cnt * U32 * absb)
        counts = cnt.cpu()

        def where(e):
            e = int(e)
            return f"grad[frame {e // 3 // Nv}, node {(e // 3) % Nv}, {'xyz'[e % 3]}] ({int(counts[e])} contributions)"
        return Out(Ref(val, bound, where), mag)

    def stats(self) -> dict:
        return {"node_frames": self.M, "rank1_family": int(self.mode2.sum()), "R_identity": int(self.zero.sum()),
                "same_axis": int(self.same_axis.sum())}


# ------------------------------------------------------------------------------------------------ KNN
class KnnVerdict(NamedTuple):
    ratio: float                # worst violation / bound (inf: a structural violation or a mismatch with bound 0)
    where: str
    unambiguous: float          # fraction of the returned ranks whose index was checked exactly
    median_rel: float           # median dist2 bound / dist2 over the non-zero distances
    checked: torch.Tensor       # [n, K] bool: the ranks whose index was checked exactly


def _exact_points(p: torch.Tensor) -> bool:
    return bool((p == p.round()).all()) and float(p.abs().max()) <= 1024


def knn_pair_bound(d64: torch.Tensor, exact: bool) -> torch.Tensor:
    if exact:
        return torch.zeros_like(d64)
    return SLACK * (KNN_EPS * d64 + torch.where(d64 > 0, torch.full_like(d64, SUBNORMAL), torch.zeros_like(d64)))


def knn_order(points: torch.Tensor, K: int, rows: Optional[torch.Tensor] = None, chunk: int = 512):
    """The float64 (distance, index) order of all points seen from each point in `rows`: (d64 [r, K+2], idx [r, K+2],
    dropped [r]) -- direct differences of the fp32 points, chunked (n = 50 000 runs on the device)."""
    p = points.to(F64)
    n = p.shape[0]
    rows = torch.arange(n, device=p.device) if rows is None else rows
    keep = min(K + 2, n)
    ds, ix, dr = [], [], []
    ar = torch.arange(n, device=p.device)
    for c0 in range(0, rows.numel(), chunk):
        r = rows[c0:c0 + chunk]
        d = ((p[r][:, None, :] - p[None, :, :]) ** 2).sum(-1)
        dd, ii = torch.sort(d, dim=1, stable=True)
        ds.append(dd[:, :keep]); ix.append(ii[:, :keep])
        dr.append(torch.where(d == 0, ar[None], torch.full_like(ar[None], n)).min(1).values)
        del d, dd, ii
    return torch.cat(ds), torch.cat(ix), torch.cat(dr)


def knn_check(points: torch.Tensor, K: int, nbr: torch.Tensor, dist2: torch.Tensor, order=None) -> KnnVerdict:
    """a3d_knn_graph's (nbr [n, K], dist2 [n, K]) for fp32 points [n, 3] against the float64 contract (module docstring)."""
    p = points.float()
    dev = p.device
    n = p.shape[0]
    exact = _exact_points(p)
    nbr = nbr.to(dev).long()
    dist2 = dist2.to(dev).to(F64)
    if order is None:
        order = knn_order(p, K)
    D, I, dropped = order
    bD = knn_pair_bound(D, exact)
    rows = torch.arange(n, device=dev)
    worst = [0.0, "ok"]

    def hit(r, where):
        if r > worst[0]:
            worst[0], worst[1] = r, where
    # structure
    if bool(((nbr < 0) | (nbr >= n)).any()):
        k = int(torch.nonzero((nbr < 0) | (nbr >= n))[0, 0])
        return KnnVerdict(math.inf, f"row {k}: index out of range {nbr[k].tolist()}", 0.0, 0.0, torch.zeros_like(nbr, dtype=torch.bool))
    srt = nbr.sort(1).values
    dup = (srt[:, 1:] == srt[:, :-1]).any(1) if K > 1 else torch.zeros(n, dtype=torch.bool, device=dev)
    if bool(dup.any()):
        k = int(torch.nonzero(dup)[0])
        hit(math.inf, f"row {k}: repeated index {nbr[k].tolist()}")
    has_drop = (nbr == dropped[:, None]).any(1)
    if bool(has_drop.any()):
        k = int(torch.nonzero(has_drop)[0])
        hit(math.inf, f"row {k}: returns the dropped first candidate {int(dropped[k])} {nbr[k].tolist()}")
    if K > 1:
        desc = dist2[:, 1:] < dist2[:, :-1]
        if bool(desc.any()):
            k = int(torch.nonzero(desc.any(1))[0])
            hit(math.inf, f"row {k}: dist2 not ascending {dist2[k].tolist()}")
    # dist2 against the float64 distance of the returned pair
    dg = ((p.to(F64)[rows][:, None, :] - p.to(F64)[nbr]) ** 2).sum(-1)
    bg = knn_pair_bound(dg, exact)
    err = (dist2 - dg).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bg)
    k = int(torch.argmax(r))
    hit(float(r.reshape(-1)[k]), f"dist2[{k // K}, {k % K}] = {float(dist2.reshape(-1)[k]):.9g} vs {float(dg.reshape(-1)[k]):.9g}")
    # completeness: the nearest point neither returned nor dropped is no nearer than the K-th returned one
    taken = (I[:, :, None] == nbr[:, None, :]).any(-1) | (I == dropped[:, None])
    first_free = torch.where(taken, torch.full_like(D, math.inf), D).min(1)
    if K + 1 < n:
        m = first_free.values
        mb = knn_pair_bound(m, exact)
        gap = dg[:, -1] - m
        viol = torch.where(gap > 0, torch.where(bg[:, -1] + mb > 0, gap / (bg[:, -1] + mb), torch.full_like(gap, math.inf)),
                           torch.zeros_like(gap))
        k = int(torch.argmax(viol))
        hit(float(viol[k]), f"row {k}: a point at d2 {float(m[k]):.9g} is missing, K-th returned at {float(dg[k, -1]):.9g}")
    # exact order where unambiguous: rank k of the row is order position k + 1
    pos = D[:, 1:K + 1]
    bpos = bD[:, 1:K + 1]
    lo, blo = D[:, 0:K], bD[:, 0:K]
    hi = D[:, 2:K + 2] if D.shape[1] >= K + 2 else torch.full_like(pos, math.inf)
    bhi = bD[:, 2:K + 2] if D.shape[1] >= K + 2 else torch.zeros_like(pos)

    def sep(x, bx, y, by):            # x < y (sorted): separated, or an exact tie of exact distances
        return (y - x > bx + by) | ((bx == 0) & (by == 0))
    unamb = sep(lo, blo, pos, bpos) & sep(pos, bpos, hi, bhi)
    want = I[:, 1:K + 1]
    bad = unamb & (want != nbr)
    if bool(bad.any()):
        rr, kk = [int(x) for x in torch.nonzero(bad)[0]]
        dn = float(dg[rr, kk])
        dw = float(pos[rr, kk])
        den = float(bg[rr, kk] + bpos[rr, kk])
        rat = abs(dn - dw) / den if den > 0 else math.inf
        hit(max(rat, 1.0 + 1e-9) if dn != dw else math.inf,
            f"row {rr} rank {kk}: index {int(nbr[rr, kk])} (d2 {dn:.9g}), the unambiguous order has {int(want[rr, kk])} (d2 {dw:.9g})")
    nzd = dg > 0
    med = float((bg[nzd] / dg[nzd]).median()) if bool(nzd.any()) else 0.0
    return KnnVerdict(worst[0], worst[1], float(unamb.double().mean()), med, unamb)



def connectivity_weight_bound(d64: torch.Tensor, count: int) -> torch.Tensor:
    """Bound on the adaptive weights w = exp(-d / mean(d)) / sum_row of cal_connectivity_from_points (util.py:95-99) when d
    is the kernel's fp32 dist2 (relative error e = SLACK KNN_EPS) and the mean is torch's fp32 reduction over `count`
    entries in an unspecified order (count u32): a = d / mean carries a (2 e + (count + 2) u32); expf adds 2 u32; the row
    normalisation adds the worst relative error of the row's terms and (K + 2) u32.  d64 [n, K]: float64 distances of the
    returned pairs; returns the bound on each weight (x SLACK)."""
    K = d64.shape[1]
    a = d64 / d64.mean()
    ex = torch.exp(-a)
    w = ex / ex.sum(1, keepdim=True)
    re = a * (2 * SLACK * KNN_EPS + (count + 2) * U32) + 2 * U32
    return SLACK * w * (re + re.amax(1, keepdim=True) + (K + 2) * U32)
