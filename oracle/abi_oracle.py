"""float64 restatement of the C ABI (include/a3d.h), with a per-element error bound for every op.

Each function takes the arguments of the matching `animate3d_b200.ops` wrapper (tensors may live on any device) and
returns a `Ref`: the expected contents of the WHOLE output span the call may write (`value`, float64, flat), a per-element
bound on |kernel - value| (`bound`) and `where(i)`, which names the row / tile / (batch, head) behind flat index i.  Elements
the call must not write carry bound 0 and the pre-call contents, so a stray store, or a read-modify-write that changes an
element it should only have read, is an error too.  `check(got_flat, ref)` returns the worst |err| / bound and its location.

Error bounds (u16 = 2^-11 and u32 = 2^-24 are the unit round-offs of fp16 and fp32; every bound is multiplied by SLACK = 2,
which covers the second-order terms dropped below and a tensor core that truncates instead of rounding):

  gemm       v = acc + bias + rowbias, the fp32 sum of K fp16 products: |dv| <= (K + 2) u32 (|A||B|^T + |bias| + |rowbias|).
             The epilogue's fp32 operations add 4 u32 (|acc_scale v| + |r1_scale R1| + |R2|); an fp16 store adds u16 |out|,
             an fp32 store u32 |out|.  GEGLU out = u gelu(g) propagates the (scaled) errors of u and g:
             |gelu(g)| du + |u| (1.13 dg + 3 u32 (|g| + |gelu(g)|)) (|gelu'| <= 1.13; erff is accurate to 2 ulp), plus the
             fp16 store.  Every store bound includes half the subnormal spacing.  CONV3 uses the im2col of |x| for |A|.
  attention  the kernels round P to fp16 before the PV product and take the row sum from the same rounded P (the ones column
             of V), so a relative error e_j of p_j moves O_c by sum_j p_j e_j (v_jc - O_c) / sum_j p_j, at most
             e (P|V| + |O|)_c with P the exact softmax.  e = u16 (P rounding) + 2^-20 (exp2 approximation) + ds, where
             ds = (d + 8) u32 scale |q|_1 max_j |k_j|_inf bounds the fp32 error of the logit and of the max subtraction.
             The fp32 PV sums add (Lk + 4) u32 (P|V| + |O|).  The result is scaled by |out_scale| and, after the optional
             add of the previous output, stored as fp16 (u16 |out|).  SIMT and the few-keys kernel keep P in fp32 and
             satisfy the same bound.
  temporal   the same bound as attention over the F frames.
  group_norm the statistics are pivoted (n, mean, M2) sums: at most 128 rows per thread, then trees, so the mean has
             |dmu| <= es D and the variance |dvar| / var <= es (1 + 4 D^2 / var), es = (128 + 4 log2 n + 16) u32, D the
             largest |x - mean| of the (sample, group).  y = x s + (beta - mean s) with s = rstd gamma adds
             3 u32 (|x s| + |mean s| + |beta|); rsqrtf adds 2 u32 to rstd; SiLU (fast exp) 1.1 dy + 2^-20 |y|; fp16 store.
  group_norm_backward  dx = rstd (g - mean(g) - xhat mean(g xhat)), g = dy gamma [silu']: the two means are fp32 sums
             (<= 128 per thread, then trees: eb = (192 + 2 log2 n) u32 relative to the mean of the absolute terms),
             g carries 2^-20 |g| (fast exp in silu'), xhat u32 (|x| + |mean|) rstd, three more fp32 operations, fp16 store.
  layer_norm the same as group_norm with one group of C channels per row (the row is summed by a warp: es = (C/32 + 16) u32).
  linear_f32 / conv_in / conv_out   fp32 dot products: (K + 2) u32 (|x||W|^T + |b|) [+ 2^-20 of the SiLU input], then the
             store (u16 for fp16 outputs, u32 for fp32) and, when accumulating, u32 |previous|.
  silu_rows  2^-20 |silu(x)| + the fp16 store.  cast_f32_f16: the fp16 store.  upsample2x: exact (bound 0).
  ddim_cfg_step  eight fp32 operations on the absolute values of the terms: 8 u32 R_abs.  Frame 0 is an exact copy.

A bound is a worst case, not a statistic: no global rel-L2 enters the verdict, so an error confined to one tile, one row or
one (batch, head) counts as much as one spread over the whole tensor."""
from __future__ import annotations

import math
from typing import Callable, NamedTuple, Tuple

import torch
import torch.nn.functional as F

U16 = 2.0 ** -11
U32 = 2.0 ** -24
EXP_APPROX = 2.0 ** -20
SLACK = 2.0
F64 = torch.float64
CHUNK = 1 << 25          # float64 elements per intermediate (256 MB)


class Ref(NamedTuple):
    value: torch.Tensor                 # float64, flat over the output span
    bound: torch.Tensor                 # float64, same shape
    where: Callable[[int], str]


class Verdict(NamedTuple):
    ratio: float                        # worst |err| / bound (inf: a mismatch where the bound is 0, or a non-finite value)
    index: int
    where: str
    got: float
    want: float
    bound: float


# ------------------------------------------------------------------------------------------------ helpers
def perm_rows(m, a, b):
    """Row permutation of a3d_gemm / a3d_group_norm: "(x a b) -> (x b a)"."""
    if a == 0:
        return m
    return (m // (a * b)) * (a * b) + (m % b) * a + (m // b) % a


def sdpa_ref(q, k, v, scale):
    """softmax(scale q k^T) v over [..., L, d] (in the dtype of q)."""
    s = torch.einsum("bhqd,bhkd->bhqk", q, k) * scale
    return torch.einsum("bhqk,bhkd->bhqd", s.softmax(-1), v)


def span_of(rows: int, cols: int, ld: int) -> int:
    return (rows - 1) * ld + cols


def flat(t: torch.Tensor, n: int, offset: int = 0) -> torch.Tensor:
    """The n elements that start `offset` elements after t's first element, as a 1-D view (what a raw pointer sees)."""
    return t.as_strided((n,), (1,), t.storage_offset() + offset)


def mat(t: torch.Tensor, rows: int, cols: int, ld: int, offset: int = 0) -> torch.Tensor:
    return t.as_strided((rows, cols), (ld, 1), t.storage_offset() + offset)


def _store(x, e, f32=False):
    """Bound after the final store: |round(x~) - x| <= e + u |x~| + h <= e (1 + u) + u |x| + h, with h half the spacing
    of the subnormals (2^-25 for fp16, 2^-150 for fp32) for values below the normal range."""
    u, h = (U32, 2.0 ** -150) if f32 else (U16, 2.0 ** -25)
    return e * (1 + u) + u * x.abs() + h


def check(got: torch.Tensor, ref: Ref) -> Verdict:
    g = got.reshape(-1).to(F64)
    want = ref.value.to(g.device)
    bound = ref.bound.to(g.device)
    assert g.numel() == want.numel(), (g.numel(), want.numel())
    err = torch.where(g == want, torch.zeros_like(g), (g - want).abs())        # equal infinities (untouched memory) match
    both_nan = torch.isnan(g) & torch.isnan(want)
    err = torch.where(both_nan, torch.zeros_like(err), err)
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)      # bound 0 and err > 0 -> inf
    i = int(torch.argmax(ratio).item())
    r = float(ratio[i].item())
    return Verdict(r, i, ref.where(i), float(g[i].item()), float(want[i].item()), float(bound[i].item()))


def assert_within(got, ref: Ref, what=""):
    v = check(got, ref)
    assert v.ratio <= 1.0, (f"{what}: |err|/bound = {v.ratio:.3g} at {v.where}: got {v.got:.6g}, want {v.want:.6g} "
                            f"+- {v.bound:.3g}")
    return v


# ------------------------------------------------------------------------------------------------ GEMM
def _conv_rows(xp, m, conv):
    """im2col rows m of the CONV3 operand from the padded image xp: [len(m), 9 C], k = (ky*3+kx)*C + c."""
    n, h, w, c, s = conv
    oh, ow = h // s, w // s
    img, oy, ox = m // (oh * ow), (m // ow) % oh, m % ow
    taps = [xp[img, oy * s + ky, ox * s + kx] for ky in range(3) for kx in range(3)]
    return torch.cat(taps, 1)


def _gelu(g):
    return 0.5 * g * (1.0 + torch.erf(g / math.sqrt(2.0)))


def gemm(A, B, out, *, M, N, K, lda=0, ldc=0, conv=None, bias=None, rowbias=None, rb_div=1, rb_mod=0, rb_ld=0,
         acc_scale=1.0, R1=None, ldr1=0, r1_scale=1.0, R2=None, ldr2=0, geglu=False, out_f32=False, perm=(0, 0), impl=0,
         conv_nopad_lo=False, rb_rows=None) -> Ref:
    """a3d_gemm.  `out` holds the output buffer BEFORE the call (read when R2 aliases it; kept where nothing is written).
    rb_ld must be given when rowbias is not a 2-D tensor whose stride(0) is the table's row stride."""
    n_out = N // 2 if geglu else N
    lda, ldc = lda or K, ldc or n_out
    ldr1, ldr2 = ldr1 or N, ldr2 or N
    dev = out.device
    pa, pb = perm
    out_rows = M
    span = span_of(out_rows, n_out, ldc)
    value = flat(out, span).to(F64).clone()
    bound = torch.zeros_like(value)
    Bd = mat(B, N, K, K).to(F64)
    Bt, Bta = Bd.t(), Bd.abs().t()
    div = rb_div if rb_div > 0 else 1
    mod = rb_mod if rb_mod > 0 else 1 << 40
    if rowbias is not None:
        rb_ld = rb_ld or rowbias.stride(0)
        rows_rb = rb_rows or min(mod, (M - 1) // div + 1)
        rbt = mat(rowbias, rows_rb, N, rb_ld).to(F64)
    bd = bias.to(F64) if bias is not None else None
    xi = None
    if conv is not None:
        n, h, w, c, s = conv
        pad = 0 if conv_nopad_lo else 1
        xi = F.pad(flat(A, n * h * w * c).to(F64).view(n, h, w, c), (0, 0, pad, 1, pad, 1))   # [n, h + pad + 1, w + pad + 1, c]
    else:
        Ad = mat(A, M, K, lda).to(F64) if M > 0 else None
    vflat = value.view(-1)
    chunk = max(1, CHUNK // max(K, N))
    for m0 in range(0, M, chunk):
        m = torch.arange(m0, min(M, m0 + chunk), device=dev)
        a = _conv_rows(xi, m, conv) if conv is not None else Ad[m]
        v = a @ Bt
        vb = a.abs() @ Bta
        if bd is not None:
            v = v + bd
            vb = vb + bd.abs()
        if rowbias is not None:
            r = rbt[(m // div) % mod]
            v = v + r
            vb = vb + r.abs()
        e = (K + 2) * U32 * vb * abs(acc_scale)
        v = v * acc_scale
        orow = perm_rows(m, pa, pb)
        if geglu:
            blk = torch.arange(n_out, device=dev)
            nu = (blk // 32) * 64 + blk % 32
            u, g = v[:, nu], v[:, nu + 32]
            eu, eg = e[:, nu], e[:, nu + 32]
            gl = _gelu(g)
            res = u * gl
            err = gl.abs() * eu + u.abs() * (1.13 * eg + 3 * U32 * (g.abs() + gl.abs())) + U32 * res.abs()
        else:
            mag = v.abs()
            if R1 is not None:
                r1 = mat(R1, M, N, ldr1)[m].to(F64) * r1_scale
                v = v + r1
                mag = mag + r1.abs()
            if R2 is not None:
                r2 = mat(R2, M, N, ldr2)[orow].to(F64)
                v = v + r2
                mag = mag + r2.abs()
            res = v
            err = e + 4 * U32 * mag
        err = SLACK * _store(res, err, out_f32)
        idx = orow[:, None] * ldc + torch.arange(n_out, device=dev)[None, :]
        vflat[idx.reshape(-1)] = res.reshape(-1)
        bound.view(-1)[idx.reshape(-1)] = err.reshape(-1)

    inv = {}

    def where(i):
        om, col = divmod(int(i), ldc)
        if col >= n_out or om >= out_rows:
            return f"flat {i}: outside the written columns (row {om}, col {col})"
        if not inv:
            mm = torch.arange(M)
            inv["m"] = torch.empty(M, dtype=torch.long)
            inv["m"][perm_rows(mm, pa, pb)] = mm
        m = int(inv["m"][om])
        return f"output row {om} (source row {m}, M-tile {m // 128} of 128 rows), col {col} (8-col group {col // 8})"

    return Ref(value, bound, where)


# ------------------------------------------------------------------------------------------------ attention
class V5(NamedTuple):
    """A rank-5 strided view (a3d_view5) over tensor t, starting `off` elements after t's first element."""
    t: torch.Tensor
    off: int
    cols: int
    s: Tuple[int, int, int, int]
    e: Tuple[int, int, int, int]

    def span(self) -> int:
        return self.off + sum((e - 1) * s for e, s in zip(self.e, self.s)) + self.cols


def _gather5(v: V5, c0: int, ncols: int) -> torch.Tensor:
    """[batches (i4*e3 + i3), L (i2*e1 + i1), ncols] starting at column c0."""
    e1, e2, e3, e4 = v.e
    s1, s2, s3, s4 = v.s
    x = v.t.as_strided((e4, e3, e2, e1, ncols), (s4, s3, s2, s1, 1), v.t.storage_offset() + v.off + c0)
    return x.reshape(e4 * e3, e2 * e1, ncols)


def out_span(e, ostr, ncols, off):
    return off + sum((a - 1) * s for a, s in zip(e, ostr)) + ncols


def _attn_core(q, k, v, scale, Lk, d):
    """q [b, h, lq, d], k / v [b, h, Lk, d] float64 -> (O, bound of O before out_scale and the store)."""
    s = torch.einsum("bhqd,bhkd->bhqk", q, k) * scale
    p = s.softmax(-1)
    o = p @ v
    pv = p @ v.abs()
    ds = (d + 8) * U32 * abs(scale) * q.abs().sum(-1, keepdim=True) * k.abs().amax(dim=(-1, -2), keepdim=True)
    eps = U16 + EXP_APPROX + ds + (Lk + 4) * U32
    return o, eps * (pv + o.abs())


def attention(q: V5, k: V5, v: V5, out, ostrides, *, heads, d, scale, kv_div=1, kv_i3_zero=False, accumulate=False,
              out_scale=1.0, impl=0, out_col_offset=0) -> Ref:
    """a3d_attention; `out` is the output buffer before the call, addressed from its first element."""
    dqk, dv = (d + 15) // 16 * 16, (d + 16) // 16 * 16
    e1, e2, e3, e4 = q.e
    Lq, batches = e1 * e2, e3 * e4
    ke1, ke2, ke3, ke4 = k.e
    Lk = ke1 * ke2
    kv_div = kv_div if kv_div > 0 else 1
    C = heads * d
    span = out_span(q.e, ostrides, C, out_col_offset)
    value = flat(out, span).to(F64).clone()
    bound = torch.zeros_like(value)
    os1, os2, os3, os4 = ostrides
    dev = value.device
    cols = torch.arange(C, device=dev)
    Q = _gather5(q, 0, heads * dqk)                                   # [batches, Lq, H*dqk]
    Kall = _gather5(k, 0, heads * dqk).view(ke4, ke3, Lk, heads * dqk)
    Vall = _gather5(v, 0, heads * dv).view(ke4, ke3, Lk, heads * dv)
    per_b = heads * Lq * max(Lk, d)
    nb = max(1, CHUNK // per_b)
    qc = Lq if per_b <= CHUNK else max(1, CHUNK // (heads * max(Lk, d)))
    for b0 in range(0, batches, nb):
        qb = torch.arange(b0, min(batches, b0 + nb), device=Q.device)
        kb = qb // kv_div
        i3 = torch.zeros_like(kb) if kv_i3_zero else kb % ke3
        kk = Kall[kb // ke3, i3].to(F64).view(-1, Lk, heads, dqk)[..., :d].permute(0, 2, 1, 3)
        vv = Vall[kb // ke3, i3].to(F64).view(-1, Lk, heads, dv)[..., :d].permute(0, 2, 1, 3)
        for l0 in range(0, Lq, qc):
            l1 = min(Lq, l0 + qc)
            qq = Q[qb, l0:l1].to(F64).view(len(qb), l1 - l0, heads, dqk)[..., :d].permute(0, 2, 1, 3)
            o, eo = _attn_core(qq, kk, vv, scale, Lk, d)
            o = o.permute(0, 2, 1, 3).reshape(len(qb), l1 - l0, C).to(dev) * out_scale
            eo = eo.permute(0, 2, 1, 3).reshape(len(qb), l1 - l0, C).to(dev) * abs(out_scale)
            bq = qb.to(dev)
            lv = torch.arange(l0, l1, device=dev)
            row = (bq // e3 * os4 + bq % e3 * os3)[:, None] + (lv // e1 * os2 + lv % e1 * os1)[None, :]
            addr = (out_col_offset + row[..., None] + cols).reshape(-1)
            res = o.reshape(-1) + (value[addr] if accumulate else 0.0)
            value[addr] = res
            bound[addr] = SLACK * _store(res, eo.reshape(-1))

    rows = None

    def where(i):
        nonlocal rows
        if rows is None:
            b = torch.arange(batches)
            l = torch.arange(Lq)
            i4, i3 = b // e3, b % e3
            i2, i1 = l // e1, l % e1
            rows = (out_col_offset + (i4 * os4 + i3 * os3)[:, None] + (i2 * os2 + i1 * os1)[None, :]).reshape(-1)
        hit = ((i - rows) >= 0) & ((i - rows) < C)
        if not bool(hit.any()):
            return f"flat {i}: outside the written rows / columns"
        r = int(torch.nonzero(hit)[0])
        b, l = divmod(r, Lq)
        c = i - int(rows[r])
        return f"(batch {b}, head {c // d}) query {l} col {c % d}"

    return Ref(value, bound, where)


def temporal_attn(qkv, out, pixels, frames, heads, d, scale, ldo=0, out_col_offset=0) -> Ref:
    """a3d_temporal_attn: qkv [P, F, 3C] (q | k | v), out rows of stride ldo starting at column out_col_offset."""
    C = heads * d
    ldo = ldo or C
    rows = pixels * frames
    span = out_col_offset + span_of(rows, C, ldo)
    value = flat(out, span).to(F64).clone()
    bound = torch.zeros_like(value)
    vo = value.as_strided((rows, C), (ldo, 1), out_col_offset)
    bo = bound.as_strided((rows, C), (ldo, 1), out_col_offset)
    x = mat(qkv, rows, 3 * C, 3 * C)
    chunk = max(1, CHUNK // (heads * frames * max(frames, d)))
    for p0 in range(0, pixels, chunk):
        p1 = min(pixels, p0 + chunk)
        t = x[p0 * frames:p1 * frames].to(F64).view(p1 - p0, frames, 3, heads, d).permute(2, 0, 3, 1, 4)
        o, eo = _attn_core(t[0], t[1], t[2], scale, frames, d)
        o = o.permute(0, 2, 1, 3).reshape(-1, C)
        vo[p0 * frames:p1 * frames] = o
        bo[p0 * frames:p1 * frames] = SLACK * _store(o, eo.permute(0, 2, 1, 3).reshape(-1, C))

    def where(i):
        r, c = divmod(i - out_col_offset, ldo)
        if c < 0 or c >= C:
            return f"flat {i}: outside the written columns"
        return f"(pixel {r // frames}, head {c // d}) frame {r % frames} col {c % d}"

    return Ref(value, bound, where)


# ------------------------------------------------------------------------------------------------ normalisation
def _rows_where(cols, what="row"):
    return lambda i: f"{what} {i // cols} col {i % cols}"


def group_norm(x1, c1, x2, c2, gamma, beta, y, samples, rows_per_sample, groups, eps, silu, ws_stats=None, perm=(0, 0)) -> Ref:
    C = c1 + (c2 if x2 is not None else 0)
    rows = samples * rows_per_sample
    x = mat(x1, rows, c1, c1).to(F64)
    if x2 is not None and c2:
        x = torch.cat([x, mat(x2, rows, c2, c2).to(F64)], 1)
    cpg = C // groups
    n = rows_per_sample * cpg
    xg = x.view(samples, rows_per_sample, groups, cpg)
    mu = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg - mu) ** 2).mean(dim=(1, 3), keepdim=True)
    D = (xg - mu).abs().amax(dim=(1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    es = (128 + 4 * math.ceil(math.log2(max(n, 2))) + 16) * U32
    dmu = es * D
    dr = 0.5 * es * (1 + 4 * D * D / (var + eps)) + 2 * U32
    gm, bt = gamma.to(F64).view(groups, cpg), beta.to(F64).view(groups, cpg)
    xh = (xg - mu) * rstd
    yp = xh * gm + bt
    e = gm.abs() * rstd * (dmu + (xg - mu).abs() * dr) + 3 * U32 * ((xg * rstd * gm).abs() + (mu * rstd * gm).abs() + bt.abs())
    if silu:
        e = 1.1 * e + EXP_APPROX * yp.abs()
        yp = F.silu(yp)
    e = SLACK * _store(yp, e)
    orow = perm_rows(torch.arange(rows, device=x.device), *perm)
    value = torch.empty(rows, C, dtype=F64, device=x.device)
    bound = torch.empty_like(value)
    value[orow] = yp.reshape(rows, C)
    bound[orow] = e.reshape(rows, C)
    return Ref(value.view(-1), bound.view(-1), _rows_where(C, "output row"))


def group_norm_backward(x, c, gamma, beta, fwd_stats, dy, dx, samples, rows_per_sample, groups, silu, ws=None) -> Ref:
    rows = samples * rows_per_sample
    cpg = c // groups
    n = rows_per_sample * cpg
    xg = mat(x, rows, c, c).to(F64).view(samples, rows_per_sample, groups, cpg)
    dyg = mat(dy, rows, c, c).to(F64).view(samples, rows_per_sample, groups, cpg)
    st = flat(fwd_stats, 2 * samples * groups).to(F64).view(samples, 1, groups, 1, 2)
    mu, rstd = st[..., 0], st[..., 1]
    gm, bt = gamma.to(F64).view(groups, cpg), beta.to(F64).view(groups, cpg)
    xh = (xg - mu) * rstd
    g = dyg * gm
    if silu:
        z = xh * gm + bt
        sg = torch.sigmoid(z)
        g = g * sg * (1 + z * (1 - sg))
    m1 = g.mean(dim=(1, 3), keepdim=True)
    m2 = (g * xh).mean(dim=(1, 3), keepdim=True)
    dxv = rstd * (g - m1 - xh * m2)
    eb = (192 + 2 * math.ceil(math.log2(max(n, 2)))) * U32
    e = rstd * (EXP_APPROX * g.abs() + eb * g.abs().mean(dim=(1, 3), keepdim=True)
                + xh.abs() * eb * (g * xh).abs().mean(dim=(1, 3), keepdim=True)
                + U32 * (xg.abs() + mu.abs()) * rstd * m2.abs() + 3 * U32 * (g.abs() + m1.abs() + (xh * m2).abs()))
    e = SLACK * _store(dxv, e)
    return Ref(dxv.reshape(-1), e.reshape(-1), _rows_where(c))


def layer_norm(x, gamma, beta, y, rows, c, eps=1e-5) -> Ref:
    xd = mat(x, rows, c, c).to(F64)
    mu = xd.mean(-1, keepdim=True)
    var = ((xd - mu) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    gm, bt = gamma.to(F64), beta.to(F64)
    yp = (xd - mu) * rstd * gm + bt
    es = (c / 32 + 16) * U32
    D = (xd - mu).abs().amax(-1, keepdim=True)
    M = xd.abs().amax(-1, keepdim=True)
    dr = 0.5 * es * (1 + 4 * (D + M) ** 2 / (var + eps)) + 2 * U32
    e = gm.abs() * rstd * (es * (D + M) + (xd - mu).abs() * dr) + 3 * U32 * ((xd * rstd * gm).abs() + (mu * rstd * gm).abs() + bt.abs())
    return Ref(yp.view(-1), (SLACK * _store(yp, e)).view(-1), _rows_where(c))


# ------------------------------------------------------------------------------------------------ small ops
def upsample2x(x, y, n, h, w, c) -> Ref:
    xd = mat(x, n * h * w, c, c).to(F64).view(n, h, w, c)
    v = xd.repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(-1)
    return Ref(v, torch.zeros_like(v), lambda i: f"(img {i // (4 * h * w * c)}) pixel {(i // c) % (4 * h * w)} col {i % c}")


def silu_rows(x, y, rows, c, rep) -> Ref:
    xd = mat(x, (rows + rep - 1) // rep, c, c).to(F64)
    v = F.silu(xd)[torch.arange(rows, device=xd.device) // rep]
    return Ref(v.reshape(-1), (SLACK * _store(v, EXP_APPROX * v.abs())).reshape(-1), _rows_where(c))


def cast_f32_f16(x, y) -> Ref:
    v = x.reshape(-1).to(F64)
    return Ref(v, _store(v, torch.zeros_like(v)), lambda i: f"element {i}")


def conv_in(sample, w, b, y, bn, cin, f, h, wd, cout) -> Ref:
    xs = flat(sample, bn * cin * f * h * wd).to(F64).view(bn, cin, f, h, wd).permute(0, 2, 1, 3, 4).reshape(bn * f, cin, h, wd)
    wt, bb = flat(w, cout * cin * 9).to(F64).view(cout, cin, 3, 3), flat(b, cout).to(F64)
    v = F.conv2d(xs, wt, bb, padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    va = F.conv2d(xs.abs(), wt.abs(), bb.abs(), padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    e = (9 * cin + 2) * U32 * va
    return Ref(v.reshape(-1), (SLACK * _store(v, e)).reshape(-1), _rows_where(cout, "pixel"))


def conv_out(x, w, b, y, bn, cin, f, h, wd, cout) -> Ref:
    xs = mat(x, bn * f * h * wd, cin, cin).to(F64).view(bn * f, h, wd, cin).permute(0, 3, 1, 2)
    wt, bb = flat(w, cout * cin * 9).to(F64).view(cout, cin, 3, 3), flat(b, cout).to(F64)
    v = F.conv2d(xs, wt, bb, padding=1).view(bn, f, cout, h, wd).permute(0, 2, 1, 3, 4)
    va = F.conv2d(xs.abs(), wt.abs(), bb.abs(), padding=1).view(bn, f, cout, h, wd).permute(0, 2, 1, 3, 4)
    e = (9 * cin + 2) * U32 * va
    return Ref(v.reshape(-1), (SLACK * _store(v, e, True)).reshape(-1),
               lambda i: "[bn, cout, f, h, w] index %s" % (tuple(int(t) for t in torch.unravel_index(torch.tensor(i), (bn, cout, f, h, wd))),))


def linear_f32(x, w, b, y, m, n, k, act_in=0, accumulate=False) -> Ref:
    """`y` is the output before the call (read when accumulating)."""
    xd = mat(x, m, k, k).to(F64)
    a = F.silu(xd) if act_in else xd
    wt = mat(w, n, k, k).to(F64)
    v = a @ wt.t()
    va = a.abs() @ wt.abs().t()
    if b is not None:
        v, va = v + b.to(F64), va + b.to(F64).abs()
    e = ((k + 2) * U32 + (EXP_APPROX if act_in else 0.0)) * va
    if accumulate:
        prev = mat(y, m, n, n).to(F64)
        v = v + prev
        e = e + U32 * (v.abs() + prev.abs())
    return Ref(v.reshape(-1), (SLACK * _store(v, e, True)).reshape(-1), _rows_where(n))


def timestep_proj(t, out, rows, half) -> Ref:
    td = flat(t, rows).to(F64)
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=F64, device=td.device) / half)
    arg = td[:, None] * freqs[None, :]
    v = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    # fp32 argument: the frequency exp(-ln(1e4) i / half) is good to ~9 u32 (argument up to 9.2), the product adds u32; sin / cos
    # are 1-Lipschitz
    e = 16 * U32 * arg.abs().repeat(1, 2) + 4 * U32
    return Ref(v.reshape(-1), (SLACK * _store(v, e, True)).reshape(-1), _rows_where(2 * half))


def ddim_cfg_step(latents, noise_pred, first_frame, bn, c, f, hw, guidance, alpha_t, alpha_prev, uncond_first=True) -> Ref:
    """`latents` is the state before the step."""
    x = flat(latents, bn * c * f * hw).to(F64).view(bn, c, f, hw)
    e2 = flat(noise_pred, 2 * bn * c * f * hw).to(F64).view(2 * bn, c, f, hw)
    ea, eb = (e2[:bn], e2[bn:]) if uncond_first else (e2[bn:], e2[:bn])
    if uncond_first:
        eps = ea + guidance * (eb - ea)
        eps_abs = ea.abs() + abs(guidance) * (eb.abs() + ea.abs())
    else:
        eps = ea + guidance * (ea - eb)
        eps_abs = ea.abs() + abs(guidance) * (eb.abs() + ea.abs())
    sa, sp = math.sqrt(alpha_t), math.sqrt(alpha_prev)
    x0 = (x - math.sqrt(1 - alpha_t) * eps) / sa
    v = sp * x0 + math.sqrt(1 - alpha_prev) * eps
    r_abs = sp / sa * (x.abs() + math.sqrt(1 - alpha_t) * eps_abs) + math.sqrt(1 - alpha_prev) * eps_abs
    e = 8 * U32 * r_abs
    if first_frame is not None:
        v[:, :, 0] = flat(first_frame, bn * c * hw).to(F64).view(bn, c, hw)
        e[:, :, 0] = 0
    return Ref(v.reshape(-1), (SLACK * _store(v, e, True)).reshape(-1),
               lambda i: "[bn, c, f, hw] index %s" % (tuple(int(t) for t in torch.unravel_index(torch.tensor(i), (bn, c, f, hw))),))
