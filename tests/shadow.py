"""Shadow check of real passes: while the context manager is active every kernel-launching function of
`animate3d_b200.ops` is wrapped.  Per call the wrapper snapshots what the call writes (the output span, and residuals that
may alias it), runs the real op, synchronises, computes oracle/abi_oracle.py on the same operands and compares element by
element against the per-element bound.  Inputs the call only reads are used in place: the oracle runs before any later launch
can overwrite them.  Each record keeps the op, the kernel path it took, its geometry, the worst |err| / bound with its location
and the caller's file:line.  No product code changes: `ops.view5` is wrapped as well, to attach the base tensor and column
offset to the returned View5 (ctypes structures take extra attributes)."""
from __future__ import annotations

import collections
import contextlib
import os
import sys

import torch

from oracle import abi_oracle as O

OPS = ("gemm", "attention", "temporal_attn", "group_norm", "group_norm_backward", "layer_norm", "upsample2x", "silu_rows",
       "conv_in", "conv_out", "timestep_proj", "linear_f32", "cast_f32_f16", "ddim_cfg_step")
_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _site():
    f = sys._getframe(2)
    here = os.path.abspath(__file__)
    while f is not None and (os.path.abspath(f.f_code.co_filename) == here or f.f_code.co_filename.endswith("ops.py")):
        f = f.f_back
    if f is None:
        return "?"
    return f"{os.path.relpath(f.f_code.co_filename, _PKG)}:{f.f_lineno}"


def _snap(t, n):
    return O.flat(t, n).clone()


# ------------------------------------------------------------------------------------------------ the wrappers
def _v5(v):
    return O.V5(v._t, v._off, v.cols, (v.s1, v.s2, v.s3, v.s4), (v.e1, v.e2, v.e3, v.e4))


def _prepare(op, a, kw):
    """-> (oracle thunk to run after the call, output tensor, output span, kernel path, geometry).  The kernel path is the
    library's own answer for these arguments (ops.*_kernel)."""
    from animate3d_b200 import ops
    if op == "gemm":
        A, B, out = a
        M, N, K = kw["M"], kw["N"], kw["K"]
        geglu = kw.get("geglu", False)
        n_out = N // 2 if geglu else N
        k2 = dict(kw)
        k2["ldc"] = kw.get("ldc", 0) or n_out
        span = O.span_of(M, n_out, k2["ldc"])
        snap = _snap(out, span)
        for r, ld in (("R1", "ldr1"), ("R2", "ldr2")):
            if kw.get(r) is not None:
                k2[ld] = kw.get(ld, 0) or N
                k2[r] = _snap(kw[r], O.span_of(M, N, k2[ld]))
        if kw.get("rowbias") is not None:
            k2["rb_ld"] = kw.get("rb_ld", 0) or kw["rowbias"].stride(0)
        path = ops.gemm_kernel(*a, **kw)
        geo = f"M={M} N={N} K={K}" + (f" conv={kw['conv']}" if kw.get("conv") else "") + \
            "".join(f" {f}" for f in ("bias", "rowbias", "R1", "R2") if kw.get(f) is not None) + \
            (f" perm={kw['perm']}" if kw.get("perm", (0, 0))[0] else "") + (" geglu" if geglu else "")
        return (lambda: O.gemm(A, B, snap, **k2)), out, span, path, geo
    if op == "attention":
        q, k, v, out, ostr = a
        heads, d = kw["heads"], kw["d"]
        off = kw.get("out_col_offset", 0)
        span = O.out_span((q.e1, q.e2, q.e3, q.e4), ostr, heads * d, off)
        snap = _snap(out, span)
        k2 = dict(kw)
        path = ops.attention_kernel(*a, **kw)
        geo = f"Lq={q.e1 * q.e2} Lk={k.e1 * k.e2} batches={q.e3 * q.e4} d={d}" + \
            "".join(f" {f}={kw[f]}" for f in ("kv_div", "kv_i3_zero", "accumulate", "out_scale", "out_col_offset") if kw.get(f))
        return (lambda: O.attention(_v5(q), _v5(k), _v5(v), snap, ostr, **k2)), out, span, path, geo
    if op == "temporal_attn":
        qkv, out, pixels, frames, heads, d, scale = a[:7]
        ldo = kw.get("ldo", a[7] if len(a) > 7 else 0) or heads * d
        off = kw.get("out_col_offset", 0)
        span = off + O.span_of(pixels * frames, heads * d, ldo)
        snap = _snap(out, span)
        path = ops.temporal_attn_kernel(*a, **kw)
        return (lambda: O.temporal_attn(qkv, snap, pixels, frames, heads, d, scale, ldo=ldo, out_col_offset=off)), out, span, \
            path, f"P={pixels} F={frames} d={d} ldo={ldo} off={off}"
    if op == "ddim_cfg_step":
        lat = a[0]
        snap = _snap(lat, lat.numel())
        return (lambda: O.ddim_cfg_step(snap, *a[1:], **kw)), lat, lat.numel(), "ddim", f"{tuple(lat.shape)}"
    if op == "linear_f32":
        y = a[3]
        m, n = a[4], a[5]
        snap = _snap(y, m * n)
        return (lambda: O.linear_f32(a[0], a[1], a[2], snap, *a[4:], **kw)), y, m * n, "fp32", f"m={m} n={n} k={a[6]}"
    out_idx = {"group_norm": 6, "group_norm_backward": 6, "layer_norm": 3, "upsample2x": 1, "silu_rows": 1, "conv_in": 3,
               "conv_out": 3, "timestep_proj": 1, "cast_f32_f16": 1}[op]
    out = a[out_idx]
    fn = getattr(O, op)
    if op == "timestep_proj":
        span = a[2] * 2 * a[3]
    else:
        span = out.numel()
    return (lambda: fn(*a, **kw)), out, span, op, f"{tuple(out.shape)}"


class Shadow:
    def __init__(self, label=""):
        self.label = label
        self.records = []
        self.calls = collections.Counter()
        self.peak_bytes = 0

    def _wrap(self, op, real):
        def run(*a, **kw):
            self.calls[op] += 1
            site = _site()
            torch.cuda.synchronize()
            thunk, out, span, path, geo = _prepare(op, a, kw)
            r = real(*a, **kw)
            torch.cuda.synchronize()
            with torch.no_grad():
                ref = thunk()
                v = O.check(O.flat(out, span), ref)
            del ref
            self.peak_bytes = max(self.peak_bytes, torch.cuda.max_memory_allocated())
            self.records.append({"op": op, "path": path, "geo": geo, "ratio": v.ratio, "where": v.where, "got": v.got,
                                 "want": v.want, "bound": v.bound, "site": site, "label": self.label})
            return r
        return run

    @contextlib.contextmanager
    def active(self):
        from animate3d_b200 import ops
        saved = {n: getattr(ops, n) for n in OPS + ("view5",)}
        real_view5 = saved["view5"]

        def view5(base, col_offset, cols, strides, extents):
            v = real_view5(base, col_offset, cols, strides, extents)
            v._t, v._off = base, col_offset
            return v

        try:
            ops.view5 = view5
            for n in OPS:
                setattr(ops, n, self._wrap(n, saved[n]))
            yield self
        finally:
            for n, f in saved.items():
                setattr(ops, n, f)

    # ------------------------------------------------------------------------------------------ reports
    def failures(self):
        return [r for r in self.records if not r["ratio"] <= 1.0]

    def table(self, rows):
        lines = [f"{'ratio':>9}  {'op':<14} {'path':<30} {'site':<34} geometry / worst element"]
        for r in rows:
            lines.append(f"{r['ratio']:9.3g}  {r['op']:<14} {r['path']:<30} {r['site']:<34} {r['geo']} | {r['where']}: "
                         f"got {r['got']:.6g} want {r['want']:.6g} +- {r['bound']:.3g}")
        return "\n".join(lines)

    def summary(self):
        agg = collections.OrderedDict()
        for r in self.records:
            k = (r["op"], r["path"])
            n, w = agg.get(k, (0, 0.0))
            agg[k] = (n + 1, max(w, r["ratio"]))
        lines = [f"{'op':<20} {'path':<34} {'launches':>8} {'worst |err|/bound':>18}"]
        for (op, path), (n, w) in sorted(agg.items()):
            lines.append(f"{op:<20} {path:<34} {n:>8} {w:>18.3g}")
        return "\n".join(lines)


@contextlib.contextmanager
def counting():
    """A plain counting patch of the same functions (no oracle): the shadow must see the same number of calls."""
    from animate3d_b200 import ops
    saved = {n: getattr(ops, n) for n in OPS}
    calls = collections.Counter()

    def wrap(n, f):
        def run(*a, **kw):
            calls[n] += 1
            return f(*a, **kw)
        return run

    try:
        for n in OPS:
            setattr(ops, n, wrap(n, saved[n]))
        yield calls
    finally:
        for n, f in saved.items():
            setattr(ops, n, f)
