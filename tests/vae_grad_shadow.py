"""Backward shadow of the VAE encoder: while the context manager is active, vae.py's five autograd Functions (`_Conv3`, `_Lin`,
`_GroupNorm`, `_ConvIn`, `_ConvOut`) are replaced by subclasses whose backward runs the parent's backward and then checks
what it returned, element by element, against oracle/vae_grad_oracle.py at the upstream gradient the call received.  The
residual gradient must be `torch.equal` to that upstream gradient, and `_GroupNorm`'s saved (mean, rstd) pairs must be the
forward's within its bound.  No product code changes: the module attributes are swapped for the length of the context.

With `images` given, every call is checked on those images only (each image's slice of g and of d/dx; NHWC rows are
image-major, `_ConvIn`'s d/dx and `_ConvOut`'s g are NCHW), so a 64-image batch costs three images of float64 work.  Each
record keeps the Function, the layer's name in `AutoencoderKL.W`, its kind and geometry, the worst |err| / bound and where
it occurs."""
from __future__ import annotations

import collections
import contextlib
import math

import torch

from animate3d_b200 import vae as V
from oracle import abi_oracle as O
from oracle import vae_grad_oracle as G

FUNCTIONS = ("_Conv3", "_Lin", "_GroupNorm", "_ConvIn", "_ConvOut")
BASE = {f: getattr(V, f) for f in FUNCTIONS}
_ACTIVE = []


def layer_names(W, prefix=""):
    """id(layer dict) / id(gamma) -> its path in AutoencoderKL.W."""
    out = {}
    if isinstance(W, dict):
        if "cin" in W:
            out[id(W)] = prefix
            return out
        for k, v in W.items():
            out.update(layer_names(v, f"{prefix}.{k}" if prefix else k))
    elif isinstance(W, list):
        for i, v in enumerate(W):
            out.update(layer_names(v, f"{prefix}.{i}"))
    elif isinstance(W, tuple) and len(W) == 2 and all(isinstance(t, torch.Tensor) for t in W):
        out[id(W[0])] = prefix
    return out


class GradShadow:
    def __init__(self, label="", model=None, n=None, images=None):
        self.label = label
        self.names = layer_names(model.W) if model is not None else {}
        self.n = n                      # batch size (the images of a _Lin call are its rows split n ways)
        self.images = images            # None: check the whole batch at once
        self.records = []
        self.calls = collections.Counter()

    # ------------------------------------------------------------------------------------------ recording
    def _ranges(self, n):
        if self.images is None:
            return [(0, n)]
        assert max(self.images) < n, (self.images, n)
        return [(i, i + 1) for i in self.images]

    def _add(self, fn, name, kind, geo, images, got, ref):
        v = O.check(got, ref)
        self.records.append({"fn": fn, "name": name, "kind": kind, "geo": geo, "images": images, "ratio": v.ratio,
                             "where": v.where, "got": v.got, "want": v.want, "bound": v.bound, "label": self.label})

    def _residual(self, fn, name, geo, g, dres, has_res):
        ok = torch.equal(dres, g) if has_res and dres is not None else (dres is None and not has_res)
        what = "is g" if ok else "missing" if has_res and dres is None else "differs from g"
        self.records.append({"fn": fn, "name": name, "kind": "residual", "geo": geo, "images": "all", "ratio": 0.0 if ok else math.inf,
                             "where": f"residual gradient {what}",
                             "got": math.nan, "want": math.nan, "bound": 0.0, "label": self.label})

    # ------------------------------------------------------------------------------------------ the checks
    def conv3(self, ctx, g, out):
        lay = ctx.lay
        n, h, w, s = ctx.geom
        name = self.names.get(id(lay), "?")
        geo = f"n={n} {h}x{w} {lay['cin']}->{lay['cout']} stride {s}" + (" res" if ctx.has_res else "")
        self._residual("_Conv3", name, geo, g, out[1], ctx.has_res)
        rg, rx = (h // s) * (w // s), h * w
        for i0, i1 in self._ranges(n):
            ref = G.conv3_backward(g[i0 * rg:i1 * rg], lay, i1 - i0, h, w, s)
            self._add("_Conv3", name, f"conv3 stride {s}" + (" res" if ctx.has_res else ""), geo, (i0, i1), out[0][i0 * rx:i1 * rx], ref)

    def lin(self, ctx, g, out):
        lay = ctx.lay
        name = self.names.get(id(lay), "?")
        m = g.shape[0]
        geo = f"M={m} {lay['cin']}->{lay['cout']}" + (" res" if ctx.has_res else "")
        self._residual("_Lin", name, geo, g, out[1], ctx.has_res)
        n = self.n or 1
        per = m // n
        for i0, i1 in (self._ranges(n) if self.n else [(0, 1)]):
            ref = G.lin_backward(g[i0 * per:i1 * per], lay)
            self._add("_Lin", name, "lin" + (" res" if ctx.has_res else ""), geo, (i0, i1), out[0][i0 * per:i1 * per], ref)

    def group_norm(self, ctx, g, out):
        x, stats = ctx.saved_tensors
        gb, n, rows, silu = ctx.meta
        name = self.names.get(id(gb[0]), "?")
        c = x.shape[1]
        geo = f"n={n} rows={rows} c={c} silu={silu}"
        for i0, i1 in self._ranges(n):
            xs, st = x[i0 * rows:i1 * rows], stats[2 * G.GROUPS * i0:2 * G.GROUPS * i1]
            self._add("_GroupNorm", name, "gn stats", geo, (i0, i1), st, G.group_norm_stats(xs, i1 - i0, rows))
            ref = G.group_norm_backward(xs, g[i0 * rows:i1 * rows], gb, i1 - i0, rows, silu, st)
            self._add("_GroupNorm", name, f"gn silu {silu}", geo, (i0, i1), out[0][i0 * rows:i1 * rows], ref)

    def conv_in(self, ctx, g, out):
        lay = ctx.lay
        n, cin, h, w = ctx.geom
        name = self.names.get(id(lay), "?")
        geo = f"n={n} {h}x{w} {cin}->{lay['cout']}"
        for i0, i1 in self._ranges(n):
            ref = G.conv_in_backward(g[i0 * h * w:i1 * h * w], lay, i1 - i0, h, w)
            self._add("_ConvIn", name, f"conv_in cin {cin}", geo, (i0, i1), out[0][i0:i1], ref)

    def conv_out(self, ctx, g, out):
        lay = ctx.lay
        n, h, w = ctx.geom
        name = self.names.get(id(lay), "?")
        geo = f"n={n} {h}x{w} {lay['cin']}->{lay['cout']}"
        for i0, i1 in self._ranges(n):
            ref = G.conv_out_backward(g[i0:i1], lay, i1 - i0, h, w)
            self._add("_ConvOut", name, f"conv_out cout {lay['cout']}", geo, (i0, i1), out[0][i0 * h * w:i1 * h * w], ref)

    @contextlib.contextmanager
    def active(self):
        _ACTIVE.append(self)
        try:
            with _patched(CHECKED):
                yield self
        finally:
            _ACTIVE.remove(self)

    # ------------------------------------------------------------------------------------------ reports
    def failures(self):
        return [r for r in self.records if not r["ratio"] <= 1.0]

    def table(self, rows):
        lines = [f"{'ratio':>9}  {'Function':<11} {'layer':<28} {'kind':<20} geometry | images | worst element"]
        for r in rows:
            lines.append(f"{r['ratio']:9.3g}  {r['fn']:<11} {r['name']:<28} {r['kind']:<20} {r['geo']} | {r['images']} | "
                         f"{r['where']}: got {r['got']:.6g} want {r['want']:.6g} +- {r['bound']:.3g}")
        return "\n".join(lines)

    def summary(self):
        agg = collections.OrderedDict()
        for r in self.records:
            n, worst = agg.get(r["kind"], (0, None))
            agg[r["kind"]] = (n + 1, r if worst is None or r["ratio"] > worst["ratio"] else worst)
        lines = [f"{'kind':<20} {'checks':>6} {'worst |err|/bound':>18}  at"]
        for kind, (n, r) in sorted(agg.items()):
            lines.append(f"{kind:<20} {n:>6} {r['ratio']:>18.3g}  {r['name']} ({r['geo']}, images {r['images']}): {r['where']}")
        return "\n".join(lines)


def _checking(fn, check):
    base = BASE[fn]

    def backward(ctx, g):
        out = base.backward(ctx, g)
        sh = _ACTIVE[-1]
        sh.calls[fn] += 1
        with torch.no_grad():
            check(sh, ctx, g, out)
        return out

    return type(f"Checked{fn}", (base,), {"backward": staticmethod(backward)})


def _counting(fn, calls):
    base = BASE[fn]

    def backward(ctx, g):
        calls[fn] += 1
        return base.backward(ctx, g)

    return type(f"Counted{fn}", (base,), {"backward": staticmethod(backward)})


CHECKED = {"_Conv3": _checking("_Conv3", GradShadow.conv3), "_Lin": _checking("_Lin", GradShadow.lin),
           "_GroupNorm": _checking("_GroupNorm", GradShadow.group_norm), "_ConvIn": _checking("_ConvIn", GradShadow.conv_in),
           "_ConvOut": _checking("_ConvOut", GradShadow.conv_out)}


@contextlib.contextmanager
def _patched(classes):
    saved = {f: getattr(V, f) for f in FUNCTIONS}
    try:
        for f, cls in classes.items():
            setattr(V, f, cls)
        yield
    finally:
        for f, cls in saved.items():
            setattr(V, f, cls)


@contextlib.contextmanager
def counting():
    """A plain counting patch of the same Functions (no oracle): the shadow must check the same number of backward calls."""
    calls = collections.Counter()
    with _patched({f: _counting(f, calls) for f in FUNCTIONS}):
        yield calls
