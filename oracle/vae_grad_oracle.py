"""float64 derivative and per-element bound for each hand-built backward of animate3d_b200/vae.py.

The VAE encoder's input gradient is assembled from five `torch.autograd.Function`s (`_Conv3`, `_Lin`, `_GroupNorm`,
`_ConvIn`, `_ConvOut`), each with its own backward recipe: flipped / transposed taps, a zero-inserted copy of the output
gradient for the stride-2 downsampler, `w^T` for the 1x1 layers, the forward's saved GroupNorm statistics, 4-channel slices of
the edge kernels.  Each function here takes what one Function call saw (the upstream gradient `g` it received, its layer dict
and geometry, plus `x` and the saved statistics for GroupNorm) and returns an `abi_oracle.Ref` over the gradient the call
returns, so `abi_oracle.check` / `assert_within` apply unchanged.

The value never reuses vae.py's recipe: it is the float64 autograd derivative of the forward op as torch writes it, evaluated
at `g`:
  _Conv3     F.conv2d(x, w16, padding=1), or F.conv2d(F.pad(x, (0, 1, 0, 1)), w16, stride=2) for the downsampler; w16 is the
             fp16 weight the forward kernel multiplies by (unpacked from the forward operand `w`, not from `wt`)
  _Lin       x @ W16^T, so the derivative is g @ W16 (W16 from the forward operand `w`)
  _ConvIn / _ConvOut   F.conv2d(x, W32, padding=1) with the fp32 weight (from the forward operand `w32`)
  _GroupNorm F.group_norm(x, 32, gamma, beta, eps=1e-6), then F.silu when the layer fuses it; eps is the model's (diffusers'
             norm_eps), not the one the call was given.
All of them but GroupNorm are linear in x, so their derivative is the same at any x; it is taken at x = 0.

Bounds follow abi_oracle's conventions (u16 = 2^-11, u32 = 2^-24, every bound times SLACK = 2, half the subnormal spacing at
each store):
  dgrad GEMMs (_Conv3, _Lin)  the input gradient is one a3d_gemm of fp16 operands: the products are exact in fp32 and the
             K-term fp32 sum errs by at most (K - 1) u32 times the sum of the absolute products; the plain epilogue (no bias, no
             residual, scale 1) rounds a few more times, each by at most u32 |value| <= u32 A, which (K + 2) and SLACK absorb
             (abi_oracle.gemm charges 4 u32 |value| for a general epilogue).  So
             |dx - value| <= SLACK ((K + 2) u32 A + u16 |value| + 2^-25), with A = |g| pushed through the same derivative with
             |w|, K = 9 cout for a 3x3 convolution (the zero-inserted copy only adds zero products) and K = cout for a linear
             layer.  A is computed from |g| and |w|, not from the operands vae.py builds.
  edge convolutions  abi_oracle's conv_in / conv_out form: fp32 products and sums, (9 cout + 2) u32 A; _ConvIn.backward
             stores fp32 (u32 |value|), _ConvOut.backward fp16 (u16 |value|).
  GroupNorm  dx = rstd (g' - mean(g') - xhat mean(g' xhat)), g' = g gamma [silu'(z)], evaluated by the kernel at the saved
             statistics.  abi_oracle.group_norm_backward bounds the kernel against that formula at the saved statistics.  The
             saved statistics differ from the exact ones by at most the forward's bound (abi_oracle.group_norm: mean
             es D, rstd (0.5 es (1 + 4 D^2 / (var + eps)) + 2 u32) relative, es = (128 + 4 log2 n + 16) u32, D the largest
             |x - mean| of the group, plus the fp32 store of each statistic, times SLACK); that difference moves dx by at most
             |d dx / d mean| dmean + |d dx / d rstd| drstd to first order, the partial derivatives taken by forward-mode
             autograd of the same formula at the exact statistics.  The bound is the sum of the two.  `group_norm_stats`
             checks the saved (mean, rstd) pairs against the forward's bound on their own.
  residuals  the gradient a residual receives is g itself, so it must be torch.equal to g (bound 0)."""
from __future__ import annotations

import math
from typing import Callable

import torch
import torch.nn.functional as F

from oracle import abi_oracle as O
from oracle.abi_oracle import F64, SLACK, U32, Ref

GROUPS = 32
EPS = 1e-6                  # diffusers AutoencoderKL norm_eps (oracle/vae_oracle.py VAEConfig.norm_eps)


# ------------------------------------------------------------------------------------------------ helpers
def _vjp(fwd: Callable[[torch.Tensor], torch.Tensor], shape, gy: torch.Tensor, at=None) -> torch.Tensor:
    """float64 autograd derivative of fwd at `at` (zeros by default: the linear maps), applied to gy."""
    x = (torch.zeros(shape, dtype=F64, device=gy.device) if at is None else at.detach().clone()).requires_grad_(True)
    with torch.enable_grad():
        (d,) = torch.autograd.grad(fwd(x), x, gy)
    return d


def _nchw(rows: torch.Tensor, n: int, h: int, w: int) -> torch.Tensor:
    """NHWC rows [n h w, c] -> float64 [n, c, h, w]."""
    return rows.reshape(n, h, w, -1).to(F64).permute(0, 3, 1, 2)


def _rows(t: torch.Tensor) -> torch.Tensor:
    """[n, c, h, w] -> flat NHWC rows."""
    return t.permute(0, 2, 3, 1).reshape(-1)


def _rows_where(n, h, w, c):
    def where(i):
        img, r = divmod(int(i), h * w * c)
        p, ch = divmod(r, c)
        return f"image {img} of {n}, pixel (y {p // w}, x {p % w}) of {h}x{w}, channel {ch} (8-col group {ch // 8})"
    return where


def _nchw_where(n, c, h, w):
    def where(i):
        img, r = divmod(int(i), c * h * w)
        ch, p = divmod(r, h * w)
        return f"image {img} of {n}, channel {ch}, pixel (y {p // w}, x {p % w}) of {h}x{w}"
    return where


def conv3_weight(lay) -> torch.Tensor:
    """The fp16 weight a3d_gemm multiplies by in the forward, [cout, cin, 3, 3] float64, from the forward operand
    [cout, (ky, kx, cin)]."""
    return lay["w"].to(F64).view(lay["cout"], 3, 3, lay["cin"]).permute(0, 3, 1, 2)


def edge_weight(lay) -> torch.Tensor:
    """The fp32 weight of an edge convolution, [cout, cin, 3, 3] float64, from the forward operand [cout, (cin, tap)]."""
    return lay["w32"].to(F64).view(lay["cout"], lay["cin"], 3, 3)


def conv3_forward(x: torch.Tensor, w: torch.Tensor, stride: int) -> torch.Tensor:
    """The forward op of `_Conv3` as torch writes it (diffusers' Downsample2D pads (0, 1, 0, 1) for stride 2)."""
    if stride == 1:
        return F.conv2d(x, w, padding=1)
    return F.conv2d(F.pad(x, (0, 1, 0, 1)), w, stride=2)


def _gemm_bound(v, va, K):
    return SLACK * O._store(v, (K + 2) * U32 * va)


# ------------------------------------------------------------------------------------------------ the five Functions
def conv3_backward(g, lay, n, h, w, stride) -> Ref:
    """`_Conv3.backward`: g [n (h/s)(w/s), cout] NHWC rows -> d/dx [n h w, cin] NHWC rows (fp16 store)."""
    cin, cout = lay["cin"], lay["cout"]
    wd = conv3_weight(lay).to(g.device)
    G = _nchw(g, n, h // stride, w // stride)
    d = lambda gy, ww: _vjp(lambda x: conv3_forward(x, ww, stride), (n, cin, h, w), gy)
    v, va = d(G, wd), d(G.abs(), wd.abs())
    return Ref(_rows(v), _rows(_gemm_bound(v, va, 9 * cout)), _rows_where(n, h, w, cin))


def lin_backward(g, lay) -> Ref:
    """`_Lin.backward`: g [M, cout] -> d/dx [M, cin] (fp16 store)."""
    cin, cout = lay["cin"], lay["cout"]
    wd = lay["w"].to(F64).view(cout, cin).to(g.device)
    gd = g.to(F64)
    d = lambda gy, ww: _vjp(lambda x: x @ ww.t(), (gd.shape[0], cin), gy)
    v, va = d(gd, wd), d(gd.abs(), wd.abs())
    return Ref(v.reshape(-1), _gemm_bound(v, va, cout).reshape(-1), lambda i: f"row {int(i) // cin} col {int(i) % cin}")


def conv_in_backward(g, lay, n, h, w) -> Ref:
    """`_ConvIn.backward`: g [n h w, cout] NHWC rows -> d/dx [n, cin, h, w] NCHW (fp32 store)."""
    cin, cout = lay["cin"], lay["cout"]
    wd = edge_weight(lay).to(g.device)
    G = _nchw(g, n, h, w)
    d = lambda gy, ww: _vjp(lambda x: F.conv2d(x, ww, padding=1), (n, cin, h, w), gy)
    v, va = d(G, wd), d(G.abs(), wd.abs())
    e = SLACK * O._store(v, (9 * cout + 2) * U32 * va, True)
    return Ref(v.reshape(-1), e.reshape(-1), _nchw_where(n, cin, h, w))


def conv_out_backward(g, lay, n, h, w) -> Ref:
    """`_ConvOut.backward`: g [n, cout, h, w] NCHW fp32 -> d/dx [n h w, cin] NHWC rows (fp16 store)."""
    cin, cout = lay["cin"], lay["cout"]
    wd = edge_weight(lay).to(g.device)
    G = g.reshape(n, cout, h, w).to(F64)
    d = lambda gy, ww: _vjp(lambda x: F.conv2d(x, ww, padding=1), (n, cin, h, w), gy)
    v, va = d(G, wd), d(G.abs(), wd.abs())
    e = SLACK * O._store(v, (9 * cout + 2) * U32 * va)
    return Ref(_rows(v), _rows(e), _rows_where(n, h, w, cin))


def _grouped(t, n, rows, c):
    return t.reshape(n, rows, c).to(F64).view(n, rows, GROUPS, c // GROUPS)


def _exact_stats(xg, eps):
    """-> mean, rstd, and the forward's bound on each (abi_oracle.group_norm, plus the fp32 store), [n, 1, G, 1]."""
    cnt = xg.shape[1] * xg.shape[3]
    mu = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg - mu) ** 2).mean(dim=(1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    D = (xg - mu).abs().amax(dim=(1, 3), keepdim=True)
    es = (128 + 4 * math.ceil(math.log2(max(cnt, 2))) + 16) * U32
    b_mu = SLACK * (es * D + U32 * mu.abs() + 2.0 ** -150)
    b_rstd = SLACK * (0.5 * es * (1 + 4 * D * D / (var + eps)) + 2 * U32 + U32) * rstd
    return mu, rstd, b_mu, b_rstd


def group_norm_stats(x, n, rows, eps=EPS) -> Ref:
    """The (mean, rstd) pairs `_GroupNorm.forward` saves, [n, G, 2] flat, against the exact statistics of x [n rows, c]."""
    c = x.shape[-1]
    mu, rstd, b_mu, b_rstd = _exact_stats(_grouped(x, n, rows, c), eps)
    v = torch.stack([mu.reshape(n, GROUPS), rstd.reshape(n, GROUPS)], -1)
    b = torch.stack([b_mu.reshape(n, GROUPS), b_rstd.reshape(n, GROUPS)], -1)
    return Ref(v.reshape(-1), b.reshape(-1),
               lambda i: f"image {int(i) // (2 * GROUPS)} group {(int(i) // 2) % GROUPS} {'rstd' if int(i) % 2 else 'mean'}")


def group_norm_forward(x4, gamma, beta, silu, eps=EPS):
    """GroupNorm(32) [+ SiLU] of the encoder as torch writes it, on [n, c, *]."""
    y = F.group_norm(x4, GROUPS, gamma, beta, eps)
    return F.silu(y) if silu else y


def group_norm_backward(x, g, gb, n, rows, silu, stats, eps=EPS) -> Ref:
    """`_GroupNorm.backward`: x, g [n rows, c] NHWC rows, gb = (gamma, beta), `stats` the saved (mean, rstd) pairs ->
    d/dx [n rows, c] (fp16 store)."""
    c = x.shape[-1]
    gamma, beta = gb[0].to(F64).to(x.device), gb[1].to(F64).to(x.device)
    to4 = lambda t: t.reshape(n, rows, c).to(F64).permute(0, 2, 1)
    v = _vjp(lambda t: group_norm_forward(t, gamma, beta, silu, eps), (n, c, rows), to4(g), at=to4(x)).permute(0, 2, 1)

    at_saved = O.group_norm_backward(x, c, gamma, beta, stats, g, None, n, rows, GROUPS, silu)
    xg, dyg = _grouped(x, n, rows, c), _grouped(g, n, rows, c)
    gm, bt = gamma.view(GROUPS, -1), beta.view(GROUPS, -1)

    def dx_at(mu, rstd):
        xh = (xg - mu) * rstd
        gg = dyg * gm
        if silu:
            z = xh * gm + bt
            s = torch.sigmoid(z)
            gg = gg * s * (1 + z * (1 - s))
        return rstd * (gg - gg.mean(dim=(1, 3), keepdim=True) - xh * (gg * xh).mean(dim=(1, 3), keepdim=True))

    mu, rstd, b_mu, b_rstd = _exact_stats(xg, eps)
    one, zero = torch.ones_like(mu), torch.zeros_like(mu)
    _, d_mu = torch.func.jvp(dx_at, (mu, rstd), (one, zero))
    _, d_rstd = torch.func.jvp(dx_at, (mu, rstd), (zero, one))
    e = at_saved.bound.view(n, rows, GROUPS, -1) + d_mu.abs() * b_mu + d_rstd.abs() * b_rstd
    return Ref(v.reshape(-1), e.reshape(-1), lambda i: f"image {int(i) // (rows * c)} of {n}, pixel {(int(i) // c) % rows}, "
                                                       f"channel {int(i) % c} (group {int(i) % c // (c // GROUPS)})")
