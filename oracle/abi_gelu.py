"""float64 restatement of a3d_gemm's GELU epilogue (geglu = 2, include/a3d.h), with the per-element bound, in the terms of
oracle/abi_oracle.py (same Ref / check / store model):

  v = acc_scale (acc + bias + rowbias), the fp32 sum of K fp16 products: |dv| <= (K + 2) u32 (|A||B|^T + |bias| + |rowbias|)
  out = gelu_erf(v): the error of v propagates through |gelu'| <= 1.13, and the erf approximation with its rcp / ex2 steps
  adds 3 u32 (|v| + |gelu(v)|) (A-S 7.1.26: |erf err| <= 1.5e-7, i.e. <= 1.3 u32 |v| after the x / 2 factor); then the
  fp16 store.  Every bound is multiplied by SLACK = 2, as in abi_oracle.

`gemm(..., gelu=True)` restates that epilogue; without `gelu` it is abi_oracle.gemm unchanged, so a per-launch checker can
route every a3d_gemm call through this function."""
from __future__ import annotations

import torch

from oracle import abi_oracle as O

_plain_gemm = O.gemm          # bound at import: callers may route abi_oracle.gemm itself through this module's gemm


def gemm(A, B, out, *, M, N, K, lda=0, ldc=0, bias=None, rowbias=None, rb_div=1, rb_mod=0, rb_ld=0, acc_scale=1.0, impl=0,
         rb_rows=None, gelu=False, **rest) -> O.Ref:
    """a3d_gemm with the GELU epilogue; `out` holds the output buffer before the call (kept where nothing is written)."""
    if not gelu:
        return _plain_gemm(A, B, out, M=M, N=N, K=K, lda=lda, ldc=ldc, bias=bias, rowbias=rowbias, rb_div=rb_div, rb_mod=rb_mod,
                           rb_ld=rb_ld, acc_scale=acc_scale, impl=impl, rb_rows=rb_rows, **rest)
    if rest.get("conv") is not None or rest.get("R1") is not None or rest.get("R2") is not None or rest.get("geglu") \
            or rest.get("out_f32") or rest.get("perm", (0, 0))[0]:
        raise ValueError("the GELU epilogue takes bias / row-bias only, a plain A operand and an fp16 output")
    lda, ldc = lda or K, ldc or N
    span = O.span_of(M, N, ldc)
    value = O.flat(out, span).to(O.F64).clone()
    bound = torch.zeros_like(value)
    dev = value.device
    Bd = O.mat(B, N, K, K).to(O.F64).to(dev)
    Bt, Bta = Bd.t(), Bd.abs().t()
    Ad = O.mat(A, M, K, lda).to(O.F64).to(dev)
    div = rb_div if rb_div > 0 else 1
    mod = rb_mod if rb_mod > 0 else 1 << 40
    if rowbias is not None:
        rb_ld = rb_ld or rowbias.stride(0)
        rbt = O.mat(rowbias, rb_rows or min(mod, (M - 1) // div + 1), N, rb_ld).to(O.F64).to(dev)
    bd = bias.to(O.F64).to(dev) if bias is not None else None
    cols = torch.arange(N, device=dev)
    chunk = max(1, O.CHUNK // max(K, N))
    for m0 in range(0, M, chunk):
        m = torch.arange(m0, min(M, m0 + chunk), device=dev)
        a = Ad[m]
        v, vb = a @ Bt, a.abs() @ Bta
        if bd is not None:
            v, vb = v + bd, vb + bd.abs()
        if rowbias is not None:
            r = rbt[(m // div) % mod]
            v, vb = v + r, vb + r.abs()
        e = (K + 2) * O.U32 * vb * abs(acc_scale)
        v = v * acc_scale
        res = O._gelu(v)
        err = O.SLACK * O._store(res, 1.13 * e + 3 * O.U32 * (v.abs() + res.abs()))
        idx = (m[:, None] * ldc + cols[None, :]).reshape(-1)
        value[idx] = res.reshape(-1)
        bound[idx] = err.reshape(-1)

    def where(i):
        r, c = divmod(int(i), ldc)
        if c >= N:
            return f"flat {i}: outside the written columns (row {r}, col {c})"
        return f"output row {r} (M-tile {r // 128} of 128 rows), col {c} (8-col group {c // 8})"

    return O.Ref(value, bound, where)
