"""Thin torch-tensor wrappers over the C ABI (include/a3d.h).  torch supplies device memory and the stream only."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib as L

HALF = torch.float16

launches = 0     # kernels enqueued through these wrappers since import; a forward's count is the change over it


def _enqueued(rc: int, kernels: int = 1) -> None:
    """Raise on an error code, else count the kernels the entry point enqueued."""
    global launches
    L.check(rc)
    launches += kernels


def _chk16(*ts):
    for t in ts:
        if t is not None:
            assert t.is_cuda and t.dtype == HALF and t.is_contiguous(), (t.dtype, t.shape, t.is_contiguous())


def gemm(A: torch.Tensor, B: torch.Tensor, out: torch.Tensor, *, M: int, N: int, K: int, lda: int = 0, ldc: int = 0,
         conv: Optional[Tuple[int, int, int, int, int]] = None, bias=None, rowbias=None, rb_div: int = 1, rb_mod: int = 0,
         rb_ld: int = 0,
         acc_scale: float = 1.0, R1=None, ldr1: int = 0, r1_scale: float = 1.0, R2=None, ldr2: int = 0, geglu: bool = False,
         out_f32: bool = False, perm: Tuple[int, int] = (0, 0), impl: int = L.IMPL_AUTO, conv_nopad_lo: bool = False,
         gelu: bool = False) -> torch.Tensor:
    """out = epilogue(A @ B^T); see a3d_gemm in include/a3d.h.  `conv` = (n_img, H, W, C, stride) selects the implicit
    3x3 convolution A operand; `gelu` applies the erf GELU to the biased value (CLIP's MLP)."""
    assert not (geglu and gelu)
    lib = L.load()
    a = L.GemmArgs()
    a.A, a.B, a.C = A.data_ptr(), B.data_ptr(), out.data_ptr()
    a.M, a.N, a.K = M, N, K
    a.lda = lda or K
    n_out = N // 2 if geglu else N
    a.ldc = ldc or n_out
    if conv is not None:
        a.a_mode = L.A_CONV3
        a.conv_n, a.conv_h, a.conv_w, a.conv_c, a.conv_stride = conv
        a.conv_nopad_lo = int(conv_nopad_lo)
    else:
        a.a_mode = L.A_PLAIN
    a.bias = L.ptr(bias)
    a.rowbias = L.ptr(rowbias)
    a.rb_ld = (rb_ld or rowbias.stride(0)) if rowbias is not None else 0
    a.rb_div, a.rb_mod = rb_div, rb_mod
    a.acc_scale = acc_scale
    a.R1, a.ldr1, a.r1_scale = L.ptr(R1), ldr1 or N, r1_scale
    a.R2, a.ldr2 = L.ptr(R2), ldr2 or N
    a.geglu = L.EPI_GEGLU if geglu else (L.EPI_GELU if gelu else 0)
    a.out_f32 = int(out_f32)
    a.perm_a, a.perm_b = perm
    a.impl = impl
    _enqueued(lib.a3d_gemm(C.byref(a), L.stream_ptr()))
    return out


def view5(base: torch.Tensor, col_offset: int, cols: int, strides, extents) -> L.View5:
    v = L.View5()
    v.base = base.data_ptr() + 2 * col_offset
    v.s1, v.s2, v.s3, v.s4 = strides
    v.cols = cols
    v.e1, v.e2, v.e3, v.e4 = extents
    return v


def attention(q: L.View5, k: L.View5, v: L.View5, out: torch.Tensor, ostrides, *, heads: int, d: int, scale: float,
              kv_div: int = 1, kv_i3_zero: bool = False, accumulate: bool = False, out_scale: float = 1.0,
              impl: int = L.IMPL_AUTO, out_col_offset: int = 0) -> None:
    lib = L.load()
    a = L.AttnArgs()
    a.q, a.k, a.v = q, k, v
    a.out = out.data_ptr() + 2 * out_col_offset
    a.os1, a.os2, a.os3, a.os4 = ostrides
    a.heads, a.d, a.scale = heads, d, scale
    a.kv_div, a.kv_i3_zero = kv_div, int(kv_i3_zero)
    a.accumulate, a.out_scale, a.impl = int(accumulate), out_scale, impl
    _enqueued(lib.a3d_attention(C.byref(a), L.stream_ptr()))


def temporal_attn(qkv: torch.Tensor, out: torch.Tensor, pixels: int, frames: int, heads: int, d: int, scale: float,
                  ldo: int = 0, out_col_offset: int = 0):
    """out rows have stride `ldo` halves (0 = heads*d) and start at column `out_col_offset` of `out`."""
    lib = L.load()
    _enqueued(lib.a3d_temporal_attn(C.c_void_p(qkv.data_ptr()), C.c_void_p(out.data_ptr() + 2 * out_col_offset), C.c_int64(pixels),
                                  frames, heads, d, C.c_float(scale), C.c_int64(ldo), L.stream_ptr()))


def group_norm_ws_floats(samples: int, rows_per_sample: int, c: int, groups: int) -> int:
    """fp32 elements of scratch a3d_group_norm needs for this geometry."""
    lib = L.load()
    return (int(lib.a3d_group_norm_ws_bytes(C.c_int64(samples), C.c_int64(rows_per_sample), c, groups)) + 3) // 4


def group_norm(x1, c1, x2, c2, gamma, beta, y, samples, rows_per_sample, groups, eps, silu, ws_stats, perm=(0, 0)):
    lib = L.load()
    assert ws_stats.numel() >= group_norm_ws_floats(samples, rows_per_sample, c1 + (c2 if x2 is not None else 0), groups)
    _enqueued(lib.a3d_group_norm(C.c_void_p(x1.data_ptr()), c1, C.c_void_p(L.ptr(x2)), c2, C.c_void_p(gamma.data_ptr()),
                               C.c_void_p(beta.data_ptr()), C.c_void_p(y.data_ptr()), C.c_int64(samples),
                               C.c_int64(rows_per_sample), groups, C.c_float(eps), int(silu), C.c_int64(perm[0]),
                               C.c_int64(perm[1]), C.c_void_p(ws_stats.data_ptr()), L.stream_ptr()), 3)
    return y


def group_norm_backward(x, c, gamma, beta, fwd_stats, dy, dx, samples, rows_per_sample, groups, silu, ws):
    lib = L.load()
    _enqueued(lib.a3d_group_norm_backward(C.c_void_p(x.data_ptr()), c, C.c_void_p(gamma.data_ptr()), C.c_void_p(beta.data_ptr()),
                                        C.c_void_p(fwd_stats.data_ptr()), C.c_void_p(dy.data_ptr()), C.c_void_p(dx.data_ptr()),
                                        C.c_int64(samples), C.c_int64(rows_per_sample), groups, int(silu), C.c_void_p(ws.data_ptr()),
                                        L.stream_ptr()), 3)
    return dx


def layer_norm(x, gamma, beta, y, rows, c, eps=1e-5):
    lib = L.load()
    _enqueued(lib.a3d_layer_norm(C.c_void_p(x.data_ptr()), C.c_void_p(gamma.data_ptr()), C.c_void_p(beta.data_ptr()),
                               C.c_void_p(y.data_ptr()), C.c_int64(rows), c, C.c_float(eps), L.stream_ptr()))
    return y


def upsample2x(x, y, n, h, w, c):
    lib = L.load()
    _enqueued(lib.a3d_upsample2x(C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), C.c_int64(n), h, w, c, L.stream_ptr()))
    return y


def silu_rows(x, y, rows, c, rep):
    lib = L.load()
    _enqueued(lib.a3d_silu_rows(C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), C.c_int64(rows), c, rep, L.stream_ptr()))
    return y


def conv_in(sample, w, b, y, bn, cin, f, h, wd, cout):
    lib = L.load()
    _enqueued(lib.a3d_conv_in(C.c_void_p(sample.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(b.data_ptr()),
                            C.c_void_p(y.data_ptr()), bn, cin, f, h, wd, cout, L.stream_ptr()))
    return y


def conv_out(x, w, b, y, bn, cin, f, h, wd, cout):
    lib = L.load()
    _enqueued(lib.a3d_conv_out(C.c_void_p(x.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(b.data_ptr()),
                             C.c_void_p(y.data_ptr()), bn, cin, f, h, wd, cout, L.stream_ptr()))
    return y


def timestep_proj(t, out, rows, half):
    lib = L.load()
    _enqueued(lib.a3d_timestep_proj(C.c_void_p(t.data_ptr()), C.c_void_p(out.data_ptr()), rows, half, L.stream_ptr()))
    return out


def linear_f32(x, w, b, y, m, n, k, act_in=0, accumulate=False):
    lib = L.load()
    _enqueued(lib.a3d_linear_f32(C.c_void_p(x.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(L.ptr(b)),
                               C.c_void_p(y.data_ptr()), m, n, k, act_in, int(accumulate), L.stream_ptr()))
    return y


def cast_f32_f16(x, y):
    lib = L.load()
    _enqueued(lib.a3d_cast_f32_f16(C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), C.c_int64(x.numel()), L.stream_ptr()))
    return y


def ddim_cfg_step(latents, noise_pred, first_frame, bn, c, f, hw, guidance, alpha_t, alpha_prev, uncond_first=True):
    lib = L.load()
    _enqueued(lib.a3d_ddim_cfg_step(C.c_void_p(latents.data_ptr()), C.c_void_p(noise_pred.data_ptr()),
                                  C.c_void_p(L.ptr(first_frame)), bn, c, f, hw, C.c_float(guidance), C.c_float(alpha_t),
                                  C.c_float(alpha_prev), int(uncond_first), L.stream_ptr()))
    return latents


def clip_resize_tables(h: int, w: int):
    """Host-built Pillow bicubic tables of the CLIP resize of an h x w image: (resize_h, resize_w, (bounds_y, coeffs_y,
    ksize_y), (bounds_x, coeffs_x, ksize_x)) with int32 CPU tensors."""
    lib = L.load(require_gpu=False)
    rh, rw, ky, kx = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    L.check(lib.a3d_clip_resize_plan(h, w, C.byref(rh), C.byref(rw), C.byref(ky), C.byref(kx)))
    tabs = []
    for n_in, n_out, k in ((h, rh.value, ky.value), (w, rw.value, kx.value)):
        b = torch.empty(n_out, 2, dtype=torch.int32)
        c = torch.empty(n_out, k, dtype=torch.int32)
        L.check(lib.a3d_clip_resize_coeffs(n_in, n_out, C.c_void_p(b.data_ptr()), C.c_void_p(c.data_ptr())))
        tabs.append((b, c, k))
    return rh.value, rw.value, tabs[0], tabs[1]


def clip_preprocess(src: torch.Tensor, src_format: int, patches: Optional[torch.Tensor], pixel_values: Optional[torch.Tensor] = None,
                    tables=None) -> None:
    """a3d_clip_preprocess.  `tables` = (resize_h, resize_w, (bounds_y, coeffs_y, ksize_y), (bounds_x, coeffs_x, ksize_x)) with
    the tensors on the device (None for CLIP_SRC_PIXELS)."""
    lib = L.load()
    a = L.ClipPrepArgs()
    a.src, a.src_format = src.data_ptr(), src_format
    a.n = src.shape[0]
    if src_format == L.CLIP_SRC_U8_NHWC:
        a.h, a.w = src.shape[1], src.shape[2]
    else:
        a.h, a.w = src.shape[2], src.shape[3]
    if tables is not None:
        a.resize_h, a.resize_w, (by, cy, a.ksize_y), (bx, cx, a.ksize_x) = tables
        a.bounds_y, a.coeffs_y, a.bounds_x, a.coeffs_x = by.data_ptr(), cy.data_ptr(), bx.data_ptr(), cx.data_ptr()
    a.patches, a.pixel_values = L.ptr(patches), L.ptr(pixel_values)
    _enqueued(lib.a3d_clip_preprocess(C.byref(a), L.stream_ptr()))
