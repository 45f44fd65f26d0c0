"""ctypes binding of liba3d.so (include/a3d.h).  There is no fallback: if the library or a CUDA device is missing the
hot path raises."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liba3d.so")

A_PLAIN, A_CONV3 = 0, 1
IMPL_AUTO, IMPL_TC, IMPL_SIMT = 0, 1, 2
EPI_GEGLU, EPI_GELU = 1, 2                       # a3d_gemm_args.geglu
CLIP_SRC_F32_NCHW, CLIP_SRC_U8_NHWC, CLIP_SRC_PIXELS = 0, 1, 2


class GemmArgs(C.Structure):
    _fields_ = [("A", C.c_void_p), ("B", C.c_void_p), ("C", C.c_void_p),
                ("M", C.c_int64), ("N", C.c_int64), ("K", C.c_int64),
                ("lda", C.c_int64), ("ldc", C.c_int64),
                ("a_mode", C.c_int),
                ("conv_n", C.c_int), ("conv_h", C.c_int), ("conv_w", C.c_int), ("conv_c", C.c_int), ("conv_stride", C.c_int),
                ("conv_nopad_lo", C.c_int),
                ("bias", C.c_void_p), ("rowbias", C.c_void_p),
                ("rb_ld", C.c_int64), ("rb_div", C.c_int64), ("rb_mod", C.c_int64),
                ("acc_scale", C.c_float),
                ("R1", C.c_void_p), ("ldr1", C.c_int64), ("r1_scale", C.c_float),
                ("R2", C.c_void_p), ("ldr2", C.c_int64),
                ("geglu", C.c_int), ("out_f32", C.c_int),
                ("perm_a", C.c_int64), ("perm_b", C.c_int64),
                ("impl", C.c_int)]


class View5(C.Structure):
    _fields_ = [("base", C.c_void_p), ("s1", C.c_int64), ("s2", C.c_int64), ("s3", C.c_int64), ("s4", C.c_int64),
                ("cols", C.c_int64), ("e1", C.c_int32), ("e2", C.c_int32), ("e3", C.c_int32), ("e4", C.c_int32)]


class AttnArgs(C.Structure):
    _fields_ = [("q", View5), ("k", View5), ("v", View5), ("out", C.c_void_p),
                ("os1", C.c_int64), ("os2", C.c_int64), ("os3", C.c_int64), ("os4", C.c_int64),
                ("heads", C.c_int), ("d", C.c_int), ("scale", C.c_float),
                ("kv_div", C.c_int), ("kv_i3_zero", C.c_int),
                ("accumulate", C.c_int), ("out_scale", C.c_float), ("impl", C.c_int)]


class ClipPrepArgs(C.Structure):
    _fields_ = [("src", C.c_void_p), ("src_format", C.c_int), ("n", C.c_int), ("h", C.c_int), ("w", C.c_int),
                ("resize_h", C.c_int), ("resize_w", C.c_int),
                ("bounds_y", C.c_void_p), ("coeffs_y", C.c_void_p), ("ksize_y", C.c_int),
                ("bounds_x", C.c_void_p), ("coeffs_x", C.c_void_p), ("ksize_x", C.c_int),
                ("patches", C.c_void_p), ("pixel_values", C.c_void_p)]


class RasterCam(C.Structure):
    _fields_ = [("viewmatrix", C.c_float * 16), ("projmatrix", C.c_float * 16), ("campos", C.c_float * 3),
                ("tanfovx", C.c_float), ("tanfovy", C.c_float)]


class RasterArgs(C.Structure):
    _fields_ = [("P", C.c_int), ("H", C.c_int), ("W", C.c_int), ("num_cams", C.c_int), ("cams", C.c_void_p),
                ("means3D", C.c_void_p), ("scales", C.c_void_p), ("rotations", C.c_void_p), ("opacities", C.c_void_p),
                ("shs", C.c_void_p), ("colors_precomp", C.c_void_p), ("sh_degree", C.c_int), ("sh_coeffs", C.c_int),
                ("per_cam_geometry", C.c_int), ("scale_modifier", C.c_float), ("bg", C.c_float * 3), ("deterministic", C.c_int)]


class SamplerStepArgs(C.Structure):
    _fields_ = [("latents", C.c_void_p), ("noise_pred", C.c_void_p), ("first_frame", C.c_void_p), ("noise", C.c_void_p),
                ("history_out", C.c_void_p), ("history_in", C.c_void_p),
                ("bn", C.c_int), ("c", C.c_int), ("f", C.c_int), ("hw", C.c_int),
                ("cfg_mode", C.c_int), ("guidance", C.c_float), ("kind", C.c_int), ("order", C.c_int),
                ("alpha_s0", C.c_float), ("sigma_s0", C.c_float), ("c_x", C.c_float), ("c_m0", C.c_float),
                ("inv_r0", C.c_float), ("c_d1", C.c_float),
                ("sigma", C.c_float), ("dt", C.c_float), ("sigma_up", C.c_float)]


_lib: Optional[C.CDLL] = None
_inited = False


class A3DError(RuntimeError):
    pass


def load(require_gpu: bool = True) -> C.CDLL:
    """dlopen liba3d.so; with require_gpu also run a3d_init() (sm_90 + TMA entry points)."""
    global _lib, _inited
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise A3DError(f"{LIB_PATH} is missing: build it with `python -m animate3d_b200.build` "
                           "(there is no CPU / PyTorch fallback for the hot path)")
        lib = C.CDLL(LIB_PATH)
        lib.a3d_last_error.restype = C.c_char_p
        lib.a3d_group_norm_ws_bytes.restype = C.c_size_t
        lib.a3d_raster_workspace_bytes.restype = C.c_size_t
        lib.a3d_raster_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]
        lib.a3d_raster_forward_rgba8_workspace_bytes.restype = C.c_size_t
        lib.a3d_raster_forward_rgba8_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]
        lib.a3d_raster_counters_offset.restype = C.c_size_t
        lib.a3d_raster_counters_offset.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]
        lib.a3d_raster_backward_scratch_bytes.restype = C.c_size_t
        lib.a3d_raster_backward_scratch_bytes.argtypes = [C.c_void_p, C.c_int64]
        lib.a3d_deform_backward_scratch_bytes.restype = C.c_size_t
        lib.a3d_deform_backward_scratch_bytes.argtypes = [C.c_void_p]
        lib.a3d_arap_scratch_bytes.restype = C.c_size_t
        lib.a3d_arap_scratch_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        lib.a3d_mesh_adjacency_scratch_bytes.restype = C.c_size_t
        lib.a3d_mesh_adjacency_scratch_bytes.argtypes = [C.c_int, C.c_int]
        lib.a3d_mesh_vertex_stats_scratch_bytes.restype = C.c_size_t
        lib.a3d_mesh_vertex_stats_scratch_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        lib.a3d_mesh_sample_neighbors.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_void_p,
                                                  C.c_void_p]
        lib.a3d_mesh_sample_neighbors_state.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.a3d_clip_resize_plan.argtypes = [C.c_int, C.c_int] + [C.POINTER(C.c_int)] * 4
        lib.a3d_clip_resize_coeffs.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _lib = lib
    if require_gpu and not _inited:
        if not torch.cuda.is_available():
            raise A3DError("animate3d_b200 needs a CUDA device (sm_90a); none is visible and there is no fallback")
        check(_lib.a3d_init())
        _inited = True
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise A3DError(f"liba3d error {rc}: {_lib.a3d_last_error().decode()}")


def stream_ptr() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def deterministic() -> int:
    """1 when torch.use_deterministic_algorithms(True) is in effect: the 4D-path kernels then sum in a fixed order."""
    return int(torch.are_deterministic_algorithms_enabled())


def scratch(nbytes: int, device) -> Optional[torch.Tensor]:
    """Caller-owned device scratch of the 4D-path entry points (None when a size query returned 0)."""
    return torch.empty(nbytes, dtype=torch.uint8, device=device) if nbytes else None
