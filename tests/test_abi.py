"""The C-ABI shared library loads without a GPU and exports every entry point include/a3d.h declares (no compute calls)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "a3d.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(a3d_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_hot_path():
    syms = declared_symbols()
    for s in ("a3d_gemm", "a3d_attention", "a3d_temporal_attn", "a3d_group_norm", "a3d_layer_norm", "a3d_ddim_cfg_step",
              "a3d_raster_forward", "a3d_raster_backward", "a3d_init", "a3d_last_error"):
        assert s in syms


def test_library_exports_every_declared_symbol():
    from animate3d_b200.build import build
    from animate3d_b200 import _lib
    build()
    lib = _lib.load(require_gpu=False)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"declared in include/a3d.h but not exported by liba3d.so: {missing}"
    assert lib.a3d_version() == 101


def test_hot_path_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from animate3d_b200 import _lib
    with pytest.raises(_lib.A3DError):
        _lib.load(require_gpu=True)
