"""Which kernel a GEMM, attention or temporal-attention call runs, asked of the library itself (a3d_*_kernel through
ops.*_kernel) without a GPU.  The queries read operand addresses only for their alignment, so the operands here are bare
addresses.  The shapes are the product's where it has them (UNet at 32^2 latents, VAE at 256^2, CLIP ViT-H/14)."""
import ctypes

import pytest

from animate3d_b200 import _lib as L
from animate3d_b200 import ops

BASE = 1 << 32                      # 256-byte aligned, never dereferenced


class Buf:
    """A device address as ops reads it: data_ptr() and, for row-bias tables, stride(0)."""

    def __init__(self, addr=BASE, ld=0):
        self.addr, self.ld = addr, ld

    def data_ptr(self):
        return self.addr

    def stride(self, dim):
        return self.ld


@pytest.fixture(scope="module", autouse=True)
def library():
    from animate3d_b200.build import build
    build()


def gemm(**kw):
    A, B, C = kw.pop("A", Buf()), kw.pop("B", Buf()), kw.pop("C", Buf())
    return ops.gemm_kernel(A, B, C, **kw)


# ------------------------------------------------------------------------------------------------ GEMM tile width
@pytest.mark.parametrize("M,N,K,bn", [
    (4096, 1280, 320, 256),         # N % 256 == 0
    (4096, 1152, 320, 256),         # short K, ragged last 256-column tile (12.5 % idle columns)
    (4096, 960, 320, 256),          # ... ahead of N % 160 == 0
    (4096, 960, 1280, 160),         # long K: N % 160 == 0
    (4096, 640, 1280, 160),
    (4096, 384, 1280, 128),
    (4096, 1152, 1280, 128),        # long K, neither 256 nor 160 divides N
    (4096, 1088, 320, 128),         # short K but the ragged tile would idle more than 12.5 %
])
def test_gemm_tile_width(M, N, K, bn):
    assert gemm(M=M, N=N, K=K, bias=Buf()) == f"tc BN{bn} plain plain"


def test_gemm_geglu_tile_width():
    assert gemm(M=2048, N=2560, K=320, geglu=True) == "tc BN256 geglu plain"
    assert gemm(M=2048, N=640, K=320, geglu=True) == "tc BN128 geglu plain"     # N % 256 == 128


def test_gemm_rowbias_table_falls_back_to_128_columns():
    """CLIP's patch GEMM: a 257-row position table puts up to 64 distinct rows in one warpgroup's epilogue buffer, which
    leaves fewer than two operand stages of the 256-column tile."""
    n = 4
    patch = dict(M=n * 257, N=1280, K=640, rowbias=Buf(ld=1280), rb_mod=257)
    assert gemm(**patch) == "tc BN128 plain plain"
    assert gemm(**dict(patch, rb_mod=16)) == "tc BN256 plain plain"                # 16 rows per warpgroup fit
    assert gemm(**dict(patch, rb_div=257, rb_mod=n)) == "tc BN256 plain plain"     # one row per image
    assert gemm(M=1028, N=5120, K=1280, bias=Buf(), rowbias=Buf(ld=5120), rb_mod=257, gelu=True) == "tc BN128 gelu plain"
    assert gemm(M=77, N=256, K=64, bias=Buf(), rowbias=Buf(ld=256), rb_mod=257, gelu=True) == "tc BN128 gelu plain"
    assert gemm(M=1028, N=5120, K=1280, bias=Buf(), gelu=True) == "tc BN256 gelu plain"      # CLIP's fc1


def test_gemm_epilogue_instance():
    k = dict(M=4096, N=320, K=1280, bias=Buf())
    assert gemm(**k) == "tc BN160 plain plain"
    assert gemm(**k, R1=Buf()) == "tc BN160 res plain"
    assert gemm(**k, R2=Buf()) == "tc BN160 res plain"
    assert gemm(**k, perm=(4, 16)) == "tc BN160 res plain"
    assert gemm(**k, out_f32=True) == "tc BN160 f32 plain"
    assert gemm(**k, gelu=True) == "tc BN160 gelu plain"
    assert gemm(M=4096, N=2560, K=320, geglu=True, bias=Buf()) == "tc BN256 geglu plain"


@pytest.mark.parametrize("conv,N,want", [
    ((1, 256, 256, 128, 1), 128, "tc BN128 plain conv-wide-rows"),       # VAE decoder at 256^2: a tile is half an output row
    ((2, 32, 32, 320, 1), 320, "tc BN160 plain conv-row-block"),         # UNet at 32^2: four output rows per tile
    ((2, 32, 32, 320, 2), 320, "tc BN160 plain conv-row-block"),         # stride-2 downsampler
    ((4, 8, 8, 1280, 1), 1280, "tc BN256 plain conv-image-block"),       # 8^2: two images per tile
])
def test_gemm_conv_geometry(conv, N, want):
    n, h, w, c, s = conv
    assert gemm(M=n * (h // s) * (w // s), N=N, K=9 * c, conv=conv) == want


@pytest.mark.parametrize("kw", [
    dict(A=Buf(BASE + 2)),                          # misaligned A
    dict(K=1000),                                   # K % 64 != 0
    dict(lda=1284),                                 # lda % 8 != 0
    dict(R2=Buf(BASE + 16)),                        # residual not 32-byte aligned
    dict(M=1 << 31),                                # row index past 32 bits
    dict(conv=(2, 32, 32, 40, 1), M=2048, K=360),   # conv channels not a multiple of 64
], ids=["misaligned_a", "k_not_64", "lda", "r2_align", "m_32bit", "conv_c"])
def test_gemm_simt_fallback_and_forced_tc(kw):
    k = dict(M=4096, N=1280, K=1280)
    k.update(kw)
    assert gemm(**k) == "simt"
    assert gemm(**k, impl=L.IMPL_SIMT) == "simt"
    with pytest.raises(L.A3DError, match="not supported by the tensor-core path"):
        gemm(**k, impl=L.IMPL_TC)


def test_gemm_invalid_arguments():
    with pytest.raises(L.A3DError, match="GEGLU epilogue takes bias"):
        gemm(M=128, N=256, K=64, geglu=True, R1=Buf())
    with pytest.raises(L.A3DError, match="conv geometry"):
        gemm(M=100, N=320, K=2880, conv=(2, 32, 32, 320, 1))
    with pytest.raises(L.A3DError, match="impl 3"):
        gemm(M=128, N=256, K=64, impl=3)
    with pytest.raises(L.A3DError, match="do not hold the name"):
        args = ops._gemm_args(Buf(), Buf(), Buf(), M=128, N=256, K=64)
        L.check(L.load(require_gpu=False).a3d_gemm_kernel(ctypes.byref(args), ctypes.create_string_buffer(8), ctypes.c_size_t(8)))


# ------------------------------------------------------------------------------------------------ attention
def attention(lk, impl=L.IMPL_AUTO, d=40, q_addr=BASE, batches=6, frames=3):
    """Text cross-attention geometry: queries [(b f), 256] of d-wide heads, keys [b, lk] shared by the frames (kv_div)."""
    heads, dqk, dv = 8, (d + 15) // 16 * 16, (d + 16) // 16 * 16
    ldq, ldk = heads * dqk, 2 * heads * dqk + heads * dv
    hw, b = 256, batches // frames
    q = ops.view5(Buf(q_addr), 0, ldq, (ldq, hw * ldq, hw * ldq, frames * hw * ldq), (hw, 1, frames, b))
    k = ops.view5(Buf(), heads * dqk, ldk, (ldk, lk * ldk, lk * ldk, lk * ldk), (lk, 1, 1, b))
    v = ops.view5(Buf(), 2 * heads * dqk, ldk, (ldk, lk * ldk, lk * ldk, lk * ldk), (lk, 1, 1, b))
    C = heads * d
    return ops.attention_kernel(q, k, v, Buf(), (C, hw * C, hw * C, frames * hw * C), heads=heads, d=d, scale=d ** -0.5,
                                kv_div=frames, impl=impl)


@pytest.mark.parametrize("lk,want", [(1, "fewkeys"), (4, "fewkeys"), (8, "fewkeys"), (9, "shortkeys"), (77, "shortkeys"),
                                     (80, "shortkeys"), (81, "tc"), (1024, "tc")])
@pytest.mark.parametrize("d", [40, 80, 160])
def test_attention_by_key_count(lk, want, d):
    assert attention(lk, d=d) == want


def test_attention_forced_tensor_core_and_fallbacks():
    assert attention(77, impl=L.IMPL_TC) == "tc"
    assert attention(4, impl=L.IMPL_TC) == "tc"
    assert attention(77, q_addr=BASE + 2) == "tc"              # short-keys kernel reads Q rows 4 bytes at a time
    with pytest.raises(L.A3DError, match="operand rows must be 16-byte aligned"):
        attention(4, q_addr=BASE + 2)                          # few-keys kernel has no fallback
    with pytest.raises(L.A3DError, match="impl 2"):
        attention(77, impl=2)


# ------------------------------------------------------------------------------------------------ temporal attention
@pytest.mark.parametrize("frames,heads,d,want", [
    (16, 8, 40, "frames16"), (16, 8, 80, "frames16"), (16, 8, 160, "frames16"),
    (16, 4, 40, "generic"),           # heads % (320 / d) != 0
    (16, 6, 80, "generic"),
    (4, 8, 40, "generic"), (24, 8, 80, "generic"),
])
def test_temporal_kernel(frames, heads, d, want):
    assert ops.temporal_attn_kernel(Buf(), Buf(), 1024, frames, heads, d, d ** -0.5) == want


def test_temporal_invalid_arguments():
    with pytest.raises(L.A3DError, match="head dim 64"):
        ops.temporal_attn_kernel(Buf(), Buf(), 1024, 16, 8, 64, 0.125)
    with pytest.raises(L.A3DError, match="frames=33"):
        ops.temporal_attn_kernel(Buf(), Buf(), 1024, 33, 8, 40, 0.1)
    with pytest.raises(L.A3DError, match="output row stride"):
        ops.temporal_attn_kernel(Buf(), Buf(BASE + 8), 1024, 16, 8, 40, 0.1)
