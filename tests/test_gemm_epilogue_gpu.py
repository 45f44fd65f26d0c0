"""The tensor-core GEMM's epilogue operands (bias slice and row-bias rows staged in shared memory per warpgroup) against the
float64 ABI oracle, element by element (oracle/abi_oracle.py: per-element bounds).  The cases walk the row-bias slot mapping:
rb_div that does not divide a warpgroup's 64 rows, tables whose rows wrap inside a warpgroup (rb_mod < 64), CLIP's 257-row
position table, ragged M and N, an odd row stride at a 4-byte-aligned pointer, and each operand alone across the epilogues
and tile widths."""
import pytest
import torch

from oracle import abi_gelu as G
from oracle import abi_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _run(M, N, K, *, bias=False, rowbias=None, epi="plain", seed=0):
    """rowbias: None or (rb_div, rb_mod, table_rows, col_offset, rb_ld); table_rows None = what the oracle needs."""
    from animate3d_b200 import ops, _lib as L
    L.load()
    g = torch.Generator(device=DEV).manual_seed(seed + M + N + K)
    geglu, f32 = epi == "geglu", epi == "f32"
    n_out = N // 2 if geglu else N
    A = (torch.randn(M, K, device=DEV, generator=g) * 0.5).half()
    B = (torch.randn(N, K, device=DEV, generator=g) * 0.05).half()
    kw = dict(M=M, N=N, K=K, bias=torch.randn(N, device=DEV, generator=g) if bias else None, geglu=geglu,
              out_f32=f32)
    if rowbias is not None:
        div, mod, rows, off, ld = rowbias
        rows = rows or min(mod, (M - 1) // div + 1)
        ld = ld or N
        # exactly `rows` table rows: the last one ends at the end of its allocation
        flat = torch.randn((rows - 1) * ld + off + N, device=DEV, generator=g)
        kw.update(rowbias=flat[off:], rb_ld=ld, rb_div=div, rb_mod=mod, rb_rows=rows)
    if epi == "res":
        kw.update(R2=torch.randn(M, N, device=DEV, generator=g).half(), R1=torch.randn(M, N, device=DEV, generator=g).half(),
                  r1_scale=0.3)
    if epi == "gelu":
        kw.update(gelu=True)
    out = torch.randn(M, n_out, device=DEV, generator=g).to(torch.float32 if f32 else torch.float16)
    rb_rows = kw.pop("rb_rows", None)
    ref = G.gemm(A, B, out.clone(), rb_rows=rb_rows, **kw)
    ops.gemm(A, B, out, impl=L.IMPL_TC, **kw)
    torch.cuda.synchronize()
    return out, ref


SLOT_CASES = [
    # M, N, K, (rb_div, rb_mod, table rows, pointer offset in floats, rb_ld)
    (1000, 1152, 320, (3, 1 << 40, None, 0, 0)),      # rb_div does not divide 64; ragged M and N at BN = 256
    (1000, 320, 320, (5, 1 << 40, None, 0, 0)),       # ... BN = 160
    (4096, 384, 64, (100, 1 << 40, None, 0, 0)),      # a warpgroup spans two quotients; BN = 128
    (2048, 1152, 320, (1, 3, None, 0, 0)),            # rb_mod < 64: the slots wrap
    (2048, 960, 320, (1, 16, None, 0, 0)),            # tqkv: 16 slots
    (2048, 1536, 320, (2, 16, None, 0, 0)),
    (1028, 1280, 640, (1, 257, None, 0, 0)),          # CLIP patch GEMM: 64 slots, the 256-column tile gives way
    (2000, 320, 320, (1, 257, None, 0, 0)),           # 64 slots at BN = 160
    (1000, 1152, 320, (16, 1 << 40, None, 0, 0)),     # M % 64 != 0, table with exactly the rows M needs
    (968, 320, 640, (64, 1 << 40, None, 0, 0)),       # conv temb: one table row per image
    (1000, 1152, 320, (16, 8, None, 1, 1155)),        # pointer one float past 16-byte alignment, odd rb_ld
    (1000, 320, 320, (7, 5, None, 1, 333)),
]


@pytest.mark.parametrize("case", SLOT_CASES, ids=lambda c: f"{c[0]}x{c[1]}x{c[2]}_div{c[3][0]}_mod{c[3][1]}_off{c[3][3]}")
@pytest.mark.parametrize("bias", [False, True], ids=["rb", "bias_rb"])
def test_rowbias_slots(case, bias):
    M, N, K, rb = case
    out, ref = _run(M, N, K, bias=bias, rowbias=rb)
    O.assert_within(O.flat(out, ref.value.numel()), ref, f"gemm {case} bias={bias}")


# (epilogue, N, K): N picks the tile width (256: N % 256 == 0 or short-K ragged; 160: N % 160 == 0; else 128)
EPI_SHAPES = [
    ("plain", 1024, 320), ("plain", 320, 320), ("plain", 384, 64),
    ("res", 1024, 320), ("res", 320, 320), ("res", 384, 64),
    ("geglu", 1024, 320), ("geglu", 384, 64),
    ("gelu", 1024, 320), ("gelu", 320, 320), ("gelu", 384, 64),
    ("f32", 1024, 320), ("f32", 320, 320), ("f32", 384, 64),
]


@pytest.mark.parametrize("operands", ["none", "bias", "rowbias", "both"])
@pytest.mark.parametrize("shape", EPI_SHAPES, ids=lambda s: f"{s[0]}_N{s[1]}")
def test_epilogue_operands(shape, operands):
    epi, N, K = shape
    M = 1000
    rb = (16, 8, None, 0, 0) if operands in ("rowbias", "both") else None
    out, ref = _run(M, N, K, bias=operands in ("bias", "both"), rowbias=rb, epi=epi)
    O.assert_within(O.flat(out, ref.value.numel()), ref, f"gemm {epi} N={N} {operands}")
