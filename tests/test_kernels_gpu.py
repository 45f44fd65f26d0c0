"""Per-kernel parity on a real H100: every CUDA kernel behind the C ABI vs a plain fp32 torch restatement of the same op
on the same seeded fp16 inputs.  Tolerances: outputs are fp16 with fp32 accumulation -> rtol 1e-2 (north_star's budget)
on top of an absolute term scaled to the output magnitude."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from animate3d_b200 import ops, _lib
    _lib.load()
    return ops, _lib


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def close(a, b, tol=4e-3, what=""):
    e = rel_err(a, b)
    mx = (a.float() - b.float()).abs().max().item()
    assert math.isfinite(e) and e < tol, f"{what}: rel-l2 {e:.3e} max-abs {mx:.3e}"
    scale = b.float().abs().max().item() + 1e-6
    assert mx < 2e-2 * scale + 1e-3, f"{what}: max-abs {mx:.3e} vs scale {scale:.3e}"


def perm_rows(m, a, b):
    if a == 0:
        return m
    return (m // (a * b)) * (a * b) + (m % b) * a + (m // b) % a


# ------------------------------------------------------------------------------------------------------------ GEMM
GEMM_CASES = [
    # M, N, K, flags
    (128, 128, 64, ""),
    (256, 256, 128, "bias"),
    (1000, 320, 320, "bias,r2"),
    (4096, 640, 640, "bias,rowbias"),
    (2048, 1280, 1280, "bias,r1,r2,scale"),
    (616, 320, 768, ""),
    (8192, 2560, 320, "geglu"),
    (1024, 10240, 1280, "geglu"),
    (4096, 1536, 320, "bias"),
    (2048, 2688, 640, ""),
    (512, 5248, 1280, ""),
    (128, 20160, 1280, "bias,f32"),
    (4096, 320, 1280, "bias,perm,r2"),
]


def gemm_ref(A, B, flags, bias, rowbias, rb_div, rb_mod, acc_scale, R1, r1s, R2, perm):
    v = A.float() @ B.float().t()
    M = A.shape[0]
    if "geglu" in flags:
        if bias is not None:
            v = v + bias
        N = v.shape[1]
        v = v.reshape(M, N // 64, 2, 32)
        return (v[:, :, 0] * F.gelu(v[:, :, 1])).reshape(M, N // 2)
    if bias is not None:
        v = v + bias
    if rowbias is not None:
        idx = (torch.arange(M, device=A.device) // rb_div) % rb_mod
        v = v + rowbias[idx]
    v = v * acc_scale
    if R1 is not None:
        v = v + r1s * R1.float()
    rows = torch.arange(M, device=A.device)
    orow = perm_rows(rows, *perm)
    out = torch.empty_like(v)
    if R2 is not None:
        v = v + R2.float()[orow]
    out[orow] = v
    return out


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: f"{c[0]}x{c[1]}x{c[2]}_{c[3] or 'plain'}")
def test_gemm(case, impl):
    ops, L = _ops()
    M, N, K, flags = case
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    A = (torch.randn(M, K, device=DEV, generator=g) * 0.5).half()
    B = (torch.randn(N, K, device=DEV, generator=g) * 0.05).half()
    bias = torch.randn(N, device=DEV, generator=g) if "bias" in flags else None
    rb_div, rb_mod = 16, 8
    rowbias = torch.randn(rb_mod, N, device=DEV, generator=g) if "rowbias" in flags else None
    acc_scale = 0.7 if "scale" in flags else 1.0
    R1 = torch.randn(M, N, device=DEV, generator=g).half() if "r1" in flags else None
    R2 = torch.randn(M, N, device=DEV, generator=g).half() if "r2" in flags else None
    perm = (64, 16) if "perm" in flags else (0, 0)
    geglu = "geglu" in flags
    f32 = "f32" in flags
    out = torch.zeros(M, N // 2 if geglu else N, device=DEV, dtype=torch.float32 if f32 else torch.float16)
    ops.gemm(A, B, out, M=M, N=N, K=K, bias=bias, rowbias=rowbias, rb_div=rb_div, rb_mod=rb_mod, acc_scale=acc_scale,
             R1=R1, r1_scale=0.3, R2=R2, geglu=geglu, out_f32=f32, perm=perm,
             impl=L.IMPL_TC if impl == "tc" else L.IMPL_SIMT)
    torch.cuda.synchronize()
    ref = gemm_ref(A, B, flags, bias, rowbias, rb_div, rb_mod, acc_scale, R1, 0.3, R2, perm)
    close(out, ref, what=f"gemm {case} {impl}")


CONV_CASES = [
    # n, H, W, C, Cout, stride
    (4, 32, 32, 64, 128, 1),
    (3, 32, 32, 320, 320, 1),
    (8, 16, 16, 128, 160, 1),
    (4, 8, 8, 64, 256, 1),
    (16, 4, 4, 64, 128, 1),
    (5, 4, 4, 128, 128, 1),
    (4, 32, 32, 64, 128, 2),
    (8, 16, 16, 128, 128, 2),
    (8, 8, 8, 64, 128, 2),
    (2, 256, 256, 128, 128, 1),      # VAE level 0: an output row (256 px) is wider than the 128-row tile
    (1, 256, 256, 64, 64, 1),
]


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "n%d_%dx%d_c%d_o%d_s%d" % c)
def test_conv3x3(case, impl):
    ops, L = _ops()
    n, H, W, Cin, Cout, s = case
    g = torch.Generator(device=DEV).manual_seed(sum(case))
    x = (torch.randn(n, H, W, Cin, device=DEV, generator=g) * 0.5).half()
    w = (torch.randn(Cout, Cin, 3, 3, device=DEV, generator=g) * 0.05)
    bias = torch.randn(Cout, device=DEV, generator=g)
    wk = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous().half()      # k = (ky*3+kx)*Cin + c
    OH, OW = H // s, W // s
    M = n * OH * OW
    out = torch.zeros(M, Cout, device=DEV, dtype=torch.float16)
    ops.gemm(x, wk, out, M=M, N=Cout, K=9 * Cin, conv=(n, H, W, Cin, s), bias=bias,
             impl=L.IMPL_TC if impl == "tc" else L.IMPL_SIMT)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wk.float().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2), bias,
                   stride=s, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(M, Cout)
    close(out, ref, what=f"conv {case} {impl}")


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("case", [(2, 256, 256, 128, 128), (3, 64, 64, 256, 256), (4, 16, 16, 64, 128)], ids=lambda c: "n%d_%dx%d_c%d_o%d" % c)
def test_conv3x3_stride2_asymmetric_padding(case, impl):
    """SD-VAE Downsample2D: F.pad(x, (0, 1, 0, 1)) then conv(stride 2, padding 0) -- `conv_nopad_lo`."""
    ops, L = _ops()
    n, H, W, Cin, Cout = case
    g = torch.Generator(device=DEV).manual_seed(sum(case))
    x = (torch.randn(n, H, W, Cin, device=DEV, generator=g) * 0.5).half()
    w = torch.randn(Cout, Cin, 3, 3, device=DEV, generator=g) * 0.05
    bias = torch.randn(Cout, device=DEV, generator=g)
    wk = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous().half()
    M = n * (H // 2) * (W // 2)
    out = torch.zeros(M, Cout, device=DEV, dtype=torch.float16)
    ops.gemm(x, wk, out, M=M, N=Cout, K=9 * Cin, conv=(n, H, W, Cin, 2), bias=bias, conv_nopad_lo=True,
             impl=L.IMPL_TC if impl == "tc" else L.IMPL_SIMT)
    torch.cuda.synchronize()
    xp = F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1))
    ref = F.conv2d(xp, wk.float().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2), bias, stride=2, padding=0)
    close(out, ref.permute(0, 2, 3, 1).reshape(M, Cout), what=f"vae downsample conv {case} {impl}")


# ------------------------------------------------------------------------------------------------------------ attention
def dqk_of(d):
    return (d + 15) // 16 * 16


def dv_of(d):
    return (d + 1 + 15) // 16 * 16


def make_qkv(rows, heads, d, gen, n_q=1):
    """Projection-layout buffer [rows, n_q*H*dqk | H*dqk | H*dv]: zero padded q/k heads, V with the ones column."""
    dqk, dv = dqk_of(d), dv_of(d)
    q = torch.zeros(rows, n_q, heads, dqk, device=DEV)
    k = torch.zeros(rows, heads, dqk, device=DEV)
    v = torch.zeros(rows, heads, dv, device=DEV)
    q[..., :d] = torch.randn(rows, n_q, heads, d, device=DEV, generator=gen)
    k[..., :d] = torch.randn(rows, heads, d, device=DEV, generator=gen)
    v[..., :d] = torch.randn(rows, heads, d, device=DEV, generator=gen)
    v[..., d] = 1.0
    buf = torch.cat([q.reshape(rows, -1), k.reshape(rows, -1), v.reshape(rows, -1)], dim=1).half().contiguous()
    return buf, q.half().float()[..., :d], k.half().float()[..., :d], v.half().float()[..., :d]


ATTN_CASES = [
    # name, B, Nv, F, hw, d
    ("l0", 1, 4, 2, 1024, 40),
    ("l1", 1, 4, 2, 256, 80),
    ("l2", 1, 4, 2, 64, 160),
    ("l3", 1, 4, 2, 16, 160),
    ("l0_nv1", 1, 1, 2, 1024, 40),
    ("l2_nv1", 2, 1, 3, 64, 160),
    ("l1_b2", 2, 4, 3, 256, 80),
]


def sdpa_ref(q, k, v, scale):
    s = torch.einsum("bhqd,bhkd->bhqk", q, k) * scale
    return torch.einsum("bhqk,bhkd->bhqd", s.softmax(-1), v)


@pytest.mark.parametrize("layout", ["spatial_tf", "motion"])
@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("case", ATTN_CASES, ids=lambda c: c[0])
def test_cross_view_attention(case, impl, layout):
    """MV attention ("(b n f) l c -> (b f) (n l) c") + the I2V branch (frame-0 keys) through the strided views."""
    ops, L = _ops()
    name, B, Nv, Fr, hw, d = case
    heads = 8
    gen = torch.Generator(device=DEV).manual_seed(hash(name) % 1000)
    dqk, dv = dqk_of(d), dv_of(d)
    rows = B * Nv * Fr * hw
    buf, q, k, v = make_qkv(rows, heads, d, gen, n_q=2)
    ld = buf.shape[1]
    C = heads * d
    if layout == "spatial_tf":   # rows ordered (b n f p)
        strides = (ld, Fr * hw * ld, hw * ld, Nv * Fr * hw * ld)
        ostr = (C, Fr * hw * C, hw * C, Nv * Fr * hw * C)
        def to_bf(t):            # [rows, H, d] -> [(b f), H, (n p), d]
            return t.reshape(B, Nv, Fr, hw, heads, d).permute(0, 2, 4, 1, 3, 5).reshape(B * Fr, heads, Nv * hw, d)
        def from_bf(o):
            return o.reshape(B, Fr, heads, Nv, hw, d).permute(0, 3, 1, 4, 2, 5).reshape(rows, C)
    else:                        # motion-module rows ordered (b n p f)
        strides = (Fr * ld, hw * Fr * ld, ld, Nv * hw * Fr * ld)
        ostr = (Fr * C, hw * Fr * C, C, Nv * hw * Fr * C)
        def to_bf(t):
            return t.reshape(B, Nv, hw, Fr, heads, d).permute(0, 3, 4, 1, 2, 5).reshape(B * Fr, heads, Nv * hw, d)
        def from_bf(o):
            return o.reshape(B, Fr, heads, Nv, hw, d).permute(0, 3, 4, 1, 2, 5).reshape(rows, C)
    ext = (hw, Nv, Fr, B)
    qoff, q2off, koff, voff = 0, heads * dqk, 2 * heads * dqk, 3 * heads * dqk
    scale = d ** -0.5
    im = L.IMPL_TC if impl == "tc" else L.IMPL_SIMT
    out = torch.zeros(rows, C, device=DEV, dtype=torch.float16)
    vq = ops.view5(buf, qoff, ld - qoff, strides, ext)
    vk = ops.view5(buf, koff, ld - koff, strides, ext)
    vv = ops.view5(buf, voff, ld - voff, strides, ext)
    ops.attention(vq, vk, vv, out, ostr, heads=heads, d=d, scale=scale, impl=im)
    ref = from_bf(sdpa_ref(to_bf(q[:, 0]), to_bf(k), to_bf(v), scale))
    torch.cuda.synchronize()
    close(out, ref, what=f"mv attention {name} {impl} {layout}")
    # I2V branch: second query set, keys/values of frame 0 only, accumulated onto the first result with a scale
    vq2 = ops.view5(buf, q2off, ld - q2off, strides, ext)
    ops.attention(vq2, vk, vv, out, ostr, heads=heads, d=d, scale=scale, kv_i3_zero=True, accumulate=True,
                  out_scale=0.5, impl=im)
    kb, vb = to_bf(k), to_bf(v)
    k0 = kb.reshape(B, Fr, heads, Nv * hw, d)[:, 0:1].expand(B, Fr, heads, Nv * hw, d).reshape_as(kb)
    v0 = vb.reshape(B, Fr, heads, Nv * hw, d)[:, 0:1].expand(B, Fr, heads, Nv * hw, d).reshape_as(vb)
    ref2 = ref + 0.5 * from_bf(sdpa_ref(to_bf(q[:, 1]), k0, v0, scale))
    torch.cuda.synchronize()
    close(out, ref2, what=f"i2v attention {name} {impl} {layout}")


@pytest.mark.parametrize("impl", ["tc", "auto", "simt"])
@pytest.mark.parametrize("case", [(2, 3, 1024, 40, 77), (2, 2, 256, 80, 77), (3, 2, 64, 160, 4), (2, 2, 16, 160, 77),
                                  (2, 3, 1024, 40, 4), (3, 2, 256, 80, 4), (2, 2, 64, 160, 8), (2, 2, 256, 40, 16)],
                         ids=lambda c: "bn%d_f%d_hw%d_d%d_k%d" % c)
def test_cross_attention_text_keys(case, impl):
    """attn2 of the spatial transformers: queries [(bn f), hw], keys [bn, Lk] shared by the F frames (kv_div = F)."""
    ops, L = _ops()
    BN, Fr, hw, d, Lk = case
    heads = 8
    gen = torch.Generator(device=DEV).manual_seed(sum(case))
    dqk, dv = dqk_of(d), dv_of(d)
    rows = BN * Fr * hw
    qbuf, q, _, _ = make_qkv(rows, heads, d, gen)
    kvbuf, _, k, v = make_qkv(BN * Lk, heads, d, gen)
    ldq, ldk = qbuf.shape[1], kvbuf.shape[1]
    C = heads * d
    vq = ops.view5(qbuf, 0, ldq, (ldq, hw * ldq, hw * ldq, Fr * hw * ldq), (hw, 1, Fr, BN))
    vk = ops.view5(kvbuf, heads * dqk, ldk - heads * dqk, (ldk, Lk * ldk, Lk * ldk, Lk * ldk), (Lk, 1, 1, BN))
    vv = ops.view5(kvbuf, 2 * heads * dqk, ldk - 2 * heads * dqk, (ldk, Lk * ldk, Lk * ldk, Lk * ldk), (Lk, 1, 1, BN))
    out = torch.zeros(rows, C, device=DEV, dtype=torch.float16)
    scale = d ** -0.5
    im = {"tc": L.IMPL_TC, "auto": L.IMPL_AUTO, "simt": L.IMPL_SIMT}[impl]   # auto = few-keys / short-keys kernels
    ops.attention(vq, vk, vv, out, (C, hw * C, hw * C, Fr * hw * C), heads=heads, d=d, scale=scale, kv_div=Fr, impl=im)
    qq = q[:, 0].reshape(BN, Fr, hw, heads, d).permute(0, 1, 3, 2, 4)                  # [BN, F, H, hw, d]
    kk = k.reshape(BN, 1, Lk, heads, d).permute(0, 1, 3, 2, 4).expand(BN, Fr, heads, Lk, d)
    vv_ = v.reshape(BN, 1, Lk, heads, d).permute(0, 1, 3, 2, 4).expand(BN, Fr, heads, Lk, d)
    ref = sdpa_ref(qq.reshape(BN * Fr, heads, hw, d), kk.reshape(BN * Fr, heads, Lk, d), vv_.reshape(BN * Fr, heads, Lk, d),
                   scale)
    ref = ref.permute(0, 2, 1, 3).reshape(rows, C)
    torch.cuda.synchronize()
    close(out, ref, what=f"cross attention {case} {impl}")
    # IP-adapter use: a second key set accumulated onto the first result with a scale (attention_processor.py:218-238)
    ops.attention(vq, vk, vv, out, (C, hw * C, hw * C, Fr * hw * C), heads=heads, d=d, scale=scale, kv_div=Fr,
                  accumulate=True, out_scale=0.25, impl=im)
    torch.cuda.synchronize()
    close(out, 1.25 * ref, what=f"accumulated cross attention {case} {impl}")


# ------------------------------------------------------------------------------------------------------------ ops
@pytest.mark.parametrize("case", [(6, 64, 320, 0), (4, 256, 640, 320), (3, 1024, 320, 0), (2, 4 * 64, 1280, 1280)],
                         ids=lambda c: "s%d_r%d_c%d+%d" % c)
@pytest.mark.parametrize("silu", [0, 1])
def test_group_norm(case, silu):
    ops, _ = _ops()
    samples, rps, c1, c2 = case
    g = torch.Generator(device=DEV).manual_seed(sum(case))
    x1 = (torch.randn(samples * rps, c1, device=DEV, generator=g) * 1.5 + 0.3).half()
    x2 = (torch.randn(samples * rps, c2, device=DEV, generator=g) * 0.7 - 0.2).half() if c2 else None
    C = c1 + c2
    gamma = torch.randn(C, device=DEV, generator=g)
    beta = torch.randn(C, device=DEV, generator=g)
    y = torch.empty(samples * rps, C, device=DEV, dtype=torch.float16)
    ws = torch.empty(ops.group_norm_ws_floats(samples, rps, C, 32), device=DEV)
    perm = (rps // 4, 4) if c2 == 0 else (0, 0)
    ops.group_norm(x1, c1, x2, c2, gamma, beta, y, samples, rps, 32, 1e-5, silu, ws, perm=perm)
    y2 = torch.empty_like(y)
    ops.group_norm(x1, c1, x2, c2, gamma, beta, y2, samples, rps, 32, 1e-5, silu, ws, perm=perm)
    assert torch.equal(y, y2), "GroupNorm statistics are reduced in a fixed order: repeated calls must be bit-identical"
    x = x1.float() if x2 is None else torch.cat([x1.float(), x2.float()], 1)
    xr = x.reshape(samples, rps, C).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, gamma, beta, 1e-5)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(samples * rps, C)
    rows = torch.arange(samples * rps, device=DEV)
    out = torch.empty_like(ref)
    out[perm_rows(rows, *perm)] = ref
    torch.cuda.synchronize()
    close(y, out, what=f"group_norm {case}")


@pytest.mark.parametrize("case", [(2, 16 * 1024, 320), (8, 16 * 256, 640), (3, 100, 1280), (2, 7, 2560)], ids=lambda c: "s%d_r%d_c%d" % c)
def test_group_norm_large_mean_small_variance(case):
    """|mean| >> std (here 200 : 0.05): the E[x^2]-E[x]^2 form loses every significant digit of the variance in fp32; the
    pivoted (n, mean, M2) merge does not.  Also covers the over-frames geometry of the motion modules (16 x 1024 rows)."""
    ops, _ = _ops()
    samples, rps, c = case
    g = torch.Generator(device=DEV).manual_seed(sum(case))
    x = (200.0 + 0.0625 * torch.randn(samples * rps, c, device=DEV, generator=g)).half()    # fp16 spacing at 200 is 0.125
    gamma = torch.randn(c, device=DEV, generator=g)
    beta = torch.randn(c, device=DEV, generator=g)
    y = torch.empty_like(x)
    ws = torch.empty(ops.group_norm_ws_floats(samples, rps, c, 32), device=DEV)
    ops.group_norm(x, c, None, 0, gamma, beta, y, samples, rps, 32, 1e-5, 0, ws)
    xr = x.double().reshape(samples, rps, c).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, gamma.double(), beta.double(), 1e-5).permute(0, 2, 1).reshape(samples * rps, c)
    torch.cuda.synchronize()
    close(y, ref.float(), what=f"group_norm large mean {case}")


@pytest.mark.parametrize("case", [(3, 1024, 128), (2, 4096, 256), (4, 256, 512), (2, 65536, 128)], ids=lambda c: "s%d_r%d_c%d" % c)
@pytest.mark.parametrize("silu", [0, 1])
def test_group_norm_backward(case, silu):
    """d/dx of GroupNorm(32, eps 1e-6)(+SiLU) -- the VAE encoder's norms on the SDS gradient path -- vs torch autograd."""
    ops, _ = _ops()
    samples, rps, c = case
    g = torch.Generator(device=DEV).manual_seed(sum(case) + silu)
    x = (torch.randn(samples * rps, c, device=DEV, generator=g) * 1.3 + 0.2).half()
    dy = torch.randn(samples * rps, c, device=DEV, generator=g).half()
    gamma = torch.randn(c, device=DEV, generator=g)
    beta = torch.randn(c, device=DEV, generator=g)
    y = torch.empty_like(x)
    ws = torch.empty(ops.group_norm_ws_floats(samples, rps, c, 32), device=DEV)
    ops.group_norm(x, c, None, 0, gamma, beta, y, samples, rps, 32, 1e-6, silu, ws)
    stats = ws[: 2 * 32 * samples].clone()
    dx = torch.empty_like(x)
    ws2 = torch.empty_like(ws)
    ops.group_norm_backward(x, c, gamma, beta, stats, dy, dx, samples, rps, 32, silu, ws2)
    xr = x.float().reshape(samples, rps, c).permute(0, 2, 1).clone().requires_grad_(True)
    ref = F.group_norm(xr, 32, gamma, beta, 1e-6)
    if silu:
        ref = F.silu(ref)
    ref.backward(dy.float().reshape(samples, rps, c).permute(0, 2, 1))
    want = xr.grad.permute(0, 2, 1).reshape(samples * rps, c)
    torch.cuda.synchronize()
    close(dx, want, what=f"group_norm backward {case} silu={silu}")
    dx2 = torch.empty_like(x)
    ops.group_norm_backward(x, c, gamma, beta, stats, dy, dx2, samples, rps, 32, silu, ws2)
    assert torch.equal(dx, dx2)


@pytest.mark.parametrize("c", [320, 640, 1280])
def test_layer_norm(c):
    ops, _ = _ops()
    g = torch.Generator(device=DEV).manual_seed(c)
    x = (torch.randn(1000, c, device=DEV, generator=g) * 2 + 0.5).half()
    gamma = torch.randn(c, device=DEV, generator=g)
    beta = torch.randn(c, device=DEV, generator=g)
    y = torch.empty_like(x)
    ops.layer_norm(x, gamma, beta, y, 1000, c)
    torch.cuda.synchronize()
    close(y, F.layer_norm(x.float(), (c,), gamma, beta, 1e-5), what="layer_norm")


@pytest.mark.parametrize("case", [(300, 16, 40), (100, 16, 80), (50, 4, 160), (70, 16, 160)], ids=lambda c: "p%d_f%d_d%d" % c)
def test_temporal_attention(case):
    ops, _ = _ops()
    P, Fr, d = case
    heads = 8
    C = heads * d
    g = torch.Generator(device=DEV).manual_seed(sum(case))
    qkv = torch.randn(P, Fr, 3 * C, device=DEV, generator=g).half()
    out = torch.empty(P, Fr, C, device=DEV, dtype=torch.float16)
    ops.temporal_attn(qkv, out, P, Fr, heads, d, d ** -0.5)
    q, k, v = [t.float().reshape(P, Fr, heads, d).permute(0, 2, 1, 3) for t in qkv.chunk(3, dim=-1)]
    ref = sdpa_ref(q, k, v, d ** -0.5).permute(0, 2, 1, 3).reshape(P, Fr, C)
    torch.cuda.synchronize()
    close(out, ref, what="temporal attention")


def test_conv_in_out_upsample_misc():
    ops, _ = _ops()
    g = torch.Generator(device=DEV).manual_seed(7)
    bn, cin, f, h, w, cout = 3, 4, 5, 16, 16, 320
    sample = torch.randn(bn, cin, f, h, w, device=DEV, generator=g)
    wt = torch.randn(cout, cin, 3, 3, device=DEV, generator=g) * 0.1
    b = torch.randn(cout, device=DEV, generator=g)
    y = torch.empty(bn * f * h * w, cout, device=DEV, dtype=torch.float16)
    ops.conv_in(sample, wt, b, y, bn, cin, f, h, w, cout)
    x = sample.permute(0, 2, 1, 3, 4).reshape(bn * f, cin, h, w)
    ref = F.conv2d(x, wt, b, padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    torch.cuda.synchronize()
    close(y, ref, what="conv_in")
    # conv_out
    xo = torch.randn(bn * f * h * w, cout, device=DEV, generator=g).half()
    wo = torch.randn(4, cout, 3, 3, device=DEV, generator=g) * 0.05
    bo = torch.randn(4, device=DEV, generator=g)
    yo = torch.empty(bn, 4, f, h, w, device=DEV)
    ops.conv_out(xo, wo, bo, yo, bn, cout, f, h, w, 4)
    refo = F.conv2d(xo.float().reshape(bn * f, h, w, cout).permute(0, 3, 1, 2), wo, bo, padding=1)
    refo = refo.reshape(bn, f, 4, h, w).permute(0, 2, 1, 3, 4)
    torch.cuda.synchronize()
    close(yo, refo, what="conv_out")
    # upsample
    xu = torch.randn(6, 8, 8, 64, device=DEV, generator=g).half()
    yu = torch.empty(6, 16, 16, 64, device=DEV, dtype=torch.float16)
    ops.upsample2x(xu, yu, 6, 8, 8, 64)
    refu = F.interpolate(xu.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    assert torch.equal(yu.float(), refu)
    # timestep projection + small linear
    t = torch.tensor([961.0, 1.0, 500.0], device=DEV)
    tp = torch.empty(3, 320, device=DEV)
    ops.timestep_proj(t, tp, 3, 160)
    from oracle.unet_oracle import timesteps_proj
    torch.cuda.synchronize()
    torch.testing.assert_close(tp.cpu(), timesteps_proj(t.cpu(), 320), rtol=1e-4, atol=2e-4)
    wl = torch.randn(1280, 320, device=DEV, generator=g) * 0.05
    bl = torch.randn(1280, device=DEV, generator=g)
    yl = torch.empty(3, 1280, device=DEV)
    ops.linear_f32(tp, wl, bl, yl, 3, 1280, 320, act_in=1)
    torch.cuda.synchronize()
    torch.testing.assert_close(yl, F.linear(F.silu(tp), wl, bl), rtol=1e-4, atol=1e-4)


def test_ddim_cfg_step():
    ops, _ = _ops()
    g = torch.Generator(device=DEV).manual_seed(3)
    bn, c, f, hw = 4, 4, 6, 64
    lat = torch.randn(bn, c, f, hw, device=DEV, generator=g)
    eps = torch.randn(2 * bn, c, f, hw, device=DEV, generator=g)
    first = torch.randn(bn, c, 1, hw, device=DEV, generator=g)
    a_t, a_p, gs = 0.37, 0.52, 7.5
    e = eps[:bn] + gs * (eps[bn:] - eps[:bn])
    x0 = (lat - (1 - a_t) ** 0.5 * e) / a_t ** 0.5
    ref = a_p ** 0.5 * x0 + (1 - a_p) ** 0.5 * e
    ref = torch.cat([first, ref[:, :, 1:]], dim=2)
    ops.ddim_cfg_step(lat, eps, first, bn, c, f, hw, gs, a_t, a_p, True)
    torch.cuda.synchronize()
    torch.testing.assert_close(lat, ref, rtol=1e-5, atol=1e-5)
