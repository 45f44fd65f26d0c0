"""The float64 ABI oracle (oracle/abi_oracle.py) against independent formulations of the same operations, and its comparator
against deliberately broken outputs: every mutation below is the kind of fault a tiled kernel makes (one k-step, one column
group, one ragged tile, one key, one (batch, head)) and must be flagged, while the fp16-rounded oracle output must pass."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import abi_oracle as O

torch.manual_seed(0)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close64(a, b, tol=1e-10):
    a, b = a.reshape(-1).double(), b.reshape(-1).double()
    assert ((a - b).abs().max() / (b.abs().max() + 1e-30)).item() < tol


def _passes(got, ref):
    v = O.check(got, ref)
    assert v.ratio <= 1.0, v
    return v


def _flagged(got, ref):
    v = O.check(got, ref)
    assert v.ratio > 1.0, f"mutation not flagged: worst ratio {v.ratio:.3g} at {v.where}"
    return v


# ------------------------------------------------------------------------------------------------ oracle vs independent forms
@pytest.mark.parametrize("case", [(2, 8, 8, 16, 24, 1, False), (2, 8, 8, 16, 24, 2, False), (1, 8, 12, 16, 8, 2, True)],
                         ids=["s1", "s2", "s2_pad0101"])
def test_gemm_conv3_matches_conv2d(case):
    n, H, W, Cin, Cout, s, nopad = case
    g = _g(sum(case[:6]))
    x = torch.randn(n, H, W, Cin, generator=g).half()
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * 0.1
    bias = torch.randn(Cout, generator=g)
    wk = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous().half()
    M = n * (H // s) * (W // s)
    out = torch.zeros(M, Cout, dtype=torch.float16)
    ref = O.gemm(x, wk, out, M=M, N=Cout, K=9 * Cin, conv=(n, H, W, Cin, s), bias=bias, conv_nopad_lo=nopad)
    xi = x.double().permute(0, 3, 1, 2)
    wf = wk.double().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2)
    if nopad:
        want = F.conv2d(F.pad(xi, (0, 1, 0, 1)), wf, bias.double(), stride=s, padding=0)
    else:
        want = F.conv2d(xi, wf, bias.double(), stride=s, padding=1)
    _close64(ref.value, want.permute(0, 2, 3, 1).reshape(M, Cout))


def test_gemm_geglu_matches_interleave_then_chunk():
    from animate3d_b200.unet import _geglu_interleave
    g = _g(1)
    M, K, N = 40, 32, 256
    A = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) * 0.2)
    b = torch.randn(N, generator=g)
    rb = torch.randn(3, N, generator=g)
    wi = _geglu_interleave(w).half()
    bi, rbi = _geglu_interleave(b), _geglu_interleave(rb.t()).t().contiguous()
    out = torch.zeros(M, N // 2, dtype=torch.float16)
    ref = O.gemm(A, wi, out, M=M, N=N, K=K, bias=bi, rowbias=rbi, rb_div=5, rb_mod=3, acc_scale=0.6, geglu=True)
    h = (A.double() @ w.half().double().t() + b.double() + rb.double()[(torch.arange(M) // 5) % 3]) * 0.6
    u, gate = h.chunk(2, dim=1)
    _close64(ref.value, u * F.gelu(gate))


def test_gemm_strides_rowbias_slice_permutation_and_aliased_residual():
    """lda > K, ldc > N, ldr1 != N, a row-bias that is a column slice of a wider table (rb_ld > N), R2 = the output
    buffer read at the permuted row: against a Python loop over rows."""
    g = _g(2)
    M, N, K, lda, ldc, ldr1 = 24, 16, 8, 12, 24, 20
    pa, pb = 3, 4
    A = torch.randn(M, lda, generator=g).half()
    B = torch.randn(N, K, generator=g).half()
    table = torch.randn(5, 40, generator=g)
    rb = table[:, 7:]                                # rb_ld = 40
    R1 = torch.randn(M, ldr1, generator=g).half()
    out = torch.randn(M, ldc, generator=g).half()
    ref = O.gemm(A, B, out, M=M, N=N, K=K, lda=lda, ldc=ldc, rowbias=rb, rb_div=2, rb_mod=5, acc_scale=0.5, R1=R1, ldr1=ldr1,
                 r1_scale=0.25, R2=out, ldr2=ldc, perm=(pa, pb))
    want = out.double().clone()
    for m in range(M):
        om = (m // (pa * pb)) * (pa * pb) + (m % pb) * pa + (m // pb) % pa
        v = A[m, :K].double() @ B.double().t() + table[(m // 2) % 5, 7:7 + N].double()
        want[om, :N] = 0.5 * v + 0.25 * R1[m, :N].double() + out[om, :N].double()
    span = (M - 1) * ldc + N                         # the output span ends at the last row's last written column
    _close64(ref.value, want.reshape(-1)[:span])
    bound = torch.zeros(M * ldc, dtype=torch.float64)
    bound[:span] = ref.bound
    assert torch.equal(bound.view(M, ldc)[:, N:], torch.zeros(M, ldc - N, dtype=torch.float64))


def test_permutation_matches_python_loop():
    a, b = 4, 6
    m = torch.arange(3 * a * b)
    got = O.perm_rows(m, a, b)
    want = []
    for x in range(3):                # "(x a b) -> (x b a)": element (x, i, j) moves to (x, j, i)
        for i in range(a):
            for j in range(b):
                want.append(x * a * b + j * a + i)
    assert got.tolist() == want
    assert sorted(got.tolist()) == list(range(3 * a * b))


def _qkv_buf(rows, heads, d, g, n_q=1):
    dqk, dv = (d + 15) // 16 * 16, (d + 16) // 16 * 16
    q = torch.zeros(rows, n_q, heads, dqk)
    k = torch.zeros(rows, heads, dqk)
    v = torch.zeros(rows, heads, dv)
    q[..., :d] = torch.randn(rows, n_q, heads, d, generator=g)
    k[..., :d] = torch.randn(rows, heads, d, generator=g)
    v[..., :d] = torch.randn(rows, heads, d, generator=g)
    v[..., d] = 1.0
    buf = torch.cat([q.reshape(rows, -1), k.reshape(rows, -1), v.reshape(rows, -1)], 1).half()
    r = lambda t: t.half().double()[..., :d]
    return buf, r(q), r(k), r(v)


@pytest.mark.parametrize("layout", ["spatial_tf", "motion"])
def test_attention_views_match_written_out_rearranges(layout):
    """The view5 addressing against the "(b n f) l c -> (b f) (n l) c" regroupings of the two product layouts, for the
    cross-view call and the I2V call (frame-0 keys, accumulated at a column offset of a [M, 2C] buffer)."""
    B, Nv, Fr, hw, d, heads = 1, 2, 3, 8, 40, 2
    g = _g(3)
    dqk = 48
    rows = B * Nv * Fr * hw
    buf, q, k, v = _qkv_buf(rows, heads, d, g, n_q=2)
    ld = buf.shape[1]
    C = heads * d
    if layout == "spatial_tf":
        st = (ld, Fr * hw * ld, hw * ld, Nv * Fr * hw * ld)
        ostr = (2 * C, 2 * Fr * hw * C, 2 * hw * C, 2 * Nv * Fr * hw * C)
        to_bf = lambda t: t.reshape(B, Nv, Fr, hw, heads, d).permute(0, 2, 4, 1, 3, 5).reshape(B * Fr, heads, Nv * hw, d)
        from_bf = lambda o: o.reshape(B, Fr, heads, Nv, hw, d).permute(0, 3, 1, 4, 2, 5).reshape(rows, C)
    else:
        st = (Fr * ld, hw * Fr * ld, ld, Nv * hw * Fr * ld)
        ostr = (2 * Fr * C, 2 * hw * Fr * C, 2 * C, 2 * Nv * hw * Fr * C)
        to_bf = lambda t: t.reshape(B, Nv, hw, Fr, heads, d).permute(0, 3, 4, 1, 2, 5).reshape(B * Fr, heads, Nv * hw, d)
        from_bf = lambda o: o.reshape(B, Fr, heads, Nv, hw, d).permute(0, 3, 4, 1, 2, 5).reshape(rows, C)
    ext = (hw, Nv, Fr, B)
    hq = heads * dqk
    vq, vqi = O.V5(buf, 0, ld, st, ext), O.V5(buf, hq, ld - hq, st, ext)
    vk, vv = O.V5(buf, 2 * hq, ld - 2 * hq, st, ext), O.V5(buf, 3 * hq, ld - 3 * hq, st, ext)
    out = torch.randn(rows, 2 * C, generator=g).half()
    r1 = O.attention(vq, vk, vv, out, ostr, heads=heads, d=d, scale=d ** -0.5)
    want = out.double().clone()
    o1 = from_bf(O.sdpa_ref(to_bf(q[:, 0]), to_bf(k), to_bf(v), d ** -0.5))
    want[:, :C] = o1
    n1 = r1.value.numel()                            # the span ends at the last written column
    _close64(r1.value, want.reshape(-1)[:n1])
    bound = torch.zeros(rows * 2 * C, dtype=torch.float64)
    bound[:n1] = r1.bound
    assert torch.equal(bound.view(rows, 2 * C)[:, C:], torch.zeros(rows, C, dtype=torch.float64))
    r2 = O.attention(vqi, vk, vv, out, ostr, heads=heads, d=d, scale=d ** -0.5, kv_i3_zero=True, accumulate=True, out_scale=0.5,
                     out_col_offset=C)
    kb, vb = to_bf(k), to_bf(v)
    k0 = kb.reshape(B, Fr, heads, Nv * hw, d)[:, :1].expand(B, Fr, heads, Nv * hw, d).reshape_as(kb)
    v0 = vb.reshape(B, Fr, heads, Nv * hw, d)[:, :1].expand(B, Fr, heads, Nv * hw, d).reshape_as(vb)
    want2 = out.double().clone()
    want2[:, C:] += 0.5 * from_bf(O.sdpa_ref(to_bf(q[:, 1]), k0, v0, d ** -0.5))
    _close64(r2.value, want2)


def test_attention_kv_div_matches_explicit_expansion():
    """Text keys shared by F frames (kv_div = F) against the keys repeated per query batch."""
    BN, Fr, hw, Lk, d, heads = 2, 3, 8, 5, 80, 2
    g = _g(4)
    qbuf, q, _, _ = _qkv_buf(BN * Fr * hw, heads, d, g)
    kvbuf, _, k, v = _qkv_buf(BN * Lk, heads, d, g)
    dqk = 80
    ldq, ldk = qbuf.shape[1], kvbuf.shape[1]
    C = heads * d
    vq = O.V5(qbuf, 0, ldq, (ldq, hw * ldq, hw * ldq, Fr * hw * ldq), (hw, 1, Fr, BN))
    stk = (ldk, Lk * ldk, Lk * ldk, Lk * ldk)
    vk = O.V5(kvbuf, heads * dqk, ldk - heads * dqk, stk, (Lk, 1, 1, BN))
    vv = O.V5(kvbuf, 2 * heads * dqk, ldk - 2 * heads * dqk, stk, (Lk, 1, 1, BN))
    out = torch.zeros(BN * Fr * hw, C, dtype=torch.float16)
    ref = O.attention(vq, vk, vv, out, (C, hw * C, hw * C, Fr * hw * C), heads=heads, d=d, scale=0.1, kv_div=Fr)
    kk = k.reshape(BN, 1, Lk, heads, d).expand(BN, Fr, Lk, heads, d).reshape(BN * Fr, Lk, heads, d).permute(0, 2, 1, 3)
    vx = v.reshape(BN, 1, Lk, heads, d).expand(BN, Fr, Lk, heads, d).reshape(BN * Fr, Lk, heads, d).permute(0, 2, 1, 3)
    qq = q[:, 0].reshape(BN * Fr, hw, heads, d).permute(0, 2, 1, 3)
    _close64(ref.value, O.sdpa_ref(qq, kk, vx, 0.1).permute(0, 2, 1, 3).reshape(-1, C))


def test_temporal_attention_ldo_and_offset():
    P, Fr, heads, d = 5, 4, 2, 40
    C = heads * d
    g = _g(5)
    qkv = torch.randn(P, Fr, 3 * C, generator=g).half()
    out = torch.randn(P * Fr, 2 * C, generator=g).half()
    ref = O.temporal_attn(qkv, out, P, Fr, heads, d, d ** -0.5, ldo=2 * C, out_col_offset=C)
    q, k, v = [t.double().reshape(P, Fr, heads, d).permute(0, 2, 1, 3) for t in qkv.chunk(3, -1)]
    want = out.double().clone()
    want[:, C:] = O.sdpa_ref(q, k, v, d ** -0.5).permute(0, 2, 1, 3).reshape(P * Fr, C)
    _close64(ref.value, want)
    assert torch.equal(ref.bound.view(P * Fr, 2 * C)[:, :C], torch.zeros(P * Fr, C, dtype=torch.float64))


@pytest.mark.parametrize("silu", [0, 1])
def test_group_norm_matches_torch(silu):
    g = _g(6)
    samples, rps, c1, c2 = 2, 12, 64, 32
    x1 = torch.randn(samples * rps, c1, generator=g).half()
    x2 = torch.randn(samples * rps, c2, generator=g).half()
    gamma, beta = torch.randn(96, generator=g), torch.randn(96, generator=g)
    y = torch.empty(samples * rps, 96, dtype=torch.float16)
    ref = O.group_norm(x1, c1, x2, c2, gamma, beta, y, samples, rps, 32, 1e-5, silu, perm=(3, 4))
    x = torch.cat([x1, x2], 1).double().reshape(samples, rps, 96).permute(0, 2, 1)
    want = F.group_norm(x, 32, gamma.double(), beta.double(), 1e-5)
    want = (F.silu(want) if silu else want).permute(0, 2, 1).reshape(samples * rps, 96)
    out = torch.empty_like(want)
    out[O.perm_rows(torch.arange(samples * rps), 3, 4)] = want
    _close64(ref.value, out)


@pytest.mark.parametrize("silu", [0, 1])
def test_group_norm_backward_matches_autograd(silu):
    g = _g(7)
    samples, rps, c = 2, 16, 64
    x = torch.randn(samples * rps, c, generator=g).half()
    dy = torch.randn(samples * rps, c, generator=g).half()
    gamma, beta = torch.randn(c, generator=g), torch.randn(c, generator=g)
    xr = x.double().reshape(samples, rps, c).permute(0, 2, 1).clone().requires_grad_(True)
    y = F.group_norm(xr, 32, gamma.double(), beta.double(), 1e-6)
    (F.silu(y) if silu else y).backward(dy.double().reshape(samples, rps, c).permute(0, 2, 1))
    xg = x.double().reshape(samples, rps, 32, 2)
    mu = xg.mean(dim=(1, 3))
    rstd = 1 / torch.sqrt(xg.var(dim=(1, 3), unbiased=False) + 1e-6)
    stats = torch.stack([mu, rstd], -1).reshape(-1).float()
    ref = O.group_norm_backward(x, c, gamma, beta, stats, dy, None, samples, rps, 32, silu)
    _close64(ref.value, xr.grad.permute(0, 2, 1).reshape(-1), tol=1e-6)     # the stats went through fp32


def test_layer_norm_linear_and_small_ops():
    g = _g(8)
    x = torch.randn(10, 64, generator=g).half()
    gamma, beta = torch.randn(64, generator=g), torch.randn(64, generator=g)
    _close64(O.layer_norm(x, gamma, beta, None, 10, 64).value, F.layer_norm(x.double(), (64,), gamma.double(), beta.double(), 1e-5))
    xf, w, b = torch.randn(3, 16, generator=g), torch.randn(8, 16, generator=g), torch.randn(8, generator=g)
    y0 = torch.randn(3, 8, generator=g)
    r = O.linear_f32(xf, w, b, y0, 3, 8, 16, act_in=1, accumulate=True)
    _close64(r.value, y0.double() + F.linear(F.silu(xf.double()), w.double(), b.double()))
    xu = torch.randn(2, 3, 4, 8, generator=g).half()
    r = O.upsample2x(xu, None, 2, 3, 4, 8)
    _close64(r.value, F.interpolate(xu.double().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1))
    r = O.silu_rows(xf, None, 6, 16, 2)
    _close64(r.value, F.silu(xf.double()).repeat_interleave(2, 0))
    from oracle.unet_oracle import timesteps_proj
    t = torch.tensor([961.0, 1.0, 500.0])
    _close64(O.timestep_proj(t, None, 3, 160).value, timesteps_proj(t, 320).double(), tol=1e-4)     # an fp32 restatement


def test_conv_in_out_match_conv2d():
    g = _g(9)
    bn, cin, f, h, w, cout = 2, 4, 3, 6, 5, 16
    s = torch.randn(bn, cin, f, h, w, generator=g)
    wt, b = torch.randn(cout, cin, 3, 3, generator=g), torch.randn(cout, generator=g)
    r = O.conv_in(s, wt, b, None, bn, cin, f, h, w, cout)
    want = F.conv2d(s.double().permute(0, 2, 1, 3, 4).reshape(bn * f, cin, h, w), wt.double(), b.double(), padding=1)
    _close64(r.value, want.permute(0, 2, 3, 1))
    xo = torch.randn(bn * f * h * w, cout, generator=g).half()
    wo, bo = torch.randn(4, cout, 3, 3, generator=g), torch.randn(4, generator=g)
    r = O.conv_out(xo, wo, bo, None, bn, cout, f, h, w, 4)
    want = F.conv2d(xo.double().reshape(bn * f, h, w, cout).permute(0, 3, 1, 2), wo.double(), bo.double(), padding=1)
    _close64(r.value, want.reshape(bn, f, 4, h, w).permute(0, 2, 1, 3, 4))


def test_ddim_cfg_step_formula():
    g = _g(10)
    bn, c, f, hw = 2, 4, 3, 8
    lat = torch.randn(bn, c, f, hw, generator=g)
    eps = torch.randn(2 * bn, c, f, hw, generator=g)
    first = torch.randn(bn, c, 1, hw, generator=g)
    r = O.ddim_cfg_step(lat, eps, first, bn, c, f, hw, 7.5, 0.37, 0.52, True)
    e = eps[:bn].double() + 7.5 * (eps[bn:].double() - eps[:bn].double())
    x0 = (lat.double() - math.sqrt(0.63) * e) / math.sqrt(0.37)
    want = math.sqrt(0.52) * x0 + math.sqrt(0.48) * e
    want[:, :, :1] = first.double()
    _close64(r.value, want)


# ------------------------------------------------------------------------------------------------ comparator mutations
def _gemm_case(M=200, N=256, K=320, seed=11, **kw):
    g = _g(seed)
    A = (torch.randn(M, K, generator=g) * 0.5).half()
    B = (torch.randn(N, K, generator=g) * 0.05).half()
    bias = torch.randn(N, generator=g)
    out = torch.zeros(M, N, dtype=torch.float16)
    ref = O.gemm(A, B, out, M=M, N=N, K=K, bias=bias, **kw)
    return A, B, bias, ref


def test_mutation_gemm_rounded_oracle_passes_dropped_kstep_and_missing_bias_fail():
    M, N, K = 200, 256, 320
    A, B, bias, ref = _gemm_case(M, N, K)
    good = ref.value.half()                      # the ideal kernel: exact sum, one fp16 rounding
    _passes(good, ref)
    # a 16-wide k-step dropped in one 128 x 256 tile (rows 128..199, k 160..175)
    v = ref.value.view(M, N).clone()
    v[128:, :] -= A[128:, 160:176].double() @ B[:, 160:176].double().t()
    bad = _flagged(v.half(), ref)
    assert "M-tile 1" in bad.where
    # the bias missing on one 8-column group
    v = ref.value.view(M, N).clone()
    v[:, 40:48] -= bias[40:48].double()
    assert "8-col group 5" in _flagged(v.half(), ref).where


def test_mutation_two_rows_swapped_in_ragged_last_tile():
    M, N = 200, 128
    _, _, _, ref = _gemm_case(M, N, 64, seed=12)
    v = ref.value.view(M, N).clone()
    v[[190, 191]] = v[[191, 190]]
    _flagged(v.half(), ref)


def _attn_case(batches, heads, Lq, Lk, d, seed, out_scale=1.0, accumulate=False):
    g = _g(seed)
    dqk, dv = (d + 15) // 16 * 16, (d + 16) // 16 * 16
    qbuf, q, _, _ = _qkv_buf(batches * Lq, heads, d, g)
    kvbuf, _, k, v = _qkv_buf(batches * Lk, heads, d, g)
    ldq, ldk = qbuf.shape[1], kvbuf.shape[1]
    C = heads * d
    vq = O.V5(qbuf, 0, ldq, (ldq, Lq * ldq, Lq * ldq, Lq * ldq), (Lq, 1, 1, batches))
    stk = (ldk, Lk * ldk, Lk * ldk, Lk * ldk)
    vk = O.V5(kvbuf, heads * dqk, ldk - heads * dqk, stk, (Lk, 1, 1, batches))
    vv = O.V5(kvbuf, 2 * heads * dqk, ldk - 2 * heads * dqk, stk, (Lk, 1, 1, batches))
    out = torch.randn(batches * Lq, C, generator=g).half()
    ref = O.attention(vq, vk, vv, out, (C, Lq * C, Lq * C, Lq * C), heads=heads, d=d, scale=d ** -0.5, accumulate=accumulate,
                      out_scale=out_scale)
    qq = q[:, 0].reshape(batches, Lq, heads, d).permute(0, 2, 1, 3)
    kk = k.reshape(batches, Lk, heads, d).permute(0, 2, 1, 3)
    vx = v.reshape(batches, Lk, heads, d).permute(0, 2, 1, 3)
    return ref, qq, kk, vx, out


def test_mutation_one_key_in_or_out_of_a_ragged_key_tile():
    """100 keys = one full 64-key step + a ragged 36-key step: key 99 dropped, or a 101st (zero-filled past the end, score
    exp(0) instead of -inf) let in."""
    batches, heads, Lq, Lk, d = 2, 2, 64, 100, 40
    ref, q, k, v, _ = _attn_case(batches, heads, Lq, Lk, d, 13)
    good = ref.value.half()
    _passes(good, ref)
    C = heads * d
    drop = O.sdpa_ref(q, k[:, :, :Lk - 1], v[:, :, :Lk - 1], d ** -0.5).permute(0, 2, 1, 3).reshape(-1)
    _flagged(drop.half(), ref)
    k1 = torch.cat([k, torch.zeros_like(k[:, :, :1])], 2)
    v1 = torch.cat([v, torch.zeros_like(v[:, :, :1])], 2)
    extra = O.sdpa_ref(q, k1, v1, d ** -0.5).permute(0, 2, 1, 3).reshape(-1)
    _flagged(extra.half(), ref)
    assert C * batches * Lq == ref.value.numel()


def test_mutation_error_confined_to_one_batch_head_of_256():
    """A 5% error in one (batch, head) of 32 x 8: the global rel-L2 moves by ~3e-3, inside the old 4e-3 budget; the
    per-element bound names the (batch, head)."""
    batches, heads, Lq, Lk, d = 32, 8, 16, 77, 40
    ref, *_ = _attn_case(batches, heads, Lq, Lk, d, 14)
    C = heads * d
    v = ref.value.view(batches, Lq, heads, d).clone()
    v[17, :, 5] *= 1.05
    got = v.reshape(-1).half()
    glob = ((got.double() - ref.value).norm() / ref.value.norm()).item()
    assert glob < 4e-3, glob
    bad = _flagged(got, ref)
    assert "(batch 17, head 5)" in bad.where


def test_mutation_out_scale_applied_twice():
    batches, heads, Lq, Lk, d = 2, 2, 32, 20, 80
    ref, q, k, v, out = _attn_case(batches, heads, Lq, Lk, d, 15, out_scale=0.5, accumulate=True)
    _passes(ref.value.half(), ref)
    o = O.sdpa_ref(q, k, v, d ** -0.5).permute(0, 2, 1, 3).reshape(-1)
    _flagged((out.double().reshape(-1) + 0.25 * o).half(), ref)
    # out_scale = 0 with accumulate: the output must come back unchanged
    ref0, *_ , out0 = _attn_case(batches, heads, Lq, Lk, d, 15, out_scale=0.0, accumulate=True)
    assert torch.equal(ref0.value, out0.double().reshape(-1))
    _flagged((out0.double().reshape(-1) + o).half(), ref0)


def test_mutation_geglu_missing_rowbias_and_acc_scale():
    """What the SIMT GEGLU epilogue used to compute (bias only) is flagged against the ABI's epilogue."""
    g = _g(16)
    M, K, N = 64, 64, 256
    A = torch.randn(M, K, generator=g).half()
    B = (torch.randn(N, K, generator=g) * 0.2).half()
    bias, rb = torch.randn(N, generator=g), torch.randn(4, N, generator=g)
    out = torch.zeros(M, N // 2, dtype=torch.float16)
    ref = O.gemm(A, B, out, M=M, N=N, K=K, bias=bias, rowbias=rb, rb_div=1, rb_mod=4, acc_scale=0.7, geglu=True)
    _passes(ref.value.half(), ref)
    old = O.gemm(A, B, out, M=M, N=N, K=K, bias=bias, geglu=True)
    _flagged(old.value.half(), ref)


def test_untouched_region_must_stay_untouched():
    P, Fr, heads, d = 3, 4, 2, 40
    C = heads * d
    g = _g(17)
    qkv = torch.randn(P, Fr, 3 * C, generator=g).half()
    out = torch.randn(P * Fr, 2 * C, generator=g).half()
    ref = O.temporal_attn(qkv, out, P, Fr, heads, d, d ** -0.5, ldo=2 * C, out_col_offset=C)
    good = ref.value.half()
    _passes(good, ref)
    bad = good.view(P * Fr, 2 * C).clone()
    bad[5, 3] += 0.5                                 # a stray store into the half the call must not write
    assert "outside" in _flagged(bad.reshape(-1), ref).where
