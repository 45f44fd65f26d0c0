"""oracle/vae_grad_oracle.py without a GPU: the oracle against independent formulations of each derivative; vae.py's own
autograd Functions, driven with float64 ABI stand-ins for the kernels (abi_oracle's values rounded into the same fp16 / fp32
buffers), within every per-call bound through a whole small encoder and within rel-L2 1e-2 of float64 autograd through
oracle/vae_oracle.py; and negative controls: each mutation of a backward recipe must be flagged at >= 10x its bound."""
import pytest
import torch
import torch.nn.functional as F

import vae_grad_shadow as S
from animate3d_b200 import ops
from animate3d_b200 import vae as V
from oracle import abi_oracle as O
from oracle import vae_grad_oracle as G
from oracle import vae_oracle as VO

F64 = torch.float64
SMALL = (32, 64, 64, 64)        # channels that are multiples of 32; three downsample levels


# ------------------------------------------------------------------------------------------------ float64 ABI stand-ins
def _gemm(A, B, out, **kw):
    ref = O.gemm(A, B, out, **kw)
    O.flat(out, ref.value.numel()).copy_(ref.value.to(out.dtype))


def _group_norm(x1, c1, x2, c2, gamma, beta, y, samples, rows, groups, eps, silu, ws, perm=(0, 0)):
    ref = O.group_norm(x1, c1, x2, c2, gamma, beta, y, samples, rows, groups, eps, silu, perm=perm)
    y.view(-1)[:ref.value.numel()].copy_(ref.value.to(y.dtype))
    xg = O.mat(x1, samples * rows, c1, c1).to(F64).view(samples, rows, groups, -1)
    mu = xg.mean(dim=(1, 3))
    rstd = 1.0 / torch.sqrt(((xg - mu[:, None, :, None]) ** 2).mean(dim=(1, 3)) + eps)
    ws[:2 * samples * groups] = torch.stack([mu, rstd], -1).reshape(-1).float()


def _group_norm_backward(x, c, gamma, beta, stats, dy, dx, samples, rows, groups, silu, ws):
    dx.view(-1).copy_(O.group_norm_backward(x, c, gamma, beta, stats, dy, dx, samples, rows, groups, silu).value.to(dx.dtype))


def _conv_in(sample, w, b, y, *a):
    y.view(-1).copy_(O.conv_in(sample, w, b, y, *a).value.to(y.dtype))


def _conv_out(x, w, b, y, *a):
    y.view(-1).copy_(O.conv_out(x, w, b, y, *a).value.to(y.dtype))


@pytest.fixture
def stand_ins(monkeypatch):
    for name, f in (("gemm", _gemm), ("group_norm", _group_norm), ("group_norm_backward", _group_norm_backward),
                    ("conv_in", _conv_in), ("conv_out", _conv_out),
                    ("group_norm_ws_floats", lambda samples, rows, c, groups: 2 * samples * groups)):
        monkeypatch.setattr(ops, name, f)


def _model(in_channels=3, seed=0):
    cfg = VO.VAEConfig(in_channels=in_channels, block_out_channels=SMALL)
    sd = VO.make_state_dict(cfg, seed)
    m = V.AutoencoderKL(in_channels=in_channels, block_out_channels=SMALL, device="cpu")
    m.load_state_dict(sd)
    return m, sd, cfg


def _rand16(*shape, gen):
    return torch.randn(*shape, generator=gen).half()


# ------------------------------------------------------------------------------------------------ the oracle itself
@pytest.mark.parametrize("stride,h,w", [(1, 6, 10), (1, 10, 6), (2, 6, 10), (2, 10, 6), (2, 8, 8)])
def test_conv3_oracle_matches_transpose_conv_zero_insert_and_fd(stride, h, w):
    gen = torch.Generator().manual_seed(h * 31 + w + stride)
    n, cin, cout = 2, 5, 7
    wt = torch.randn(cout, cin, 3, 3, generator=gen, dtype=F64)
    lay = {"w": wt.permute(0, 2, 3, 1).reshape(cout, -1), "cin": cin, "cout": cout}
    g = torch.randn(n * (h // stride) * (w // stride), cout, generator=gen, dtype=F64)
    ref = G.conv3_backward(g, lay, n, h, w, stride)
    v = ref.value.view(n, h, w, cin).permute(0, 3, 1, 2)
    Gy = g.view(n, h // stride, w // stride, cout).permute(0, 3, 1, 2)
    if stride == 1:
        tc = F.conv_transpose2d(Gy, wt, padding=1)
    else:
        tc = F.conv_transpose2d(Gy, wt, stride=2)[:, :, :h, :w]          # gradient of the (h+1) x (w+1) padded input, cropped
        u = torch.zeros(n, cout, h, w, dtype=F64)                         # vae.py's formulation: dY at the odd positions
        u[:, :, 1::2, 1::2] = Gy
        zi = F.conv2d(u, wt.flip(2, 3).transpose(0, 1), padding=1)
        assert torch.allclose(zi, v, rtol=0, atol=1e-12)
    assert torch.allclose(tc, v, rtol=0, atol=1e-12)
    x0 = torch.randn(n, cin, h, w, generator=gen, dtype=F64)
    loss = lambda x: (G.conv3_forward(x, wt, stride) * Gy).sum()
    for (i, c, y, xx) in [(0, 0, 0, 0), (1, cin - 1, h - 1, w - 1), (0, 2, h - 1, 0), (1, 3, 1, w - 2)]:
        dx = torch.zeros_like(x0)
        dx[i, c, y, xx] = 1e-3
        fd = (loss(x0 + dx) - loss(x0 - dx)) / 2e-3
        assert abs(fd.item() - v[i, c, y, xx].item()) < 1e-8, (i, c, y, xx, fd.item(), v[i, c, y, xx].item())
    assert (ref.bound > 0).all()


def test_lin_and_edge_oracles_match_transposes():
    gen = torch.Generator().manual_seed(3)
    cin, cout, m = 24, 40, 11
    W = torch.randn(cout, cin, generator=gen, dtype=F64)
    g = torch.randn(m, cout, generator=gen, dtype=F64)
    assert torch.allclose(G.lin_backward(g, {"w": W, "cin": cin, "cout": cout}).value.view(m, cin), g @ W, rtol=0, atol=1e-12)
    n, h, w = 2, 6, 10
    for cin, cout in ((3, 32), (64, 8)):
        W = torch.randn(cout, cin, 3, 3, generator=gen, dtype=F64)
        lay = {"w32": W.reshape(cout, -1), "cin": cin, "cout": cout}
        Gy = torch.randn(n, cout, h, w, generator=gen, dtype=F64)
        want = F.conv_transpose2d(Gy, W, padding=1)
        got_in = G.conv_in_backward(Gy.permute(0, 2, 3, 1).reshape(-1, cout), lay, n, h, w).value.view(n, cin, h, w)
        got_out = G.conv_out_backward(Gy, lay, n, h, w).value.view(n, h, w, cin).permute(0, 3, 1, 2)
        assert torch.allclose(got_in, want, rtol=0, atol=1e-12) and torch.allclose(got_out, want, rtol=0, atol=1e-12)


@pytest.mark.parametrize("silu", [0, 1])
def test_group_norm_oracle_matches_formula_and_fd(silu):
    gen = torch.Generator().manual_seed(7 + silu)
    n, rows, c = 2, 12, 64
    x = _rand16(n * rows, c, gen=gen) + 0.3
    g = _rand16(n * rows, c, gen=gen)
    gb = (1 + 0.1 * torch.randn(c, generator=gen), 0.1 * torch.randn(c, generator=gen))
    st = G.group_norm_stats(x, n, rows)
    ref = G.group_norm_backward(x, g, gb, n, rows, silu, st.value.float())
    # the ABI formula at the exact statistics is an independent formulation of the same derivative
    formula = O.group_norm_backward(x, c, gb[0], gb[1], st.value, g, None, n, rows, G.GROUPS, silu)
    assert torch.allclose(formula.value, ref.value, rtol=0, atol=1e-10 * ref.value.abs().max().item())
    x4 = x.to(F64).view(n, rows, c).permute(0, 2, 1)
    g4 = g.to(F64).view(n, rows, c).permute(0, 2, 1)
    gm, bt = gb[0].to(F64), gb[1].to(F64)
    loss = lambda t: (G.group_norm_forward(t, gm, bt, silu) * g4).sum()
    v = ref.value.view(n, rows, c)
    for (i, r, ch) in [(0, 0, 0), (1, rows - 1, c - 1), (0, 5, 33), (1, 7, 2)]:
        d = torch.zeros_like(x4)
        d[i, ch, r] = 1e-5
        fd = (loss(x4 + d) - loss(x4 - d)) / 2e-5
        assert abs(fd.item() - v[i, r, ch].item()) < 1e-7 * max(1.0, abs(v[i, r, ch].item())), (i, r, ch, fd.item())
    rel = (ref.bound / ref.value.abs().clamp_min(1e-3 * ref.value.abs().max())).median().item()
    assert 0 < rel < 1e-2, rel                      # a bound, not a tolerance as large as the value


# ------------------------------------------------------------------------------------------------ vae.py's recipes, stand-ins
@pytest.mark.parametrize("h,w", [(64, 64), (32, 128), (128, 32)])
def test_stand_in_encoder_within_every_bound(stand_ins, h, w):
    torch.set_num_threads(min(16, torch.get_num_threads()))
    model, sd, cfg = _model()
    gen = torch.Generator().manual_seed(h + 3 * w)
    n = 2
    x = torch.rand(n, 3, h, w, generator=gen) * 2 - 1
    dm = torch.randn(n, 8, h // 8, w // 8, generator=gen)
    with S.counting() as calls:
        xc = x.clone().requires_grad_(True)
        (model.encode_moments(xc) * dm).sum().backward()
    sh = S.GradShadow(f"stand-in {h}x{w}", model=model, n=n)
    xe = x.clone().requires_grad_(True)
    with sh.active():
        (model.encode_moments(xe) * dm).sum().backward()
    assert torch.equal(xe.grad, xc.grad)
    print(f"\nstand-in encoder {n} x {h}x{w}: {sum(sh.calls.values())} backward calls checked\n{sh.summary()}")
    assert dict(sh.calls) == dict(calls), (dict(sh.calls), dict(calls))
    bad = sh.failures()
    assert not bad, sh.table(sorted(bad, key=lambda r: -r["ratio"])[:20])
    sd64 = {k: v.to(F64) for k, v in sd.items()}
    xo = x.to(F64).requires_grad_(True)
    (VO.encode_moments(sd64, cfg, xo) * dm.to(F64)).sum().backward()
    rel = ((xe.grad.to(F64) - xo.grad).norm() / xo.grad.norm()).item()
    mx = ((xe.grad.to(F64) - xo.grad).abs().max() / xo.grad.abs().max()).item()
    print(f"input gradient vs float64 autograd through vae_oracle: rel-L2 {rel:.2e}, max-abs/max-ref {mx:.2e}")
    assert rel < 1e-2, rel
    kinds = {r["kind"] for r in sh.records}
    assert {"conv3 stride 1", "conv3 stride 1 res", "conv3 stride 2", "lin", "lin res", "gn silu 0", "gn silu 1", "gn stats",
            "residual", "conv_in cin 3", "conv_out cout 8"} <= kinds, kinds


# ------------------------------------------------------------------------------------------------ negative controls
def _conv3_even(ctx, g):
    lay = ctx.lay
    n, h, w, stride = ctx.geom
    cin, cout = lay["cin"], lay["cout"]
    u = torch.zeros(n, h, w, cout, device=g.device, dtype=V.HALF)
    u[:, 0::2, 0::2] = g.contiguous().view(n, h // 2, w // 2, cout)
    dx = torch.empty(n * h * w, cin, device=g.device, dtype=V.HALF)
    ops.gemm(u.view(n * h * w, cout), lay["wt"], dx, M=n * h * w, N=cin, K=9 * cout, conv=(n, h, w, cout, 1))
    return dx, None, None, None, None, None, None


def _conv3_hw_swapped(ctx, g):
    lay = ctx.lay
    n, h, w, stride = ctx.geom
    cin, cout = lay["cin"], lay["cout"]
    u = torch.zeros(n, w, h, cout, device=g.device, dtype=V.HALF)
    u[:, 1::2, 1::2] = g.contiguous().view(n, w // 2, h // 2, cout)
    dx = torch.empty(n * h * w, cin, device=g.device, dtype=V.HALF)
    ops.gemm(u.view(n * h * w, cout), lay["wt"], dx, M=n * h * w, N=cin, K=9 * cout, conv=(n, h, w, cout, 1))
    return dx, None, None, None, None, None, None


_CONV3_BACKWARD = V._Conv3.backward


def _conv3_residual_dropped(ctx, g):
    return (_CONV3_BACKWARD(ctx, g)[0],) + (None,) * 6


def _lin_w_not_wt(ctx, g):
    lay = ctx.lay
    g = g.contiguous()
    dx = torch.empty(g.shape[0], lay["cin"], device=g.device, dtype=V.HALF)
    ops.gemm(g, lay["w"], dx, M=g.shape[0], N=lay["cin"], K=lay["cout"])
    return dx, (g if ctx.has_res else None), None


def _gn_no_silu(ctx, g):
    x, stats = ctx.saved_tensors
    gb, n, rows, silu = ctx.meta
    c = x.shape[1]
    dx = torch.empty_like(x)
    ws = torch.empty(ops.group_norm_ws_floats(n, rows, c, V.GROUPS), device=x.device, dtype=torch.float32)
    ops.group_norm_backward(x, c, gb[0], gb[1], stats, g.contiguous(), dx, n, rows, V.GROUPS, 0, ws)
    return dx, None, None, None, None, None


def _conv_in_slice_offset(ctx, g):
    lay = ctx.lay
    n, cin, h, w = ctx.geom
    dx = torch.zeros(n, cin, 1, h, w, device=g.device, dtype=torch.float32)
    for c0 in range(0, cin, 4):
        c1 = min(c0 + 4, cin)
        part = torch.empty(n, c1 - c0, 1, h, w, device=g.device, dtype=torch.float32)
        ops.conv_out(g.contiguous(), lay["wt32"][c0:c1].contiguous(), lay["zero_b"], part, n, lay["cout"], 1, h, w, c1 - c0)
        o = max(c0 - 1, 0)                                      # the second slice lands one channel early
        dx[:, o:o + c1 - c0] = part
    return dx.reshape(n, cin, h, w), None


def _pack_unflipped(w):
    fwd = w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)
    bwd = w.permute(1, 2, 3, 0).reshape(w.shape[1], -1)
    return fwd.to(V.HALF).contiguous(), bwd.to(V.HALF).contiguous()


def _run(model, fn, n, h, w, gen):
    """One Function call of `model` (forward + backward with a random upstream gradient) under the shadow."""
    W = model.W
    sh = S.GradShadow(fn, model=model, n=n)
    with sh.active():
        if fn in ("conv3", "conv3 res", "down"):
            lay = W["enc_down"][0]["down"] if fn == "down" else W["enc_down"][0]["res"][0]["conv2"]
            x = _rand16(n * h * w, lay["cin"], gen=gen).requires_grad_(True)
            res = _rand16(n * h * w, lay["cout"], gen=gen).requires_grad_(True) if fn == "conv3 res" else None
            s = 2 if fn == "down" else 1
            y = V._Conv3.apply(x, res, lay, n, h, w, s)
        elif fn == "lin res":
            lay = W["enc_mid"]["out"]                           # square, residual output projection
            x = _rand16(n * h * w, lay["cin"], gen=gen).requires_grad_(True)
            y = V._Lin.apply(x, _rand16(n * h * w, lay["cout"], gen=gen).requires_grad_(True), lay)
        elif fn.startswith("gn"):
            gb = W["enc_down"][0]["res"][0]["norm1"]
            c = gb[0].numel()
            if fn == "gn small variance":                       # 1 + k 2^-10, k in -3..3: group variance ~4e-6
                k = torch.randint(-3, 4, (n * h * w, c), generator=gen)
                x = (1.0 + k * 2.0 ** -10).half()
            else:
                x = _rand16(n * h * w, c, gen=gen)
            x.requires_grad_(True)
            y = V._GroupNorm.apply(x, gb, n, h * w, 1, model.eps)
        elif fn == "conv_in":
            lay = W["enc_in"]
            x = torch.randn(n, lay["cin"], h, w, generator=gen).requires_grad_(True)
            y = V._ConvIn.apply(x, lay)
        y.backward(torch.randn(y.shape, generator=gen).to(y.dtype))
    assert sum(sh.calls.values()) == 1 and sh.records
    return max(r["ratio"] for r in sh.records), sh


CONTROLS = {
    # name: (Function call, image h x w, what to patch: (object, attribute, value))
    "taps not flipped (square conv)": ("conv3", 8, 12, ("vae", "_pack_conv", _pack_unflipped)),
    "zero insertion at the even positions": ("down", 8, 12, ("_Conv3", "backward", staticmethod(_conv3_even))),
    "h and w swapped in the zero insertion": ("down", 8, 16, ("_Conv3", "backward", staticmethod(_conv3_hw_swapped))),
    "w instead of w^T (square _Lin)": ("lin res", 8, 8, ("_Lin", "backward", staticmethod(_lin_w_not_wt))),
    "residual gradient dropped": ("conv3 res", 8, 8, ("_Conv3", "backward", staticmethod(_conv3_residual_dropped))),
    "SiLU factor missing in the GroupNorm backward": ("gn", 8, 8, ("_GroupNorm", "backward", staticmethod(_gn_no_silu))),
    "_ConvIn channel slice at the wrong offset": ("conv_in", 8, 12, ("_ConvIn", "backward", staticmethod(_conv_in_slice_offset))),
    "eps 1e-5 instead of 1e-6": ("gn small variance", 8, 8, ("model", "eps", 1e-5)),
}


@pytest.mark.parametrize("mutated", [False, True], ids=["recipe", "mutated"])
@pytest.mark.parametrize("control", list(CONTROLS))
def test_negative_control(stand_ins, monkeypatch, control, mutated):
    fn, h, w, (obj, attr, value) = CONTROLS[control]
    if mutated and obj == "vae":
        monkeypatch.setattr(V, attr, value)
    if mutated and obj.startswith("_"):
        monkeypatch.setattr(S.BASE[obj], attr, value)
    model, _, _ = _model(in_channels=6 if fn == "conv_in" else 3)
    if mutated and obj == "model":
        monkeypatch.setattr(model, attr, value)
    ratio, sh = _run(model, fn, 2, h, w, torch.Generator().manual_seed(5))
    worst = max(sh.records, key=lambda r: r["ratio"])
    print(f"\n{control} ({'mutated' if mutated else 'as shipped'}): worst |err|/bound {ratio:.3g} [{worst['kind']}] at {worst['where']}")
    if mutated:
        assert ratio >= 10, sh.table([worst])
    else:
        assert ratio <= 1, sh.table(sh.failures())
