"""CPU checks of animate3d_b200/processor_exec.py, the one implementation of the three attention processors that both the UNet
forward and the processor protocol run: the packed operands' algebra, the UNet's packing when the motion modules have their
own head count, and the kernel-launch count of a forward (liba3d.so replaced by a stub that enqueues nothing)."""
import ctypes

import pytest
import torch

from animate3d_b200 import _lib as L
from animate3d_b200 import modules as Mo
from animate3d_b200 import ops
from animate3d_b200 import processor_exec as P


def _attn(c, kv_dim, proc, heads=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    attn = Mo.AttentionNode(heads, c // heads)
    attn.to_q, attn.to_k, attn.to_v = Mo._linear(c, c, False, "cpu"), Mo._linear(c, kv_dim, False, "cpu"), Mo._linear(c, kv_dim, False, "cpu")
    attn.to_out = Mo.Node()
    attn.to_out.add_module("0", Mo._linear(c, c, True, "cpu"))
    attn.processor = proc
    with torch.no_grad():
        for name, p in attn.named_parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (0.3 if name.endswith("mix_factor") else 0.05))
    return attn


def _heads(w, heads, dp, d):
    """[heads*dp, K] -> ([heads*d, K] real rows, padding rows)."""
    w = w.reshape(heads, dp, -1)
    return w[:, :d].reshape(heads * d, -1), w[:, d:]


def _check_ones_column(b, offset, heads, d, dv):
    want = torch.zeros(heads, dv)
    want[:, d] = 1
    assert torch.equal(b[offset:offset + heads * dv].reshape(heads, dv), want)


@pytest.mark.parametrize("c,heads", [(320, 8), (640, 4)])
def test_pack_mv_i2v(c, heads):
    proc = Mo.MVDreamI2VXFormersAttnProcessor(hidden_size=c, device="cpu")
    attn = _attn(c, c, proc, heads)
    p = P.pack_mv_i2v(proc, attn, "cpu")
    d = c // heads
    dqk, dv = P._dqk(d), P._dv(d)
    assert (p["heads"], p["d"], p["hq"]) == (heads, d, heads * dqk)
    w, hq = p["qkv"].w, p["hq"]
    for i, src in enumerate((attn.to_q, proc.to_q_i2v, attn.to_k)):
        real, pad = _heads(w[i * hq:(i + 1) * hq], heads, dqk, d)
        assert torch.equal(real, src.weight.half()) and not pad.any()
    real, pad = _heads(w[3 * hq:], heads, dv, d)
    assert torch.equal(real, attn.to_v.weight.half()) and not pad.any()
    assert not p["qkv"].b[:3 * hq].any()
    _check_ones_column(p["qkv"].b, 3 * hq, heads, d, dv)
    # [O1 | O2] [W_out | W_out W_i2v]^T + b == to_out(O1 + to_out_i2v(O2))
    o1, o2 = torch.randn(5, c), torch.randn(5, c)
    got = torch.cat([o1, o2], 1) @ p["out"].w.float().t() + p["out"].b
    lin = lambda m, x: x @ m.weight.t() + m.bias
    torch.testing.assert_close(got, lin(attn.to_out[0], o1 + lin(proc.to_out_i2v, o2)), rtol=1e-2, atol=2e-3)


def test_pack_ip_adapter():
    c, heads = 320, 8
    proc = Mo.IPAdapterXFormersAttnProcessor(hidden_size=c, cross_attention_dim=64, num_tokens=(4,), scale=0.7, device="cpu")
    attn = _attn(c, 64, proc, heads)
    p = P.pack_ip_adapter(proc, attn, "cpu")
    d = c // heads
    dqk, dv = P._dqk(d), P._dv(d)
    hq = p["hq"]
    assert p["scale"] == 0.7 and p["q"].b is None
    assert torch.equal(_heads(p["q"].w, heads, dqk, d)[0], attn.to_q.weight.half())
    for key, k, v in (("kv", attn.to_k, attn.to_v), ("ip", proc.to_k_ip[0], proc.to_v_ip[0])):
        lin = p[key]
        assert torch.equal(_heads(lin.w[:hq], heads, dqk, d)[0], k.weight.half())
        assert torch.equal(_heads(lin.w[hq:], heads, dv, d)[0], v.weight.half())
        _check_ones_column(lin.b, hq, heads, d, dv)
    assert torch.equal(p["out"].w, attn.to_out[0].weight.half()) and torch.equal(p["out"].b, attn.to_out[0].bias)


@pytest.mark.parametrize("c,heads,fs", [(320, 8, 8), (640, 4, 4)])
def test_pack_spatiotemporal(c, heads, fs):
    proc = Mo.SpatioTemporalI2VXFormersAttnProcessor(hidden_size=c, feature_size=fs, use_alpha_blender=True, device="cpu")
    attn = _attn(c, c, proc, heads)
    p = P.pack_spatiotemporal(proc, attn, "cpu")
    d = c // heads
    dqk, dv = P._dqk(d), P._dv(d)
    hq = p["hq"]
    # temporal table: table[f] == pe[f] W_qkv^T
    wt = torch.cat([attn.to_q.weight, attn.to_k.weight, attn.to_v.weight], 0)
    torch.testing.assert_close(p["t_table"], proc.time_pos_embed.pe[0] @ wt.t(), rtol=1e-5, atol=1e-6)
    # spatial table: table[p] == pos2d[p] W_sp^T, per head (padding columns zero); V's ones column in the bias
    pos2d = P._sine_pos_enc_2d(c // 2, fs, fs)
    assert p["s_table"].shape[0] == fs * fs
    for i, (src, dp) in enumerate(((proc.to_q_sp, dqk), (proc.to_k_sp, dqk), (proc.to_v_sp, dv))):
        cols = p["s_table"][:, i * hq:i * hq + heads * dp].reshape(fs * fs, heads, dp)
        torch.testing.assert_close(cols[..., :d].reshape(fs * fs, c), pos2d @ src.weight.t(), rtol=1e-5, atol=1e-5)
        assert not cols[..., d:].any()
    _check_ones_column(p["s_qkv"].b, 2 * hq, heads, d, dv)
    # AlphaBlender: [S | T] [a W_sp | (1 - a) W_t]^T + b == a to_out_sp(S) + (1 - a) to_out(T)
    a = torch.sigmoid(proc.alpha_blender.mix_factor)
    s, t = torch.randn(5, c), torch.randn(5, c)
    got = torch.cat([s, t], 1) @ p["out"].w.float().t() + p["out"].b
    lin = lambda m, x: x @ m.weight.t() + m.bias
    torch.testing.assert_close(got, a * lin(proc.to_out_sp, s) + (1 - a) * lin(attn.to_out[0], t), rtol=1e-2, atol=2e-3)


class _StubLib:
    """liba3d.so stand-in: every entry point succeeds and enqueues nothing."""

    def __getattr__(self, name):
        return lambda *a: 0


@pytest.fixture
def stub_lib(monkeypatch):
    monkeypatch.setattr(L, "load", lambda require_gpu=True: _StubLib())
    monkeypatch.setattr(L, "stream_ptr", lambda: ctypes.c_void_p(0))


def _model(**kw):
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig, key_plan
    cfg = UNetConfig(cross_attention_dim=64, ip_image_embed_dim=32, **kw)
    m = MVUNetMotionModel(cfg, device="cpu")
    m._loaded.update(key_plan(cfg))          # built-in initial values stand in for a checkpoint
    return m


def test_prepare_motion_heads_differ_from_spatial(stub_lib):
    """Motion modules pack and attend with their own head count (here 4 against 8 spatial heads: head dims 40, 80, 160)."""
    m = _model(block_out_channels=(320, 640, 640, 640), motion_num_attention_heads=4, num_views=1, num_frames=2)
    m._prepare()
    for lay, c in ((m.W["down"][0]["layers"][0], 320), (m.W["down"][1]["layers"][1], 640)):
        for a in ("attn1", "attn2"):
            p = lay["motion"][a]
            d = c // 4
            assert (p["heads"], p["d"], p["hq"]) == (4, d, 4 * P._dqk(d))
            assert p["s_qkv"].n == 2 * p["hq"] + 4 * P._dv(d) and p["s_table"].shape[1] == p["s_qkv"].n
        assert lay["attn"]["attn1"]["heads"] == 8 and lay["attn"]["attn1"]["d"] == c // 8


def test_launch_count_matches_the_ops_calls(stub_lib):
    """launches_per_forward is the kernels the ops wrappers enqueued: 3 per GroupNorm, 1 per other call; the
    i2v_cond_time_zero embedding path adds its four launches."""
    import shadow as S
    m = _model(block_out_channels=(64, 128, 256, 256), num_views=2, num_frames=2)
    m.use_cuda_graph = False
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 2, 32, 32, generator=g)
    counts = []
    for cond_zero in (False, True):
        with S.counting() as calls:
            m(x, 500, torch.randn(2, 77, 64, generator=g), camera=torch.randn(2, 16, generator=g),
              added_cond_kwargs={"image_embeds": torch.randn(2, 32, generator=g)}, num_views=2, i2v_cond_time_zero=cond_zero)
        assert m.launches_per_forward == sum(n * (3 if op == "group_norm" else 1) for op, n in calls.items())
        counts.append(m.launches_per_forward)
    assert counts[1] == counts[0] + 4
