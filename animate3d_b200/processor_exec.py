"""Stand-alone execution of the three released attention processors through the diffusers attention-processor protocol

    processor(attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None) -> Tensor

(animatediff/models/attention_processor.py:39-48, 169-178, 325-334, 541-550) on the sm_90a kernels of liba3d.so: one fused
projection GEMM, the strided-view attention kernel (the "(b n f) l c -> (b f) (n l) c" regroupings are TMA strides, never copies),
one merged output GEMM.  `MVUNetMotionModel.forward` fuses the same arithmetic into the whole-network schedule; this module is the
boundary for code that drives a single `Attention` layer with one of the processors -- e.g. a diffusers `Attention.forward`, or
the per-processor parity tests (tests/test_processors_gpu.py) that compare against oracle/unet_oracle.py's pinned restatements.

`attn` supplies what the reference processors read from a diffusers `Attention`: to_q / to_k / to_v / to_out[0] (Linear-like:
.weight [, .bias]) and heads.  Only the released call patterns are served: no attention mask, no spatial / group / cross norm,
residual_connection False, rescale_output_factor 1 (SURVEY 8b)."""
from __future__ import annotations

from typing import Dict, Tuple

import torch

from . import _lib as L
from . import ops
from .unet import HALF, _Lin, _dqk, _dv, _ones_bias, _pad_heads, _sine_pos_enc_2d

_cache: Dict[Tuple, dict] = {}


def _w(mod, name="weight"):
    t = getattr(mod, name, None)
    return None if t is None else t.detach().float()


def _key(proc, attn, dev):
    ts = [p for p in list(proc.parameters()) + [attn.to_q.weight, attn.to_k.weight, attn.to_v.weight, attn.to_out[0].weight]]
    return (id(proc), id(attn), str(dev), tuple((t.data_ptr(), t._version) for t in ts))


def _check_common(attn, attention_mask):
    if attention_mask is not None:
        raise NotImplementedError("attention masks are never passed on the reference's call paths")
    if getattr(attn, "spatial_norm", None) is not None or getattr(attn, "group_norm", None) is not None or getattr(attn, "norm_cross", None):
        raise NotImplementedError("spatial_norm / group_norm / norm_cross are None in the released model")
    if getattr(attn, "residual_connection", False) or getattr(attn, "rescale_output_factor", 1.0) != 1.0:
        raise NotImplementedError("residual_connection / rescale_output_factor are unused in the released model")


def _buf(shape, dev, dtype=HALF):
    return torch.empty(*shape, device=dev, dtype=dtype)


# ---------------------------------------------------------------------------------------------------- MVDream I2V (attn1)
def _mv_i2v(proc, attn, x, **_):
    """attention_processor.py:325-445.  x [(b n f), l, c]."""
    dev = x.device
    heads, nv, nf = attn.heads, proc.num_views, proc.num_frames
    bnf, l, c = x.shape
    if bnf % (nv * nf):
        raise ValueError(f"batch {bnf} is not a multiple of num_views*num_frames = {nv * nf}")
    b = bnf // (nv * nf)
    d = c // heads
    dqk, dv = _dqk(d), _dv(d)
    k = _key(proc, attn, dev)
    W = _cache.get(k)
    if W is None:
        wq = _pad_heads(_w(attn.to_q), heads, d, dqk)
        wqi = _pad_heads(_w(proc.to_q_i2v), heads, d, dqk)
        wk = _pad_heads(_w(attn.to_k), heads, d, dqk)
        wv = _pad_heads(_w(attn.to_v), heads, d, dv)
        wqkv = torch.cat([wq, wqi, wk, wv], 0)
        w_out, b_out = _w(attn.to_out[0]), _w(attn.to_out[0], "bias")
        w_i2v, b_i2v = _w(proc.to_out_i2v), _w(proc.to_out_i2v, "bias")
        W = {"qkv": _Lin(wqkv, _ones_bias(heads, d, dv, 3 * heads * dqk, wqkv.shape[0], "cpu"), dev),
             "out": _Lin(torch.cat([w_out, w_out @ w_i2v], 1), b_out + w_out @ b_i2v, dev)}
        _cache.clear()
        _cache[k] = W
    M = bnf * l
    xin = x.reshape(M, c).to(HALF).contiguous()
    nq = W["qkv"].n
    hq = heads * dqk
    qkv = _buf((M, nq), dev)
    ops.gemm(xin, W["qkv"].w, qkv, M=M, N=nq, K=c, bias=W["qkv"].b)
    st = (nq, nf * l * nq, l * nq, nv * nf * l * nq)                     # rows ordered (b n f p)
    ext = (l, nv, nf, b)
    vq, vqi = ops.view5(qkv, 0, nq, st, ext), ops.view5(qkv, hq, nq - hq, st, ext)
    vk, vv = ops.view5(qkv, 2 * hq, nq - 2 * hq, st, ext), ops.view5(qkv, 3 * hq, nq - 3 * hq, st, ext)
    o12 = _buf((M, 2 * c), dev)
    ostr = (2 * c, 2 * nf * l * c, 2 * l * c, 2 * nv * nf * l * c)
    ops.attention(vq, vk, vv, o12, ostr, heads=heads, d=d, scale=d ** -0.5)
    ops.attention(vqi, vk, vv, o12, ostr, heads=heads, d=d, scale=d ** -0.5, kv_i3_zero=True, out_col_offset=c)
    out = _buf((M, c), dev)
    ops.gemm(o12, W["out"].w, out, M=M, N=c, K=2 * c, bias=W["out"].b)
    return out.reshape(bnf, l, c).to(x.dtype)


# ---------------------------------------------------------------------------------------------------- IP-Adapter (attn2)
def _ip_adapter(proc, attn, x, encoder_hidden_states=None, **_):
    """attention_processor.py:169-298.  x [(b n f), l, c]; encoder_hidden_states = (text [(bnf), 77, 768], [image tokens
    [(bnf), 4, 768]]) -- the tuple form the reference UNet passes (unet_motion_mv_model.py:757-765)."""
    if not isinstance(encoder_hidden_states, (tuple, list)) or len(encoder_hidden_states) != 2:
        raise ValueError("IPAdapter processor expects encoder_hidden_states = (text_states, [ip_states])")
    text, ips = encoder_hidden_states
    ip = ips[0] if isinstance(ips, (tuple, list)) else ips
    dev = x.device
    heads = attn.heads
    bnf, l, c = x.shape
    d = c // heads
    dqk, dv = _dqk(d), _dv(d)
    k = _key(proc, attn, dev)
    W = _cache.get(k)
    if W is None:
        ob = None
        wkv = torch.cat([_pad_heads(_w(attn.to_k), heads, d, dqk), _pad_heads(_w(attn.to_v), heads, d, dv)], 0)
        wip = torch.cat([_pad_heads(_w(proc.to_k_ip[0]), heads, d, dqk), _pad_heads(_w(proc.to_v_ip[0]), heads, d, dv)], 0)
        ob = _ones_bias(heads, d, dv, heads * dqk, wkv.shape[0], "cpu")
        W = {"q": _Lin(_pad_heads(_w(attn.to_q), heads, d, dqk), None, dev), "kv": _Lin(wkv, ob, dev), "ip": _Lin(wip, ob, dev),
             "out": _Lin(_w(attn.to_out[0]), _w(attn.to_out[0], "bias"), dev)}
        _cache.clear()
        _cache[k] = W
    M = bnf * l
    hq = heads * dqk
    xin = x.reshape(M, c).to(HALF).contiguous()
    q = _buf((M, hq), dev)
    ops.gemm(xin, W["q"].w, q, M=M, N=hq, K=c)
    out_attn = _buf((M, c), dev)
    vq = ops.view5(q, 0, hq, (hq, l * hq, l * hq, l * hq), (l, 1, 1, bnf))
    ostr = (c, l * c, l * c, l * c)
    scale = proc.scale[0] if isinstance(proc.scale, (list, tuple)) else proc.scale
    for tokens, lin, acc, sc in ((text, W["kv"], False, 1.0), (ip, W["ip"], True, float(scale))):
        lk = tokens.shape[1]
        t16 = tokens.reshape(bnf * lk, -1).to(HALF).contiguous()
        kv = _buf((bnf * lk, lin.n), dev)
        ops.gemm(t16, lin.w, kv, M=bnf * lk, N=lin.n, K=lin.k, bias=lin.b)
        ld = lin.n
        stk = (ld, lk * ld, lk * ld, lk * ld)
        ops.attention(vq, ops.view5(kv, 0, ld, stk, (lk, 1, 1, bnf)), ops.view5(kv, hq, ld - hq, stk, (lk, 1, 1, bnf)), out_attn, ostr,
                      heads=heads, d=d, scale=d ** -0.5, accumulate=acc, out_scale=sc)
    out = _buf((M, c), dev)
    ops.gemm(out_attn, W["out"].w, out, M=M, N=c, K=c, bias=W["out"].b)
    return out.reshape(bnf, l, c).to(x.dtype)


# ---------------------------------------------------------------------------------------------------- SpatioTemporal I2V
def _spatiotemporal(proc, attn, x, **_):
    """attention_processor.py:541-723, released configuration.  x [(b n hw), f, c] (motion-module token layout)."""
    dev = x.device
    heads, nv, nf, fs = attn.heads, proc.num_views, proc.num_frames, proc.feature_size
    rows, f, c = x.shape
    hw = fs * fs
    if f != nf or rows % (nv * hw):
        raise ValueError(f"expected [(b*{nv}*{hw}), {nf}, c] tokens, got {tuple(x.shape)}")
    b = rows // (nv * hw)
    d = c // heads
    dqk, dv = _dqk(d), _dv(d)
    k = _key(proc, attn, dev)
    W = _cache.get(k)
    if W is None:
        wt = torch.cat([_w(attn.to_q), _w(attn.to_k), _w(attn.to_v)], 0)
        pe = proc.time_pos_embed.pe.detach().float()[0]
        wsp = torch.cat([_pad_heads(_w(proc.to_q_sp), heads, d, dqk), _pad_heads(_w(proc.to_k_sp), heads, d, dqk),
                         _pad_heads(_w(proc.to_v_sp), heads, d, dv)], 0)
        pos2d = _sine_pos_enc_2d(c // 2, fs, fs).to(wsp.device)
        alpha = torch.sigmoid(proc.alpha_blender.mix_factor.detach().float()).reshape(())
        w_sp, b_sp = _w(proc.to_out_sp), _w(proc.to_out_sp, "bias")
        w_t, b_t = _w(attn.to_out[0]), _w(attn.to_out[0], "bias")
        W = {"t_qkv": _Lin(wt, None, dev), "t_table": (pe @ wt.t()).to(dev).contiguous(),
             "s_qkv": _Lin(wsp, _ones_bias(heads, d, dv, 2 * heads * dqk, wsp.shape[0], "cpu"), dev),
             "s_table": (pos2d @ wsp.t()).to(dev).contiguous(),
             "out": _Lin(torch.cat([alpha * w_sp, (1 - alpha) * w_t], 1), alpha * b_sp + (1 - alpha) * b_t, dev)}
        _cache.clear()
        _cache[k] = W
    M = rows * f
    hq = heads * dqk
    xin = x.reshape(M, c).to(HALF).contiguous()
    tq = _buf((M, 3 * c), dev)
    ops.gemm(xin, W["t_qkv"].w, tq, M=M, N=3 * c, K=c, rowbias=W["t_table"], rb_div=1, rb_mod=f)
    st2 = _buf((M, 2 * c), dev)                                               # [S | T]
    ops.temporal_attn(tq, st2, M // f, f, heads, d, d ** -0.5, ldo=2 * c, out_col_offset=c)
    ns = W["s_qkv"].n
    sq = _buf((M, ns), dev)
    ops.gemm(xin, W["s_qkv"].w, sq, M=M, N=ns, K=c, bias=W["s_qkv"].b, rowbias=W["s_table"], rb_div=f, rb_mod=hw)
    st = (f * ns, hw * f * ns, ns, nv * hw * f * ns)                          # rows ordered (b n p f)
    ext = (hw, nv, f, b)
    ops.attention(ops.view5(sq, 0, ns, st, ext), ops.view5(sq, hq, ns - hq, st, ext), ops.view5(sq, 2 * hq, ns - 2 * hq, st, ext), st2,
                  (2 * f * c, 2 * hw * f * c, 2 * c, 2 * nv * hw * f * c), heads=heads, d=d, scale=d ** -0.5)
    out = _buf((M, c), dev)
    ops.gemm(st2, W["out"].w, out, M=M, N=c, K=2 * c, bias=W["out"].b)
    return out.reshape(rows, f, c).to(x.dtype)


_DISPATCH = {"MVDreamI2VXFormersAttnProcessor": _mv_i2v, "IPAdapterXFormersAttnProcessor": _ip_adapter,
             "SpatioTemporalI2VXFormersAttnProcessor": _spatiotemporal}


@torch.no_grad()
def run(proc, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, **kwargs):
    L.load()
    if not hidden_states.is_cuda:
        raise L.A3DError("the attention processors run on an sm_90a device only; there is no CPU path")
    _check_common(attn, attention_mask)
    if hidden_states.ndim != 3:
        raise NotImplementedError("4-D (b, c, h, w) inputs never reach these processors in the reference (Transformer2DModel "
                                  "flattens to tokens first)")
    fn = _DISPATCH[proc.kind]
    return fn(proc, attn, hidden_states, encoder_hidden_states=encoder_hidden_states)
