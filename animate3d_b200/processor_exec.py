"""The three released attention processors on the sm_90a kernels of liba3d.so: weight packing (`pack_*`) and launch stages.

`MVUNetMotionModel` packs every attention layer at load and runs the stages on its graph-stable activation arena; `run` is the
diffusers protocol `processor(attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None)`
(animatediff/models/attention_processor.py:39-48, 169-178, 325-334, 541-550) over the same packers and stages on fresh tensors,
so the per-processor parity tests (tests/test_processors_gpu.py) cover the UNet's code.  Per processor: one fused projection
GEMM, the strided-view attention kernel (the "(b n f) l c -> (b f) (n l) c" regroupings are TMA strides, never copies), one
merged output GEMM.  `attn` supplies what the reference processors read from a diffusers `Attention`: to_q / to_k / to_v /
to_out[0] (.weight [, .bias]) and heads.  Only the released call patterns are served: no attention mask, no spatial / group /
cross norm, residual_connection False, rescale_output_factor 1 (SURVEY 8b)."""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch

from . import _lib as L
from . import ops

HALF = torch.float16


def _sine_pos_enc_2d(num_feats: int, h: int, w: int, temperature=10000, scale=2 * math.pi, eps=1e-6) -> torch.Tensor:
    """[h*w, 2*num_feats] table of SinePositionalEncoding2D(num_feats, normalize=True) (animatediff/models/embeddings.py:58-96)."""
    y = torch.arange(1, h + 1, dtype=torch.float32)[:, None].expand(h, w)
    x = torch.arange(1, w + 1, dtype=torch.float32)[None, :].expand(h, w)
    y = y / (y[-1:, :] + eps) * scale
    x = x / (x[:, -1:] + eps) * scale
    dim_t = torch.arange(num_feats, dtype=torch.float32)
    dim_t = temperature ** (2 * (dim_t // 2) / num_feats)
    px = x[:, :, None] / dim_t
    py = y[:, :, None] / dim_t
    px = torch.stack((px[:, :, 0::2].sin(), px[:, :, 1::2].cos()), dim=3).reshape(h, w, -1)
    py = torch.stack((py[:, :, 0::2].sin(), py[:, :, 1::2].cos()), dim=3).reshape(h, w, -1)
    return torch.cat((py, px), dim=2).reshape(h * w, -1)


def _dqk(d):
    return (d + 15) // 16 * 16


def _dv(d):
    return (d + 1 + 15) // 16 * 16


def _pad_heads(w: torch.Tensor, heads: int, d: int, dp: int) -> torch.Tensor:
    """[heads*d, K] -> [heads*dp, K] with zero rows after each head's d rows."""
    k = w.shape[1]
    out = torch.zeros(heads, dp, k, dtype=w.dtype, device=w.device)
    out[:, :d] = w.reshape(heads, d, k)
    return out.reshape(heads * dp, k)


def _ones_bias(heads: int, d: int, dv: int, offset: int, total: int, device) -> torch.Tensor:
    b = torch.zeros(total, dtype=torch.float32, device=device)
    idx = offset + torch.arange(heads, device=device) * dv + d
    b[idx] = 1.0
    return b


class _Lin:
    """fp16 weight [N, K] + fp32 bias on device."""
    __slots__ = ("w", "b", "n", "k")

    def __init__(self, w: torch.Tensor, b: Optional[torch.Tensor], device):
        self.w = w.to(device=device, dtype=HALF).contiguous()
        self.b = None if b is None else b.to(device=device, dtype=torch.float32).contiguous()
        self.n, self.k = self.w.shape

    def rows(self, a: int, b: int) -> "_Lin":
        """Row slice [a, b) of the weight (and bias) without copying -- used to split a fused projection."""
        o = object.__new__(_Lin)
        o.w, o.b = self.w[a:b], None if self.b is None else self.b[a:b]
        o.n, o.k = b - a, self.k
        return o


def linear(A, lin: _Lin, out, M, residual=None, **kw):
    """out = A @ lin.w^T + lin.b over M rows (+ a residual with the output's row pitch); kw: the GEMM's other epilogue options."""
    if residual is not None:
        kw.update(R2=residual, ldr2=residual.shape[1])
    ops.gemm(A, lin.w, out, M=M, N=lin.n, K=lin.k, bias=kw.pop("bias", lin.b), **kw)


def _w(mod, name="weight"):
    t = getattr(mod, name, None)
    return None if t is None else t.detach().float()


def _geometry(proc, attn, n_q, frame_major) -> dict:
    """n_q query blocks ahead of [k | v] in the fused projection; rows ordered (b n f p) when frame_major, else (b n p f)."""
    heads = attn.heads
    d = proc.hidden_size // heads
    return {"heads": heads, "d": d, "hq": heads * _dqk(d), "n_q": n_q, "frame_major": frame_major}


# ---------------------------------------------------------------------------------------------------- packers
# Each head of a projection is padded to a multiple of 16 columns; V gets one more column whose bias is 1, so the attention
# kernel's P.V also yields the softmax row sums.  Products of two weights are formed in fp32 and rounded to fp16 once.
def pack_mv_i2v(proc, attn, dev) -> dict:
    """attention_processor.py:325-445: the fused [q | q_i2v | k | v] projection and to_out(O1 + to_out_i2v(O2)) as ONE GEMM
    over [O1 | O2] with K = 2C:  [O1 | O2] [W_out | W_out W_i2v]^T + (b_out + W_out b_i2v)."""
    p = _geometry(proc, attn, 2, True)
    heads, d = p["heads"], p["d"]
    dqk, dv = _dqk(d), _dv(d)
    w = torch.cat([_pad_heads(_w(attn.to_q), heads, d, dqk), _pad_heads(_w(proc.to_q_i2v), heads, d, dqk),
                   _pad_heads(_w(attn.to_k), heads, d, dqk), _pad_heads(_w(attn.to_v), heads, d, dv)], 0)
    w_out, b_out = _w(attn.to_out[0]), _w(attn.to_out[0], "bias")
    w_i2v, b_i2v = _w(proc.to_out_i2v), _w(proc.to_out_i2v, "bias")
    p["qkv"] = _Lin(w, _ones_bias(heads, d, dv, 3 * p["hq"], w.shape[0], "cpu"), dev)
    p["out"] = _Lin(torch.cat([w_out, w_out @ w_i2v], 1), b_out + w_out @ b_i2v, dev)
    return p


def pack_ip_adapter(proc, attn, dev) -> dict:
    """attention_processor.py:169-298: the query projection, the [k | v] projections of the text ("kv") and of the image tokens
    ("ip"), the output projection and the image branch's scale."""
    p = _geometry(proc, attn, 1, True)
    heads, d = p["heads"], p["d"]
    dqk, dv = _dqk(d), _dv(d)
    wkv = torch.cat([_pad_heads(_w(attn.to_k), heads, d, dqk), _pad_heads(_w(attn.to_v), heads, d, dv)], 0)
    wip = torch.cat([_pad_heads(_w(proc.to_k_ip[0]), heads, d, dqk), _pad_heads(_w(proc.to_v_ip[0]), heads, d, dv)], 0)
    ob = _ones_bias(heads, d, dv, p["hq"], wkv.shape[0], "cpu")
    scale = proc.scale[0] if isinstance(proc.scale, (list, tuple)) else proc.scale
    p.update(q=_Lin(_pad_heads(_w(attn.to_q), heads, d, dqk), None, dev), kv=_Lin(wkv, ob, dev), ip=_Lin(wip, ob, dev),
             out=_Lin(_w(attn.to_out[0]), _w(attn.to_out[0], "bias"), dev), scale=float(scale))
    return p


def pack_spatiotemporal(proc, attn, dev) -> dict:
    """attention_processor.py:541-723, released configuration.  (x + pe) W = x W + (pe W): the temporal and 2-D sinusoid encodings
    are row-bias tables.  AlphaBlender (700-713) + both output projections = ONE GEMM over [S | T] with K = 2C: weights
    [a W_sp | (1 - a) W_t], bias a b_sp + (1 - a) b_t (a stays a tensor: a sigmoid that underflows to 0 or 1 stays exact)."""
    p = _geometry(proc, attn, 1, False)
    heads, d = p["heads"], p["d"]
    dqk, dv = _dqk(d), _dv(d)
    fs = proc.feature_size
    wt = torch.cat([_w(attn.to_q), _w(attn.to_k), _w(attn.to_v)], 0)                                   # [3c, c]
    pe = proc.time_pos_embed.pe.detach().float()[0]                                                      # [32, c]
    wsp = torch.cat([_pad_heads(_w(proc.to_q_sp), heads, d, dqk), _pad_heads(_w(proc.to_k_sp), heads, d, dqk),
                     _pad_heads(_w(proc.to_v_sp), heads, d, dv)], 0)
    pos2d = _sine_pos_enc_2d(proc.hidden_size // 2, fs, fs).to(wsp.device)                              # [hw, c]
    alpha = torch.sigmoid(proc.alpha_blender.mix_factor.detach().float()).reshape(())
    w_sp, b_sp = _w(proc.to_out_sp), _w(proc.to_out_sp, "bias")
    w_t, b_t = _w(attn.to_out[0]), _w(attn.to_out[0], "bias")
    p.update(t_qkv=_Lin(wt, None, dev), t_table=(pe @ wt.t()).to(dev).contiguous(),
             s_qkv=_Lin(wsp, _ones_bias(heads, d, dv, 2 * p["hq"], wsp.shape[0], "cpu"), dev),
             s_table=(pos2d @ wsp.t()).to(dev).contiguous(),
             out=_Lin(torch.cat([alpha * w_sp, (1 - alpha) * w_t], 1), alpha * b_sp + (1 - alpha) * b_t, dev))
    return p


# ---------------------------------------------------------------------------------------------------- launch stages
# Activations are [rows, n] fp16 buffers.  The attention kernel reads them through rank-5 views whose four row axes are
# (position, view, frame, group); `_rows` gives their strides in rows.
def _rows(frame_major: bool, hw: int, frames: int, views: int, view_rows: Optional[int] = None) -> Tuple[int, int, int, int]:
    """`views` views of `frames` x `hw` tokens per group; view_rows: an all-gather [V, view_rows, n] of one view per rank."""
    pos, frame = (1, hw) if frame_major else (frames, 1)
    if view_rows is None:
        return pos, frames * hw, frame, views * frames * hw
    return pos, view_rows, frame, frames * hw


def _view(buf, col: int, rows, ext) -> L.View5:
    ld = buf.shape[-1]
    return ops.view5(buf, col, ld - col, tuple(r * ld for r in rows), ext)


def _out_strides(p, vq: L.View5, out):
    return tuple(r * out.shape[1] for r in _rows(p["frame_major"], vq.e1, vq.e3, vq.e2))


def qkv_views(p, q, kv, hw, frames, groups, views, kv_view_rows=None):
    """Views of the fused projection: the query blocks (q, q_i2v for MVDreamI2V) from column 0 of `q`, then k and v -- after
    them when `kv` is `q`, else from column 0 of `kv`, the all-gather [V, kv_view_rows, n] of one view per rank."""
    rq, ext = _rows(p["frame_major"], hw, frames, views), (hw, views, frames, groups)
    rk, ext_k = rq, ext
    if kv_view_rows is not None:
        rk, ext_k = _rows(p["frame_major"], hw, frames, 1, kv_view_rows), (hw, kv.shape[0], frames, groups)
    hq = p["hq"]
    kv_col = p["n_q"] * hq if kv is q else 0
    return tuple(_view(q, i * hq, rq, ext) for i in range(p["n_q"])) + (_view(kv, kv_col, rk, ext_k), _view(kv, kv_col + hq, rk, ext_k))


def mv_i2v_attend(p, views, o12, out, residual=None):
    """Cross-view self attention and the I2V attention against frame 0's keys (kv_i3_zero) side by side into [O1 | O2], then
    to_out(O1 + to_out_i2v(O2)) (+ residual) into out [rows, C]."""
    vq, vqi, vk, vv = views
    c, d = out.shape[1], p["d"]
    ostr = _out_strides(p, vq, o12)
    ops.attention(vq, vk, vv, o12, ostr, heads=p["heads"], d=d, scale=d ** -0.5)
    ops.attention(vqi, vk, vv, o12, ostr, heads=p["heads"], d=d, scale=d ** -0.5, kv_i3_zero=True, out_col_offset=c)
    linear(o12, p["out"], out, out.shape[0], residual=residual)


def ip_adapter_attend(p, q, kv, kv_col, o, hw, frames, image: bool):
    """One of the two cross attentions into o [rows, C]: the text keys, or (image) the image tokens accumulated with the
    processor's scale.  q [rows, heads*dqk]: padded queries, rows ordered (G, F', hw); kv [(G tokens), ld]: this layer's [k | v]
    at column kv_col, shared by the F' = frames frames of a group (kv_div)."""
    d, hq = p["d"], p["hq"]
    groups = q.shape[0] // (frames * hw)
    lk = kv.shape[0] // groups
    rk, ext_k = (1, lk, lk, lk), (lk, 1, 1, groups)
    vq = _view(q, 0, (1, hw, hw, frames * hw), (hw, 1, frames, groups))
    ops.attention(vq, _view(kv, kv_col, rk, ext_k), _view(kv, kv_col + hq, rk, ext_k), o,
                  tuple(r * o.shape[1] for r in (1, hw, hw, frames * hw)),
                  heads=p["heads"], d=d, scale=d ** -0.5, kv_div=frames, accumulate=image, out_scale=p["scale"] if image else 1.0)


def spatiotemporal_temporal(p, x, tq, st2, frames):
    """Temporal branch: (x + pe) W_qkv, then attention over the frames of each pixel into the right half T of st2 [S | T]."""
    M, c = x.shape
    linear(x, p["t_qkv"], tq, M, rowbias=p["t_table"], rb_div=1, rb_mod=frames)
    ops.temporal_attn(tq, st2, M // frames, frames, p["heads"], p["d"], p["d"] ** -0.5, ldo=2 * c, out_col_offset=c)


def spatiotemporal_project(p, x, sq, hw, frames, groups, views):
    """Spatial (cross-view) branch projection (x + pos2d) W_sp into sq, and its views."""
    linear(x, p["s_qkv"], sq, x.shape[0], rowbias=p["s_table"], rb_div=frames, rb_mod=hw)
    return qkv_views(p, sq, sq, hw, frames, groups, views)


def spatiotemporal_attend(p, views, st2, out, residual=None):
    """Cross-view attention into the left half S of st2, then the AlphaBlender of both branches' output projections
    (+ residual) as one K = 2C GEMM into out."""
    vq, vk, vv = views
    ops.attention(vq, vk, vv, st2, _out_strides(p, vq, st2), heads=p["heads"], d=p["d"], scale=p["d"] ** -0.5)
    linear(st2, p["out"], out, out.shape[0], residual=residual)


# ---------------------------------------------------------------------------------------------------- processor protocol
_cache: Dict[Tuple, dict] = {}


def _packed(pack, proc, attn, dev) -> dict:
    ts = list(proc.parameters()) + [attn.to_q.weight, attn.to_k.weight, attn.to_v.weight, attn.to_out[0].weight]
    k = (id(proc), id(attn), str(dev), tuple((t.data_ptr(), t._version) for t in ts))
    p = _cache.get(k)
    if p is None:
        p = pack(proc, attn, dev)
        _cache.clear()
        _cache[k] = p
    return p


def _check_common(attn, attention_mask):
    if attention_mask is not None:
        raise NotImplementedError("attention masks are never passed on the reference's call paths")
    if getattr(attn, "spatial_norm", None) is not None or getattr(attn, "group_norm", None) is not None or getattr(attn, "norm_cross", None):
        raise NotImplementedError("spatial_norm / group_norm / norm_cross are None in the released model")
    if getattr(attn, "residual_connection", False) or getattr(attn, "rescale_output_factor", 1.0) != 1.0:
        raise NotImplementedError("residual_connection / rescale_output_factor are unused in the released model")


def _buf(shape, dev, dtype=HALF):
    return torch.empty(*shape, device=dev, dtype=dtype)


def _mv_i2v(p, proc, xin, bnf, l, _):
    """attention_processor.py:325-445.  x [(b n f), l, c]."""
    nv, nf = proc.num_views, proc.num_frames
    if bnf % (nv * nf):
        raise ValueError(f"batch {bnf} is not a multiple of num_views*num_frames = {nv * nf}")
    (M, c), dev = xin.shape, xin.device
    qkv = _buf((M, p["qkv"].n), dev)
    linear(xin, p["qkv"], qkv, M)
    o12, out = _buf((M, 2 * c), dev), _buf((M, c), dev)                        # [O1 | O2], output
    mv_i2v_attend(p, qkv_views(p, qkv, qkv, l, nf, bnf // (nv * nf), nv), o12, out)
    return out


def _ip_adapter(p, proc, xin, bnf, l, encoder_hidden_states):
    """attention_processor.py:169-298.  x [(b n f), l, c]; encoder_hidden_states = (text [(bnf), 77, 768], [image tokens
    [(bnf), 4, 768]]) -- the tuple form the reference UNet passes (unet_motion_mv_model.py:757-765)."""
    if not isinstance(encoder_hidden_states, (tuple, list)) or len(encoder_hidden_states) != 2:
        raise ValueError("IPAdapter processor expects encoder_hidden_states = (text_states, [ip_states])")
    text, ips = encoder_hidden_states
    ip = ips[0] if isinstance(ips, (tuple, list)) else ips
    (M, c), dev = xin.shape, xin.device
    q = _buf((M, p["hq"]), dev)
    linear(xin, p["q"], q, M)
    o = _buf((M, c), dev)
    for tokens, lin, image in ((text, p["kv"], False), (ip, p["ip"], True)):
        rows = bnf * tokens.shape[1]
        kv = _buf((rows, lin.n), dev)
        linear(tokens.reshape(rows, -1).to(HALF).contiguous(), lin, kv, rows)
        ip_adapter_attend(p, q, kv, 0, o, l, 1, image)
    out = _buf((M, c), dev)
    linear(o, p["out"], out, M)
    return out


def _spatiotemporal(p, proc, xin, rows, f, _):
    """attention_processor.py:541-723, released configuration.  x [(b n hw), f, c] (motion-module token layout)."""
    nv, nf, hw = proc.num_views, proc.num_frames, proc.feature_size ** 2
    if f != nf or rows % (nv * hw):
        raise ValueError(f"expected [(b*{nv}*{hw}), {nf}, c] tokens, got {(rows, f, xin.shape[1])}")
    (M, c), dev = xin.shape, xin.device
    tq, st2 = _buf((M, 3 * c), dev), _buf((M, 2 * c), dev)                    # temporal q|k|v, [S | T]
    spatiotemporal_temporal(p, xin, tq, st2, f)
    views = spatiotemporal_project(p, xin, _buf((M, p["s_qkv"].n), dev), hw, f, rows // (nv * hw), nv)
    out = _buf((M, c), dev)
    spatiotemporal_attend(p, views, st2, out)
    return out


_DISPATCH = {"MVDreamI2VXFormersAttnProcessor": (pack_mv_i2v, _mv_i2v), "IPAdapterXFormersAttnProcessor": (pack_ip_adapter, _ip_adapter),
             "SpatioTemporalI2VXFormersAttnProcessor": (pack_spatiotemporal, _spatiotemporal)}


@torch.no_grad()
def run(proc, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, **kwargs):
    L.load()
    x = hidden_states
    if not x.is_cuda:
        raise L.A3DError("the attention processors run on an sm_90a device only; there is no CPU path")
    _check_common(attn, attention_mask)
    if x.ndim != 3:
        raise NotImplementedError("4-D (b, c, h, w) inputs never reach these processors in the reference (Transformer2DModel "
                                  "flattens to tokens first)")
    if x.shape[-1] != proc.hidden_size:
        raise ValueError(f"hidden_states have {x.shape[-1]} channels, the processor was built for {proc.hidden_size}")
    pack, fn = _DISPATCH[proc.kind]
    p = _packed(pack, proc, attn, x.device)
    out = fn(p, proc, x.reshape(-1, x.shape[-1]).to(HALF).contiguous(), x.shape[0], x.shape[1], encoder_hidden_states)
    return out.reshape(x.shape).to(x.dtype)
