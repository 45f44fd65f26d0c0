"""Key-tile geometry of the tensor-core attention kernel (csrc/a3d_attn.cu, attn_tc_kernel<D>) against the float64 ABI
oracle's per-element bound (oracle/abi_oracle.py).  The key loop runs S steps per trip (S = 4 ring stages at head_dim
40 / 80, 3 at 160) and masks key columns only in the last tile, or in every tile when a TMA box holds fewer than 64 keys.
These cases cover what that loop adds over test_attention_adversarial_gpu.py (ragged last tiles, rescale patterns):

  * every tile partial   key views with e1 < 64 whose boxes hold 48 keys (e1 = 48, e2 = 4 and e1 = 16, e2 = 3)
  * tile counts          n = 1, 2, S - 1, S, S + 1 and 2S + r for every r: the trip remainder and the first / last trip
  * frame-0 keys         kv_i3_zero + accumulate + out_scale (the MVDreamI2V second attention) with n % S != 0
  * rescale position     the row maximum jumps on one tile at every position of a trip; the debug counter must see exactly
                         one rescale per consumer warp"""
import ctypes as C

import pytest
import torch

from oracle import abi_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
HEADS = 8
STAGES = {40: 4, 80: 4, 160: 3}


def _dqk(d):
    return (d + 15) // 16 * 16


def _dv(d):
    return (d + 1 + 15) // 16 * 16


def _buffers(lq_rows, lk_rows, d, gen):
    """Q rows [lq_rows, H*dqk] and K|V rows [lk_rows, H*dqk | H*dv] in the projection layout (zero padding, ones column)."""
    dqk, dv = _dqk(d), _dv(d)
    q = torch.zeros(lq_rows, HEADS, dqk, device=DEV)
    k = torch.zeros(lk_rows, HEADS, dqk, device=DEV)
    v = torch.zeros(lk_rows, HEADS, dv, device=DEV)
    q[..., :d] = torch.randn(lq_rows, HEADS, d, device=DEV, generator=gen)
    k[..., :d] = torch.randn(lk_rows, HEADS, d, device=DEV, generator=gen)
    v[..., :d] = torch.randn(lk_rows, HEADS, d, device=DEV, generator=gen)
    v[..., d] = 1.0
    return q, k, v


def _attend(qbuf, kvbuf, d, q_s, q_e, k_s, k_e, out, ostr, *, kv_i3_zero=False, accumulate=False, out_scale=1.0):
    """One tensor-core launch through ops.attention, checked against the oracle; returns the rescale count."""
    from animate3d_b200 import _lib as L
    from animate3d_b200 import ops
    lib = L.load()
    koff, voff = HEADS * _dqk(d), 2 * HEADS * _dqk(d)
    ldq, ldk = qbuf.shape[1], kvbuf.shape[1]
    vq = ops.view5(qbuf, 0, ldq, q_s, q_e)
    vk = ops.view5(kvbuf, 0, koff, k_s, k_e)
    vv = ops.view5(kvbuf, koff, ldk - koff, k_s, k_e)
    kw = dict(heads=HEADS, d=d, scale=d ** -0.5, kv_i3_zero=kv_i3_zero, accumulate=accumulate, out_scale=out_scale)
    ref = O.attention(O.V5(qbuf, 0, ldq, q_s, q_e), O.V5(kvbuf, 0, koff, k_s, k_e), O.V5(kvbuf, koff, ldk - koff, k_s, k_e),
                      out.clone(), ostr, **kw)
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    lib.a3d_debug_set_attn_trace(C.c_void_p(counter.data_ptr()))
    try:
        ops.attention(vq, vk, vv, out, ostr, impl=L.IMPL_TC, **kw)
        torch.cuda.synchronize()
    finally:
        lib.a3d_debug_set_attn_trace(C.c_void_p(None))
    what = f"d={d} q_e={q_e} k_e={k_e} kv_i3_zero={kv_i3_zero} accumulate={accumulate}"
    O.assert_within(O.flat(out, ref.value.numel()), ref, what)
    return int(counter.item())


def _dense(d, lq, lk, batches, gen, boost_tile=None):
    """batches x (lq queries, lk keys), rows contiguous per batch; boost_tile raises every row's logits on that 64-key
    tile by ~+20 nats."""
    q, k, v = _buffers(batches * lq, batches * lk, d, gen)
    if boost_tile is not None:
        A = 4.0
        q[:, :, 0] = A
        k[:, :, 0] = 0.0
        k.view(batches, lk, HEADS, -1)[:, 64 * boost_tile:64 * boost_tile + 64, :, 0] = 20.0 / (A * d ** -0.5)
    qbuf = q.reshape(batches * lq, -1).half().contiguous()
    kvbuf = torch.cat([k.reshape(batches * lk, -1), v.reshape(batches * lk, -1)], 1).half().contiguous()
    ldq, ldk = qbuf.shape[1], kvbuf.shape[1]
    C_ = HEADS * d
    out = torch.randn(batches * lq, C_, device=DEV, generator=gen).half()
    q_s = (ldq, lq * ldq, lq * ldq, batches * lq * ldq)
    k_s = (ldk, lk * ldk, lk * ldk, batches * lk * ldk)
    ostr = (C_, lq * C_, lq * C_, batches * lq * C_)
    return qbuf, kvbuf, q_s, k_s, out, ostr


def _tile_counts():
    cases = []
    for d, S in STAGES.items():
        for n in sorted({1, 2, S - 1, S, S + 1} | {2 * S + r for r in range(1, S)}):
            cases.append((d, n))
    return cases


@pytest.mark.parametrize("d,n", _tile_counts(), ids=lambda x: str(x))
def test_key_tile_counts(d, n):
    """n full 64-key tiles, and the same with the last tile ragged (64 n - 7 keys)."""
    gen = torch.Generator(device=DEV).manual_seed(100 * d + n)
    for lk in (64 * n, 64 * n - 7):
        batches, lq = 2, 128
        qbuf, kvbuf, q_s, k_s, out, ostr = _dense(d, lq, lk, batches, gen)
        _attend(qbuf, kvbuf, d, q_s, (lq, 1, batches, 1), k_s, (lk, 1, batches, 1), out, ostr)


@pytest.mark.parametrize("d", sorted(STAGES))
@pytest.mark.parametrize("e1,e2", [(48, 4), (16, 3)], ids=lambda x: str(x))
def test_every_key_tile_partial(d, e1, e2):
    """Keys in [e2, e1] views with e1 < 64: every TMA box holds fewer than 64 keys (48), so every step masks."""
    gen = torch.Generator(device=DEV).manual_seed(d + e1 + e2)
    batches, L = 3, e1 * e2
    q, k, v = _buffers(batches * L, batches * L, d, gen)
    qbuf = q.reshape(batches * L, -1).half().contiguous()
    kvbuf = torch.cat([k.reshape(batches * L, -1), v.reshape(batches * L, -1)], 1).half().contiguous()
    ldq, ldk = qbuf.shape[1], kvbuf.shape[1]
    C_ = HEADS * d
    out = torch.zeros(batches * L, C_, device=DEV, dtype=torch.float16)
    ext = (e1, e2, batches, 1)
    _attend(qbuf, kvbuf, d, (ldq, e1 * ldq, L * ldq, batches * L * ldq), ext,
            (ldk, e1 * ldk, L * ldk, batches * L * ldk), ext, out, (C_, e1 * C_, L * C_, batches * L * C_))


@pytest.mark.parametrize("d", sorted(STAGES))
def test_frame0_keys_accumulate(d):
    """MVDreamI2V second attention: queries of every frame attend to frame 0's keys (kv_i3_zero) of Nv = 5 views x 128
    tokens (n = 10 tiles: 10 % 4 = 2, 10 % 3 = 1), added onto the first output with out_scale."""
    gen = torch.Generator(device=DEV).manual_seed(7 * d)
    B, Nv, Fr, hw = 1, 5, 2, 128
    rows = B * Nv * Fr * hw
    q, k, v = _buffers(rows, rows, d, gen)
    buf = torch.cat([q.reshape(rows, -1), k.reshape(rows, -1), v.reshape(rows, -1)], 1).half().contiguous()
    ld = buf.shape[1]
    qoff = 0
    kvbuf = buf[:, HEADS * _dqk(d):]           # K | V columns: the same rows, column offset HEADS * dqk
    strides = (ld, Fr * hw * ld, hw * ld, Nv * Fr * hw * ld)   # rows ordered (b n f p)
    ext = (hw, Nv, Fr, B)
    C_ = HEADS * d
    out = torch.randn(rows, C_, device=DEV, generator=gen).half()
    ostr = (C_, Fr * hw * C_, hw * C_, Nv * Fr * hw * C_)
    _attend(buf[:, qoff:], kvbuf, d, strides, ext, strides, ext, out, ostr, kv_i3_zero=True, accumulate=True,
            out_scale=0.5)


@pytest.mark.parametrize("d", sorted(STAGES))
def test_rescale_at_each_trip_position(d):
    """The row maximum rises once, on tile j_up, for j_up at positions 1 and S - 1 of the first trip and 0 and 1 of the
    second: every consumer warp of every CTA takes the lazy-rescale branch exactly once."""
    S = STAGES[d]
    batches, lq, n = 2, 128, 2 * S + 1
    for j_up in (1, S - 1, S, S + 1):
        gen = torch.Generator(device=DEV).manual_seed(31 * d + j_up)
        qbuf, kvbuf, q_s, k_s, out, ostr = _dense(d, lq, 64 * n, batches, gen, boost_tile=j_up)
        count = _attend(qbuf, kvbuf, d, q_s, (lq, 1, batches, 1), k_s, (64 * n, 1, batches, 1), out, ostr)
        ctas = batches * HEADS * (lq // 128)
        assert count == 8 * ctas, f"d={d} j_up={j_up}: {count} rescales, want one per consumer warp ({8 * ctas})"
