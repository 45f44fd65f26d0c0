"""Adversarial inputs for the single-pass ("stale stabiliser") softmax of the tensor-core attention kernel
(csrc/a3d_attn.cu): the fast path keeps the running row maximum of the PREVIOUS key steps as the exponent offset and only
redoes a step / rescales O when a later key tile raises the maximum by more than kRescaleLog2.  `randn` logits
almost never reach that branch after the first steps, so these cases construct logits that must:

  * ascending     key norms grow with the key index: the row maximum keeps climbing -> periodic rescales
  * late_outliers a few keys far down the sequence carry +-30-logit outliers -> redo-this-step + rescale in one go
  * step_up       the second half of the keys is ~+25 logits above the first half
  * ragged keys   a key count that is not a multiple of 64, including a fully masked second half-tile at j > 0

Each case is checked against an fp32 softmax(QK^T)V of the same fp16 inputs and -- for the cases built to trigger it --
asserts through the debug counter (a3d_debug_set_attn_trace) that the lazy-rescale branch really ran.
Shapes follow the reference's cross-view attention (attention_processor.py:405-420, 656-669): L = 4 views x 32x32 at
head_dim 40, L = 4 x 16x16 at head_dim 80, L = 4 x 8x8 at head_dim 160."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
HEADS = 8


def _dqk(d):
    return (d + 15) // 16 * 16


def _dv(d):
    return (d + 1 + 15) // 16 * 16


def _pack(x, dp, ones_at=None):
    """[rows, heads, d] fp32 -> [rows, heads*dp] with zero padding (and the ones column of V)."""
    rows, h, d = x.shape
    o = torch.zeros(rows, h, dp, device=x.device)
    o[..., :d] = x
    if ones_at is not None:
        o[..., ones_at] = 1.0
    return o.reshape(rows, h * dp)


def _run(q, k, v, batches, lq, lk, d, scale):
    """q [batches*lq, H, d], k/v [batches*lk, H, d] (fp32 values already rounded to fp16) -> (out [batches*lq, H*d], count)."""
    from animate3d_b200 import _lib as L
    from animate3d_b200 import ops
    lib = L.load()
    dqk, dv = _dqk(d), _dv(d)
    qb = _pack(q, dqk).half().contiguous()
    kvb = torch.cat([_pack(k, dqk), _pack(v, dv, ones_at=d)], 1).half().contiguous()
    ldq, ldk = qb.shape[1], kvb.shape[1]
    cdim = HEADS * d
    out = torch.zeros(batches * lq, cdim, device=DEV, dtype=torch.float16)
    vq = ops.view5(qb, 0, ldq, (ldq, lq * ldq, lq * ldq, lq * ldq), (lq, 1, 1, batches))
    vk = ops.view5(kvb, 0, ldk, (ldk, lk * ldk, lk * ldk, lk * ldk), (lk, 1, 1, batches))
    vv = ops.view5(kvb, HEADS * dqk, ldk - HEADS * dqk, (ldk, lk * ldk, lk * ldk, lk * ldk), (lk, 1, 1, batches))
    counter = torch.zeros(8 + 4 * 32 * 8 + 32, dtype=torch.int64, device=DEV)   # [0] = rescale count, [8:] = timeline words
    lib.a3d_debug_set_attn_trace(C.c_void_p(counter.data_ptr()))
    try:
        ops.attention(vq, vk, vv, out, (cdim, lq * cdim, lq * cdim, lq * cdim), heads=HEADS, d=d, scale=scale, impl=L.IMPL_TC)
        torch.cuda.synchronize()
    finally:
        lib.a3d_debug_set_attn_trace(C.c_void_p(None))
    return out, int(counter[0].item())


def _ref(q, k, v, batches, lq, lk, d, scale):
    qq = q.reshape(batches, lq, HEADS, d).permute(0, 2, 1, 3)
    kk = k.reshape(batches, lk, HEADS, d).permute(0, 2, 1, 3)
    vv = v.reshape(batches, lk, HEADS, d).permute(0, 2, 1, 3)
    s = torch.einsum("bhqd,bhkd->bhqk", qq, kk) * scale
    o = torch.einsum("bhqk,bhkd->bhqd", s.softmax(-1), vv)
    return o.permute(0, 2, 1, 3).reshape(batches * lq, HEADS * d)


def _check(out, ref, what, tol=4e-3):
    e = ((out.float() - ref).norm() / (ref.norm() + 1e-12)).item()
    mx = (out.float() - ref).abs().max().item()
    sc = ref.abs().max().item() + 1e-6
    assert math.isfinite(e) and e < tol, f"{what}: rel-l2 {e:.3e}"
    assert mx < 2e-2 * sc + 1e-3, f"{what}: max-abs {mx:.3e} vs scale {sc:.3e}"


def _base(batches, lq, lk, d, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    r16 = lambda t: t.half().float()
    q = r16(torch.randn(batches * lq, HEADS, d, device=DEV, generator=g))
    k = r16(torch.randn(batches * lk, HEADS, d, device=DEV, generator=g))
    v = r16(torch.randn(batches * lk, HEADS, d, device=DEV, generator=g))
    return q, k, v, g


SHAPES = [("l0_d40", 4096, 40), ("l1_d80", 1024, 80), ("l2_d160", 256, 160)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: s[0])
@pytest.mark.parametrize("pattern", ["ascending", "late_outliers", "step_up", "descending"])
def test_softmax_rescale_branch(shape, pattern):
    name, L_, d = shape
    batches = 2
    scale = d ** -0.5
    q, k, v, g = _base(batches, L_, L_, d, 7 + d)
    # every query gets a common component A along e0; keys get a pattern-dependent component along e0, so
    # logit(q, k_j) = scale * (A * c_j + noise)
    A = 6.0
    q[:, :, 0] = A
    pos = (torch.arange(L_, device=DEV).float() / L_).repeat(batches)            # key position in [0, 1)
    if pattern == "ascending":        # row max climbs by ~60 nats over the sequence: a rescale every few key tiles
        c = pos * 60.0 / (A * scale)
    elif pattern == "descending":     # the maximum is in the first tile: the fast path must never rescale afterwards
        c = (1.0 - pos) * 200.0 / (A * scale)
    elif pattern == "step_up":        # second half +25 nats
        c = (pos >= 0.5).float() * 25.0 / (A * scale)
    else:                             # a handful of +-30-nat outliers in the last quarter of the keys
        c = torch.zeros_like(pos)
        idx = torch.randint(int(0.75 * L_), L_, (batches, 6), device=DEV, generator=g)
        sign = torch.tensor([1.0, -1.0, 1.0, 1.0, -1.0, 1.0], device=DEV)
        for b in range(batches):
            c[b * L_ + idx[b]] = sign * 30.0 / (A * scale)
    k[:, :, 0] = (c[:, None]).half().float()
    out, count = _run(q, k, v, batches, L_, L_, d, scale)
    ref = _ref(q, k, v, batches, L_, L_, d, scale)
    _check(out, ref, f"{name} {pattern}")
    print(f"{name} {pattern}: lazy-rescale branch taken {count} times")
    if pattern == "descending":
        assert count == 0, f"{name}: a descending maximum must stay on the fast path ({count} rescales)"
    else:
        assert count > 0, f"{name} {pattern}: the rescale branch was never taken -- the input does not test it"


@pytest.mark.parametrize("case", [("d40_k992", 1024, 992, 40), ("d40_k1000", 1024, 1000, 40), ("d40_k4070", 4096, 4070, 40),
                                  ("d80_k992", 1024, 992, 80), ("d80_k1000", 256, 1000, 80), ("d160_k77", 64, 77, 160),
                                  ("d40_k100", 128, 100, 40)], ids=lambda c: c[0])
def test_ragged_key_count(case):
    """Key counts that are not a multiple of the 64-key step: 992 leaves a fully masked second half-tile in the last step
    (j = 15 > 0), 1000 / 4070 / 100 a partially masked one.  Rows past the key extent are zero-filled by TMA and must get
    zero weight (score -inf), not exp(0)."""
    name, lq, lk, d = case
    batches = 3
    scale = d ** -0.5
    q, k, v, g = _base(batches, lq, lk, d, 11 + lk)
    # also make the LAST keys the largest, so the ragged step is the one that raises the maximum
    k[:, :, 0] = 0.0
    q[:, :, 0] = 4.0
    pos = (torch.arange(lk, device=DEV).float() / lk).repeat(batches)
    k[:, :, 0] = ((pos > 0.9).float() * 20.0 / (4.0 * scale))[:, None].half().float()
    out, count = _run(q, k, v, batches, lq, lk, d, scale)
    ref = _ref(q, k, v, batches, lq, lk, d, scale)
    _check(out, ref, name)
    print(f"{name}: lazy-rescale branch taken {count} times")
    if lk > 128:      # with at most two 64-key steps the maximum may already sit in the first one
        assert count > 0


def test_counter_is_off_by_default():
    q, k, v, _ = _base(1, 128, 128, 40, 3)
    from animate3d_b200 import _lib as L
    lib = L.load()
    lib.a3d_debug_set_attn_trace(C.c_void_p(None))
    out, _ = _run(q, k, v, 1, 128, 128, 40, 40 ** -0.5)
    _check(out, _ref(q, k, v, 1, 128, 128, 40, 40 ** -0.5), "plain")
