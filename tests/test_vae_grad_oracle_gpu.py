"""The VAE encoder's input gradient, one autograd Function call at a time, over real passes of the SD-1.5 encoder
(block_out_channels (128, 256, 512, 512)) on the engine's kernels: every backward call of `_Conv3`, `_Lin`, `_GroupNorm`,
`_ConvIn` and `_ConvOut` is checked element by element against oracle/vae_grad_oracle.py (tests/vae_grad_shadow.py), at the
SDS image size (2 x 256^2), on non-square images (64x256 and 256x64) and at the 4D-SDS batch of 64 views at 256^2 (images
0, 31 and 63 of every call).  Each pass checks as many backward calls as a plain counting pass sees; the last test asserts
that together the passes reached every Function in every role the encoder uses."""
import time

import pytest
import torch

import vae_grad_shadow as S

pytestmark = pytest.mark.gpu

RECORDS = []


def _model():
    from animate3d_b200.vae import AutoencoderKL
    from oracle import vae_oracle as VO
    vae = AutoencoderKL()
    vae.load_state_dict(VO.make_state_dict(VO.VAEConfig(), 0))
    return vae


def _inputs(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, 3, h, w, generator=g) * 2 - 1).cuda()
    dm = torch.randn(n, 8, h // 8, w // 8, generator=g).cuda()
    return x, dm


def _pass(vae, x, dm):
    xg = x.clone().requires_grad_(True)
    (vae.encode_moments(xg) * dm).sum().backward()
    return xg.grad


def _check(vae, n, h, w, seed, images=None):
    x, dm = _inputs(n, h, w, seed)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    with S.counting() as calls:
        _pass(vae, x, dm)
    torch.cuda.synchronize()
    engine_s, engine_peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated()
    what = f"{n} x {h}x{w}" + (f", images {list(images)}" if images else "")
    sh = S.GradShadow(what, model=vae, n=n, images=images)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    with sh.active():
        _pass(vae, x, dm)
    torch.cuda.synchronize()
    checked_s, checked_peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated()
    RECORDS.extend(sh.records)
    same = dict(sh.calls) == dict(calls)
    print(f"\n[{what}] on {torch.cuda.get_device_name()}: {sum(sh.calls.values())} backward calls checked "
          f"({'equal to' if same else 'DIFFERENT FROM'} the counting pass's {sum(calls.values())}), {len(sh.records)} checks\n"
          f"forward + backward alone {engine_s:.2f} s, peak device memory {engine_peak / 2**30:.2f} GiB; "
          f"with the checks {checked_s:.1f} s, peak {checked_peak / 2**30:.2f} GiB\n{sh.summary()}")
    assert same, (dict(sh.calls), dict(calls))
    bad = sh.failures()
    assert not bad, f"{what}: {len(bad)} checks exceed their bound\n" + sh.table(sorted(bad, key=lambda r: -r["ratio"])[:40])
    return sh


def test_sds_image_size():
    _check(_model(), 2, 256, 256, 1)


@pytest.mark.parametrize("h,w", [(64, 256), (256, 64)])
def test_non_square(h, w):
    """The last downsample level of a 64-wide image is 8 pixels wide."""
    _check(_model(), 1, h, w, h + w)


def test_sds_batch_of_64_views():
    """The 4D-SDS step's batch: 64 views at 256^2.  Image 63's rows start near element 2^29 of the widest activations."""
    sh = _check(_model(), 64, 256, 256, 64, images=(0, 31, 63))
    assert {r["images"] for r in sh.records if r["kind"] != "residual"} == {(0, 1), (31, 32), (63, 64)}


def test_coverage():
    """Together the passes above reached every Function in every role of the encoder."""
    if not RECORDS:
        pytest.skip("run together with the passes above")
    kinds = {r["kind"] for r in RECORDS}
    want = {"conv3 stride 1", "conv3 stride 1 res", "conv3 stride 2", "lin", "lin res", "gn silu 0", "gn silu 1", "gn stats",
            "residual", "conv_in cin 3", "conv_out cout 8"}
    assert want <= kinds, want - kinds
    names = {r["name"] for r in RECORDS}
    assert "?" not in names
    assert {f"enc_down.{i}.down" for i in range(3)} <= names, sorted(names)
    lin = {(r["name"].rsplit(".", 1)[-1], r["kind"]) for r in RECORDS if r["fn"] == "_Lin" and r["kind"] != "residual"}
    assert {("sc", "lin"), ("qkv", "lin"), ("out", "lin res")} <= lin, lin
    print(f"\n{len(RECORDS)} checks over all passes, worst |err|/bound {max(r['ratio'] for r in RECORDS):.3g}")
