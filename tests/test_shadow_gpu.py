"""Every kernel launch of real passes checked against the float64 ABI oracle (tests/shadow.py): the UNet at the headline
configuration, the 1-view x 4-frame plumbing configuration through one sampler step, the VAE encoder (forward and input
gradient) and decoder at 256^2, and the three attention processors.  A launch fails when any element leaves its bound; the
last test asserts that together the passes reached every wrapped op and every kernel path."""
import time

import pytest
import torch

import shadow as S

pytestmark = pytest.mark.gpu

RECORDS = []


def _finish(sh, what, t0):
    wall = time.perf_counter() - t0
    RECORDS.extend(sh.records)
    print(f"\n[{what}] {len(sh.records)} launches checked on {torch.cuda.get_device_name()} in {wall:.1f} s, "
          f"peak device memory {sh.peak_bytes / 2**30:.1f} GiB\n{sh.summary()}")
    bad = sh.failures()
    assert not bad, f"{what}: {len(bad)} launches exceed their bound\n" + sh.table(sorted(bad, key=lambda r: -r["ratio"])[:40])


def _unet(nv, nf, seed):
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from oracle import unet_oracle as O
    ocfg = O.UNetConfig(num_views=nv, num_frames=nf)
    sd = O.make_state_dict(ocfg, seed)
    model = MVUNetMotionModel(UNetConfig(num_views=nv, num_frames=nf))
    model.load_state_dict(sd)
    model.use_cuda_graph = False
    return model, O.synthetic_inputs(ocfg, 2, nv, nf, seed)


def test_shadow_unet_headline():
    """2 CFG x 4 views x 16 frames x 32^2 latents, eager; the number of checked launches equals what a plain counting patch
    sees for the same forward, so nothing bypassed the shadow."""
    torch.cuda.reset_peak_memory_stats()
    nv, nf = 4, 16
    model, (sample, text, camera, img) = _unet(nv, nf, 21)
    img[:nv] = 0
    args = (sample.cuda(), 961, text.cuda())
    kw = dict(camera=camera.cuda(), added_cond_kwargs={"image_embeds": img.cuda()}, num_views=nv)
    with S.counting() as calls:
        model(*args, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sh = S.Shadow("unet headline")
    with sh.active():
        model(*args, **kw)
    assert dict(sh.calls) == dict(calls), (dict(sh.calls), dict(calls))
    assert len(sh.records) == sum(calls.values())
    _finish(sh, "UNet 2 CFG x 4 views x 16 frames", t0)


def test_shadow_plumbing_sampler_step():
    """1 view x 4 frames (generic temporal kernel, single-view attention) through one CFG + DDIM sampler step."""
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    from animate3d_b200.scheduler import DDIMScheduler
    torch.cuda.reset_peak_memory_stats()
    nv, nf = 1, 4
    model, (sample, text, camera, img) = _unet(nv, nf, 5)
    sched = DDIMScheduler()
    t = int(sched.set_timesteps(25)[5])
    pipe = AnimateDiffMVI2VPipeline(unet=model, scheduler=sched)
    lat = sample[:nv].cuda().contiguous()
    first = lat[:, :, :1].clone()
    t0 = time.perf_counter()
    sh = S.Shadow("plumbing")
    with sh.active():
        pipe.denoise_step(lat, t, text.cuda(), camera.cuda(), img.cuda(), first, 7.5, num_views=nv)
    _finish(sh, "UNet 1 view x 4 frames + DDIM step", t0)


def test_shadow_vae():
    from animate3d_b200.vae import AutoencoderKL
    from oracle import vae_oracle as VO
    torch.cuda.reset_peak_memory_stats()
    vae = AutoencoderKL()
    vae.load_state_dict(VO.make_state_dict(VO.VAEConfig(), 0))
    g = torch.Generator().manual_seed(1)
    x = (torch.rand(2, 3, 256, 256, generator=g) * 2 - 1).cuda().requires_grad_(True)
    dm = torch.randn(2, 8, 32, 32, generator=g).cuda()
    z = torch.randn(2, 4, 32, 32, generator=g).cuda()
    t0 = time.perf_counter()
    sh = S.Shadow("vae")
    with sh.active():
        (vae.encode_moments(x) * dm).sum().backward()
        with torch.no_grad():
            vae.decode(z)
    _finish(sh, "VAE encoder + input gradient + decoder at 256^2", t0)


def test_shadow_processors():
    from animate3d_b200 import modules as Mo
    from test_processors_gpu import _attn_and_sd
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator().manual_seed(4)
    t0 = time.perf_counter()
    sh = S.Shadow("processors")
    c = 320
    mv = Mo.MVDreamI2VXFormersAttnProcessor(hidden_size=c, num_views=4, num_frames=3, device="cuda")
    a_mv, _ = _attn_and_sd(c, c, 1, mv)
    ip = Mo.IPAdapterXFormersAttnProcessor(hidden_size=c, cross_attention_dim=768, num_tokens=(4,), scale=0.7, device="cuda")
    a_ip, _ = _attn_and_sd(c, 768, 2, ip)
    stp = Mo.SpatioTemporalI2VXFormersAttnProcessor(hidden_size=c, feature_size=16, num_views=4, num_frames=16,
                                                    use_alpha_blender=True, device="cuda")
    a_st, _ = _attn_and_sd(c, c, 3, stp)
    with sh.active():
        mv(a_mv, torch.randn(2 * 4 * 3, 256, c, generator=g).cuda())
        ip(a_ip, torch.randn(6, 256, c, generator=g).cuda(),
           encoder_hidden_states=(torch.randn(6, 77, 768, generator=g).cuda(), [torch.randn(6, 4, 768, generator=g).cuda()]))
        stp(a_st, torch.randn(4 * 256, 16, c, generator=g).cuda())
    _finish(sh, "MVDreamI2V + IPAdapter + SpatioTemporalI2V processors", t0)


def test_shadow_coverage():
    """Together the passes above reached every wrapped op and every kernel path."""
    if not RECORDS:
        pytest.skip("run together with the shadow passes above")
    ops = {r["op"] for r in RECORDS}
    missing = [o for o in S.OPS if o not in ops]
    assert not missing, f"never called: {missing}"
    attn_lk = [int(r["geo"].split("Lk=")[1].split()[0]) for r in RECORDS if r["op"] == "attention"]
    assert min(attn_lk) <= 8 and any(9 <= k <= 80 for k in attn_lk) and max(attn_lk) > 80, sorted(set(attn_lk))
    apaths = {r["path"] for r in RECORDS if r["op"] == "attention"}
    assert {"fewkeys", "shortkeys", "tc"} <= apaths, apaths
    tpaths = {r["path"] for r in RECORDS if r["op"] == "temporal_attn"}
    assert tpaths == {"frames16", "generic"}, tpaths
    gpaths = {r["path"] for r in RECORDS if r["op"] == "gemm"}
    print("GEMM paths:", sorted(gpaths))
    for bn in ("BN128", "BN160", "BN256"):
        assert any(bn in p for p in gpaths), (bn, sorted(gpaths))
    for geom in ("conv-wide-rows", "conv-row-block", "conv-image-block"):
        assert any(geom in p for p in gpaths), (geom, sorted(gpaths))
    for epi in (" plain ", " res ", " geglu ", " f32 "):
        assert any(epi in p for p in gpaths), (epi, sorted(gpaths))
