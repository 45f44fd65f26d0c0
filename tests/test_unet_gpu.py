"""End-to-end parity of the H100 UNet engine against the fp32 CPU oracle (same seeded random weights and inputs).
north_star tolerance: fp16 latents within 1e-2 relative (rel-L2 and max-abs/max-ref both asserted)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(nv, nf, groups, seed=0, cond_zero=False, t=500, graph=True, ip_scale=1.0, **geometry):
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from oracle import unet_oracle as O
    ocfg = O.UNetConfig(num_views=nv, num_frames=nf, ip_scale=ip_scale, **geometry)
    sd = O.make_state_dict(ocfg, seed)
    sample, text, camera, img = O.synthetic_inputs(ocfg, groups, nv, nf, seed)
    torch.set_num_threads(min(16, os.cpu_count() or 1))   # many-core hosts: the fp32 oracle is fastest far below cpu_count
    with torch.no_grad():
        ref = O.unet_forward(sd, ocfg, sample, t, text, camera, img, nv, i2v_cond_time_zero=cond_zero)
    model = MVUNetMotionModel(UNetConfig(num_views=nv, num_frames=nf, ip_scale=ip_scale, **geometry))
    model.use_cuda_graph = graph
    missing, unexpected = model.load_state_dict(sd)
    assert not missing and not unexpected
    outs = []
    for _ in range(3 if graph else 1):   # eager, then graph replays
        out = model(sample.cuda(), t, text.cuda(), camera=camera.cuda(), added_cond_kwargs={"image_embeds": img.cuda()},
                    num_views=nv, i2v_cond_time_zero=cond_zero).sample
        outs.append(out.float().cpu())
    return ref, outs, model


def _check(ref, out, what):
    rel = ((out - ref).norm() / ref.norm()).item()
    mx = ((out - ref).abs().max() / ref.abs().max()).item()
    print(f"{what}: rel-l2 {rel:.3e}  max-abs/max-ref {mx:.3e}")
    assert rel < 1e-2, f"{what}: rel-l2 {rel}"
    assert mx < 2e-2, f"{what}: max-abs rel {mx}"


def test_unet_plumbing_config_matches_oracle():
    """BASELINE config 1: 1 view x 4 frames, 32x32x4 latent."""
    ref, outs, model = _run(1, 4, 1)
    for i, o in enumerate(outs):
        assert o.shape == ref.shape
        _check(ref, o, f"plumbing call {i}")
    # no float atomics anywhere on the path (GroupNorm statistics are a fixed-order tree): replays are bit-identical
    assert torch.equal(outs[1], outs[2])
    assert model.launches_per_forward > 500


def test_unet_ip_scale_zero_matches_oracle():
    """ip_scale = 0 turns the IP-adapter image branch off (attention_processor.py:283: hidden + scale * ip_hidden); the
    accumulated attention call must add nothing, not the branch at full weight."""
    ref, outs, _ = _run(1, 4, 1, seed=6, graph=False, ip_scale=0.0)
    _check(ref, outs[0], "ip_scale = 0")
    ref1, _, _ = _run(1, 4, 1, seed=6, graph=False, ip_scale=1.0)
    assert ((ref1 - ref).norm() / ref.norm()).item() > 1e-2, "the image branch must matter for this check to mean anything"


def test_unet_multiview_cfg_batch_matches_oracle():
    """2 groups (CFG-like batch) x 2 views x 3 frames: exercises cross-view attention, I2V frame-0 keys, GN-over-frames."""
    ref, outs, _ = _run(2, 3, 2, seed=3, t=961)
    _check(ref, outs[-1], "2 groups x 2 views x 3 frames")


def test_unet_i2v_cond_time_zero():
    ref, outs, _ = _run(1, 4, 1, seed=5, cond_zero=True, graph=False)
    _check(ref, outs[0], "i2v_cond_time_zero")


def test_unet_motion_heads_differ_from_spatial():
    """Motion modules with 4 heads next to 8 spatial heads (head dims 40, 80 and 160): every processor packs and attends with
    its own layer's head count."""
    ref, outs, _ = _run(2, 3, 1, seed=8, graph=False, motion_num_attention_heads=4, block_out_channels=(320, 640, 640, 640))
    _check(ref, outs[0], "motion heads 4, spatial heads 8")


def _oracle_threads():
    torch.set_num_threads(min(32, os.cpu_count() or 1))


def test_unet_headline_config_matches_oracle():
    """BASELINE configs[1] -- the configuration every bench number is quoted on: (uncond, cond) CFG batch x 4 views x 16
    frames x 32x32x4 latents (L = 4096 tokens in the level-0 cross-view attention), CUDA-graph replay.  The fp32 oracle runs
    the two CFG branches as two forwards (they never interact: SURVEY 8e) to bound host memory."""
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from oracle import unet_oracle as O
    nv, nf, groups, seed, t = 4, 16, 2, 21, 961
    ocfg = O.UNetConfig(num_views=nv, num_frames=nf)
    sd = O.make_state_dict(ocfg, seed)
    sample, text, camera, img = O.synthetic_inputs(ocfg, groups, nv, nf, seed)
    img[:nv] = 0          # the unconditional branch of the sampler carries zero image embeds (pipeline.py:537)
    model = MVUNetMotionModel(UNetConfig(num_views=nv, num_frames=nf))
    model.load_state_dict(sd)
    outs = []
    for _ in range(3):    # eager + capture, then two graph replays
        outs.append(model(sample.cuda(), t, text.cuda(), camera=camera.cuda(), added_cond_kwargs={"image_embeds": img.cuda()},
                          num_views=nv).sample.float().cpu())
    assert model._graphs, "the headline forward must run as a captured CUDA graph"
    _oracle_threads()
    refs = []
    import time
    with torch.no_grad():
        for g in range(groups):
            s = slice(g * nv, (g + 1) * nv)
            t0 = time.perf_counter()
            refs.append(O.unet_forward(sd, ocfg, sample[s], t, text[s], camera[s], img[s], nv))
            print(f"CPU oracle, one full 4-view x 16-frame CFG branch (25.97 TFLOP): {time.perf_counter() - t0:.1f} s on "
                  f"{torch.get_num_threads()} threads -> {2 * (time.perf_counter() - t0):.0f} s per CFG denoise step")
    ref = torch.cat(refs, 0)
    for i, o in enumerate(outs):
        _check(ref, o, f"headline 2x4vx16f call {i}")
    for g in range(groups):                                  # per CFG branch as well: one branch must not hide the other
        s = slice(g * nv, (g + 1) * nv)
        _check(ref[s], outs[-1][s], f"headline branch {g}")
    assert torch.equal(outs[1], outs[2]), "graph replays of the same inputs must be bit-identical"


def test_three_denoise_steps_match_oracle_sampler():
    """Three consecutive iterations of the sampler loop (pipeline.py:1006-1031): CFG UNet call, guidance combine, DDIM
    update, frame-0 re-injection -- the engine's `denoise_step` vs oracle UNet + oracle scheduler, to catch drift that a
    single forward cannot show.  2 views x 4 frames keeps the six oracle forwards within a minute."""
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    from animate3d_b200.scheduler import DDIMScheduler
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from oracle import unet_oracle as O
    from oracle.scheduler_oracle import DDIMOracle, denoise_step
    nv, nf, seed, gscale = 2, 4, 9, 7.5
    ocfg = O.UNetConfig(num_views=nv, num_frames=nf)
    sd = O.make_state_dict(ocfg, seed)
    sample, text, camera, img = O.synthetic_inputs(ocfg, 2, nv, nf, seed)
    img[:nv] = 0
    lat0 = sample[:nv].clone()
    first = lat0[:, :, :1].clone()
    model = MVUNetMotionModel(UNetConfig(num_views=nv, num_frames=nf))
    model.load_state_dict(sd)
    sched = DDIMScheduler()
    pipe = AnimateDiffMVI2VPipeline(unet=model, scheduler=sched)
    ts = [int(t) for t in sched.set_timesteps(25)][:3]
    osched = DDIMOracle()
    osched.set_timesteps(25)
    lat = lat0.cuda().contiguous()
    ref = lat0.clone()
    _oracle_threads()
    for i, t in enumerate(ts):
        pipe.denoise_step(lat, t, text.cuda(), camera.cuda(), img.cuda(), first.cuda(), gscale, num_views=nv)
        with torch.no_grad():
            x2 = torch.cat([ref, ref])
            eps2 = O.unet_forward(sd, ocfg, x2, t, text, camera, img, nv)
        ref = denoise_step(ref, eps2, first, gscale, osched, t)
        got = lat.float().cpu()
        rel = ((got - ref).norm() / ref.norm()).item()
        print(f"denoise step {i} (t={t}): rel-l2 {rel:.3e}")
        assert rel < 1e-2, f"step {i}: {rel}"
        torch.testing.assert_close(got[:, :, :1], first, rtol=0, atol=0)      # frame 0 is re-injected exactly


def test_arena_growth_invalidates_captured_graphs():
    """A later, larger forward makes the activation arena reallocate; graphs captured for other shapes hold the old
    pointers and must be dropped (ADVICE r1): small -> large -> small must still match the eager result."""
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from oracle import unet_oracle as O
    ocfg = O.UNetConfig(num_views=1, num_frames=2)
    sd = O.make_state_dict(ocfg, 4)
    model = MVUNetMotionModel(UNetConfig(num_views=1, num_frames=2))
    model.load_state_dict(sd)

    def call(groups, seed):
        s, t, c, i = O.synthetic_inputs(ocfg, groups, 1, 2, seed)
        return model(s.cuda(), 300, t.cuda(), camera=c.cuda(), added_cond_kwargs={"image_embeds": i.cuda()}, num_views=1).sample

    a0 = call(1, 1).clone()
    a1 = call(1, 1).clone()           # graph replay for the small shape
    call(3, 2)                        # grows every arena buffer
    torch.cuda.synchronize()
    junk = [torch.randn(1 << 22, device="cuda") for _ in range(8)]   # reuse whatever the allocator got back
    a2 = call(1, 1).clone()
    torch.cuda.synchronize()
    assert torch.equal(a0, a1)
    assert torch.equal(a0, a2), "stale graph replayed after the arena was reallocated"
    del junk
