"""Sampler options on the H100: a3d_ddim_step per element against its float64 oracle, the released step unchanged, and the
whole `__call__` (no guidance, eta = 1, i2v_similarity_init) against the oracle UNet driven by the reference's sampler loop
with a copy of the same seeded CPU generator."""
import os

import pytest
import torch

import sampler_oracle as SO
from oracle import abi_oracle as A

pytestmark = pytest.mark.gpu


def _ops():
    from animate3d_b200 import _lib, ops
    return ops, _lib


def _step_inputs(cfg_mode, bn=3, c=4, f=5, hw=37, seed=0):
    """bn * c * f * hw = 2220 elements: not a multiple of the 256-thread block."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    lat = torch.randn(bn, c, f, hw, device="cuda", generator=g)
    eps = torch.randn((2 if cfg_mode else 1) * bn, c, f, hw, device="cuda", generator=g)
    first = torch.randn(bn, c, 1, hw, device="cuda", generator=g)
    z = torch.randn(bn, c, f, hw, device="cuda", generator=g)
    return lat, eps, first, z, (bn, c, f, hw)


@pytest.mark.parametrize("cfg_mode", [0, 1, 2])
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_ddim_step_kernel_matches_oracle(cfg_mode, eta):
    from animate3d_b200.scheduler import DDIMScheduler
    ops, _ = _ops()
    s = DDIMScheduler()
    s.set_timesteps(25)
    for t in (961, 481, 1):                                       # t = 1 is the last step: alpha_prev = 1, std_dev = 0
        a_t, a_p, dc, sd = s.step_coefficients(t, eta)
        for with_first in (True, False):
            lat, eps, first, z, (bn, c, f, hw) = _step_inputs(cfg_mode, seed=t)
            zz = z if eta > 0 else None                               # eta 0: NULL variance noise
            ff = first if with_first else None
            ref = SO.ddim_step(lat.clone(), eps, ff, zz, bn, c, f, hw, cfg_mode, 7.5, a_t, a_p, dc, sd)
            ops.ddim_step(lat, eps, ff, zz, bn, c, f, hw, cfg_mode, 7.5, a_t, a_p, dc, sd)
            torch.cuda.synchronize()
            v = A.check(lat, ref)
            assert v.ratio <= 1.0, (t, with_first, v)
            if with_first:
                assert torch.equal(lat[:, :, 0], first[:, :, 0])
    assert sd == 0.0


def test_ddim_step_rejects_missing_noise_and_bad_mode():
    ops, L = _ops()
    lat, eps, first, z, (bn, c, f, hw) = _step_inputs(1)
    with pytest.raises(L.A3DError, match="variance_noise"):
        ops.ddim_step(lat, eps, first, None, bn, c, f, hw, 1, 7.5, 0.3, 0.4, 0.7, 0.1)
    with pytest.raises(L.A3DError, match="cfg_mode"):
        ops.ddim_step(lat, eps, first, z, bn, c, f, hw, 3, 7.5, 0.3, 0.4, 0.7, 0.1)


def test_released_step_is_unchanged():
    """eta 0 with guidance through a3d_ddim_step (the scheduler's coefficients) is bit-identical to a3d_ddim_cfg_step."""
    from animate3d_b200.scheduler import DDIMScheduler
    ops, _ = _ops()
    s = DDIMScheduler()
    for t in s.set_timesteps(25).tolist():
        a_t, a_p, dc, sd = s.step_coefficients(t, 0.0)
        for mode in (1, 2):
            lat, eps, first, _, (bn, c, f, hw) = _step_inputs(mode, bn=4, c=4, f=16, hw=1024, seed=t)
            old = lat.clone()
            ops.ddim_cfg_step(old, eps, first, bn, c, f, hw, 7.5, a_t, a_p, uncond_first=mode == 1)
            ops.ddim_step(lat, eps, first, None, bn, c, f, hw, mode, 7.5, a_t, a_p, dc, sd)
            torch.cuda.synchronize()
            assert torch.equal(lat, old), (t, mode)


# ------------------------------------------------------------------------------------------------ whole sampler
NV, NF, SEED = 2, 4, 9


@pytest.fixture(scope="module")
def setup():
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    from animate3d_b200.scheduler import DDIMScheduler
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from oracle import unet_oracle as O
    ocfg = O.UNetConfig(num_views=NV, num_frames=NF)
    sd = O.make_state_dict(ocfg, SEED)
    sample, text, _, img = O.synthetic_inputs(ocfg, 2, NV, NF, SEED)
    model = MVUNetMotionModel(UNetConfig(num_views=NV, num_frames=NF))
    model.load_state_dict(sd)
    pipe = AnimateDiffMVI2VPipeline(unet=model, scheduler=DDIMScheduler())
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    cond = dict(first=sample[:, :, :1][:NV].clone(), neg=text[:NV], pos=text[NV:], image=img[NV:])
    return pipe, sd, ocfg, cond


@pytest.mark.parametrize("case", [
    dict(name="no CFG", guidance_scale=1.0, eta=0.0, steps=3),
    dict(name="eta 1 with CFG", guidance_scale=7.5, eta=1.0, steps=3),
    dict(name="similarity init", guidance_scale=7.5, eta=0.0, steps=25, similarity={"strength": 0.15, "origin_prob": 0.3}),
], ids=lambda c: c["name"].replace(" ", "_"))
def test_pipeline_matches_oracle_sampler(setup, case):
    pipe, sd, ocfg, cond = setup
    gen = torch.Generator().manual_seed(1234)
    gen_ref = torch.Generator()
    gen_ref.set_state(gen.get_state())
    out = pipe(num_frames=NF, height=256, width=256, num_inference_steps=case["steps"], guidance_scale=case["guidance_scale"],
               num_videos_per_prompt=NV, eta=case["eta"], generator=gen, prompt_embeds=cond["pos"],
               negative_prompt_embeds=cond["neg"], ip_adapter_image_embeds=cond["image"], output_type="latent",
               first_frame_latents=cond["first"], i2v_similarity_init=case.get("similarity")).frames
    ref = SO.sampler(sd, ocfg, cond["first"], cond["pos"], cond["neg"], cond["image"], NF, case["steps"],
                     case["guidance_scale"], case["eta"], gen_ref, case.get("similarity"))
    got = out.float().cpu()
    assert got.shape == ref.shape == (NV, 4, NF, 32, 32)
    rel = ((got - ref).norm() / ref.norm()).item()
    print(f"{case['name']}: rel-l2 {rel:.3e}")
    assert rel < 1e-2, (case["name"], rel)
    assert torch.equal(got[:, :, :1], cond["first"])
    # both sides consumed the generator draw for draw
    assert torch.equal(torch.randn(4, generator=gen), torch.randn(4, generator=gen_ref))


def test_freeinit_with_similarity_init_raises(setup):
    pipe, _, _, cond = setup
    pipe.enable_free_init(num_iters=2)
    try:
        with pytest.raises(ValueError, match="FreeInit"):
            pipe(num_frames=NF, height=256, width=256, num_inference_steps=25, num_videos_per_prompt=NV,
                 prompt_embeds=cond["pos"], negative_prompt_embeds=cond["neg"], ip_adapter_image_embeds=cond["image"],
                 first_frame_latents=cond["first"], output_type="latent",
                 i2v_similarity_init={"strength": 0.15, "origin_prob": 0.3})
    finally:
        pipe.disable_free_init()
