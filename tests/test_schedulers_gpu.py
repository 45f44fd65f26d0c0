"""DPM-Solver++, Euler and Euler-ancestral on the H100, through the C ABI: a3d_sampler_step per element against its float64
oracle, its argument checks, and the whole `__call__` against the reference's sampler loop with a copy of the same seeded
CPU generator.  The loop's model is the fp32 oracle UNet for a 4-step DPM-Solver++ case; an oracle UNet forward takes
tens of seconds on the host, so the other cases run the loop around the engine's own UNet (checked against the oracle in
test_unet_gpu.py), which isolates the scheduler, the step kernel and the random draws."""
import ctypes as C
import inspect
import os

import pytest
import torch

import solver_oracle as SV
from oracle import abi_oracle as A

pytestmark = pytest.mark.gpu


def _inputs(cfg_mode, bn=3, c=4, f=5, hw=37, seed=0):
    """bn * c * f * hw = 2220 elements: not a multiple of the 256-thread block."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    return dict(lat=r(bn, c, f, hw), eps=r((2 if cfg_mode else 1) * bn, c, f, hw), first=r(bn, c, 1, hw), z=r(bn, c, f, hw),
                m1=r(bn, c, f, hw)), (bn, c, f, hw)


def _steps():
    """(label, SolverStep) for every kind, order and solver type, including the last step (sigma = 0, always first order:
    its h is infinite) and a second-order last step to sigma_min."""
    from animate3d_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                          EulerDiscreteScheduler)
    out = []
    for kw in (dict(), dict(solver_type="heun"), dict(use_karras_sigmas=True, timestep_spacing="leading", steps_offset=1),
               dict(final_sigmas_type="sigma_min", solver_type="heun")):
        s = DPMSolverMultistepScheduler(**kw)
        s.set_timesteps(10)
        for i in (0, 4, 9):
            for order in ((1,) if i == 0 or float(s.sigmas[i + 1]) == 0.0 else (1, 2)):
                out.append((f"dpm {kw} i={i} order={order}", s._coefficients(i, order)))
    for cls in (EulerDiscreteScheduler, EulerAncestralDiscreteScheduler):
        s = cls()
        s.set_timesteps(25)
        for i in (0, 12, 24):
            out.append((f"{cls.__name__} i={i}", s._update(i)))
    return out


def test_sampler_step_symbol_is_exported():
    from animate3d_b200 import _lib
    assert hasattr(_lib.load(require_gpu=False), "a3d_sampler_step")


@pytest.mark.parametrize("cfg_mode", [0, 1, 2])
def test_sampler_step_kernel_matches_oracle(cfg_mode):
    from animate3d_b200 import ops
    steps = _steps()
    assert any(s.c_x == 0.0 and s.c_m0 == -1.0 for _, s in steps)          # the last DPM step (sigma = 0): x' = m0
    for k, (label, step) in enumerate(steps):
        for with_first in (True, False):
            x, (bn, c, f, hw) = _inputs(cfg_mode, seed=k)
            ff = x["first"] if with_first else None
            dpm = step.kind == SV.DPMPP
            hist = torch.zeros_like(x["lat"]) if dpm else None
            m1 = x["m1"] if dpm and step.order == 2 else None
            z = x["z"] if step.sigma_up != 0.0 else None
            ref, m0 = SV.sampler_step(x["lat"].clone(), x["eps"], ff, z, hist, m1, bn, c, f, hw, cfg_mode, 7.5, step)
            ops.sampler_step(x["lat"], x["eps"], ff, bn, c, f, hw, cfg_mode, 7.5, step, noise=z, history_out=hist,
                             history_in=m1)
            torch.cuda.synchronize()
            A.assert_within(x["lat"], ref, f"{label} cfg_mode={cfg_mode} first={with_first}")
            if dpm:
                A.assert_within(hist, m0, f"m0 of {label}")
                if with_first:
                    assert torch.count_nonzero(hist[:, :, 0]) == 0          # frame 0 is neither computed nor stored
            if with_first:
                assert torch.equal(x["lat"][:, :, 0], x["first"][:, :, 0])
            if step.c_x == 0.0 and step.c_m0 == -1.0:
                assert torch.equal(x["lat"][:, :, 1:], hist[:, :, 1:])        # x' = m0 exactly


def test_sampler_step_rejects_bad_arguments():
    from animate3d_b200 import _lib as L
    from animate3d_b200 import ops
    from animate3d_b200.scheduler import SAMPLER_DPMPP, SAMPLER_EULER, SolverStep
    x, (bn, c, f, hw) = _inputs(1)
    before = x["lat"].clone()
    cases = [(SolverStep(SAMPLER_DPMPP, 1, order=2, alpha_s0=0.9, sigma_s0=0.4, c_x=0.9, c_m0=-0.1, inv_r0=1.0, c_d1=0.1),
              dict(history_in=None), "history_in"),
             (SolverStep(SAMPLER_EULER, 1, sigma=2.0, dt=-0.5, sigma_up=0.3), dict(noise=None), "needs noise"),
             (SolverStep(7, 1), {}, "kind"),
             (SolverStep(SAMPLER_DPMPP, 1, order=3, alpha_s0=0.9, sigma_s0=0.4), {}, "order"),
             (SolverStep(SAMPLER_EULER, 1, sigma=2.0, dt=-0.5), dict(cfg_mode=3), "cfg_mode")]
    for step, kw, msg in cases:
        mode = kw.pop("cfg_mode", 1)
        with pytest.raises(L.A3DError, match=msg) as e:
            ops.sampler_step(x["lat"], x["eps"], x["first"], bn, c, f, hw, mode, 7.5, step, **kw)
        assert "error -1" in str(e.value)                                  # A3D_EINVAL
    lib = L.load()
    a = L.SamplerStepArgs()
    assert lib.a3d_sampler_step(C.byref(a), L.stream_ptr()) == -1          # kind 0 / order 0, NULL buffers
    assert lib.a3d_sampler_step(None, L.stream_ptr()) == -1
    torch.cuda.synchronize()
    assert torch.equal(x["lat"], before)                                   # nothing was launched


# ------------------------------------------------------------------------------------------------ whole sampler
NV, NF, SEED = 2, 4, 9


@pytest.fixture(scope="module")
def setup():
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from oracle import unet_oracle as O
    ocfg = O.UNetConfig(num_views=NV, num_frames=NF)
    sd = O.make_state_dict(ocfg, SEED)
    sample, text, _, img = O.synthetic_inputs(ocfg, 2, NV, NF, SEED)
    model = MVUNetMotionModel(UNetConfig(num_views=NV, num_frames=NF))
    model.load_state_dict(sd)
    pipe = AnimateDiffMVI2VPipeline(unet=model)
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    cond = dict(first=sample[:, :, :1][:NV].clone(), neg=text[:NV], pos=text[NV:], image=img[NV:])
    return pipe, sd, ocfg, cond


CASES = [
    dict(name="dpm 4 oracle unet", cls="DPMSolverMultistepScheduler", kw={}, steps=4, oracle_unet=True),
    dict(name="dpm 10", cls="DPMSolverMultistepScheduler", kw={}, steps=10),
    dict(name="dpm 25 heun", cls="DPMSolverMultistepScheduler", kw=dict(solver_type="heun"), steps=25),
    dict(name="dpm 25 midpoint karras", cls="DPMSolverMultistepScheduler", kw=dict(use_karras_sigmas=True), steps=25),
    dict(name="dpm 10 leading sigma_min", cls="DPMSolverMultistepScheduler",
         kw=dict(timestep_spacing="leading", steps_offset=1, final_sigmas_type="sigma_min", beta_start=0.00085,
                 beta_end=0.012), steps=10),
    dict(name="euler 25", cls="EulerDiscreteScheduler", kw={}, steps=25),
    dict(name="euler ancestral 25", cls="EulerAncestralDiscreteScheduler", kw={}, steps=25),
    dict(name="dpm 10 freeinit 3", cls="DPMSolverMultistepScheduler", kw={}, steps=10, free_init=3),
    dict(name="dpm 25 similarity init", cls="DPMSolverMultistepScheduler", kw={}, steps=25,
         similarity={"strength": 0.2, "origin_prob": 0.3}),
]
ORACLES = {"DPMSolverMultistepScheduler": SV.DPMSolverOracle, "EulerDiscreteScheduler": SV.EulerOracle,
           "EulerAncestralDiscreteScheduler": SV.EulerAncestralOracle}


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"].replace(" ", "_"))
def test_pipeline_matches_oracle_sampler(setup, case):
    from animate3d_b200 import scheduler as S
    pipe, sd, ocfg, cond = setup
    pipe.scheduler = getattr(S, case["cls"]).from_config(S.DDIMScheduler().config, **case["kw"])
    takes = inspect.signature(ORACLES[case["cls"]]).parameters
    okw = {k: v for k, v in pipe.scheduler.config.items() if k in takes}
    if case.get("free_init"):
        pipe.enable_free_init(num_iters=case["free_init"])
    gen = torch.Generator().manual_seed(1234)
    gen_ref = torch.Generator()
    gen_ref.set_state(gen.get_state())
    try:
        out = pipe(num_frames=NF, height=256, width=256, num_inference_steps=case["steps"], guidance_scale=7.5,
                   num_videos_per_prompt=NV, generator=gen, prompt_embeds=cond["pos"], negative_prompt_embeds=cond["neg"],
                   ip_adapter_image_embeds=cond["image"], output_type="latent", first_frame_latents=cond["first"],
                   i2v_similarity_init=case.get("similarity")).frames
    finally:
        pipe.disable_free_init()
        pipe.scheduler = S.DDIMScheduler()
    def engine_unet(x, t, pe, cam, ie, nv):
        return pipe.unet(x.cuda(), float(t), pe.cuda(), camera=cam.cuda(), added_cond_kwargs={"image_embeds": ie.cuda()},
                         num_views=nv).sample.float().cpu()
    ref = SV.sampler(sd, ocfg, cond["first"], cond["pos"], cond["neg"], cond["image"], NF, case["steps"], 7.5,
                     ORACLES[case["cls"]](**okw), gen_ref, case.get("similarity"), case.get("free_init", 1),
                     model=None if case.get("oracle_unet") else engine_unet)
    got = out.float().cpu()
    assert got.shape == ref.shape == (NV, 4, NF, 32, 32)
    rel = ((got - ref).norm() / ref.norm()).item()
    print(f"{case['name']}: rel-l2 {rel:.3e}")
    assert rel < 1e-2, (case["name"], rel)
    assert torch.equal(got[:, :, :1], cond["first"])
    assert torch.equal(torch.randn(4, generator=gen), torch.randn(4, generator=gen_ref))


def test_ddim_call_launches_only_the_ddim_cfg_step(setup, monkeypatch):
    """The default scheduler keeps its path: one a3d_ddim_cfg_step per step and no a3d_sampler_step / a3d_ddim_step."""
    from animate3d_b200 import ops
    from animate3d_b200.scheduler import DDIMScheduler
    pipe, _, _, cond = setup
    assert isinstance(pipe.scheduler, DDIMScheduler)
    calls = {"ddim_cfg_step": 0, "ddim_step": 0, "sampler_step": 0}
    for name in calls:
        real = getattr(ops, name)

        def counted(*a, _real=real, _name=name, **k):
            calls[_name] += 1
            return _real(*a, **k)
        monkeypatch.setattr(ops, name, counted)
    pipe(num_frames=NF, height=256, width=256, num_inference_steps=3, guidance_scale=7.5, num_videos_per_prompt=NV,
         generator=torch.Generator().manual_seed(0), prompt_embeds=cond["pos"], negative_prompt_embeds=cond["neg"],
         ip_adapter_image_embeds=cond["image"], output_type="latent", first_frame_latents=cond["first"])
    assert calls == {"ddim_cfg_step": 3, "ddim_step": 0, "sampler_step": 0}
