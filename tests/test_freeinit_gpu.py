"""FreeInit's filters and coarse-to-fine sampling, and per-view generator lists, on the H100: the whole `__call__` (engine
UNet and step kernels) against the reference loop of tests/freeinit_oracle.py run around the same engine UNet (checked
against the oracle in test_unet_gpu.py) with copies of the same seeded CPU generators, as test_multistep_gpu.py does; and
the released configuration (DDIM, butterworth FreeInit without fast sampling, one generator or none) bit for bit against
the code path it had before these options existed."""
import inspect
import math
import os

import pytest
import torch

import freeinit_oracle as FO
import multistep_oracle as MO
import solver_oracle as SV

pytestmark = pytest.mark.gpu

NV, NF, SEED = 4, 4, 9


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
    return pipe, cond


ORACLES = {"DDIMScheduler": FO.DDIMLoop, "DPMSolverMultistepScheduler": SV.DPMSolverOracle,
           "EulerAncestralDiscreteScheduler": FO.EulerAncestralLists, "PNDMScheduler": MO.PNDMOracle}
CASES = [
    dict(name="ddim 10 gaussian fast", cls="DDIMScheduler", steps=10,
         free_init=dict(num_iters=3, method="gaussian", use_fast_sampling=True)),
    dict(name="dpm 10 ideal", cls="DPMSolverMultistepScheduler", steps=10, free_init=dict(num_iters=3, method="ideal")),
    dict(name="pndm prk 12 butterworth fast", cls="PNDMScheduler", steps=12,
         free_init=dict(num_iters=3, method="butterworth", use_fast_sampling=True)),
    dict(name="ddim 10 eta 0.5 generator list gaussian fast", cls="DDIMScheduler", steps=10, eta=0.5, gens=NV,
         free_init=dict(num_iters=3, method="gaussian", use_fast_sampling=True)),
    dict(name="euler ancestral 10 generator list", cls="EulerAncestralDiscreteScheduler", steps=10, gens=NV,
         kw=dict(timestep_spacing="linspace", steps_offset=0)),
    dict(name="ddim 10 cpu generator freeinit", cls="DDIMScheduler", steps=10, free_init=dict(num_iters=3)),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"].replace(" ", "_"))
def test_pipeline_matches_oracle_sampler(setup, case):
    from animate3d_b200 import scheduler as S
    pipe, cond = setup
    if case["cls"] == "DDIMScheduler":
        pipe.scheduler = S.DDIMScheduler()
        oracle = FO.DDIMLoop(eta=case.get("eta", 0.0))
    else:
        pipe.scheduler = getattr(S, case["cls"]).from_config(S.DDIMScheduler().config, **case.get("kw", {}))
        takes = inspect.signature(ORACLES[case["cls"]]).parameters
        oracle = ORACLES[case["cls"]](**{k: v for k, v in pipe.scheduler.config.items() if k in takes})
    if case.get("free_init"):
        pipe.enable_free_init(**case["free_init"])
    seeds = range(1234, 1234 + case["gens"]) if case.get("gens") else [1234]
    gen = [torch.Generator().manual_seed(s) for s in seeds]
    gen_ref = [torch.Generator() for _ in seeds]
    for a, b in zip(gen_ref, gen):
        a.set_state(b.get_state())
    pick = (lambda g: g) if case.get("gens") else (lambda g: g[0])
    try:
        out = pipe(num_frames=NF, height=256, width=256, num_inference_steps=case["steps"], guidance_scale=7.5,
                   num_videos_per_prompt=NV, eta=case.get("eta", 0.0), generator=pick(gen), prompt_embeds=cond["pos"],
                   negative_prompt_embeds=cond["neg"], ip_adapter_image_embeds=cond["image"], output_type="latent",
                   first_frame_latents=cond["first"]).frames
    finally:
        pipe.disable_free_init()
        pipe.scheduler = S.DDIMScheduler()

    def engine_unet(x, t, pe, cam, ie, nv):
        return pipe.unet(x.cuda(), float(t), pe.cuda(), camera=cam.cuda(), added_cond_kwargs={"image_embeds": ie.cuda()},
                         num_views=nv).sample.float().cpu()
    ref, calls = FO.sampler(cond["first"], cond["pos"], cond["neg"], cond["image"], NF, case["steps"], 7.5, oracle,
                            pick(gen_ref), engine_unet, case.get("free_init"))
    got = out.float().cpu()
    assert got.shape == ref.shape == (NV, 4, NF, 32, 32)
    rel = ((got - ref).norm() / ref.norm()).item()
    print(f"{case['name']}: rel-l2 {rel:.3e}, {calls} UNet calls")
    assert rel < 1e-2, (case["name"], rel)
    assert torch.equal(got[:, :, :1], cond["first"])
    for a, b in zip(gen, gen_ref):
        assert torch.equal(torch.randn(4, generator=a), torch.randn(4, generator=b))


# ------------------------------------------------------------------------------------------------ the released path
def _previous_randn_tensor(shape, generator, device):
    """pipeline.randn_tensor as it was before generator lists: one generator, drawn on its device."""
    rand_device = generator.device if generator is not None else device
    return torch.randn(shape, generator=generator, device=rand_device, dtype=torch.float32).to(device)


def _previous_apply_free_init(self, latents, it, num_inference_steps, generator):
    """pipeline._apply_free_init as it was before the filter and fast-sampling options (DDIM branch)."""
    from animate3d_b200.pipeline import _butterworth_lpf
    if it == 0:
        self._free_init_initial_noise = latents.detach().clone()
    else:
        order, ds, dt = self._fi
        a = float(self.scheduler.alphas_cumprod[self.scheduler.num_train_timesteps - 1])
        z_T = math.sqrt(a) * latents + math.sqrt(1 - a) * self._free_init_initial_noise
        z_rand = torch.randn(latents.shape, generator=generator, device=latents.device, dtype=torch.float32)
        lpf = _butterworth_lpf(latents.shape, order, ds, dt, latents.device)
        dims = (-3, -2, -1)
        zf = torch.fft.fftshift(torch.fft.fftn(z_T, dim=dims), dim=dims)
        rf = torch.fft.fftshift(torch.fft.fftn(z_rand, dim=dims), dim=dims)
        latents = torch.fft.ifftn(torch.fft.ifftshift(zf * lpf + rf * (1 - lpf), dim=dims), dim=dims).real.contiguous()
    self.scheduler.set_timesteps(num_inference_steps)
    return latents, self.scheduler.timesteps


@pytest.mark.parametrize("generator", ["none", "cuda"])
def test_released_configuration_is_unchanged(setup, monkeypatch, generator):
    """DDIM 25 steps, CFG 7.5, three butterworth FreeInit iterations (inference.py:243-245): with the global seed (as
    inference.py seeds it) or one CUDA generator, the latents equal those of the previous code path bit for bit."""
    from animate3d_b200 import pipeline as P
    from animate3d_b200.scheduler import DDIMScheduler
    pipe, cond = setup

    def run():
        torch.manual_seed(7)
        g = torch.Generator(device="cuda").manual_seed(7) if generator == "cuda" else None
        pipe.scheduler = DDIMScheduler()
        pipe.enable_free_init(num_iters=3, method="butterworth", use_fast_sampling=False)
        try:
            return pipe(num_frames=NF, height=256, width=256, num_inference_steps=25, guidance_scale=7.5,
                        num_videos_per_prompt=NV, generator=g, prompt_embeds=cond["pos"],
                        negative_prompt_embeds=cond["neg"], ip_adapter_image_embeds=cond["image"], output_type="latent",
                        first_frame_latents=cond["first"]).frames.clone()
        finally:
            pipe.disable_free_init()
    now = run()
    with monkeypatch.context() as m:
        m.setattr(P, "randn_tensor", _previous_randn_tensor)
        m.setattr(P.AnimateDiffMVI2VPipeline, "_apply_free_init", _previous_apply_free_init)
        before = run()
    assert torch.isfinite(now).all()
    assert torch.equal(now, before)
