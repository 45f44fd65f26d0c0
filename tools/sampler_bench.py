"""Sampling time per scheduler: one full latent-output `__call__` at 4 views x 16 frames x 32^2 latents with CFG, random
weights and FreeInit off, for DDIM 25 steps, DPM-Solver++ 25 and 15 steps, Euler 25 steps, PNDM 25 steps with and without
its PRK steps and LMS 25 steps, then DDIM 25 steps with three butterworth FreeInit iterations, with and without
coarse-to-fine sampling (wall clock ending on a device synchronise, after one untimed warm-up call of each; each leg also
reports how many times the last call ran the UNet); then the step kernels alone, a3d_sampler_step (DPM-Solver++
order 2 and Euler-ancestral) and a3d_multistep_step (four-term PLMS and LMS, and a PRK sub-step) against a3d_ddim_step,
timed with CUDA events over many launches.  Prints one JSON line with the card's name and power limit.
`python tools/sampler_bench.py [--reps 3] [--out DIR]`."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from animate3d_b200 import ops                                                     # noqa: E402
from animate3d_b200 import scheduler as S                                          # noqa: E402
from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline                       # noqa: E402
from animate3d_b200.unet import MVUNetMotionModel                                  # noqa: E402
from animate3d_b200.unet_config import UNetConfig                                  # noqa: E402
from animate3d_b200.weights import random_state_dict                               # noqa: E402

NV, NF, LAT = 4, 16, 32


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def time_calls(pipe, sched, steps, reps, cond, free_init=None):
    pipe.scheduler = sched
    if free_init is not None:
        pipe.enable_free_init(**free_init)
    forward, unet_calls = pipe.unet.forward, [0]

    def counted(*a, **k):
        unet_calls[0] += 1
        return forward(*a, **k)
    pipe.unet.forward = counted

    def call(seed):
        return pipe(num_frames=NF, height=8 * LAT, width=8 * LAT, num_inference_steps=steps, guidance_scale=7.5,
                    num_videos_per_prompt=NV, generator=torch.Generator().manual_seed(seed), output_type="latent", **cond).frames
    call(0)
    torch.cuda.synchronize()
    out = []
    for r in range(reps):
        unet_calls[0] = 0
        t0 = time.perf_counter()
        call(r + 1)
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    del pipe.unet.forward
    pipe.disable_free_init()
    return out, unet_calls[0]


def time_kernel(fn, iters=2000):
    for _ in range(50):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters                                      # microseconds per launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cfg = UNetConfig()
    model = MVUNetMotionModel(cfg)
    model.load_state_dict(random_state_dict(cfg, 0, "cuda"))
    pipe = AnimateDiffMVI2VPipeline(unet=model)
    g = torch.Generator(device="cuda").manual_seed(1)
    cond = dict(prompt_embeds=torch.randn(NV, 77, 768, device="cuda", generator=g),
                negative_prompt_embeds=torch.randn(NV, 77, 768, device="cuda", generator=g),
                ip_adapter_image_embeds=torch.randn(NV, 1024, device="cuda", generator=g),
                first_frame_latents=torch.randn(NV, 4, 1, LAT, LAT, device="cuda", generator=g))
    ddim_cfg = S.DDIMScheduler().config
    runs = [("DDIM", 25, lambda: S.DDIMScheduler()),
            ("DPM-Solver++", 25, lambda: S.DPMSolverMultistepScheduler.from_config(ddim_cfg)),
            ("DPM-Solver++", 15, lambda: S.DPMSolverMultistepScheduler.from_config(ddim_cfg)),
            ("Euler", 25, lambda: S.EulerDiscreteScheduler.from_config(ddim_cfg)),
            ("PNDM (PLMS only)", 25, lambda: S.PNDMScheduler.from_config(ddim_cfg, skip_prk_steps=True)),
            ("PNDM (PRK + PLMS)", 25, lambda: S.PNDMScheduler.from_config(ddim_cfg)),
            ("LMS", 25, lambda: S.LMSDiscreteScheduler.from_config(ddim_cfg)),
            ("DDIM, FreeInit 3", 25, lambda: S.DDIMScheduler(), dict(num_iters=3)),
            ("DDIM, FreeInit 3, coarse-to-fine", 25, lambda: S.DDIMScheduler(), dict(num_iters=3, use_fast_sampling=True))]
    calls = []
    for name, steps, make, *free_init in runs:
        secs, unet_calls = time_calls(pipe, make(), steps, args.reps, cond, *free_init)
        med = sorted(secs)[len(secs) // 2]
        calls.append(dict(scheduler=name, steps=steps, unet_calls=unet_calls, seconds=[round(s, 3) for s in secs],
                          median_s=round(med, 3), ms_per_step=round(1e3 * med / steps, 1),
                          ms_per_unet_call=round(1e3 * med / unet_calls, 1)))
        print(json.dumps(calls[-1]), flush=True)

    # the step kernels alone, at the same latent size
    shape = (NV, 4, NF, LAT * LAT)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    lat, eps, first, z, h0, h1 = r(*shape), r(2 * NV, 4, NF, LAT * LAT), r(NV, 4, 1, LAT * LAT), r(*shape), r(*shape), r(*shape)
    ring, saved, acc = [r(*shape) for _ in range(S.RING)], r(*shape), r(*shape)
    dpm = S.DPMSolverMultistepScheduler.from_config(ddim_cfg)
    dpm.set_timesteps(25)
    eul = S.EulerAncestralDiscreteScheduler.from_config(ddim_cfg)
    eul.set_timesteps(25)
    s2, se = dpm._coefficients(10, 2), eul._update(10)
    dd = S.DDIMScheduler()
    dd.set_timesteps(25)
    a_t, a_p, dc, sd = dd.step_coefficients(561, 0.0)
    pndm = S.PNDMScheduler.from_config(ddim_cfg)
    pndm_steps = [pndm.next_step(t) for t in pndm.set_timesteps(25)]
    plms4, prk2 = pndm_steps[20], pndm_steps[1]
    lms = S.LMSDiscreteScheduler.from_config(ddim_cfg)
    lms_steps = [lms.next_step(t) for t in lms.set_timesteps(25)]
    lms4 = lms_steps[10]
    assert (plms4.terms, prk2.prk, lms4.terms) == (4, 2, 4)
    multistep = lambda s: (lambda: ops.multistep_step(lat, eps, first, NV, 4, NF, LAT * LAT, 1, 7.5, s, ring, saved, acc))
    kernels = {
        "a3d_ddim_step": time_kernel(lambda: ops.ddim_step(lat, eps, first, None, NV, 4, NF, LAT * LAT, 1, 7.5, a_t, a_p, dc, sd)),
        "a3d_sampler_step dpm++ order 2": time_kernel(lambda: ops.sampler_step(lat, eps, first, NV, 4, NF, LAT * LAT, 1, 7.5, s2,
                                                                                history_out=h0, history_in=h1)),
        "a3d_sampler_step euler ancestral": time_kernel(lambda: ops.sampler_step(lat, eps, first, NV, 4, NF, LAT * LAT, 1, 7.5,
                                                                                  se, noise=z)),
        "a3d_multistep_step plms 4 terms": time_kernel(multistep(plms4)),
        "a3d_multistep_step prk sub-step 2": time_kernel(multistep(prk2)),
        "a3d_multistep_step lms 4 terms": time_kernel(multistep(lms4)),
    }
    result = dict(card=card(), workload=f"{NV} views x {NF} frames x {LAT}^2 latents, CFG 7.5, random weights",
                  calls=calls, kernel_us={k: round(v, 2) for k, v in kernels.items()})
    print(json.dumps(result), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sampler_bench.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
