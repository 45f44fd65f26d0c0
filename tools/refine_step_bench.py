"""ms per 4D-SDS refine step, eager versus replayed from a CUDA graph (animate3d_b200/capture.py) with the UNet, the CLIP
tower and the VAE recorded inside the step, measured in the same process in alternating blocks, with CUDA events and the
wall clock.

    python -m tools.refine_step_bench [--steps 200] [--block 20] [--out result.json]

Workload (refine_frame_16.yaml; systems/animate3d.py:120-244 with guidance):
  * 50 000 gaussians with the deformation field;
  * reconstruction batch: 4 views x frames 1-15 = 60 cameras at 1024^2, rgb / mask MSE against fixed targets (closed over
    by the step body, not copied in);
  * random-camera batch: 4 views x 16 frames = 64 cameras at 256^2, a fresh seeded `tools.splat_bench.cameras(seed=step)`
    per step, its camera rows computed outside the graph;
  * SDS: CLIP image tower (ViT-H/14) on frame 0 of each view, VAE encoder forward and backward on the 64 renders, one CFG
    UNet evaluation over 2 x 4 views x 16 frames, all random-init;
  * ARAP from the random-camera render's means3D[:15] (radius 0.01, K 3, 512 samples); fused Adam.
Reported: median block and block range in ms/step, overflow and pointer recaptures of the replayed steps, the peak
`max_memory_reserved` of the eager phase (before any capture) and of the replay blocks, the card name and power limit.
At this size the graph pool and an eager step's working set do not fit in 80 GB together, so each eager block runs after
`StepGraphs.release()` and each replay block after one untimed capture (those captures are not counted as recaptures)."""
from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np
import torch
import torch.nn.functional as F

N_VIEW, N_FRAME, REC, RND = 4, 16, 1024, 256
VIT_H = dict(hidden_size=1280, intermediate_size=5120, num_attention_heads=16, num_hidden_layers=32, image_size=224,
             patch_size=14, projection_dim=1024, layer_norm_eps=1e-5, hidden_act="gelu")


class Refine:
    def __init__(self, gaussians: int = 50000):
        from animate3d_b200 import arap as AP
        from animate3d_b200.clip import CLIPImageProcessor, CLIPVisionModelWithProjection, IPAdapterImageProcessor
        from animate3d_b200.guidance import AnimateMVDiffusionGuidance, PrecomputedPromptUtils
        from animate3d_b200.renderer import camera_rows, make_renderer, timestamp_layout
        from animate3d_b200.unet import MVUNetMotionModel
        from animate3d_b200.unet_config import UNetConfig
        from animate3d_b200.vae import AutoencoderKL
        from animate3d_b200.weights import random_state_dict
        from oracle import clip_oracle as CO
        from oracle import vae_oracle as VO
        from tools.splat_bench import cameras, synthetic_model
        cfg = UNetConfig(num_views=N_VIEW, num_frames=N_FRAME)
        unet = MVUNetMotionModel(cfg)
        unet.load_state_dict(random_state_dict(cfg, seed=0))
        vae = AutoencoderKL()
        vae.load_state_dict(VO.make_state_dict(VO.VAEConfig(), 0))
        enc = CLIPVisionModelWithProjection(VIT_H, "cuda").load_state_dict(CO.random_state_dict(VIT_H, 0))
        self.guide = AnimateMVDiffusionGuidance({"n_view": N_VIEW, "n_frame": N_FRAME, "guidance_scale": 5.0,
                                                 "recon_std_rescale": 0.5, "min_step_percent": 0.02, "max_step_percent": 0.98},
                                                unet=unet, vae=vae,
                                                ip_image_processor=IPAdapterImageProcessor(CLIPImageProcessor("cuda"), enc))
        self.model = synthetic_model(gaussians, seed=0)
        self.rend = make_renderer(self.model).train()
        params = [p for p in self.model.parameters() if p.requires_grad]
        self.opt = torch.optim.Adam([{"params": params, "lr": torch.tensor(1e-3, device="cuda")}], eps=1e-15, fused=True,
                                    capturable=True)
        c2w, fovy, ts = cameras(n_views=N_VIEW, n_frames=N_FRAME, seed=1000)
        idx = [v * N_FRAME + f for v in range(N_VIEW) for f in range(1, N_FRAME)]
        rec_rows, rec_ts = camera_rows(c2w[idx], fovy[idx]), ts[idx]
        rec_layout = timestamp_layout(ts.cpu()[idx].numpy())
        layout = timestamp_layout(ts.cpu().numpy())
        g = torch.Generator(device="cuda").manual_seed(1)
        mask = (torch.rand(len(idx), REC, REC, 1, device="cuda", generator=g) > 0.3).float()
        gt = torch.rand(len(idx), REC, REC, 3, device="cuda", generator=g) * mask + 0.5 * (1 - mask)
        pu = PrecomputedPromptUtils(torch.randn(77, 768, device="cuda", generator=g), torch.randn(77, 768, device="cuda", generator=g))
        z = torch.zeros(N_VIEW * N_FRAME, device="cuda")
        guide, rend, model = self.guide, self.rend, self.model

        def body(inp):
            rec = rend.batch_forward({"camera_rows": rec_rows, "timestamps": rec_ts, "timestamp_layout": rec_layout,
                                      "width": REC, "height": REC, "do_guidance": True, "do_reconstruction": True})
            loss = 100.0 * F.mse_loss(gt, rec["comp_rgb"]) + 100.0 * F.mse_loss(mask, rec["comp_mask"])
            out = rend.batch_forward({"camera_rows": inp["rows"], "timestamps": ts, "timestamp_layout": layout, "width": RND,
                                      "height": RND, "do_guidance": True, "do_reconstruction": True})
            loss = loss + 0.1 * guide(out["comp_rgb"], pu, z, z, z, inp["c2w"])["loss_sds"]
            nodes = torch.stack([model._xyz] + out["means3D"][:15])
            ii, jj, nn, _ = AP.cal_connectivity_from_points(nodes[:1], radius=0.01, K=3)
            loss = loss + 12.0 * AP.cal_arap_error(nodes, ii, jj, nn, K=3, sample_num=512)
            loss.backward()
        self.body = body
        self.step_no = 0

    def inputs(self):
        """A fresh seeded random-camera batch; its rows are computed here, outside the graph."""
        from animate3d_b200.renderer import camera_rows
        from tools.splat_bench import cameras
        self.step_no += 1
        c2w, fovy, _ = cameras(n_views=N_VIEW, n_frames=N_FRAME, seed=self.step_no)
        return {"rows": camera_rows(c2w, fovy), "c2w": c2w}


def _block(run, n):
    """n steps; (CUDA-event ms, wall ms) per step and the peak reserved bytes.  The wall clock ends on a device synchronise."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    e0.record()
    for _ in range(n):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, (time.perf_counter() - t0) * 1e3 / n, torch.cuda.max_memory_reserved()


def measure(steps: int, block: int) -> dict:
    from animate3d_b200.capture import StepGraphs
    r = Refine()
    graphs = StepGraphs(r.body, r.opt)
    eager = lambda: graphs.eager(r.inputs())
    replay = lambda: graphs.step("refine", r.inputs())
    out = {"workload": "refine step: 50k gaussians, 60 x 1024^2 recon + 64 x 256^2 random cameras, CLIP ViT-H/14, VAE "
                       "encoder fwd+bwd (64 x 256^2), CFG UNet 2 x 4 views x 16 frames, ARAP 512 samples, fused Adam"}
    for _ in range(2):                                    # eager warm-up (first calls pack weights and capture inner graphs)
        eager()
    out["eager_peak_reserved_gib_before_capture"] = _block(eager, 2)[2] / 2**30
    graphs.step("refine", r.inputs())                     # eager first step of the layout
    graphs.step("refine", r.inputs())                     # capture + first replay
    rec0 = (graphs.recaptures, graphs.pointer_recaptures)
    rec = {"eager": [], "graph": []}
    for _ in range(max(1, steps // block)):
        # the graph pool (about the step's working set) and an eager step's working set do not both fit in 80 GB at this
        # size: the pool is released for the eager block and the step captured again, untimed, before the replay block
        graphs.release()
        rec["eager"].append(_block(eager, block))
        graphs.step("refine", r.inputs())
        rec["graph"].append(_block(replay, block))
    out.update({"steps_each": block * len(rec["eager"]), "replayed_steps": block * len(rec["graph"]),
                "overflow_recaptures": graphs.recaptures - rec0[0], "pointer_recaptures": graphs.pointer_recaptures - rec0[1],
                "recaptures_during_first_replay": list(rec0)})
    for k, v in rec.items():
        ev, wall, peak = np.array(v).T
        out[f"{k}_ms_event"] = float(np.median(ev))
        out[f"{k}_ms_event_range"] = [float(ev.min()), float(ev.max())]
        out[f"{k}_ms_wall"] = float(np.median(wall))
        out[f"{k}_ms_wall_range"] = [float(wall.min()), float(wall.max())]
        out[f"{k}_peak_reserved_gib"] = float(peak.max()) / 2**30
    out["speedup_wall"] = out["eager_ms_wall"] / out["graph_ms_wall"]
    out["blocks"] = {k: [[float(x) for x in b] for b in v] for k, v in rec.items()}    # (event ms, wall ms, peak bytes)
    return out


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--block", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("refine_step_bench needs a CUDA device: there is nothing to measure without one")
    np.random.seed(0)
    torch.manual_seed(0)
    res = {"card": card(), "result": measure(a.steps, a.block)}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
