"""ms per optimisation step of the motion-reconstruction and mesh-animation stages, eager versus replayed from a CUDA graph
(animate3d_b200/capture.py), measured in the same process in alternating blocks, with CUDA events and the wall clock.

    python -m tools.recon_step_bench [--steps 200] [--block 20] [--out result.json]

Configs (the two stages that take 1 600 of the workflow's 1 800 steps):
  * recon: motion_recon_frame_16.yaml at start_index 14 -- 50 000 gaussians, 4 views x 15 frames = 60 cameras at 256^2,
    use_global_trans, ARAP K = 3 on 512 sampled nodes;
  * mesh:  mesh_animation_frame_16.yaml ("light" strategy: 2 frames x 4 views) on a 163 842-vertex icosphere, mesh-edge ARAP
    with a fresh neighbour draw per step.
Both use fused Adam with the config's learning rates.  The card name and power limit are printed with the numbers."""
from __future__ import annotations

import argparse
import json
import random
import subprocess
import time

import numpy as np
import torch
import torch.nn.functional as F

N_VIEW, N_FRAME, RES = 4, 16, 256


def icosphere(level: int):
    """Vertices [10 * 4^level + 2, 3] and faces of a subdivided icosahedron on the unit sphere."""
    t = (1 + 5 ** 0.5) / 2
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
                  [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
                  [8, 6, 7], [9, 8, 1]], np.int64)
    for _ in range(level):
        e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
        uniq, inv = np.unique(e, axis=0, return_inverse=True)
        mid = len(v) + inv.reshape(3, -1)
        v = np.concatenate([v, (v[uniq[:, 0]] + v[uniq[:, 1]]) / 2])
        a, b, c = f[:, 0], f[:, 1], f[:, 2]
        ab, bc, ca = mid
        f = np.concatenate([np.stack([a, ab, ca], 1), np.stack([b, bc, ab], 1), np.stack([c, ca, bc], 1), np.stack([ab, bc, ca], 1)])
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32), f


def _model(xyz: torch.Tensor):
    from animate3d_b200.gaussian4d import Gaussian4DModel
    from oracle import raster_oracle as R
    _, s, q, o, sh = R.synthetic_scene(xyz.shape[0], 5)
    return Gaussian4DModel(xyz, torch.log(s), q, o, sh[:, 0], use_global_trans=True)


def _optimizer(model):
    lr = lambda v: torch.tensor(v, device="cuda")
    groups = [{"params": [p for pl in model.grids for p in pl], "lr": lr(0.01)},
              {"params": [p for n in ("delta_xyz_network", "delta_rot_network", "delta_scaling_network")
                          for p in getattr(model, n)], "lr": lr(1e-4)},
              {"params": [p for n in ("global_rot_network", "global_trans_network") for p in getattr(model, n)], "lr": lr(1e-3)}]
    return torch.optim.Adam(groups, eps=1e-15, fused=True, capturable=True)


class Stage:
    """The step body of systems/animate3d.py:120-244 (no guidance) for one config."""

    def __init__(self, mode: str):
        from animate3d_b200 import arap as AP
        from animate3d_b200.mesh import MeshGraph, edge_list
        from animate3d_b200.renderer import camera_rows, make_renderer, timestamp_layout
        from oracle import raster_oracle as R
        from tools.splat_bench import cameras
        self.mode = mode
        if mode == "recon":
            xyz = R.synthetic_scene(50000, 5)[0]
            self.graph, self.lam = None, 12.0
            self.frames = lambda: list(range(1, 16))                           # start_index 14, "normal"
        else:
            verts, faces = icosphere(7)
            xyz = torch.from_numpy(verts) * 0.6
            self.graph = MeshGraph.from_faces(torch.from_numpy(faces).cuda(), verts.shape[0])
            self.graph.set_sample_state(random.getrandbits(62))
            self.lam = 4.0
            self.frames = lambda: [random.randint(1, 14), 15]                  # "light": animate3d.py:144-150
        self.model = _model(xyz)
        self.rend = make_renderer(self.model).train()
        self.opt = _optimizer(self.model)
        c2w, fovy, ts = cameras(n_views=N_VIEW, n_frames=N_FRAME)
        self.rows, self.ts = camera_rows(c2w, fovy), ts
        g = torch.Generator(device="cuda").manual_seed(1)
        n = N_VIEW * N_FRAME
        self.mask = (torch.rand(n, RES, RES, 1, device="cuda", generator=g) > 0.3).float()
        self.rgb = torch.rand(n, RES, RES, 3, device="cuda", generator=g)
        nf = len(self.frames())
        idx = [v * N_FRAME + f for v in range(N_VIEW) for f in self.frames()]
        self.layout = timestamp_layout(self.ts.cpu()[idx].numpy())
        self.key = (mode, nf, self.layout)

        def step_fn(inp):
            batch = {"camera_rows": inp["rows"], "timestamps": inp["ts"], "timestamp_layout": self.layout, "width": RES,
                     "height": RES, "do_guidance": False, "do_reconstruction": True}
            out = self.rend.batch_forward(batch)
            gt = inp["rgb"] * inp["mask"] + 0.5 * (1 - inp["mask"])
            loss = 100.0 * F.mse_loss(gt, out["comp_rgb"]) + 100.0 * F.mse_loss(inp["mask"], out["comp_mask"])
            nodes = torch.stack([self.model._xyz] + out["means3D"][:nf])
            if self.graph is not None:
                ii, jj, nn = edge_list(self.graph.sample(3))
            else:
                ii, jj, nn, _ = AP.cal_connectivity_from_points(nodes[:1], radius=0.01, K=3)
            loss = loss + self.lam * AP.cal_arap_error(nodes, ii, jj, nn, K=3, sample_num=512)
            loss.backward()
        self.step_fn = step_fn

    def inputs(self):
        idx = [v * N_FRAME + f for v in range(N_VIEW) for f in self.frames()]
        return {"ts": self.ts[idx], "rows": self.rows[idx], "rgb": self.rgb[idx], "mask": self.mask[idx]}


def _block(run, n):
    """n steps; (CUDA-event ms, wall ms) per step.  The wall clock ends on a device synchronise."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    for _ in range(n):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, (time.perf_counter() - t0) * 1e3 / n


def measure(mode: str, steps: int, block: int) -> dict:
    from animate3d_b200.capture import StepGraphs
    st = Stage(mode)
    graphs = StepGraphs(st.step_fn, st.opt)
    for _ in range(3):                                   # eager warm-up, capture, first replays
        graphs.step(st.key, st.inputs())
    eager = lambda: graphs.eager(st.inputs())
    replay = lambda: graphs.step(st.key, st.inputs())
    for _ in range(3):
        eager()
    rec = {"eager": [], "graph": []}
    for _ in range(max(1, steps // block)):
        rec["eager"].append(_block(eager, block))
        rec["graph"].append(_block(replay, block))
    out = {"mode": mode, "steps_each": block * len(rec["eager"]), "recaptures": graphs.recaptures}
    for k, v in rec.items():
        ev, wall = np.array(v).T
        out[f"{k}_ms_event"] = float(np.median(ev))
        out[f"{k}_ms_wall"] = float(np.median(wall))
        out[f"{k}_ms_wall_spread"] = [float(wall.min()), float(wall.max())]
    out["speedup_wall"] = out["eager_ms_wall"] / out["graph_ms_wall"]
    return out


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--block", type=int, default=20)
    ap.add_argument("--modes", default="recon,mesh")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("recon_step_bench needs a CUDA device: there is nothing to measure without one")
    random.seed(0)
    torch.manual_seed(0)
    res = {"card": card(), "results": [measure(m, a.steps, a.block) for m in a.modes.split(",")]}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
