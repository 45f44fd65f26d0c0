"""Mesh animation timings on the GPU (one JSON line):

* conversion: vertex graph + per-vertex statistics + corner-colour sampling of a subdivided icosphere (level 8:
  1 310 720 faces, 655 362 vertices) with a 1024 x 1024 texture, i.e. the GPU part of `mesh.mesh_to_gaussians`;
* one mesh-mode ARAP step (systems/animate3d.py:222-244): sample K = 3 neighbours, `cal_arap_error` over 16 deformed
  frames plus the static frame with sample_num 512, and its backward, on an icosphere of level 7 (163 842 vertices).

Both are timed with CUDA events after warm-up; the card's name and power limit are read in the same run.

    python tools/mesh_bench.py [--reps 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from animate3d_b200 import arap  # noqa: E402
from animate3d_b200 import mesh as MS  # noqa: E402


def icosphere(level: int):
    t = (1 + 5 ** 0.5) / 2
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
                  [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
                  [8, 6, 7], [9, 8, 1]], np.int64)
    for _ in range(level):
        e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
        uniq, inv = np.unique(e[:, 0] * len(v) + e[:, 1], return_inverse=True)
        mid = len(v) + inv.reshape(3, -1).T                                   # midpoints of edges (01, 12, 20)
        a, b = uniq // len(v), uniq % len(v)
        v = np.concatenate([v, (v[a] + v[b]) / 2])
        f = np.concatenate([np.stack([f[:, 0], mid[:, 0], mid[:, 2]], 1), np.stack([f[:, 1], mid[:, 1], mid[:, 0]], 1),
                            np.stack([f[:, 2], mid[:, 2], mid[:, 1]], 1), mid])
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return v.astype(np.float32), f


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    rng = np.random.default_rng(0)
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": card}

    v, f = icosphere(8)
    verts, faces = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    tex = torch.rand(1024, 1024, 3, device="cuda")
    uvs = torch.from_numpy(rng.random((v.shape[0], 2), dtype=np.float32)).cuda()

    def convert():
        g = MS.MeshGraph.from_faces(faces, v.shape[0])
        crgb = MS.corner_colours(tex, uvs, faces)
        MS.vertex_stats(verts, g, faces, crgb)
    out["convert_faces"], out["convert_verts"] = int(f.shape[0]), int(v.shape[0])
    out["convert_ms"] = timed(convert, max(1, args.reps // 4))

    v7, f7 = icosphere(7)
    graph = MS.MeshGraph.from_faces(torch.from_numpy(f7).cuda(), v7.shape[0])
    base = torch.from_numpy(v7).cuda()
    frames = torch.stack([base] + [base + 0.01 * t * torch.randn_like(base) for t in range(1, 17)])
    sample = torch.from_numpy(rng.choice(v7.shape[0], 512)).cuda()

    def step():
        nodes = frames.clone().requires_grad_(True)
        ii, jj, nn = MS.edge_list(graph.sample(3))
        arap.cal_arap_error(nodes, ii, jj, nn, K=3, sample_num=512, sample_idx=sample).backward()
    out["arap_verts"], out["arap_frames"] = int(v7.shape[0]), int(frames.shape[0])
    out["arap_step_ms"] = timed(step, args.reps)
    out["sample_k3_ms"] = timed(lambda: graph.sample(3), args.reps * 5)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
