"""Test-view renders of the visualize configs (animate3d_b200/visualize.py) against the reference's per-camera test path.

    python -m tools.visualize_bench [--sets four_view,testset] [--out result.json]

Scene: BASELINE config 3 -- 50 000 synthetic gaussians with the deformation field and the global motion branch (non-zero
last layers, so every frame moves) -- rendered at 1024^2 for `four_view` (64 items) and `testset` (192 items).
Per set it reports:
  * engine: device time of `render_views` (CUDA events; the deformation, every chunk's RGBA8 render and its one sync),
    the D2H bytes (4 per pixel), PNG encode + write wall time per encoder thread count, and the wall time of `save_views`
    end to end (render, pinned copies and encoding overlapped);
  * per camera, as `test_step` does it (animate3d.py:427-463): one `batch_forward` per item, `.cpu()` of the float
    rgb + mask (16 B per pixel), numpy `* 255` / `astype(uint8)`, PIL save -- render + copy and PNG wall time.
The two paths' bytes are compared.  The card's name and power limit are printed with the numbers."""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch


def scene(P: int = 50000, seed: int = 5):
    from animate3d_b200.gaussian4d import Gaussian4DModel
    from oracle import raster_oracle as R
    xyz, s, q, o, sh = R.synthetic_scene(P, seed)
    model = Gaussian4DModel(xyz, torch.log(s), q, torch.logit(o), sh[:, 0], use_global_trans=True)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name in ("delta_xyz_network", "delta_rot_network", "delta_scaling_network", "global_rot_network", "global_trans_network"):
            net = getattr(model, name)
            net[1].copy_((torch.randn(net[1].shape, generator=g) * 0.05).cuda())
    return model


def _png_wall(rgba: np.ndarray, threads: int, folder: str) -> float:
    from PIL import Image
    t0 = time.perf_counter()
    with ThreadPoolExecutor(max_workers=threads) as pool:
        list(pool.map(lambda i: Image.fromarray(rgba[i]).save(os.path.join(folder, f"{i}.png")), range(len(rgba))))
    return time.perf_counter() - t0


def engine(model, views, threads_list, save_threads, tmp):
    from animate3d_b200 import visualize as V
    from animate3d_b200.rasterizer import RGBA8Renderer
    r = RGBA8Renderer()
    V.render_views(model, views, renderer=r)                       # warm-up: modules, workspace, pair capacity
    times = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        rgba = V.render_views(model, views, renderer=r)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    host = rgba.cpu().numpy()
    png = {}
    for t in threads_list:
        d = tempfile.mkdtemp(dir=tmp)
        png[t] = _png_wall(host, t, d)
        shutil.rmtree(d)
    d = tempfile.mkdtemp(dir=tmp)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    V.save_views(model, views, d, threads=save_threads, renderer=r)
    total = time.perf_counter() - t0
    shutil.rmtree(d)
    return rgba, {"render_ms_device": sorted(times)[1], "render_ms_all": times, "d2h_bytes": int(rgba.numel()),
                  "png_s_by_threads": png, "save_views_s": total, "save_views_threads": save_threads,
                  "overflow_rerenders": r.overflows}


def per_camera(model, views, tmp):
    from PIL import Image

    from animate3d_b200.renderer import make_renderer
    ren = make_renderer(model, back_ground_color=views.background)
    d = tempfile.mkdtemp(dir=tmp)
    out = np.empty((len(views), views.height, views.width, 4), np.uint8)
    render_s = png_s = 0.0
    d2h = 0
    torch.cuda.synchronize()
    t_all = time.perf_counter()
    for i in range(len(views)):
        t0 = time.perf_counter()
        batch = {"c2w": views.c2w[i:i + 1].cuda(), "fovy": views.fovy[i:i + 1].cuda(), "height": views.height,
                 "width": views.width, "do_guidance": False, "do_reconstruction": True}
        if views.timestamps is not None:
            batch["timestamps"] = views.timestamps[i:i + 1].cuda()
        o = ren.batch_forward(batch)
        rgba = torch.cat([o["comp_rgb"], o["comp_mask"]], dim=-1)[0].detach().cpu().numpy()
        d2h += rgba.nbytes
        t1 = time.perf_counter()
        out[i] = (rgba * 255).astype(np.uint8)
        Image.fromarray(out[i]).save(os.path.join(d, f"{i}.png"))
        t2 = time.perf_counter()
        render_s += t1 - t0
        png_s += t2 - t1
    total = time.perf_counter() - t_all
    shutil.rmtree(d)
    return out, {"render_and_copy_s": render_s, "png_s": png_s, "total_s": total, "d2h_bytes": d2h}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--sets", default="four_view,testset")
    p.add_argument("--threads", default="1,4,8,16", help="PNG encoder thread counts timed on pre-rendered images")
    p.add_argument("--save_threads", type=int, default=8, help="encoder threads of the timed save_views (its default)")
    p.add_argument("--out", default=None)
    a = p.parse_args()
    from animate3d_b200 import visualize as V
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    res = {"card": card[0] if card else "unknown", "cpus": os.cpu_count(), "sets": {}}
    model = scene()
    threads = [int(t) for t in a.threads.split(",")]
    tmp = tempfile.mkdtemp()
    try:
        for name in a.sets.split(","):
            views = V.camera_set(name)
            with torch.no_grad():
                mine, eng = engine(model, views, threads, a.save_threads, tmp)
                ref, pc = per_camera(model, views, tmp)
            res["sets"][name] = {"items": len(views), "resolution": [views.height, views.width], "engine": eng, "per_camera": pc,
                                 "bytes_identical": bool(np.array_equal(mine.cpu().numpy(), ref))}
            print(json.dumps({name: res["sets"][name]}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
