"""Test-view renders and the multi-view image loader: the engine's counterpart of threestudio's `launch.py --test` with the
visualize configs, and of the refine stage's data module.

* Camera sets (`camera_set`): `four_view` and `testset` restate `HybridRandomCameraTestDataset`
  (custom/threestudio-animate3d/data/uncond_hybrid.py:560-700) with the values of visualize_four_view_frame_16.yaml /
  visualize_testset_frame_16.yaml; `static` restates the test split of `RandomCameraDataset` (threestudio/data/uncond.py:
  346-430) with the values of visualize_four_view_static.yaml.  Item i of a set is one (camera, timestamp) test batch.
* `render_views` renders a set through the forward-only RGBA8 rasterizer entry point (`a3d_raster_forward_rgba8`): the
  bytes the reference's `test_step` saves (systems/animate3d.py:427-463), without autograd, float planes or a host copy per
  camera.  `save_views` writes them in the reference's folder layout with PIL, PNG encoding in a thread pool overlapped with
  the next chunk's render.
* `load_multiview_images` restates `SimpleMultiImageDataBase` (custom/threestudio-animate3d/data/simple_multi_image.py:
  91-226, 271-289): the reconstruction / refine targets and their cameras.

Command line: python -m animate3d_b200.visualize --ply G.ply [--state deform.pt] --option four_view|testset|static --out DIR
"""
from __future__ import annotations

import argparse
import math
import os
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass
from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from .rasterizer import PairBudgetExceeded, RGBA8Renderer
from .renderer import camera_rows, timestamp_layout

OPTIONS = ("four_view", "testset", "static")


@dataclass
class ViewSet:
    """One test set: per item (the reference's test batch `index`) a camera, a timestamp and an output file."""
    option: str
    c2w: torch.Tensor                   # [N, 4, 4] float32
    fovy: torch.Tensor                  # [N] float32, radians
    timestamps: Optional[torch.Tensor]  # [N] float32, or None for the static gaussians
    height: int
    width: int
    background: Tuple[float, float, float]
    files: List[str]                    # path of item i relative to the output directory

    def __len__(self) -> int:
        return len(self.files)


def orbit_c2w(elevation_deg: torch.Tensor, azimuth_deg: torch.Tensor, distance: float) -> torch.Tensor:
    """[B, 4, 4] camera-to-world of cameras on a sphere looking at the origin, +z up, in float32 and in the operation order
    of uncond_hybrid.py:581-623 (= uncond.py:367-409, simple_multi_image.py:96-124)."""
    camera_distances = torch.full_like(elevation_deg, distance)
    elevation = elevation_deg * math.pi / 180
    azimuth = azimuth_deg * math.pi / 180
    camera_positions = torch.stack([camera_distances * torch.cos(elevation) * torch.cos(azimuth),
                                    camera_distances * torch.cos(elevation) * torch.sin(azimuth),
                                    camera_distances * torch.sin(elevation)], dim=-1)
    center = torch.zeros_like(camera_positions)
    up = torch.as_tensor([0, 0, 1], dtype=torch.float32)[None, :].expand_as(camera_positions)
    lookat = F.normalize(center - camera_positions, dim=-1)
    right = F.normalize(torch.linalg.cross(lookat, up, dim=-1), dim=-1)
    up = F.normalize(torch.linalg.cross(right, lookat, dim=-1), dim=-1)
    c2w3x4 = torch.cat([torch.stack([right, up, -lookat], dim=-1), camera_positions[:, :, None]], dim=-1)
    c2w = torch.cat([c2w3x4, torch.zeros_like(c2w3x4[:, :1])], dim=1)
    c2w[:, 3, 3] = 1.0
    return c2w


def _hybrid_test_set(option: str, elevation_deg: Sequence[float], azimuth_deg: Sequence[Sequence[float]], height: int,
                     width: int, total_frame: int, distance: float, fovy_deg: float) -> ViewSet:
    # uncond_hybrid.py:577-579: the azimuth rows flattened against each elevation repeated once per azimuth of a row
    azi = torch.tensor(azimuth_deg).reshape(-1)
    elv = torch.tensor(elevation_deg).repeat_interleave(len(azimuth_deg[0]))
    c2w = orbit_c2w(elv, azi, distance)
    fovy = torch.full_like(elv, fovy_deg) * math.pi / 180
    ts = torch.linspace(-1, 1, steps=total_frame)                            # 659
    n = len(azi) * total_frame                                               # __len__, 669-670
    cam = torch.arange(n) // total_frame                                     # __getitem__, 672-695
    if option == "four_view":                                                # animate3d.py:454-456
        files = [f"images/{i}.png" for i in range(n)]
    else:                                                                    # animate3d.py:448-452 (4 azimuths hard-coded)
        files = [f"images/elv_{i // (total_frame * 4)}_azi_{(i // total_frame) % 4}/{i % total_frame}.png" for i in range(n)]
    return ViewSet(option, c2w[cam].contiguous(), fovy[cam].contiguous(), ts[torch.arange(n) % total_frame].contiguous(),
                   height, width, (0.5, 0.5, 0.5), files)


def four_view_cameras(height: int = 1024, width: int = 1024, total_frame: int = 16) -> ViewSet:
    """visualize_four_view_frame_16.yaml: elevation 15, azimuths 0/90/180/270, distance 3, fovy 40, 64 items
    (camera i // 16, timestamp linspace(-1, 1, 16)[i % 16]) saved as images/{i}.png."""
    return _hybrid_test_set("four_view", [15.0], [[0.0, 90.0, 180.0, 270.0]], height, width, total_frame, 3.0, 40.0)


def testset_cameras(height: int = 1024, width: int = 1024, total_frame: int = 16) -> ViewSet:
    """visualize_testset_frame_16.yaml: elevations 15 / 0 / 30, each with its own row of 4 azimuths, 192 items saved as
    images/elv_{i // 64}_azi_{(i // 16) % 4}/{i % 16}.png."""
    return _hybrid_test_set("testset", [15.0, 0.0, 30.0], [[0.0, 90.0, 180.0, 270.0], [30.0, 120.0, 210.0, 300.0],
                                                           [-45.0, 45.0, 135.0, 225.0]], height, width, total_frame, 3.0, 40.0)


def static_cameras(height: int = 512, width: int = 512, n_views: int = 5) -> ViewSet:
    """visualize_four_view_static.yaml through uncond.py:363: azimuths linspace(0, 360, 5), so view 4 repeats view 0 (kept:
    inference.py:274 reads views 0-3), elevation 15, distance 3, fovy 40, no timestamps, background 0.498; images/{i}.png."""
    azi = torch.linspace(0, 360.0, n_views)
    elv = torch.full_like(azi, 15.0)
    fovy = torch.full_like(elv, 40.0) * math.pi / 180
    return ViewSet("static", orbit_c2w(elv, azi, 3.0), fovy, None, height, width, (0.498, 0.498, 0.498),
                   [f"images/{i}.png" for i in range(n_views)])


def camera_set(option: str, height: Optional[int] = None, width: Optional[int] = None) -> ViewSet:
    """The views of one visualize config; height / width default to the config's (1024² for the 4D sets, 512² static)."""
    if option not in OPTIONS:
        raise ValueError(f"option must be one of {OPTIONS}, got {option!r}")
    make = {"four_view": four_view_cameras, "testset": testset_cameras, "static": static_cameras}[option]
    default = 512 if option == "static" else 1024
    return make(height=height or default, width=width or default)


# ---------------------------------------------------------------------------------------------------------------- render

def _render_chunks(geometry, views: ViewSet, deform_scale: bool, first_frame_trainable: bool, max_pixels: int,
                   renderer: RGBA8Renderer, out_for) -> Iterator[Tuple[int, torch.Tensor]]:
    """Yields (first item, rgba [n, H, W, 4] on the device) over chunks of at most max_pixels pixels (and the renderer's
    pair budget: a chunk that exceeds it is split in halves).  out_for(first, n) gives the tensor a chunk renders into."""
    pc = geometry
    dev = pc._xyz.device
    H, W, N = views.height, views.width, len(views)
    rows = camera_rows(views.c2w.to(dev), views.fovy.to(dev))
    opacity, shs = pc.get_opacity.contiguous(), pc.get_features.contiguous()
    if views.timestamps is None:
        static = (pc._xyz.contiguous(), torch.exp(pc._scaling).contiguous(),
                  F.normalize(pc._rotation, dim=-1).contiguous())
    else:
        # every distinct timestamp deformed once (diff_gaussian_rasterizer_advanced_4d.py:77-83, 119-135)
        uniq, inverse = torch.unique(views.timestamps.to(dev).float(), return_inverse=True)
        frames = pc.deform_frames(uniq, deform_scale=deform_scale, first_frame_trainable=first_frame_trainable)
    chunk = max(1, max_pixels // (H * W))
    i = 0
    while i < N:
        n = min(chunk, N - i)
        if views.timestamps is None:
            geo, per_cam = static, False
        else:
            idx = inverse[i:i + n]
            geo, per_cam = tuple(t[idx].contiguous() for t in frames), True
        try:
            rgba = renderer.render(rows[i:i + n], H, W, *geo, opacity, shs, None, int(pc.active_sh_degree), per_cam,
                                   views.background, out=out_for(i, n))
        except PairBudgetExceeded:
            chunk = max(1, n // 2)
            continue
        yield i, rgba
        i += n


@torch.no_grad()
def render_views(geometry, views: ViewSet, deform_scale: bool = False, first_frame_trainable: bool = False,
                 max_pixels: int = 1 << 24, renderer: Optional[RGBA8Renderer] = None) -> torch.Tensor:
    """RGBA8 renders [N, H, W, 4] (device) of every item of `views`: per pixel (clamp(C + T·bg, 0, 1), alpha) × 255
    truncated to uint8, byte for byte what `test_step` saves (animate3d.py:439-445).

    deform_scale: the reference renders its test views with `do_guidance = load_guidance` (animate3d.py:429-435), and every
    visualize config sets `load_guidance: false`, so its test renders use the static scales with the deformed means and
    rotations (diff_gaussian_rasterizer_advanced_4d.py:130-133).  False keeps that; True applies the scale deltas, as the
    refine stage's training renders do.  No autograd and no reconstruction-stage gradient gate: the gate changes no value."""
    renderer = renderer or RGBA8Renderer()
    out = torch.empty(len(views), views.height, views.width, 4, dtype=torch.uint8, device=geometry._xyz.device)
    for _ in _render_chunks(geometry, views, deform_scale, first_frame_trainable, max_pixels, renderer,
                            lambda i, n: out[i:i + n]):
        pass
    return out


def _write_png(path: str, rgba: np.ndarray) -> None:
    from PIL import Image
    Image.fromarray(rgba).save(path)          # animate3d.py:445, 463


@torch.no_grad()
def save_views(geometry, views: ViewSet, out_dir: str, threads: int = 8, deform_scale: bool = False,
               first_frame_trainable: bool = False, save_gaussian_trajectory: bool = False, max_pixels: int = 1 << 24,
               renderer: Optional[RGBA8Renderer] = None) -> List[str]:
    """Render `views` and write item i to out_dir/views.files[i] (the reference's `test_step` layout).  Each chunk is copied
    to pinned host memory on the render stream and PNG-encoded by `threads` workers (zlib releases the GIL) while the next
    chunk renders; at most two chunks are in flight.  save_gaussian_trajectory also writes mesh_trajectory/{i}.npy, the
    means of frame i (animate3d.py:465-471).  Returns the written image paths."""
    renderer = renderer or RGBA8Renderer()
    H, W = views.height, views.width
    dev = geometry._xyz.device
    paths = [os.path.join(out_dir, f) for f in views.files]
    for d in sorted({os.path.dirname(p) for p in paths}):
        os.makedirs(d, exist_ok=True)
    chunk_buf: Dict[int, torch.Tensor] = {}

    def device_chunk(i, n):      # one device buffer: a chunk's D2H copy is ordered before the next render on the stream
        if n not in chunk_buf:
            chunk_buf.clear()
            chunk_buf[n] = torch.empty(n, H, W, 4, dtype=torch.uint8, device=dev)
        return chunk_buf[n]

    def encode(ev, host, j, path):
        ev.synchronize()
        _write_png(path, host[j].numpy())

    inflight: List[list] = []
    with ThreadPoolExecutor(max_workers=max(1, threads)) as pool:
        for i, rgba in _render_chunks(geometry, views, deform_scale, first_frame_trainable, max_pixels, renderer, device_chunk):
            n = rgba.shape[0]
            host = torch.empty(n, H, W, 4, dtype=torch.uint8, pin_memory=True)
            host.copy_(rgba, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            inflight.append([pool.submit(encode, ev, host, j, paths[i + j]) for j in range(n)])
            if len(inflight) > 1:
                for f in inflight.pop(0):
                    f.result()
        for fs in inflight:
            for f in fs:
                f.result()
    if save_gaussian_trajectory and views.timestamps is not None:
        from .mesh import save_mesh_trajectory
        n_frame = int(torch.unique(views.timestamps).numel())
        save_mesh_trajectory(geometry, os.path.join(out_dir, "mesh_trajectory"), n_frame=n_frame,
                             first_frame_trainable=first_frame_trainable)
    return paths


# ---------------------------------------------------------------------------------------------------------------- load

def load_multiview_images(image_root: str, n_view: int = 4, total_frame: int = 16, height: int = 256, width: int = 256,
                          elevation_deg: float = 15.0, azimuth_deg: Sequence[float] = (0.0, 90.0, 180.0, 270.0),
                          camera_distance: float = 3.0, fovy_deg: float = 40.0, device="cuda") -> Dict:
    """`SimpleMultiImageDataBase` of the reconstruction / refine configs (simple_multi_image.py:91-226): every image of
    image_root sorted by int(name[:-4]) (view-major: item i is view i // total_frame at frame i % total_frame), read with
    cv2 IMREAD_UNCHANGED, BGRA -> RGBA, INTER_AREA-resized to (width, height), / 255 in float32; mask = alpha > 0.5.

    Returns the keys of `collate` (271-289) the gaussian renderer and the losses read -- rgb [N,H,W,3], mask [N,H,W,1] bool,
    c2w [N,4,4], fovy [N], timestamps [N,1], elevation, azimuth, camera_distances, camera_positions, light_positions,
    height, width, ref_depth (None) -- plus `camera_rows` and `timestamp_layout` for a captured step (INTEGRATION §3e).
    rays_o / rays_d / mvp_mtx are left out: the gaussian renderer never reads them."""
    import cv2
    n = n_view * total_frame
    names = sorted(os.listdir(image_root), key=lambda x: int(x[:-4]))
    if len(names) != n:
        raise ValueError(f"{image_root}: {len(names)} images, expected n_view * total_frame = {n}")
    rgbs, masks = [], []
    for name in names:
        img = cv2.imread(os.path.join(image_root, name), cv2.IMREAD_UNCHANGED)
        if img is None or img.ndim != 3 or img.shape[2] != 4:
            raise ValueError(f"{os.path.join(image_root, name)}: not a 4-channel image")
        rgba = cv2.cvtColor(img, cv2.COLOR_BGRA2RGBA)
        rgba = cv2.resize(rgba, (width, height), interpolation=cv2.INTER_AREA).astype(np.float32) / 255.0
        rgbs.append(rgba[..., :3])
        masks.append(rgba[..., 3:] > 0.5)
    # cameras, 91-131
    elevation = torch.FloatTensor([elevation_deg] * n)
    azimuth = (torch.FloatTensor(list(azimuth_deg)).unsqueeze(-1).repeat(1, total_frame).reshape(-1)
               if len(azimuth_deg) // n_view < total_frame else torch.FloatTensor(list(azimuth_deg)))
    if azimuth.numel() != n:
        raise ValueError(f"{len(azimuth_deg)} azimuths for {n_view} views x {total_frame} frames")
    c2w = orbit_c2w(elevation, azimuth, camera_distance)
    positions = c2w[:, :3, 3].clone()
    fovy = torch.deg2rad(torch.FloatTensor([fovy_deg] * n))
    ts = torch.linspace(-1, 1, steps=total_frame).unsqueeze(-1).repeat(1, n_view).permute(1, 0).reshape(-1, 1)     # 167
    dev = torch.device(device)
    c2w_d, fovy_d = c2w.to(dev), fovy.to(dev)
    return {"rgb": torch.from_numpy(np.stack(rgbs)).to(dev), "mask": torch.from_numpy(np.stack(masks)).to(dev),
            "ref_depth": None, "height": height, "width": width, "c2w": c2w_d, "fovy": fovy_d,
            "timestamps": ts.to(dev), "elevation": elevation.to(dev), "azimuth": azimuth.to(dev),
            "camera_distances": torch.full_like(elevation, camera_distance).to(dev), "camera_positions": positions.to(dev),
            "light_positions": positions.to(dev), "camera_rows": camera_rows(c2w_d, fovy_d),
            "timestamp_layout": timestamp_layout(ts.reshape(-1).numpy())}


# ---------------------------------------------------------------------------------------------------------------- CLI

def _load_geometry(ply: str, state: Optional[str], rot_x_degree: float, rot_z_degree: float, scale_factor: float, device):
    """Gaussian4DModel.from_ply applies the load_ply_cfg transform of gaussian_4d.py:177-306, which is the same as
    gaussian_3d_vis.py:48-172 (the static config's geometry): positions rotated by Rz·Rx then scaled, log-scales
    + log(scale_factor), orientations left-multiplied by Rz·Rx through scipy.  `state` is a Gaussian4DModel state_dict
    (torch.save(model.state_dict())); the global-motion branch is enabled when it holds its weights."""
    from .gaussian4d import Gaussian4DModel
    sd = torch.load(state, map_location=device, weights_only=True) if state else None
    use_global = sd is not None and any(k.startswith("global_rot_network") for k in sd)
    model = Gaussian4DModel.from_ply(ply, rot_x_degree=rot_x_degree, rot_z_degree=rot_z_degree, scale_factor=scale_factor,
                                     device=device, use_global_trans=use_global)
    if sd is not None:
        model.load_state_dict(sd)
    return model


def main(argv: Optional[Sequence[str]] = None) -> None:
    p = argparse.ArgumentParser(description="Render a visualize config's test views of a 4D (or static) gaussian scene")
    p.add_argument("--ply", required=True)
    p.add_argument("--state", default=None, help="Gaussian4DModel state_dict (deformation field); static gaussians without")
    p.add_argument("--option", required=True, choices=OPTIONS)
    p.add_argument("--out", required=True, help="output directory (images/... and mesh_trajectory/ go under it)")
    p.add_argument("--rot_x_degree", type=float, default=0.0)
    p.add_argument("--rot_z_degree", type=float, default=0.0)
    p.add_argument("--scale_factor", type=float, default=1.0)
    p.add_argument("--height", type=int, default=None)
    p.add_argument("--width", type=int, default=None)
    p.add_argument("--save_gaussian_trajectory", action="store_true")
    p.add_argument("--deform_scale", action="store_true", help="apply the scale deltas (the reference's test renders do not)")
    p.add_argument("--threads", type=int, default=8, help="PNG encoder threads")
    a = p.parse_args(argv)
    geometry = _load_geometry(a.ply, a.state, a.rot_x_degree, a.rot_z_degree, a.scale_factor, "cuda")
    views = camera_set(a.option, a.height, a.width)
    paths = save_views(geometry, views, a.out, threads=a.threads, deform_scale=a.deform_scale,
                       save_gaussian_trajectory=a.save_gaussian_trajectory)
    print(f"{len(paths)} images ({views.width}x{views.height}) under {os.path.join(a.out, 'images')}")


if __name__ == "__main__":
    main()
