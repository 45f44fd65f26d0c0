"""Forward-only RGBA8 renders (a3d_raster_forward_rgba8) and the test-view pipeline of animate3d_b200/visualize.py on the
GPU.  The RGBA8 bytes must equal quantising the float forward of a3d_raster_forward exactly:
(cat(color.clamp(0, 1), alpha) * 255).to(uint8), the reference's test_step arithmetic (animate3d.py:439-445)."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _quantise(color, alpha):
    """[cams,3,H,W], [cams,1,H,W] float -> [cams,H,W,4] uint8, as the reference saves its test renders."""
    return (torch.cat([color.clamp(0, 1), alpha], dim=1).permute(0, 2, 3, 1) * 255).to(torch.uint8).contiguous()


def _scene(P, seed, sh_degree):
    from oracle import raster_oracle as R
    xyz, s, q, o, sh = R.synthetic_scene(P, seed, sh_degree)
    return [t.cuda().contiguous() for t in (xyz, s, q, o, sh)]


def _rows(option, H, W, away=False):
    from animate3d_b200 import visualize as V
    from animate3d_b200.renderer import camera_rows
    views = V.camera_set(option, H, W)
    c2w = views.c2w[::16].clone() if option != "static" else views.c2w.clone()
    if away:                                   # turned 180 degrees about the up axis: looks away from the scene
        c2w[:, :3, 0] *= -1
        c2w[:, :3, 2] *= -1
    return camera_rows(c2w.cuda(), views.fovy[:c2w.shape[0]].cuda())


def _float_forward(rows, H, W, xyz, s, q, o, sh, deg, bg):
    from animate3d_b200.rasterizer import _RasterizeBatch
    meta = (H, W, deg, False, 1.0, [float(b) for b in bg])
    with torch.no_grad():
        color, radii, depth, alpha = _RasterizeBatch.apply(xyz, None, s, q, o, sh, None, rows, meta)
    return color, radii, alpha


@pytest.mark.parametrize("P,H,W,deg,bg,away", [
    (50000, 1024, 1024, 0, 0.5, False),      # config-3 scene at the test-render resolution
    (50000, 1024, 1024, 3, 1.0, False),
    (20000, 1000, 760, 3, 0.5, False),       # ragged tiles in both directions
    (20000, 1000, 760, 0, 1.0, False),
    (20000, 512, 512, 0, 0.5, True),         # every camera sees nothing: background and alpha 0
])
def test_rgba8_equals_quantised_float_forward(P, H, W, deg, bg, away):
    from animate3d_b200.rasterizer import RGBA8Renderer
    xyz, s, q, o, sh = _scene(P, 7 + deg, deg)
    rows = _rows("four_view", H, W, away)
    bgv = (bg, bg, bg)
    color, radii, alpha = _float_forward(rows, H, W, xyz, s, q, o, sh, deg, bgv)
    ref = _quantise(color, alpha)
    r = RGBA8Renderer()
    got = r.render(rows, H, W, xyz, s, q, o, sh, None, deg, False, bgv)
    assert got.shape == (4, H, W, 4) and got.dtype == torch.uint8
    assert torch.equal(got, ref), f"{int((got != ref).sum())} bytes differ"
    if away:
        assert r.last_total == 0 and int(radii.max()) == 0
        assert bool((got[..., 3] == 0).all()) and bool((got[..., :3] == int(bg * 255)).all())
    else:
        assert r.last_total > 0 and bool((got[..., 3] > 0).any())


def _model(P=50000, seed=11):
    from animate3d_b200.gaussian4d import Gaussian4DModel
    from oracle import raster_oracle as R
    pts, s, q, o, sh = R.synthetic_scene(P, seed)
    model = Gaussian4DModel(pts, torch.log(s), q, torch.logit(o), sh[:, 0], use_global_trans=True)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name in ("delta_xyz_network", "delta_rot_network", "delta_scaling_network", "global_rot_network", "global_trans_network"):
            net = getattr(model, name)
            net[1].copy_((torch.randn(net[1].shape, generator=g) * 0.05).cuda())
    return model


@pytest.fixture(scope="module")
def model():
    return _model()


def test_chunked_equals_one_shot_and_overflow_retry(model):
    from animate3d_b200 import visualize as V
    from animate3d_b200.rasterizer import RGBA8Renderer
    views = V.camera_set("four_view", 384, 384)
    one = V.render_views(model, views, max_pixels=1 << 30)
    chunked = V.render_views(model, views, max_pixels=384 * 384 * 5)          # 13 chunks, the last of 4 cameras
    assert torch.equal(one, chunked)
    r = RGBA8Renderer()
    r.pairs_per_cam = 1.0                                                     # capacity far too small: the first call overflows
    again = V.render_views(model, views, max_pixels=384 * 384 * 16, renderer=r)
    assert r.overflows >= 1 and torch.equal(one, again)
    tight = RGBA8Renderer(max_pairs=1 << 16)                                  # pair budget: chunks are halved down to 1 camera
    assert torch.equal(one, V.render_views(model, views, max_pixels=384 * 384 * 16, renderer=tight))
    assert tight.overflows >= 1 and tight.last_total > 0


def test_four_view_equals_batch_forward_without_scale_deltas(model):
    """The reference's test batches: do_guidance False (load_guidance false), so the deformed means and rotations with the
    static scales; batch_forward's gradient gate changes no value."""
    from animate3d_b200 import visualize as V
    from animate3d_b200.renderer import make_renderer
    views = V.camera_set("four_view", 256, 256)
    got = V.render_views(model, views)
    ren = make_renderer(model, back_ground_color=(0.5, 0.5, 0.5))
    with torch.no_grad():
        out = ren.batch_forward({"c2w": views.c2w.cuda(), "fovy": views.fovy.cuda(), "timestamps": views.timestamps.cuda(),
                                 "height": 256, "width": 256, "do_guidance": False, "do_reconstruction": True})
    ref = (torch.cat([out["comp_rgb"], out["comp_mask"]], dim=-1) * 255).to(torch.uint8)
    assert torch.equal(got, ref)
    scaled = V.render_views(model, views, deform_scale=True)
    assert not torch.equal(got, scaled)                                       # the scale deltas do move the splats


def test_static_equals_batch_forward_without_timestamps(model):
    from animate3d_b200 import visualize as V
    from animate3d_b200.renderer import make_renderer
    views = V.camera_set("static")
    got = V.render_views(model, views)
    ren = make_renderer(model, back_ground_color=(0.498, 0.498, 0.498))
    with torch.no_grad():
        out = ren.batch_forward({"c2w": views.c2w.cuda(), "fovy": views.fovy.cuda(), "height": 512, "width": 512})
    ref = (torch.cat([out["comp_rgb"], out["comp_mask"]], dim=-1) * 255).to(torch.uint8)
    assert got.shape == (5, 512, 512, 4) and torch.equal(got, ref)


@pytest.mark.parametrize("option,n_files,n_dirs", [("four_view", 64, 1), ("testset", 192, 12), ("static", 5, 1)])
def test_save_views_layout(model, tmp_path, option, n_files, n_dirs):
    from animate3d_b200 import visualize as V
    views = V.camera_set(option, 64, 64)
    paths = V.save_views(model, views, str(tmp_path), threads=4, save_gaussian_trajectory=True)
    files = sorted(os.path.relpath(os.path.join(d, f), tmp_path) for d, _, fs in os.walk(tmp_path / "images") for f in fs)
    assert len(files) == n_files == len(paths) and sorted(views.files) == files
    assert len({os.path.dirname(f) for f in files}) == n_dirs
    if option == "testset":
        assert sorted(os.listdir(tmp_path / "images")) == sorted(f"elv_{e}_azi_{a}" for e in range(3) for a in range(4))
        assert sorted(os.listdir(tmp_path / "images" / "elv_2_azi_3")) == sorted(f"{i}.png" for i in range(16))
    traj = tmp_path / "mesh_trajectory"
    assert (sorted(os.listdir(traj)) == sorted(f"{i}.npy" for i in range(16))) if option != "static" else not traj.exists()


def test_round_trip_render_save_load(model, tmp_path):
    """render -> save_views -> load_multiview_images gives back rgba[..., :3] / 255 and alpha > 0.5 exactly: the four_view
    renders are the refine stage's reconstruction targets."""
    from PIL import Image

    from animate3d_b200 import visualize as V
    views = V.camera_set("four_view", 128, 128)
    rgba = V.render_views(model, views)
    V.save_views(model, views, str(tmp_path), threads=4)
    first = np.asarray(Image.open(tmp_path / "images" / "0.png"))
    assert first.dtype == np.uint8 and first.shape == (128, 128, 4) and np.array_equal(first, rgba[0].cpu().numpy())
    data = V.load_multiview_images(str(tmp_path / "images"), n_view=4, total_frame=16, height=128, width=128)
    host = rgba.cpu().numpy().astype(np.float32)       # true division (torch's CUDA division by a scalar multiplies by 1/255)
    assert np.array_equal(data["rgb"].cpu().numpy(), host[..., :3] / 255)
    assert np.array_equal(data["mask"].cpu().numpy(), host[..., 3:] / 255 > 0.5)
    assert bool(data["mask"].any()) and not bool(data["mask"].all())
    assert data["timestamp_layout"] == V.timestamp_layout(views.timestamps.numpy())
    torch.testing.assert_close(data["c2w"].cpu(), views.c2w, rtol=0, atol=1e-6)
