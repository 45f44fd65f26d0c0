"""Test-view camera sets, the multi-view image loader and the RGBA8 quantiser (animate3d_b200/visualize.py,
a3d_raster_math.h) without a GPU.  The camera sets are checked against a line-by-line restatement of the reference's
datasets and `test_step` file naming, kept below; the loader against cv2 itself; the quantiser, compiled from the header the
kernel includes, against numpy's `(np.float32(x) * 255).astype(np.uint8)`."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from animate3d_b200 import visualize as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ reference restatement
def _ref_orbit(elevation_deg, azimuth_deg, camera_distance, fovy_deg_value, up_rows):
    """uncond_hybrid.py:581-623 / uncond.py:367-409 (the two are the same code): c2w and fovy."""
    camera_distances = torch.full_like(elevation_deg, camera_distance)
    elevation = elevation_deg * math.pi / 180
    azimuth = azimuth_deg * math.pi / 180
    camera_positions = torch.stack([camera_distances * torch.cos(elevation) * torch.cos(azimuth),
                                    camera_distances * torch.cos(elevation) * torch.sin(azimuth),
                                    camera_distances * torch.sin(elevation)], dim=-1)
    center = torch.zeros_like(camera_positions)
    up = torch.as_tensor([0, 0, 1], dtype=torch.float32)[None, :].repeat(up_rows, 1)
    fovy_deg = torch.full_like(elevation_deg, fovy_deg_value)
    fovy = fovy_deg * math.pi / 180
    lookat = F.normalize(center - camera_positions, dim=-1)
    right = F.normalize(torch.linalg.cross(lookat, up.expand_as(lookat)), dim=-1)
    up = F.normalize(torch.linalg.cross(right, lookat), dim=-1)
    c2w3x4 = torch.cat([torch.stack([right, up, -lookat], dim=-1), camera_positions[:, :, None]], dim=-1)
    c2w = torch.cat([c2w3x4, torch.zeros_like(c2w3x4[:, :1])], dim=1)
    c2w[:, 3, 3] = 1.0
    return c2w, fovy


def _ref_hybrid_test(eval_elevation_deg, eval_azimuth_deg, total_frame=16, n_frame=16, test_option="four_view"):
    """HybridRandomCameraTestDataset (uncond_hybrid.py:560-700, eval_batch_size 1) and the file name test_step gives each
    batch (animate3d.py:446-462)."""
    azimuth_deg = torch.tensor(eval_azimuth_deg).reshape(-1)
    elevation_deg = torch.tensor(eval_elevation_deg).repeat_interleave(len(eval_azimuth_deg[0]))
    c2w, fovy = _ref_orbit(elevation_deg, azimuth_deg, 3.0, 40.0, 1)
    timestamps = torch.linspace(-1, 1, steps=total_frame).unsqueeze(-1)
    items = []
    for origin_index in range(len(eval_azimuth_deg[0]) * len(eval_elevation_deg) * total_frame):
        time_index = origin_index % total_frame
        index = int(origin_index // total_frame)
        batch_index = origin_index
        if test_option == "testset":
            elv_index = batch_index // (n_frame * 4)
            azi_index = (batch_index // n_frame) % 4
            path = os.path.join("images", f"elv_{elv_index}_azi_{azi_index}", f"{batch_index % n_frame}.png")
        else:
            path = os.path.join("images", f"{batch_index}.png")
        items.append((c2w[index], fovy[index], timestamps[time_index], path))
    return items


def _ref_static():
    """RandomCameraDataset test split (uncond.py:347-409) with visualize_four_view_static.yaml (n_test_views 5); test_step
    with test_option four_view and n_frame 1 saves batch i as images/{i}.png."""
    azimuth_deg = torch.linspace(0, 360.0, 5)
    elevation_deg = torch.full_like(azimuth_deg, 15.0)
    c2w, fovy = _ref_orbit(elevation_deg, azimuth_deg, 3.0, 40.0, 1)
    return [(c2w[i], fovy[i], None, os.path.join("images", f"{i}.png")) for i in range(5)]


def _check_set(views, items):
    assert len(views) == len(items)
    for i, (c2w, fovy, ts, path) in enumerate(items):
        assert torch.equal(views.c2w[i], c2w), i
        assert torch.equal(views.fovy[i], fovy), i
        if ts is None:
            assert views.timestamps is None
        else:
            assert torch.equal(views.timestamps[i].reshape(1), ts.reshape(1)), i
        assert os.path.normpath(views.files[i]) == os.path.normpath(path), (i, views.files[i], path)


def test_four_view_set_matches_reference():
    views = V.camera_set("four_view")
    _check_set(views, _ref_hybrid_test([15.0], [[0.0, 90.0, 180.0, 270.0]]))
    assert (views.height, views.width, views.background) == (1024, 1024, (0.5, 0.5, 0.5))
    assert len(set(views.files)) == 64


def test_testset_matches_reference():
    views = V.camera_set("testset")
    _check_set(views, _ref_hybrid_test([15.0, 0.0, 30.0], [[0.0, 90.0, 180.0, 270.0], [30.0, 120.0, 210.0, 300.0],
                                                            [-45.0, 45.0, 135.0, 225.0]], test_option="testset"))
    assert len(set(views.files)) == 192 and len({os.path.dirname(f) for f in views.files}) == 12
    # item 70 is camera 4 (azimuth 30, the first of the elevation-0 row) at frame 6
    assert views.c2w[70].equal(views.c2w[64]) and float(views.timestamps[70]) == float(torch.linspace(-1, 1, 16)[6])
    assert views.files[70] == "images/elv_1_azi_0/6.png"


def test_static_set_matches_reference():
    views = V.camera_set("static")
    _check_set(views, _ref_static())
    assert (views.height, views.width, views.background) == (512, 512, (0.498, 0.498, 0.498))
    assert torch.allclose(views.c2w[4], views.c2w[0], atol=1e-5)      # linspace(0, 360, 5): view 4 repeats view 0


def test_camera_set_rejects_unknown_option():
    with pytest.raises(ValueError):
        V.camera_set("test_set")


# ------------------------------------------------------------------------------------------------ loader
def _write_synthetic(root, n, h, w, seed):
    import cv2
    g = np.random.default_rng(seed)
    imgs = []
    for i in g.permutation(n):                                # creation order unrelated to the index
        rgba = g.integers(0, 256, size=(h, w, 4), dtype=np.uint8)
        rgba[0, :4, 3] = [127, 128, 0, 255]                   # alpha straddling the 0.5 threshold
        imgs.append((int(i), rgba))
        assert cv2.imwrite(os.path.join(root, f"{i}.png"), cv2.cvtColor(rgba, cv2.COLOR_RGBA2BGRA))
    return dict(imgs)


def test_loader_sorts_converts_resizes_like_cv2(tmp_path):
    import cv2
    n_view, total_frame, h, w = 2, 6, 40, 52                  # 12 files: "10.png" sorts after "9.png"
    imgs = _write_synthetic(str(tmp_path), n_view * total_frame, h, w, 0)
    kw = dict(n_view=n_view, total_frame=total_frame, azimuth_deg=(0.0, 180.0), device="cpu")
    out = V.load_multiview_images(str(tmp_path), height=24, width=30, **kw)
    assert out["rgb"].shape == (12, 24, 30, 3) and out["mask"].dtype == torch.bool
    for i in range(12):
        ref = cv2.resize(imgs[i], (30, 24), interpolation=cv2.INTER_AREA).astype(np.float32) / 255.0
        assert np.array_equal(out["rgb"][i].numpy(), ref[..., :3]), i
        assert np.array_equal(out["mask"][i].numpy(), ref[..., 3:] > 0.5), i
    same = V.load_multiview_images(str(tmp_path), height=h, width=w, **kw)
    for i in range(12):
        assert np.array_equal(same["rgb"][i].numpy(), imgs[i][..., :3].astype(np.float32) / 255.0)
        assert same["mask"][i, 0, :4, 0].tolist() == [False, True, False, True]


def test_loader_cameras_and_timestamps(tmp_path):
    n_view, total_frame = 4, 16
    _write_synthetic(str(tmp_path), n_view * total_frame, 8, 8, 1)
    out = V.load_multiview_images(str(tmp_path), n_view=n_view, total_frame=total_frame, height=8, width=8, device="cpu")
    # simple_multi_image.py:91-131: each azimuth repeated total_frame times (view-major), up [1, 3] broadcast
    azimuth_deg = torch.FloatTensor([0.0, 90.0, 180.0, 270.0]).unsqueeze(-1).repeat(1, total_frame).reshape(-1)
    elevation_deg = torch.FloatTensor([15.0] * 64)
    c2w, _ = _ref_orbit(elevation_deg, azimuth_deg, 3.0, 40.0, 1)
    assert torch.equal(out["c2w"], c2w)
    assert torch.equal(out["fovy"], torch.deg2rad(torch.FloatTensor([40.0] * 64)))
    ts = torch.linspace(-1, 1, steps=total_frame).unsqueeze(-1).repeat(1, n_view).permute(1, 0).reshape(-1, 1)   # 167
    assert torch.equal(out["timestamps"], ts)
    assert out["timestamp_layout"] == tuple(list(range(16)) * 4)
    assert out["camera_rows"].shape == (64, 37)
    assert torch.equal(out["azimuth"], azimuth_deg) and torch.equal(out["camera_positions"], c2w[:, :3, 3])


def test_loader_rejects_wrong_count(tmp_path):
    _write_synthetic(str(tmp_path), 5, 8, 8, 2)
    with pytest.raises(ValueError):
        V.load_multiview_images(str(tmp_path), n_view=4, total_frame=2, height=8, width=8, device="cpu")


# ------------------------------------------------------------------------------------------------ quantiser
@pytest.fixture(scope="module")
def quant(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("q") / "quant_cpu.so")
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(ROOT, "tests", "cpu_harness", "quant_cpu.cpp"), "-o", out])
    lib = C.CDLL(out)
    lib.quant_cpu.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int]
    return lib


def _run(lib, x, clamp):
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty(x.shape, np.uint8)
    lib.quant_cpu(x.ctypes.data, out.ctypes.data, x.size, int(clamp))
    return out


def test_quantiser_bit_equal_to_numpy(quant):
    k = np.arange(256, dtype=np.float32) / np.float32(255)
    edges = np.concatenate([k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(2))])
    extra = np.array([0.0, -0.0, 1.0, 1.0000001, 1.002, 1.5, 2.0, 3.7, 100.0, 8e6, -1e-7, -0.001, -0.3, -0.5, -1.0, -100.0,
                      np.float32(0.5) / 255], np.float32)
    rng = np.random.default_rng(0)
    x = np.concatenate([edges, extra, rng.random(100000, dtype=np.float32), rng.uniform(-3, 3, 100000).astype(np.float32)])
    with np.errstate(invalid="ignore"):
        ref = (x * np.float32(255)).astype(np.uint8)
    got = _run(quant, x, False)
    bad = np.nonzero(got != ref)[0]
    assert bad.size == 0, [(float(x[i]), int(got[i]), int(ref[i])) for i in bad[:10]]
    # the alpha above 1 and the negative values wrap as numpy's cast does; colours are clamped first
    assert _run(quant, np.array([1.5, -0.5], np.float32), False).tolist() == [126, 129]
    assert np.array_equal(_run(quant, x, True), (np.clip(x, 0, 1) * np.float32(255)).astype(np.uint8))
