"""Mesh animation kernels (a3d_mesh_adjacency / a3d_mesh_vertex_stats / a3d_mesh_sample_neighbors) against
oracle/mesh_oracle.py, and the OBJ -> PLY + JSON -> 4D model -> mesh-edge ARAP -> trajectory flow end to end."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from animate3d_b200 import mesh as MS  # noqa: E402
from oracle import mesh_oracle as M    # noqa: E402


def _random_mesh(nf=100_000, nv=30_000, seed=3):
    rng = np.random.default_rng(seed)
    faces = rng.integers(0, nv - 10, size=(nf, 3))           # the last 10 vertices stay unreferenced
    faces[:50, 1] = faces[:50, 0]                              # a few degenerate faces: self-edges, as in the reference
    faces[100:400, 0] = 7                                      # a fan vertex of degree > 300
    return rng.normal(size=(nv, 3)).astype(np.float32), faces


def _fixture(golden_dir):
    d = torch.load(os.path.join(golden_dir, "ref_mesh.pt"), weights_only=False)
    return d["verts"].numpy(), d["faces"].numpy(), d["corner_rgb"].numpy()


def test_adjacency_bit_exact(golden_dir):
    for verts, faces in (_fixture(golden_dir)[:2], _random_mesh()):
        g = MS.MeshGraph.from_faces(torch.from_numpy(faces).cuda(), verts.shape[0])
        row_ptr, col = M.csr_from_faces(faces, verts.shape[0])
        assert torch.equal(g.row_ptr.cpu(), torch.from_numpy(row_ptr))
        assert torch.equal(g.col.cpu(), torch.from_numpy(col))
        g2 = MS.MeshGraph.from_faces(torch.from_numpy(faces).cuda(), verts.shape[0])
        assert torch.equal(g.col, g2.col) and torch.equal(g.row_ptr, g2.row_ptr)


def test_vertex_stats_against_oracle(golden_dir):
    vf, ff, cf = _fixture(golden_dir)
    rv, rf = _random_mesh()
    rc = np.random.default_rng(4).random((rf.shape[0], 3, 3)).astype(np.float32)
    eps = 2.0 ** -24
    for verts, faces, crgb in ((vf, ff, cf), (rv, rf, rc)):
        nv = verts.shape[0]
        g = MS.MeshGraph.from_faces(torch.from_numpy(faces).cuda(), nv)
        mae, rgb = MS.vertex_stats(torch.from_numpy(verts).cuda(), g, torch.from_numpy(faces).cuda(), torch.from_numpy(crgb).cuda())
        row_ptr, col = M.csr_from_faces(faces, nv)
        deg = np.diff(row_ptr)
        # float64 sums; an fp32 sum of n terms then one division is within (n + 1) eps of it, relative to the sum of |terms|
        v64 = verts.astype(np.float64)
        src = np.repeat(np.arange(nv), deg)
        s64 = np.zeros((nv, 3))
        np.add.at(s64, src, np.abs(v64[col] - v64[src]))
        want = np.where(deg[:, None] > 0, s64 / np.maximum(deg, 1)[:, None], 0)
        bound = (deg[:, None] + 1) * eps * want + 1e-30
        assert (np.abs(mae.cpu().numpy() - want) <= bound).all()
        cnt = np.bincount(faces.reshape(-1), minlength=nv)
        c64 = np.zeros((nv, 3))
        for k in range(3):
            np.add.at(c64, faces[:, k], crgb[:, k].astype(np.float64))
        want_rgb = c64 / np.maximum(cnt, 1)[:, None]
        assert (np.abs(rgb.cpu().numpy() - want_rgb) <= (cnt[:, None] + 1) * eps * want_rgb + 1e-30).all()
        # the fp32 restatement in the kernel's order is bit-equal
        assert np.array_equal(mae.cpu().numpy(), M.edge_stats(verts, row_ptr, col))
        assert np.array_equal(rgb.cpu().numpy(), M.vertex_rgb(faces, crgb, nv))


@pytest.mark.parametrize("K", [1, 3, 12])
def test_sample_neighbors_bit_exact(K):
    rng = np.random.default_rng(K)
    nv = 5000
    deg = rng.integers(0, 30, size=nv)
    deg[:6] = [0, 1, K - 1 if K > 1 else 0, K, K + 1, 400]
    col = np.concatenate([np.sort(rng.choice(nv, d, replace=False)) for d in deg]).astype(np.int32)
    row_ptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
    g = MS.MeshGraph(torch.from_numpy(row_ptr).cuda(), torch.from_numpy(col).cuda())
    for seed, offset in ((0, 0), (1234567, 3), (2 ** 40 + 17, 2 ** 33 + 5), (2 ** 62 - 1, 1)):
        got = g.sample(K, seed=seed, offset=offset).cpu().numpy()
        assert np.array_equal(got, M.sample_csr(row_ptr, col, K, seed, offset)), (seed, offset)


def test_sample_matrix_vectorized_dropin(golden_dir):
    d = torch.load(os.path.join(golden_dir, "ref_mesh.pt"), weights_only=False)
    nn_idx, max_idx = d["nn_idx"].cuda(), d["max_idx"].cuda()
    out = MS.sample_matrix_vectorized(nn_idx, 3, max_idx)
    assert out.dtype == torch.int64 and out.shape == (nn_idx.shape[0], 3)
    deg = max_idx.sum(1)
    for i in range(nn_idx.shape[0]):
        row = out[i][out[i] >= 0].tolist()
        assert len(row) == min(3, int(deg[i])) and len(set(row)) == len(row)
        assert set(row) <= set(nn_idx[i][max_idx[i]].tolist())
    assert MS.sample_matrix_vectorized(nn_idx, nn_idx.shape[1] + 2, max_idx).shape == tuple(nn_idx.shape)


def _flow(tmp_path, deterministic):
    from animate3d_b200 import arap
    from animate3d_b200.gaussian4d import Gaussian4DModel
    from animate3d_b200.io import load_gaussian_ply
    from animate3d_b200.mesh2gaussian import main
    obj = M.write_fixture_obj(str(tmp_path / "in"))
    main(["--input_obj", obj, "--output_dir", str(tmp_path / "out"), "--output_name", "dragon"])
    ply, js = str(tmp_path / "out" / "dragon.ply"), str(tmp_path / "out" / "dragon.json")
    nv = load_gaussian_ply(ply)["_xyz"].shape[0]
    graph = MS.MeshGraph.from_connected_vertices(js, nv)
    model = Gaussian4DModel.from_ply(ply, rot_x_degree=90, rot_z_degree=90, scale_factor=0.76,
                                     grid_size=((8, 8, 8, 4), (16, 16, 16, 8)))
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for net in (model.delta_xyz_network, model.delta_rot_network, model.delta_scaling_network):
            net[1].copy_(torch.randn(net[1].shape, generator=g) * 0.05)
    torch.use_deterministic_algorithms(deterministic)
    try:
        means, _, _ = model.deform_all(torch.linspace(-1, 1, 4).cuda())
        nodes = torch.cat([model._xyz[None], means])
        torch.manual_seed(11)
        nbr = graph.sample(3)
        ii, jj, nn = MS.edge_list(nbr)
        loss = arap.cal_arap_error(nodes, ii, jj, nn, K=3, sample_num=512)
        loss.backward()
    finally:
        torch.use_deterministic_algorithms(False)
    grads = [p.grad.clone() for p in model.parameters() if p.grad is not None]
    return model, graph, nodes.detach(), nbr, loss.detach(), grads


def test_end_to_end_mesh_arap(tmp_path):
    from oracle import arap_oracle as A
    model, graph, nodes, nbr, loss, _ = _flow(tmp_path / "a", False)
    # the graph read back from the JSON equals the faces' graph; the PLY is the oracle's gaussians
    ref = MS.load_obj(str(tmp_path / "a" / "in" / "mesh.obj"))
    fg = MS.MeshGraph.from_faces(torch.from_numpy(ref.faces).cuda(), ref.verts.shape[0])
    assert torch.equal(fg.row_ptr, graph.row_ptr) and torch.equal(fg.col, graph.col)
    ii, jj, nn = MS.edge_list(nbr.cpu())
    want = A.arap_error(nodes.cpu(), ii, jj, nn, 3)
    assert float(want) > 0
    assert abs(float(loss) - float(want)) <= 5e-4 * abs(float(want)), (float(loss), float(want))
    # deterministic mode: two runs are bit-identical
    _, _, _, nbr1, l1, g1 = _flow(tmp_path / "b", True)
    _, _, _, nbr2, l2, g2 = _flow(tmp_path / "c", True)
    assert torch.equal(nbr1, nbr2) and torch.equal(l1, l2)
    assert len(g1) > 0 and all(torch.equal(a, b) for a, b in zip(g1, g2))


def test_save_mesh_trajectory(tmp_path):
    from animate3d_b200.io import load_mesh_trajectory
    model, *_ = _flow(tmp_path / "a", False)
    folder = str(tmp_path / "traj")
    MS.save_mesh_trajectory(model, folder)
    assert sorted(os.listdir(folder)) == sorted(f"{i}.npy" for i in range(16))
    traj = torch.from_numpy(load_mesh_trajectory(folder, 16))
    with torch.no_grad():
        means, _, _ = model.deform_all(torch.linspace(-1, 1, 16).cuda())
    assert torch.equal(traj[0], model._xyz.cpu())
    assert torch.equal(traj[1:], means[1:].cpu())
    assert not torch.equal(traj[0], means[0].cpu())      # the static first frame is a real substitution
