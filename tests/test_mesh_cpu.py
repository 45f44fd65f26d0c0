"""Mesh animation host side (SURVEY 8f-5): the oracle against the reference's own mesh2gaussian / util.py functions
(ref_mesh.pt), the OBJ reader, the JSON round trip, the graph loader's checks and the sampler's statistics."""
import json
import os

import numpy as np
import pytest
import torch

from animate3d_b200 import mesh as MS
from oracle import mesh_oracle as M


@pytest.fixture(scope="module")
def ref(golden_dir):
    return torch.load(os.path.join(golden_dir, "ref_mesh.pt"), weights_only=False)


def fp32_close(a, b, rtol=4e-7, atol=1e-7):
    np.testing.assert_allclose(np.asarray(a, np.float64), np.asarray(b, np.float64), rtol=rtol, atol=atol)


def test_oracle_reproduces_reference_stats_and_fields(ref):
    verts, faces = ref["verts"].numpy(), ref["faces"].numpy()
    v = verts.shape[0]
    row_ptr, col = M.csr_from_faces(faces, v)
    mae = M.edge_stats(verts, row_ptr, col)
    fp32_close(mae, ref["mean_abs_edge"])
    assert not mae[-1].any() and np.diff(row_ptr)[-1] == 0          # the unreferenced last vertex
    rgb = M.vertex_rgb(faces, ref["corner_rgb"].numpy(), v)
    fp32_close(rgb, ref["vertex_rgb"])
    fields = M.gaussian_fields(verts, rgb, mae)
    ply = {k: t.numpy() for k, t in ref["ply"].items()}
    cols = {"xyz": ["x", "y", "z"], "f_dc": ["f_dc_0", "f_dc_1", "f_dc_2"], "opacity": ["opacity"],
            "scale": ["scale_0", "scale_1", "scale_2"], "rotation": ["rot_0", "rot_1", "rot_2", "rot_3"]}
    for k, names in cols.items():
        want = np.stack([ply[n] for n in names], 1)
        got = fields[k]
        assert np.array_equal(np.isinf(got), np.isinf(want)), k
        fin = np.isfinite(want)
        fp32_close(got[fin], want[fin], rtol=2e-6)
    assert np.isneginf(fields["scale"][-1]).all()                    # log(0): the reference's behaviour, kept
    assert not any(ply[n].any() for n in ("nx", "ny", "nz"))


def test_oracle_reproduces_reference_json_and_util(ref):
    verts, faces = ref["verts"].numpy(), ref["faces"].numpy()
    table = M.json_roundtrip(M.connected_vertices(verts, faces))
    want = ref["table"]
    assert set(table) == set(want)
    for k in want:
        assert set(table[k]) == set(want[k])
        for n in want[k]:
            assert abs(table[k][n] - want[k][n]) <= 2e-7 * max(1.0, want[k][n])
    nn_idx, max_idx = M.prepare_arap_from_mesh_vertices(want)
    assert torch.equal(nn_idx, ref["nn_idx"]) and torch.equal(max_idx, ref["max_idx"])
    e_idx, e_max = MS.prepare_arap_from_mesh_vertices(want)
    assert torch.equal(e_idx, ref["nn_idx"]) and torch.equal(e_max, ref["max_idx"])
    got = M.sample_with_keys(ref["nn_idx"], ref["P"], ref["max_idx"], ref["keys"])
    assert torch.equal(got, ref["sampled"])
    # P above the widest row: the reference returns only D columns
    d = ref["nn_idx"].shape[1]
    assert M.sample_with_keys(ref["nn_idx"], d + 3, ref["max_idx"], ref["keys"]).shape == (ref["nn_idx"].shape[0], d)


def test_engine_json_writer_round_trip(ref):
    """engine writer (CSR -> table) -> reference-shaped reader -> the same dense table as the reference's own JSON."""
    verts, faces = ref["verts"].numpy(), ref["faces"].numpy()
    row_ptr, col = M.csr_from_faces(faces, verts.shape[0])
    graph = MS.MeshGraph(torch.from_numpy(row_ptr), torch.from_numpy(col))
    table = json.loads(json.dumps(MS.connected_vertices(verts, graph), indent=2))
    want = ref["table"]
    assert set(table) == set(want)
    for k in want:
        assert set(table[k]) == set(want[k])
        for n in want[k]:
            assert abs(table[k][n] - want[k][n]) <= 2e-7 * max(1.0, want[k][n])
    got_idx, got_max = MS.prepare_arap_from_mesh_vertices(table)
    # same neighbour set per row (the reference's column order is first appearance, the engine's ascending)
    assert torch.equal(got_max, ref["max_idx"])
    assert torch.equal(got_idx.sort(1).values, ref["nn_idx"].sort(1).values)
    back = MS.MeshGraph.from_connected_vertices(table, verts.shape[0], device="cpu")
    assert torch.equal(back.row_ptr, torch.from_numpy(row_ptr)) and torch.equal(back.col, torch.from_numpy(col))


def test_graph_loader_rejects_out_of_range():
    with pytest.raises(ValueError, match="vertex 5"):
        MS.MeshGraph.from_connected_vertices({"0": {"1": 1.0}, "1": {"0": 1.0}, "5": {"0": 1.0}}, 5, device="cpu")
    with pytest.raises(ValueError, match="neighbour 9"):
        MS.MeshGraph.from_connected_vertices({"0": {"9": 1.0}}, 5, device="cpu")
    with pytest.raises(ValueError, match="key 3"):
        MS.prepare_arap_from_mesh_vertices({"0": {"3": 1.0}, "3": {"0": 1.0}})


def test_obj_reader_on_fixture(tmp_path, ref):
    path = M.write_fixture_obj(str(tmp_path))
    mesh = MS.load_obj(path)
    assert np.array_equal(mesh.verts, ref["verts"].numpy())
    assert np.array_equal(mesh.faces, ref["faces"].numpy())          # the quad is fanned (v0, v1, v2), (v0, v2, v3)
    assert np.array_equal(mesh.faces_uvs, ref["faces_uvs"].numpy())
    assert np.array_equal(mesh.verts_uvs, ref["verts_uvs"].numpy())
    assert np.array_equal(mesh.texture, ref["texture"].numpy().astype(np.float32) / 255)
    crgb = MS.corner_colours(torch.from_numpy(mesh.texture), torch.from_numpy(mesh.verts_uvs), torch.from_numpy(mesh.faces_uvs))
    fp32_close(crgb, ref["corner_rgb"], rtol=1e-5, atol=1e-6)


def _obj(tmp_path, body, texture=True, mtl="newmtl a\nmap_Kd t.png\n"):
    from PIL import Image
    if texture:
        Image.fromarray(np.zeros((2, 2, 3), np.uint8)).save(tmp_path / "t.png")
        (tmp_path / "m.mtl").write_text(mtl)
        body = "mtllib m.mtl\n" + body
    p = tmp_path / "x.obj"
    p.write_text(body)
    return str(p)


VT = "vt 0 0\nvt 1 0\nvt 1 1\nvt 0 1\nvt 0.5 0.5\n"
V5 = "v 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nv 0.5 0.5 1\n"


def test_obj_face_forms_fan_and_negative_indices(tmp_path):
    body = V5 + VT + "vn 0 0 1\nf 1/1 2/2 3/3 4/4 5/5\nf -5/-5/-1 -3/-3/-1 -1/-1/-1\nf 2/2/1 3/3/1 5/5/1\n"
    m = MS.load_obj(_obj(tmp_path, body))
    assert m.faces.tolist() == [[0, 1, 2], [0, 2, 3], [0, 3, 4], [0, 2, 4], [1, 2, 4]]
    assert m.faces_uvs.tolist() == m.faces.tolist()
    # v and v//vn forms parse (and are then rejected on a textured mesh, see below); without a texture they fail loudly too
    for face in ("f 1 2 3\n", "f 1//1 2//1 3//1\n"):
        with pytest.raises(ValueError, match="without texture coordinates"):
            MS.load_obj(_obj(tmp_path, V5 + VT + "vn 0 0 1\n" + face))
    with pytest.raises(ValueError, match="no texture"):
        MS.load_obj(_obj(tmp_path, V5 + "f 1 2 3\n", texture=False))


def test_obj_loud_rejections(tmp_path):
    with pytest.raises(ValueError, match="textured materials"):
        MS.load_obj(_obj(tmp_path, V5 + VT + "f 1/1 2/2 3/3\n", mtl="newmtl a\nmap_Kd t.png\nnewmtl b\nmap_Kd u.png\n"))
    with pytest.raises(ValueError, match="negative index followed by more"):
        MS.load_obj(_obj(tmp_path, V5 + VT + "f -1/1 -2/2 -3/3\nv 2 2 2\n"))
    with pytest.raises(ValueError, match="outside"):
        MS.load_obj(_obj(tmp_path, V5 + VT + "f 1/1 2/2 9/3\n"))


def test_philox_known_answer():
    """Random123's published known-answer vectors for philox4x32-10 (word 0)."""
    assert int(M.philox_word0(0, 0, 0, 0, 0, 0)) == 0x6627E8D5
    assert int(M.philox_word0(0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF)) == 0x408F276D
    assert int(M.philox_word0(0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344, 0xA4093822, 0x299F31D0)) == 0xD16CFE09


def _ragged_graph(v=300, seed=0):
    rng = np.random.default_rng(seed)
    deg = rng.integers(0, 20, size=v)
    deg[:4] = [0, 1, 3, 12]
    col = np.concatenate([np.sort(rng.choice(v, d, replace=False)) for d in deg]).astype(np.int32)
    row_ptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
    return row_ptr, col, deg


@pytest.mark.parametrize("K", [1, 3, 12])
def test_sampler_rows(K):
    row_ptr, col, deg = _ragged_graph()
    nbr = M.sample_csr(row_ptr, col, K, seed=123, offset=5)
    for i in range(len(deg)):
        row = nbr[i]
        got = row[row >= 0]
        assert len(got) == min(K, deg[i])                       # -1 exactly when the degree is below K
        assert (row[len(got):] == -1).all()
        assert len(set(got.tolist())) == len(got)               # no repeats
        assert set(got.tolist()) <= set(col[row_ptr[i]:row_ptr[i + 1]].tolist())


def test_sampler_frequencies_chi_square():
    """Over 3000 offsets every neighbour of a degree-d row is picked K/d of the time: Pearson's statistic over the d cells
    stays below the 99.9 % quantile of chi-square with d - 1 degrees of freedom."""
    from scipy.stats import chi2
    row_ptr, col, deg = _ragged_graph(60, 1)
    K, n = 3, 3000
    counts = [np.zeros(d) for d in deg]
    for off in range(n):
        nbr = M.sample_csr(row_ptr, col, K, seed=99, offset=off)
        for i in range(len(deg)):
            if deg[i] > K:
                slot = np.searchsorted(col[row_ptr[i]:row_ptr[i + 1]], nbr[i])
                counts[i][slot] += 1
    tested = 0
    for i, d in enumerate(deg):
        if d > K:
            exp = n * K / d
            stat = ((counts[i] - exp) ** 2 / exp).sum()
            assert stat < chi2.ppf(0.999, d - 1), (i, d, stat)
            tested += 1
    assert tested > 20
