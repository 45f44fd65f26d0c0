"""Generate tests/golden/ref_mesh.pt by RUNNING THE REFERENCE'S OWN SOURCE (read from /root/reference at generation time,
never copied), in the manner of gen_reference_goldens.py.  Run in the build container only:

    python tests/golden/gen_mesh_goldens.py        ->  tests/golden/ref_mesh.pt

What is real and what is stubbed
  real   : tools/mesh_animation/mesh2gaussian.py (convert_to_textureVertex_with_average, compute_edge_distances,
           find_and_save_connected_vertices, convert_point_cloud_to_gaussian and its helpers) and
           custom/threestudio-animate3d/systems/util.py:300-344 (prepare_arap_from_mesh_vertices, sample_matrix_vectorized),
           exec'd from the files' AST
  stubbed: pytorch3d's Meshes / TexturesVertex / packed_to_list (the mesh is oracle.mesh_oracle's fixture, its corner
           colours from oracle.mesh_oracle.corner_colours), plyfile's PlyElement / PlyData writer; `.cuda()` is dropped.
The GPU box has no /root/reference; only the emitted .pt fixture travels.
"""
import ast
import os
import sys
from types import SimpleNamespace

import torch

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))


def run_reference_mesh():
    """exec the mesh functions of tools/mesh_animation/mesh2gaussian.py and prepare_arap_from_mesh_vertices /
    sample_matrix_vectorized of systems/util.py:300-344 on the CPU, on oracle.mesh_oracle's seeded fixture (a UV sphere
    with a texture seam, one fanned quad, one unreferenced last vertex).  pytorch3d's Meshes / TexturesVertex /
    packed_to_list and plyfile's writer are stubbed, `.cuda()` is dropped, torch.rand is recorded."""
    import json
    import tempfile
    import numpy as np
    sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))
    from oracle import mesh_oracle as M
    verts_np, uvs, polys, tex = M.fixture_mesh(0)
    faces_np, fuvs = [], []
    for p in polys:                                      # fan (v0, vk, vk+1), as pytorch3d's load_obj
        for k in range(1, len(p) - 1):
            faces_np.append([p[0][0], p[k][0], p[k + 1][0]])
            fuvs.append([p[0][1], p[k][1], p[k + 1][1]])
    verts, faces = torch.from_numpy(verts_np), torch.tensor(faces_np, dtype=torch.int64)
    corner_rgb = torch.from_numpy(M.corner_colours(tex.astype(np.float32) / 255.0, uvs, np.asarray(fuvs)))

    def functions(path, want, no_cuda=False):
        src = open(os.path.join(REF, path)).read()
        body = [n for n in ast.parse(src).body if (isinstance(n, ast.FunctionDef) and n.name in want) or
                (isinstance(n, ast.Assign) and any(getattr(t, "id", None) in want for t in n.targets))]

        class NoCuda(ast.NodeTransformer):
            def visit_Call(self, node):
                self.generic_visit(node)
                if isinstance(node.func, ast.Attribute) and node.func.attr == "cuda" and not node.args:
                    return node.func.value
                return node
        mod = ast.Module(body=body, type_ignores=[])
        return ast.fix_missing_locations(NoCuda().visit(mod) if no_cuda else mod)

    captured = {}

    class PlyElement:
        @staticmethod
        def describe(elements, name):
            captured["ply"] = {n: np.array(elements[n]) for n in elements.dtype.names}
            return elements

    class PlyData:
        def __init__(self, els):
            pass

        def write(self, path):
            pass

    class TexturesVertex:
        def __init__(self, feats):
            self.feats = feats

        def verts_features_packed(self):
            return torch.cat(self.feats)
    ns = {"torch": torch, "np": np, "json": json, "PlyElement": PlyElement, "PlyData": PlyData, "TexturesVertex": TexturesVertex,
          "packed_to_list": lambda x, sizes: list(x.split(sizes.tolist() if torch.is_tensor(sizes) else sizes))}
    exec(compile(functions("tools/mesh_animation/mesh2gaussian.py",
                           {"convert_to_textureVertex_with_average", "compute_edge_distances", "find_and_save_connected_vertices",
                            "C0", "construct_list_of_attributes", "RGB2SH", "inverse_sigmoid", "convert_point_cloud_to_gaussian"}),
                 "mesh2gaussian", "exec"), ns)
    meshes = SimpleNamespace(verts_packed=lambda: verts, faces_packed=lambda: faces,
                             textures=SimpleNamespace(faces_verts_textures_packed=lambda: corner_rgb),
                             num_verts_per_mesh=lambda: torch.tensor([verts.shape[0]]))
    # main() (141-177) on the stubbed mesh
    rgb = ns["convert_to_textureVertex_with_average"](meshes).verts_features_packed()
    mae = ns["compute_edge_distances"](meshes)
    ns["convert_point_cloud_to_gaussian"](verts.numpy(), rgb.numpy(), mae.numpy() / 1.1, "unused.ply")
    with tempfile.TemporaryDirectory() as d:
        ns["find_and_save_connected_vertices"](meshes, os.path.join(d, "cv.json"))
        table = json.load(open(os.path.join(d, "cv.json")))

    class RecordingTorch:
        def __getattr__(self, name):
            return getattr(torch, name)

        @staticmethod
        def rand(*shape):
            captured["keys"] = torch.rand(*shape)
            return captured["keys"].clone()
    uns = {"torch": RecordingTorch()}
    exec(compile(functions("custom/threestudio-animate3d/systems/util.py",
                           {"prepare_arap_from_mesh_vertices", "sample_matrix_vectorized"}, no_cuda=True), "util_mesh", "exec"), uns)
    nn_idx, max_idx = uns["prepare_arap_from_mesh_vertices"](table)
    torch.manual_seed(7)
    sampled = uns["sample_matrix_vectorized"](nn_idx, 3, max_idx)
    torch.save({"verts": verts, "faces": faces, "verts_uvs": torch.from_numpy(uvs), "faces_uvs": torch.tensor(fuvs),
                "texture": torch.from_numpy(tex), "corner_rgb": corner_rgb, "vertex_rgb": rgb, "mean_abs_edge": mae,
                "ply": {k: torch.from_numpy(v) for k, v in captured["ply"].items()}, "table": table, "nn_idx": nn_idx,
                "max_idx": max_idx, "P": 3, "keys": captured["keys"], "sampled": sampled}, os.path.join(OUT, "ref_mesh.pt"))


if __name__ == "__main__":
    run_reference_mesh()
