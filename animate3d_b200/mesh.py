"""Mesh animation on the engine (SURVEY 8f-5): what tools/mesh_animation/mesh2gaussian.py and the mesh mode of
custom/threestudio-animate3d/systems/animate3d.py (78-89, 222-234, 465-471) do around the recon and refine loops.

* `load_obj` + `corner_colours` + `mesh_to_gaussians`: mesh2gaussian.py:141-177.  The vertex graph and the per-vertex
  statistics run on the GPU (`a3d_mesh_adjacency`, `a3d_mesh_vertex_stats`) instead of the reference's per-corner `.item()`
  loops; the PLY goes through `io.write_gaussian_ply`, the adjacency JSON keeps find_and_save_connected_vertices' shape.
* `MeshGraph`: the mesh-edge ARAP graph as CSR on the device; `sample(K)` is the per-step neighbour draw
  (`a3d_mesh_sample_neighbors`), whose [V, K] output feeds `arap.cal_arap_error` through `edge_list`.
* `prepare_arap_from_mesh_vertices` / `sample_matrix_vectorized`: drop-ins with the signatures of systems/util.py:300-344.
* `save_mesh_trajectory`: the `mesh_trajectory/{i}.npy` export of animate3d.py:465-471.

The bindings call liba3d.so directly, like arap.py."""
from __future__ import annotations

import ctypes as C
import json
import os
from dataclasses import dataclass
from typing import Dict, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib as L
from .arap import drop_missing_edges

C0 = 0.28209479177387814
MAX_K = 12


# ---------------------------------------------------------------- OBJ reader

@dataclass
class ObjMesh:
    verts: np.ndarray                  # [V,3] float32
    faces: np.ndarray                  # [F,3] int64, fan-triangulated
    verts_uvs: np.ndarray              # [T,2] float32
    faces_uvs: np.ndarray              # [F,3] int64
    texture: np.ndarray                # [H,W,3] float32 in [0,1]


def _index(tok: str, count: int, total_ref: list, line_no: int, path: str) -> int:
    i = int(tok)
    if i == 0:
        raise ValueError(f"{path}:{line_no}: OBJ indices start at 1")
    if i < 0:
        total_ref.append((count, line_no))
        i = count + i
    else:
        i -= 1
    if not 0 <= i < count:
        raise ValueError(f"{path}:{line_no}: index {tok} is outside the {count} entries read so far")
    return i


def _read_mtl(path: str) -> Dict[str, str]:
    """{material name: map_Kd path} of a .mtl file (materials without map_Kd are left out)."""
    maps, cur = {}, None
    with open(path) as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "newmtl":
                cur = " ".join(tok[1:])
            elif tok[0] == "map_Kd" and cur is not None:
                maps[cur] = os.path.join(os.path.dirname(path), tok[-1])
    return maps


def load_obj(path: str) -> ObjMesh:
    """`pytorch3d.io.load_objs_as_meshes([path])` for a single-texture mesh: `v`, `vt` (first two components) and `f` in the
    `v`, `v/vt`, `v/vt/vn` and `v//vn` forms, 1-based or negative (relative) indices, polygons fanned as (v0, vk, vk+1).
    The texture is the `map_Kd` of the mtllib, loaded as PIL RGB / 255.  Raises ValueError where pytorch3d would not
    give the same mesh: no texture, more than one textured material, a face without `vt` while a texture is present, or a
    negative index followed by more vertices (pytorch3d counts those from the end of the file)."""
    verts, uvs, faces, fuvs = [], [], [], []
    mtllibs, no_vt_line, negs_v, negs_t = [], None, [], []
    with open(path) as f:
        for line_no, line in enumerate(f, 1):
            tok = line.split()
            if not tok or tok[0].startswith("#"):
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "vt":
                uvs.append([float(x) for x in tok[1:3]])
            elif tok[0] == "mtllib":
                mtllibs.append(os.path.join(os.path.dirname(path), " ".join(tok[1:])))
            elif tok[0] == "f":
                if len(tok) < 4:
                    raise ValueError(f"{path}:{line_no}: a face needs at least 3 corners")
                vi, ti = [], []
                for corner in tok[1:]:
                    parts = corner.split("/")
                    vi.append(_index(parts[0], len(verts), negs_v, line_no, path))
                    if len(parts) > 1 and parts[1]:
                        ti.append(_index(parts[1], len(uvs), negs_t, line_no, path))
                if ti and len(ti) != len(vi):
                    raise ValueError(f"{path}:{line_no}: some corners of the face have a vt and some do not")
                if not ti and no_vt_line is None:
                    no_vt_line = line_no
                for k in range(1, len(vi) - 1):
                    faces.append([vi[0], vi[k], vi[k + 1]])
                    fuvs.append([ti[0], ti[k], ti[k + 1]] if ti else [-1, -1, -1])
    for negs, total, what in ((negs_v, len(verts), "vertices"), (negs_t, len(uvs), "texture coordinates")):
        for count, line_no in negs:
            if count != total:
                raise ValueError(f"{path}:{line_no}: negative index followed by more {what}; pytorch3d would count it from "
                                 "the end of the file")
    if not faces:
        raise ValueError(f"{path}: no faces")
    maps: Dict[str, str] = {}
    for lib in mtllibs:
        if not os.path.exists(lib):
            raise ValueError(f"{path}: material library {lib} is missing")
        maps.update(_read_mtl(lib))
    if not maps:
        raise ValueError(f"{path}: the mesh has no texture (no map_Kd in its material library); mesh2gaussian needs one")
    if len(set(maps.values())) > 1:
        raise ValueError(f"{path}: {len(maps)} textured materials; only single-texture meshes are supported")
    if no_vt_line is not None:
        raise ValueError(f"{path}:{no_vt_line}: face without texture coordinates on a textured mesh")
    from PIL import Image
    with Image.open(next(iter(maps.values()))) as im:
        tex = np.asarray(im.convert("RGB"), np.float32) / 255.0
    return ObjMesh(np.asarray(verts, np.float32).reshape(-1, 3), np.asarray(faces, np.int64), np.asarray(uvs, np.float32).reshape(-1, 2),
                   np.asarray(fuvs, np.int64), tex)


def corner_colours(texture: torch.Tensor, verts_uvs: torch.Tensor, faces_uvs: torch.Tensor) -> torch.Tensor:
    """pytorch3d v0.7.6 `TexturesUV.faces_verts_textures_packed` with TexturesUV's defaults: bilinear grid_sample of the
    y-flipped texture at 2 uv - 1, align_corners=True, padding_mode="border".  texture [H,W,3] -> [F,3,3]."""
    maps = torch.flip(texture.float().permute(2, 0, 1)[None], [2])                        # [1,3,H,W]
    grid = (verts_uvs.float()[faces_uvs.long()] * 2 - 1)[None]                             # [1,F,3,2]
    out = torch.nn.functional.grid_sample(maps, grid, mode="bilinear", align_corners=True, padding_mode="border")
    return out[0].permute(1, 2, 0).contiguous()                                           # [F,3,3]


# ---------------------------------------------------------------- device graph

class MeshGraph:
    """CSR vertex graph on the device: row_ptr [V+1], col [E] int32, unique neighbours in ascending order per row."""

    def __init__(self, row_ptr: torch.Tensor, col: torch.Tensor):
        self.row_ptr = row_ptr.to(torch.int32).contiguous()
        self.col = col.to(torch.int32).contiguous()
        self.num_points = self.row_ptr.numel() - 1

    @property
    def degree(self) -> torch.Tensor:
        return self.row_ptr[1:] - self.row_ptr[:-1]

    @classmethod
    def from_faces(cls, faces: torch.Tensor, num_points: int) -> "MeshGraph":
        """a3d_mesh_adjacency: faces [F,3] (device) -> graph.  One host sync (the edge count)."""
        lib = L.load()
        f = faces.to(torch.int32).contiguous()
        nf = f.shape[0]
        if nf < 1 or num_points < 1:
            raise ValueError("a mesh graph needs at least one face and one vertex")
        if bool(((f < 0) | (f >= num_points)).any()):
            raise ValueError(f"face indices must lie in [0, {num_points})")
        row_ptr = torch.empty(num_points + 1, dtype=torch.int32, device=f.device)
        col = torch.empty(6 * nf, dtype=torch.int32, device=f.device)
        nbytes = lib.a3d_mesh_adjacency_scratch_bytes(num_points, nf)
        scratch = L.scratch(nbytes, f.device)
        count = torch.zeros(1, dtype=torch.int64).pin_memory()
        L.check(lib.a3d_mesh_adjacency(C.c_void_p(f.data_ptr()), nf, num_points, C.c_void_p(row_ptr.data_ptr()),
                                       C.c_void_p(col.data_ptr()), C.c_void_p(count.data_ptr()), C.c_void_p(L.ptr(scratch)),
                                       C.c_size_t(nbytes), L.stream_ptr()))
        torch.cuda.current_stream().synchronize()
        return cls(row_ptr, col[:int(count[0])])

    @classmethod
    def from_connected_vertices(cls, path_or_dict: Union[str, dict], num_points: int, device="cuda") -> "MeshGraph":
        """The adjacency JSON of mesh2gaussian (`{v: {n: distance}}`).  Vertices absent from it get empty rows."""
        info = path_or_dict
        if isinstance(info, str):
            with open(info) as f:
                info = json.load(f)
        keys = np.fromiter((int(k) for k in info), np.int64, len(info))
        lens = np.fromiter((len(v) for v in info.values()), np.int64, len(info))
        nbrs = np.fromiter((int(n) for v in info.values() for n in v), np.int64, int(lens.sum()))
        for what, arr in (("vertex", keys), ("neighbour", nbrs)):
            bad = arr[(arr < 0) | (arr >= num_points)]
            if bad.size:
                raise ValueError(f"connected-vertices table names {what} {int(bad[0])}, outside [0, {num_points})")
        key = np.unique(np.repeat(keys, lens) * num_points + nbrs)
        row_ptr = np.zeros(num_points + 1, np.int64)
        np.cumsum(np.bincount(key // num_points, minlength=num_points), out=row_ptr[1:])
        return cls(torch.from_numpy(row_ptr.astype(np.int32)).to(device), torch.from_numpy((key % num_points).astype(np.int32)).to(device))

    sample_state: Optional[torch.Tensor] = None     # device int64 [2] (seed, next offset) of captured draws

    def set_sample_state(self, seed: int, offset: int = 0) -> None:
        """Seed the draws of `sample` inside CUDA-graph captures: replay k of a graph that captured one `sample(K)` writes
        the table of the eager `sample(K, seed, offset + k)`.  Call it outside the capture; `sample_offset()` reads where
        the state has got to."""
        if not (0 <= seed < 2 ** 63 and 0 <= offset < 2 ** 63):
            raise ValueError("seed and offset must lie in [0, 2^63)")
        self.sample_state = torch.tensor([seed, offset], dtype=torch.int64, device=self.row_ptr.device)

    def sample_offset(self) -> int:
        """The offset the next captured draw will use (one host read)."""
        return int(self.sample_state[1])

    def sample(self, K: int, seed: Optional[int] = None, offset: int = 0) -> torch.Tensor:
        """K <= 12 distinct random neighbours per vertex -> nbr [V, K] int32, -1 past the degree (a3d_mesh_sample_neighbors).
        `seed` defaults to a draw from torch's default CPU generator (no device sync), so torch.manual_seed fixes a run.
        Inside a CUDA-graph capture the (seed, offset) come from the device state of `set_sample_state`, and every
        replay advances its offset (a3d_mesh_sample_neighbors_state)."""
        if not 1 <= K <= MAX_K:
            raise ValueError(f"K must be in [1, {MAX_K}], got {K}")
        capturing = torch.cuda.is_current_stream_capturing()
        if capturing and (seed is not None or offset or self.sample_state is None):
            raise ValueError("a captured MeshGraph.sample draws from the device state: call set_sample_state(seed, offset) "
                             "before the capture and pass neither seed nor offset")
        if seed is None and not capturing:
            seed = int(torch.randint(0, 2 ** 62, (1,)))
        lib = L.load()
        nbr = torch.empty(self.num_points, K, dtype=torch.int32, device=self.row_ptr.device)
        col = self.col if self.col.numel() else self.row_ptr       # any valid pointer: an edgeless graph reads no col entry
        if capturing:
            L.check(lib.a3d_mesh_sample_neighbors_state(C.c_void_p(self.row_ptr.data_ptr()), C.c_void_p(col.data_ptr()),
                                                        self.num_points, K, C.c_void_p(self.sample_state.data_ptr()),
                                                        C.c_void_p(nbr.data_ptr()), L.stream_ptr()))
        else:
            L.check(lib.a3d_mesh_sample_neighbors(C.c_void_p(self.row_ptr.data_ptr()), C.c_void_p(col.data_ptr()), self.num_points,
                                                  K, seed, offset, C.c_void_p(nbr.data_ptr()), L.stream_ptr()))
        return nbr


def edge_list(nbr: torch.Tensor):
    """(ii, jj, nn) of a sampled [V, K] table, as systems/animate3d.py:227-234 builds them for cal_arap_error."""
    nv, K = nbr.shape
    ii = torch.arange(nv, device=nbr.device)[:, None].expand(nv, K).reshape(-1)
    jj = nbr.long().reshape(-1)
    nn = torch.arange(K, device=nbr.device)[None].expand(nv, K).reshape(-1)
    return drop_missing_edges(ii, jj, nn)


def vertex_stats(verts: torch.Tensor, graph: MeshGraph, faces: Optional[torch.Tensor] = None,
                 corner_rgb: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """a3d_mesh_vertex_stats -> (mean_abs_edge [V,3], vertex_rgb [V,3] or None when corner_rgb is None)."""
    lib = L.load()
    v = verts.float().contiguous()
    nv = v.shape[0]
    if nv != graph.num_points:
        raise ValueError(f"{nv} vertices for a graph of {graph.num_points}")
    mae = torch.empty(nv, 3, device=v.device)
    rgb = f = cr = None
    nf = 0
    if corner_rgb is not None:
        f = faces.to(torch.int32).contiguous()
        nf = f.shape[0]
        cr = corner_rgb.float().contiguous()
        if cr.shape != (nf, 3, 3):
            raise ValueError(f"corner colours must be [F,3,3] = [{nf},3,3], got {tuple(cr.shape)}")
        rgb = torch.empty(nv, 3, device=v.device)
    nbytes = lib.a3d_mesh_vertex_stats_scratch_bytes(nv, nf, int(cr is not None))
    scratch = L.scratch(nbytes, v.device)
    col = graph.col if graph.col.numel() else graph.row_ptr
    L.check(lib.a3d_mesh_vertex_stats(C.c_void_p(v.data_ptr()), nv, C.c_void_p(graph.row_ptr.data_ptr()), C.c_void_p(col.data_ptr()),
                                      C.c_void_p(L.ptr(f)), nf, C.c_void_p(L.ptr(cr)), C.c_void_p(mae.data_ptr()),
                                      C.c_void_p(L.ptr(rgb)), C.c_void_p(L.ptr(scratch)), C.c_size_t(nbytes), L.stream_ptr()))
    return mae, rgb


# ---------------------------------------------------------------- mesh2gaussian

def mesh_to_gaussians(obj_path: str, device="cuda") -> Tuple[Dict[str, np.ndarray], MeshGraph]:
    """mesh2gaussian.py:141-177: one gaussian per vertex.  Returns the PLY fields (float32, `io.write_gaussian_ply`'s
    arguments) and the vertex graph.  xyz = vertices, f_dc = (rgb - 0.5) / C0, scale = log(mean |edge| / 1.1), identity
    rotation, opacity = logit(1 - 1e-5).  As in the reference, a vertex no face references has scale -inf."""
    mesh = load_obj(obj_path)
    verts = torch.from_numpy(mesh.verts).to(device)
    faces = torch.from_numpy(mesh.faces).to(device)
    graph = MeshGraph.from_faces(faces, verts.shape[0])
    crgb = corner_colours(torch.from_numpy(mesh.texture).to(device), torch.from_numpy(mesh.verts_uvs).to(device),
                          torch.from_numpy(mesh.faces_uvs).to(device))
    mae, rgb = vertex_stats(verts, graph, faces, crgb)
    mae, rgb = mae.cpu().numpy(), rgb.cpu().numpy()
    n = mesh.verts.shape[0]
    with np.errstate(divide="ignore"):
        scale = np.log(mae / 1.1)                     # float32 like the reference's numpy arithmetic
    x = np.ones((n, 1)) - 0.00001
    fields = {"xyz": mesh.verts, "f_dc": ((rgb - 0.5) / C0).astype(np.float32), "opacity": np.log(x / (1 - x)).astype(np.float32),
              "scale": scale.astype(np.float32), "rotation": np.tile(np.array([[1, 0, 0, 0]], np.float32), (n, 1))}
    return fields, graph


def connected_vertices(verts: np.ndarray, graph: MeshGraph) -> dict:
    """find_and_save_connected_vertices' table {str(v): {str(n): |v - n|}} for every vertex with an edge (ascending)."""
    row_ptr, col = graph.row_ptr.cpu().numpy().astype(np.int64), graph.col.cpu().numpy().astype(np.int64)
    v = np.asarray(verts, np.float32)
    src = np.repeat(np.arange(graph.num_points), np.diff(row_ptr))
    d = v[src] - v[col]
    dist = np.sqrt((d * d).sum(-1, dtype=np.float32)).tolist()
    cols = col.tolist()
    out = {}
    for i in np.nonzero(np.diff(row_ptr))[0].tolist():
        b, e = int(row_ptr[i]), int(row_ptr[i + 1])
        out[str(i)] = {str(cols[k]): dist[k] for k in range(b, e)}
    return out


def write_mesh_gaussians(obj_path: str, output_dir: str, output_name: str, device="cuda") -> Tuple[str, str]:
    """mesh2gaussian.py main(): `{output_name}.ply` and `{output_name}.json` under output_dir; returns both paths."""
    from .io import write_gaussian_ply
    os.makedirs(output_dir, exist_ok=True)
    fields, graph = mesh_to_gaussians(obj_path, device)
    ply = os.path.join(output_dir, f"{output_name}.ply")
    js = os.path.join(output_dir, f"{output_name}.json")
    write_gaussian_ply(ply, fields["xyz"], fields["f_dc"], fields["opacity"], fields["scale"], fields["rotation"])
    with open(js, "w") as f:
        json.dump(connected_vertices(fields["xyz"], graph), f, indent=2)
    return ply, js


# ---------------------------------------------------------------- drop-ins for systems/util.py:300-344

def prepare_arap_from_mesh_vertices(connected_vertices_info: dict) -> Tuple[torch.Tensor, torch.Tensor]:
    """util.py:300-318 (host): (nn_idx [Nv, max_degree] int64, -1 padded, neighbours in the table's order; nn_idx != -1),
    with Nv = the number of keys.  Raises ValueError where the reference raises IndexError (a key >= Nv)."""
    nv = len(connected_vertices_info)
    width = max((len(v) for v in connected_vertices_info.values()), default=0)
    nn_idx = np.full((nv, width), -1, np.int64)
    for key, val in connected_vertices_info.items():
        k = int(key)
        if not 0 <= k < nv:
            raise ValueError(f"connected-vertices key {k} outside [0, {nv}) (the table has {nv} keys)")
        nn_idx[k, :len(val)] = [int(t) for t in val.keys()]
    nn_idx = torch.from_numpy(nn_idx)
    return nn_idx, nn_idx != -1


def sample_matrix_vectorized(input_matrix: torch.Tensor, P: int, max_index: torch.Tensor) -> torch.Tensor:
    """util.py:320-344 on the kernel: min(P, D) distinct valid entries of every row of the dense table, in random order,
    -1 where the row has fewer -> [N, min(P, D)] int64 on the table's device (CUDA)."""
    n, d = input_matrix.shape
    k = min(P, d)
    mask = max_index.to(input_matrix.device).bool()
    row_ptr = torch.zeros(n + 1, dtype=torch.int32, device=input_matrix.device)
    row_ptr[1:] = torch.cumsum(mask.sum(1), 0)
    graph = MeshGraph(row_ptr, input_matrix[mask])
    return graph.sample(k).long()


# ---------------------------------------------------------------- trajectory export

@torch.no_grad()
def save_mesh_trajectory(geometry, folder: str, n_frame: int = 16, first_frame_trainable: bool = False) -> None:
    """animate3d.py:465-471: `{i}.npy` = float32 [P,3] means of frame i for timestamps linspace(-1, 1, n_frame)
    (data/simple_multi_image.py:167); frame 0 is the static `_xyz` unless the first frame is trainable."""
    os.makedirs(folder, exist_ok=True)
    ts = torch.linspace(-1, 1, n_frame, device=geometry._xyz.device)
    means, _, _ = geometry.deform_frames(ts, first_frame_trainable=first_frame_trainable)
    means = means.float().cpu().numpy()
    for i in range(n_frame):
        np.save(os.path.join(folder, f"{i}.npy"), means[i])
