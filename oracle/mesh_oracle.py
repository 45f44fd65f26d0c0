"""ORACLE (test infrastructure) -- mesh animation support (SURVEY 8f-5): tools/mesh_animation/mesh2gaussian.py (15-33
convert_to_textureVertex_with_average, 36-63 compute_edge_distances, 66-88 find_and_save_connected_vertices, 114-139
convert_point_cloud_to_gaussian, 141-177 main) and custom/threestudio-animate3d/systems/util.py:300-344
(prepare_arap_from_mesh_vertices, sample_matrix_vectorized), restated in numpy / torch on the CPU.

PINNED: the graph, statistics, gaussian fields, JSON table and both util.py functions are checked against the reference's
own functions executed on the CPU (pytorch3d / plyfile stubbed, `.cuda()` dropped) in
tests/golden/gen_mesh_goldens.py::run_reference_mesh -> ref_mesh.pt.

Neighbour sampling is restated twice: `sample_with_keys` takes the key matrix the reference draws with torch.rand and must
equal sample_matrix_vectorized; `sample_csr` draws the keys the kernel draws (Philox4x32-10 of (seed, offset, row, slot))
and must equal a3d_mesh_sample_neighbors bit for bit.  Both keep the K smallest keys in ascending order, ties by slot.

PARITY-UNPINNED: the corner colours.  The reference gets them from pytorch3d v0.7.6
`TexturesUV.faces_verts_textures_packed` (pytorch3d is not installed here, so this is not executed against it).  Restated
from that version: TexturesUV's defaults `sampling_mode="bilinear"`, `align_corners=True`, `padding_mode="border"`; the
uv coordinates map to grid_sample's [-1, 1] as 2 uv - 1 and the texture image is flipped in y first (uv origin at the
bottom-left, image rows top-down), as in its `sample_textures`.  The image is PIL RGB / 255 (pytorch3d.io.obj_io)."""
from __future__ import annotations

import json
import os
from typing import Dict, Tuple

import numpy as np
import torch

C0 = 0.28209479177387814

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def philox_word0(c0, c1, c2, c3, k0, k1) -> np.ndarray:
    """Philox4x32-10, word 0 of the output block, vectorised over numpy arrays (uint32 semantics)."""
    m32 = np.uint64(0xFFFFFFFF)
    c = [np.asarray(x, np.uint64) & m32 for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0) & m32, np.uint64(k1) & m32
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(_W0)) & m32, (k1 + np.uint64(_W1)) & m32
        p0, p1 = c[0] * np.uint64(_M0), c[2] * np.uint64(_M1)
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & m32, p1 >> np.uint64(32), p1 & m32
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return c[0].astype(np.uint32)


# ---------------------------------------------------------------- graph and statistics

def csr_from_faces(faces: np.ndarray, num_verts: int) -> Tuple[np.ndarray, np.ndarray]:
    """Unique undirected neighbours of every vertex (both directions of every face edge), ascending -> (row_ptr, col) int32."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a = np.concatenate([f[:, 0], f[:, 1], f[:, 2], f[:, 1], f[:, 2], f[:, 0]])
    b = np.concatenate([f[:, 1], f[:, 2], f[:, 0], f[:, 0], f[:, 1], f[:, 2]])
    key = np.unique(a * num_verts + b)
    src, dst = key // num_verts, key % num_verts
    row_ptr = np.zeros(num_verts + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=num_verts), out=row_ptr[1:])
    return row_ptr.astype(np.int32), dst.astype(np.int32)


def edge_stats(verts: np.ndarray, row_ptr: np.ndarray, col: np.ndarray) -> np.ndarray:
    """compute_edge_distances: mean |v_j - v_i| per axis over the row (fp32, summed in CSR order); 0 for an empty row."""
    v = np.asarray(verts, np.float32)
    deg = np.diff(row_ptr)
    s = np.zeros_like(v)
    for k in range(int(deg.max(initial=0))):
        rows = np.nonzero(deg > k)[0]
        s[rows] += np.abs(v[col[row_ptr[rows] + k]] - v[rows])
    out = np.zeros_like(v)
    nz = deg > 0
    out[nz] = s[nz] / deg[nz, None].astype(np.float32)
    return out


def vertex_rgb(faces: np.ndarray, corner_rgb: np.ndarray, num_verts: int) -> np.ndarray:
    """convert_to_textureVertex_with_average: fp32 index_add over corner slot 0, 1, 2 in face order, / count.clamp(min=1)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    cr = np.asarray(corner_rgb, np.float32).reshape(-1, 3, 3)
    s = np.zeros((num_verts, 3), np.float32)
    cnt = np.zeros(num_verts, np.float32)
    for k in range(3):
        np.add.at(s, f[:, k], cr[:, k])
        np.add.at(cnt, f[:, k], 1.0)
    return s / np.maximum(cnt, 1.0)[:, None]


def gaussian_fields(verts: np.ndarray, rgb: np.ndarray, mean_abs_edge: np.ndarray) -> Dict[str, np.ndarray]:
    """convert_point_cloud_to_gaussian called as main() calls it (max_lengths / 1.1), in the reference's dtypes; the values
    the PLY stores (float32).  A vertex no face references has mean_abs_edge 0 and scale -inf, as in the reference."""
    v = np.asarray(verts, np.float32)
    n = v.shape[0]
    with np.errstate(divide="ignore"):
        scale = np.log(np.asarray(mean_abs_edge, np.float32) / 1.1)
    rot = np.zeros((n, 4))
    rot[:, 0] = 1.0
    x = np.ones((n, 1)) - 0.00001
    return {"xyz": v, "f_dc": ((np.asarray(rgb, np.float32) - 0.5) / C0).astype(np.float32),
            "opacity": np.log(x / (1 - x)).astype(np.float32), "scale": scale.astype(np.float32),
            "rotation": rot.astype(np.float32)}


def connected_vertices(verts: np.ndarray, faces: np.ndarray) -> dict:
    """find_and_save_connected_vertices before json.dump: {v: {n: |v - n|}} in the reference's insertion order."""
    v = torch.as_tensor(np.asarray(verts, np.float32))
    out: dict = {}
    for face in np.asarray(faces, np.int64).reshape(-1, 3):
        for i in range(3):
            a, b = int(face[i]), int(face[(i + 1) % 3])
            d = torch.norm(v[a] - v[b]).item()
            out.setdefault(a, {})[b] = d
            out.setdefault(b, {})[a] = d
    return out


def json_roundtrip(table: dict) -> dict:
    """What json.dump / json.load make of a table: string keys."""
    return json.loads(json.dumps(table, indent=2))


# ---------------------------------------------------------------- util.py:300-344

def prepare_arap_from_mesh_vertices(info: dict) -> Tuple[torch.Tensor, torch.Tensor]:
    """util.py:300-318: dense [Nv, max_degree] int64 table (-1 padded, neighbours in the JSON's order), Nv = number of keys."""
    width = max((len(v) for v in info.values()), default=0)
    nn_idx = -torch.ones(len(info), width, dtype=torch.int64)
    for key, val in info.items():
        nn_idx[int(key)][:len(val)] = torch.tensor([int(t) for t in val.keys()], dtype=torch.int64)
    return nn_idx, nn_idx != -1


def sample_with_keys(input_matrix: torch.Tensor, P: int, max_index: torch.Tensor, keys: torch.Tensor) -> torch.Tensor:
    """util.py:320-344 given its torch.rand(N, D) draw `keys`: invalid slots get +1000, a row sort (ties by slot), sorted
    slots with a key >= 1000 become -1, which indexes the row's LAST column (-1 whenever the row has a free column)."""
    n = input_matrix.shape[0]
    k = keys.clone()
    k[~max_index] += 1000.0
    val, index = torch.sort(k, dim=1, stable=True)
    index[val >= 1000.0] = -1
    col = index[:, :P]
    return input_matrix[torch.arange(n)[:, None].expand(-1, col.shape[1]), col]


def sample_csr(row_ptr: np.ndarray, col: np.ndarray, K: int, seed: int, offset: int) -> np.ndarray:
    """a3d_mesh_sample_neighbors: slot j of row i keyed by philox_word0(i, j, offset_lo, offset_hi; seed_lo, seed_hi); the K
    smallest (key, j) in ascending order; -1 past the degree.  -> [V, K] int32."""
    row_ptr = np.asarray(row_ptr, np.int64)
    v = row_ptr.shape[0] - 1
    deg = np.diff(row_ptr)
    width = max(int(deg.max(initial=0)), K)
    i, j = np.meshgrid(np.arange(v), np.arange(width), indexing="ij")
    keys = philox_word0(i, j, offset & 0xFFFFFFFF, offset >> 32, seed & 0xFFFFFFFF, seed >> 32).astype(np.int64)
    keys[j >= deg[:, None]] = 1 << 40
    order = np.argsort(keys, axis=1, kind="stable")[:, :K]
    taken = np.take_along_axis(j, order, 1)
    ok = taken < deg[:, None]
    out = np.full((v, K), -1, np.int32)
    out[ok] = np.asarray(col)[(row_ptr[:-1, None] + taken)[ok]]
    return out


# ---------------------------------------------------------------- corner colours (parity-unpinned, see above)

def corner_colours(image: np.ndarray, verts_uvs: np.ndarray, faces_uvs: np.ndarray) -> np.ndarray:
    """Bilinear sample of image [H,W,3] at every face corner's uv (align_corners=True, border clamp, v = 0 at the bottom
    row) -> [F,3,3] float32, in float64 arithmetic."""
    img = np.asarray(image, np.float64)[::-1]
    h, w = img.shape[:2]
    uv = np.asarray(verts_uvs, np.float64)[np.asarray(faces_uvs, np.int64)]          # [F,3,2]
    x = np.clip(uv[..., 0] * (w - 1), 0, w - 1)
    y = np.clip(uv[..., 1] * (h - 1), 0, h - 1)
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
    fx, fy = (x - x0)[..., None], (y - y0)[..., None]
    out = (img[y0, x0] * (1 - fx) * (1 - fy) + img[y0, x1] * fx * (1 - fy) + img[y1, x0] * (1 - fx) * fy + img[y1, x1] * fx * fy)
    return out.astype(np.float32)


# ---------------------------------------------------------------- test fixture

def fixture_mesh(seed: int = 0, n_lat: int = 8, n_lon: int = 12):
    """A seeded textured mesh: a jittered UV sphere (poles as fans, a texture seam where u wraps from 1 back to 0), one
    quad floating beside it, and one last vertex no face references.  Returns (verts [V,3] f32, verts_uvs [T,2] f32,
    polygons: list of lists of (v, vt) 0-based, texture [H,W,3] uint8)."""
    rng = np.random.default_rng(seed)
    verts = [[0.0, 0.0, 1.0]]
    for a in range(1, n_lat):
        th = np.pi * a / n_lat
        for b in range(n_lon):
            ph = 2 * np.pi * b / n_lon
            verts.append([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
    verts.append([0.0, 0.0, -1.0])
    verts = np.asarray(verts) * (1 + 0.05 * rng.standard_normal((len(verts), 1)))
    uvs = [[(b + 0.5) / n_lon, 1.0] for b in range(n_lon)]                              # north pole, one per segment
    for a in range(1, n_lat):
        uvs += [[b / n_lon, 1 - a / n_lat] for b in range(n_lon + 1)]                   # u = 1 duplicates u = 0: the seam
    uvs += [[(b + 0.5) / n_lon, 0.0] for b in range(n_lon)]
    ring = lambda a, b: 1 + (a - 1) * n_lon + b % n_lon
    ring_uv = lambda a, b: n_lon + (a - 1) * (n_lon + 1) + b
    south, south_uv = len(verts) - 1, n_lon + (n_lat - 1) * (n_lon + 1)
    polys = []
    for b in range(n_lon):
        polys.append([(0, b), (ring(1, b), ring_uv(1, b)), (ring(1, b + 1), ring_uv(1, b + 1))])
        for a in range(1, n_lat - 1):
            q = [(ring(a, b), ring_uv(a, b)), (ring(a + 1, b), ring_uv(a + 1, b)), (ring(a + 1, b + 1), ring_uv(a + 1, b + 1)),
                 (ring(a, b + 1), ring_uv(a, b + 1))]
            polys += [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
        polys.append([(ring(n_lat - 1, b + 1), ring_uv(n_lat - 1, b + 1)), (ring(n_lat - 1, b), ring_uv(n_lat - 1, b)),
                      (south, south_uv + b)])
    nv, nt = len(verts), len(uvs)
    quad = np.array([[1.5, 0, 0], [2.0, 0.1, 0], [2.1, 0.6, 0.2], [1.6, 0.5, 0.1]])
    verts = np.concatenate([verts, quad, [[3.0, 3.0, 3.0]]])
    uvs += [[0.1, 0.1], [0.9, 0.15], [0.85, 0.9], [0.2, 0.8]]
    polys.append([(nv + k, nt + k) for k in range(4)])
    tex = rng.integers(0, 256, size=(8, 16, 3), dtype=np.uint8)
    return verts.astype(np.float32), np.asarray(uvs, np.float32), polys, tex


def write_fixture_obj(folder: str, seed: int = 0) -> str:
    """Writes fixture_mesh as mesh.obj + mesh.mtl + tex.png; faces in the v/vt and v/vt/vn forms, the quad with negative
    indices.  Returns the OBJ path."""
    from PIL import Image
    verts, uvs, polys, tex = fixture_mesh(seed)
    os.makedirs(folder, exist_ok=True)
    Image.fromarray(tex).save(os.path.join(folder, "tex.png"))
    with open(os.path.join(folder, "mesh.mtl"), "w") as f:
        f.write("newmtl skin\nKd 1 1 1\nmap_Kd tex.png\n")
    lines = ["# fixture", "mtllib mesh.mtl"]
    lines += [f"v {x:.9g} {y:.9g} {z:.9g}" for x, y, z in verts[:-5]]
    lines += [f"vt {u:.9g} {v:.9g}" for u, v in uvs[:-4]]
    lines += ["vn 0 0 1", "usemtl skin"]
    for n, p in enumerate(polys[:-1]):
        lines.append("f " + " ".join(f"{a + 1}/{t + 1}" if n % 2 else f"{a + 1}/{t + 1}/1" for a, t in p))
    lines += [f"v {x:.9g} {y:.9g} {z:.9g}" for x, y, z in verts[-5:]]                  # the quad, then the lone vertex
    lines += [f"vt {u:.9g} {v:.9g}" for u, v in uvs[-4:]]
    lines.append("f " + " ".join(f"{k - 1}/{k}" for k in (-4, -3, -2, -1)))
    path = os.path.join(folder, "mesh.obj")
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
    return path
