"""The float64 ARAP / KNN oracle (oracle/arap_abi_oracle.py) without a GPU: it matches the reference-pinned
oracle/arap_oracle.py at float64 inputs, float64 Horn equals the reference's SVD rotation with its reflection fix, the
kernel's own arithmetic (a3d_arap_math.h through tests/cpu_harness/arap_cpu.cpp) passes every bound on the inputs of the
GPU cases (tests/test_arap_abi_oracle_gpu.py imports them from here), and the comparator rejects wrong kernels by a wide
margin.  The case generators live here so that both files run the same inputs."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import arap_abi_oracle as O
from oracle import arap_oracle as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ inputs
def rot(axis, angle):
    a = torch.as_tensor(axis, dtype=torch.float64)
    a = a / a.norm()
    k = torch.tensor([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]], dtype=torch.float64)
    return torch.eye(3, dtype=torch.float64) + math.sin(angle) * k + (1 - math.cos(angle)) * (k @ k)


def knn_table(x: torch.Tensor, K: int) -> torch.Tensor:
    """The K nearest other points of a small cloud in float64, (distance, index) order: [n, K] int32."""
    d = torch.cdist(x.double(), x.double())
    return torch.sort(d, dim=1, stable=True)[1][:, 1:K + 1].to(torch.int32).contiguous()


def grid_case(Nv=50000, Nt=16, Ns=512, seed=0):
    """Shipped size: 50 000 nodes on a jittered 37^3 grid, K = 3 neighbours (the next grid point along x, y and z, or the
    previous one at the far faces), 16 frames of a smooth deformation, 512 samples with repeats."""
    g = torch.Generator().manual_seed(seed)
    m = 37
    ar = torch.arange(Nv)
    cx, cy = ar % m, (ar // m) % m
    x = torch.stack([cx, cy, ar // (m * m)], 1).double() / m + 0.004 * torch.randn(Nv, 3, generator=g, dtype=torch.float64)
    nbr = torch.stack([torch.where(cx < m - 1, ar + 1, ar - 1), torch.where(cy < m - 1, ar + m, ar - m),
                       torch.where(ar + m * m < Nv, ar + m * m, ar - m * m)], 1).to(torch.int32)
    frames = [x]
    for t in range(1, Nt):
        r = rot([1, 2, 3], 0.02 * t)
        frames.append(x @ r.T + 0.01 * torch.sin(3 * x + t) + 0.002 * torch.randn(Nv, 3, generator=g, dtype=torch.float64))
    sample = torch.randint(0, Nv, (Ns,), generator=g)
    sample[:40] = sample[40:80]                   # repeated samples
    return dict(nodes=torch.stack(frames).float(), nbr=nbr, weight=None, sample=sample.to(torch.int32))


def cloud(n, seed, spread=(1.0, 1.0, 1.0)):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, generator=g, dtype=torch.float64) * torch.tensor(spread, dtype=torch.float64)


def motion(x, Nt, kind, seed, noise=0.003):
    g = torch.Generator().manual_seed(seed)
    out = [x]
    for t in range(1, Nt):
        if kind == "smooth":
            y = x @ rot([0.3, -1, 0.5], 0.15 * t).T + 0.02 * torch.sin(4 * x + t) + noise * torch.randn(x.shape, generator=g, dtype=torch.float64)
        elif kind == "unmoved":
            y = x
        elif kind == "axis":          # x unchanged, y and z move
            y = x.clone()
            y[:, 1:] = x[:, 1:] @ rot([1, 0, 0], 0.2 * t)[1:, 1:].T + 0.01 * torch.randn(x.shape[0], 2, generator=g, dtype=torch.float64)
        elif kind == "rigid":
            ang = [math.radians(179.9), math.pi, 1.0, math.radians(179.99)][(t - 1) % 4]
            y = x @ rot([1, 1, -2 + t], ang).T + torch.tensor([0.3, -0.2, 0.1 * t], dtype=torch.float64)
        elif kind == "mirror":
            y = x * torch.tensor([1.0, 1.0, -1.0], dtype=torch.float64) + 0.002 * t * torch.randn(x.shape, generator=g, dtype=torch.float64)
        elif kind == "affine":        # keeps collinear edges collinear and coplanar ones coplanar
            y = x @ (rot([1, 2, 0.5], 0.4 * t) * (1 + 0.1 * t)).T + 0.1 * t
        else:
            raise ValueError(kind)
        out.append(y)
    return torch.stack(out)


def small_case(kind="smooth", n=600, Nt=3, K=3, seed=1, scale=1.0, offset=0.0, spread=(1.0, 1.0, 1.0), weight=None,
               sample=None):
    """A random cloud of n nodes, its K-nearest table, `kind` of motion; the whole sequence is then scaled by `scale` and
    shifted by `offset`."""
    x = cloud(n, seed, spread)
    nodes = motion(x, Nt, kind, seed + 1) * scale + offset
    return dict(nodes=nodes.float(), nbr=knn_table(x, K), weight=weight, sample=sample)


def line_case(Nt=4, seed=3):
    """Collinear frame-0 edges (points on a line, neighbours along it) moved by an affine map: rank-1 S, K = 3."""
    g = torch.Generator().manual_seed(seed)
    lam = torch.sort(torch.rand(300, generator=g, dtype=torch.float64))[0]
    x = torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64) + lam[:, None] * torch.tensor([0.6, -0.3, 0.2], dtype=torch.float64)
    return dict(nodes=motion(x, Nt, "affine", seed).float(), nbr=knn_table(x, 3), weight=None, sample=None)


def plane_case(Nt=4, seed=4):
    """Coplanar frame-0 edges (z = 0.5), rank-2 S, under smooth motion (K = 4)."""
    x = cloud(500, seed)
    x[:, 2] = 0.5
    return dict(nodes=motion(x, Nt, "smooth", seed).float(), nbr=knn_table(x, 4), weight=None, sample=None)


def graph_case(seed=5, Nt=4, K=6):
    """-1 at interior slots, entries >= Nv, self-edges, a hub node that ~500 nodes point to, explicit weights with zeros
    and with non-zero weights on absent slots, and a sample with repeats, -1 and Nv entries."""
    n = 1500
    x = cloud(n, seed)
    nbr = knn_table(x, K).clone()
    g = torch.Generator().manual_seed(seed)
    nbr[0::7, 1] = -1
    nbr[3::11, 2] = n + 5
    nbr[5::13, 0] = torch.arange(5, n, 13, dtype=torch.int32)        # self-edges
    nbr[1:1000:2, K - 1] = 7                                          # hub node 7
    w = torch.rand(n, K, generator=g) + 0.2
    w[2::9, 3] = 0.0
    nodes = motion(x, Nt, "smooth", seed + 1).float()
    sample = torch.randint(0, n, (700,), generator=g)
    sample[:50] = sample[50:100]
    sample[100] = -1
    sample[101] = n
    sample[102:110] = 7
    return dict(nodes=nodes, nbr=nbr, weight=w, sample=sample.to(torch.int32))


def arap_cases(big=True):
    """(name, inputs) of every ARAP case that needs no device-side input."""
    c = []
    if big:
        c.append(("shipped 50k x 16, K 3, 512 samples", grid_case()))
        c.append(("shipped 50k x 16, sample NULL", dict(grid_case(), sample=None)))
    for K in (1, 2, 10, 12):
        c.append((f"K={K}", small_case(K=K, n=800, Nt=3, seed=10 + K)))
    c.append(("Nt=1", small_case(Nt=1, seed=20)))
    c.append(("Nt=2", small_case(Nt=2, seed=21)))
    c.append(("Ns > Nv", small_case(n=300, seed=22, sample=torch.randint(0, 300, (1000,), generator=torch.Generator().manual_seed(1)).to(torch.int32))))
    c.append(("one node x 64", small_case(n=300, seed=23, sample=torch.full((64,), 17, dtype=torch.int32))))
    c.append(("entries -1 and Nv only", small_case(n=300, seed=24, sample=torch.tensor([-1, 300, -1, 300], dtype=torch.int32))))
    c.append(("graph edges", graph_case()))
    gw = graph_case(seed=6)
    c.append(("graph, weight NULL", dict(gw, weight=None)))
    c.append(("weights all zero", dict(gw, weight=torch.zeros_like(gw["weight"]))))
    c.append(("unmoved", small_case("unmoved", seed=30)))
    c.append(("one axis unchanged", small_case("axis", seed=31)))
    c.append(("rigid 179.9 / 180 deg", small_case("rigid", Nt=5, seed=32)))
    c.append(("mirror", small_case("mirror", seed=33, spread=(1.0, 1.0, 0.2))))
    c.append(("collinear (rank 1)", line_case()))
    c.append(("coplanar (rank 2)", plane_case()))
    c.append(("offset 1e3, edges 1e-3", small_case(seed=34, scale=0.02, offset=1000.0)))
    c.append(("scale 1e-4", small_case(seed=35, scale=1e-4)))
    return c


# ------------------------------------------------------------------------------------------------ mesh (CPU CSR)
def mesh_csr(level=7, dangling=96, seed=7):
    """Icosphere (numpy, tools/mesh_bench.py's construction) plus `dangling` extra vertices of degree 1 or 2: vertices
    [V], CSR row_ptr / col (unique neighbours, ascending)."""
    from tools.mesh_bench import icosphere
    v, f = icosphere(level)
    V0 = v.shape[0]
    rng = np.random.default_rng(seed)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    extra_v, extra_e = [], []
    for k in range(dangling):
        a = int(rng.integers(V0))
        nv = V0 + k
        extra_v.append(v[a] * 1.02 + 0.001 * rng.standard_normal(3))
        extra_e.append([nv, a])
        if k % 2:                                      # degree 2: also a mesh neighbour of a
            b = e[e[:, 0] == a][0, 1]
            extra_e.append([nv, int(b)])
    v = np.concatenate([v, np.array(extra_v, np.float32)]).astype(np.float32)
    e = np.concatenate([e, np.array(extra_e)])
    e = np.unique(np.concatenate([e, e[:, ::-1]]), axis=0)
    V = v.shape[0]
    row_ptr = np.zeros(V + 1, np.int64)
    np.add.at(row_ptr, e[:, 0] + 1, 1)
    return v, np.cumsum(row_ptr).astype(np.int32), e[:, 1].astype(np.int32), V0


def mesh_nodes(v, Nt=17, seed=8):
    """Smooth motion with per-vertex noise well below the level-7 edge length (about 0.01)."""
    x = torch.from_numpy(v).double()
    return motion(x, Nt, "smooth", seed, noise=3e-4).float()


def mesh_sample_cpu(row_ptr, col, K, seed):
    """K distinct random neighbours per vertex, -1 past the degree (the layout of a3d_mesh_sample_neighbors)."""
    rng = np.random.default_rng(seed)
    V = row_ptr.size - 1
    out = np.full((V, K), -1, np.int32)
    for i in range(V):
        nb = col[row_ptr[i]:row_ptr[i + 1]]
        pick = rng.permutation(nb)[:K]
        out[i, :pick.size] = pick
    return torch.from_numpy(out)


def mesh_sample_idx(V, V0, seed=9):
    g = torch.Generator().manual_seed(seed)
    s = torch.randint(0, V, (512,), generator=g)
    return torch.cat([s, torch.arange(V0, V)]).to(torch.int32)         # plus every dangling vertex


# ------------------------------------------------------------------------------------------------ harness
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("h") / "arap_cpu.so")
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", os.path.join(ROOT, "tests", "cpu_harness", "arap_cpu.cpp"), "-o", out])
    lib = C.CDLL(out)
    lib.arap_cpu.restype = C.c_double
    return lib


def fp(a):
    return a.ctypes.data_as(C.c_void_p)


def run_harness(lib, case):
    nodes = np.ascontiguousarray(case["nodes"].numpy().astype(np.float32))
    nt, nv, _ = nodes.shape
    nbr = np.ascontiguousarray(case["nbr"].numpy().astype(np.int32))
    K = nbr.shape[1]
    w = None if case["weight"] is None else np.ascontiguousarray(case["weight"].numpy().astype(np.float32))
    s = np.arange(nv, dtype=np.int32) if case["sample"] is None else np.ascontiguousarray(case["sample"].numpy().astype(np.int32))
    grad = np.zeros_like(nodes)
    e = lib.arap_cpu(fp(nodes), nt, nv, fp(nbr), K, None if w is None else fp(w), fp(s), s.size, fp(grad))
    return torch.tensor([e], dtype=torch.float64), torch.from_numpy(grad)


def verdicts(case, err, grad, *, deterministic, what):
    """Every output against the oracle; asserts the bound and its tightness, returns {output: (Verdict, Tightness)}."""
    o = O.Arap(case["nodes"], case["nbr"], case["weight"], case["sample"])
    res = {}
    outs = {"err": (err, o.err(deterministic))}
    if grad is not None:
        outs["grad"] = (grad, o.grad())
    for name, (got, out) in outs.items():
        v = O.assert_within(got, out.ref, f"{what}: {name}")
        t = O.tightness(out)
        assert t.vacuous == 0, f"{what}: {name}: {t.vacuous} vacuous bounds (worst bound / magnitude {t.worst_mag:.3g})"
        res[name] = (v, t)
    return res, o.stats()


def line(what, res, stats):
    return f"{what} {stats}: " + "; ".join(
        f"{n} |err|/bound {v.ratio:.3g}, bound/|value| median {t.median_rel:.2g}, bound/magnitude worst {t.worst_mag:.2g}"
        for n, (v, t) in res.items())


# ------------------------------------------------------------------------------------------------ pins
def _dense(ii, jj, nn, nv, K):
    nbr = torch.full((nv, K), -1, dtype=torch.int32)
    nbr[ii, nn] = jj.to(torch.int32)
    return nbr


def _edge_list(nbr):
    nv, K = nbr.shape
    ii = torch.arange(nv)[:, None].expand(nv, K).reshape(-1)
    jj = nbr.long().reshape(-1)
    nn = torch.arange(K)[None].expand(nv, K).reshape(-1)
    keep = jj >= 0
    return ii[keep], jj[keep], nn[keep]


def _pin(nodes64, nbr, sample, weight=None):
    ii, jj, nn = _edge_list(nbr)
    K = nbr.shape[1]
    x = nodes64.clone().requires_grad_(True)
    e = A.arap_error(x, ii, jj, nn, K, weight=weight, sample_idx=None if sample is None else sample.long())
    e.backward()
    o = O.Arap(nodes64, nbr, weight, sample)
    got_e, got_g = o.err(True).ref.value, o.grad().ref.value.reshape(nodes64.shape)
    e = float(e.detach())
    assert abs(float(got_e[0]) - e) <= 1e-10 * abs(e), (float(got_e[0]), e)
    assert (got_g - x.grad).abs().max() <= 1e-10 * x.grad.abs().max(), float((got_g - x.grad).abs().max())


def test_float64_matches_pinned_oracle_on_golden(golden_dir):
    d = torch.load(os.path.join(golden_dir, "ref_arap.pt"), weights_only=False)
    nodes, K = d["nodes"].double(), d["K"]
    nbr = _dense(d["ii"], d["jj"], d["nn"], nodes.shape[1], K)
    _pin(nodes, nbr, None)
    _pin(nodes, nbr, d["sample_idx"].to(torch.int32))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_float64_matches_pinned_oracle_on_random(seed):
    x = cloud(400, 40 + seed)
    nodes = motion(x, 4, "smooth", seed)
    nbr = knn_table(x, 3 + seed).clone()
    nbr[::5, 1] = -1
    g = torch.Generator().manual_seed(seed)
    w = (torch.rand(400, nbr.shape[1], generator=g) + 0.1).double()
    _pin(nodes, nbr, torch.randint(0, 400, (300,), generator=g).to(torch.int32), weight=w)
    _pin(nodes, nbr, None)


def test_horn_equals_svd_with_reflection_fix():
    """float64 Horn == the reference's SVD + reflection fix on random S with det < 0, rank-2 S and 180-degree rotations."""
    g = torch.Generator().manual_seed(3)
    m = torch.randn(500, 3, 3, generator=g, dtype=torch.float64)
    neg = torch.det(m) > 0
    m[neg, :, 0] *= -1                                          # det < 0: the reflection branch
    u, _, vh = torch.linalg.svd(torch.randn(300, 3, 3, generator=g, dtype=torch.float64))
    sig = torch.rand(300, 3, generator=g, dtype=torch.float64) + 0.2
    sig[:, 2] = 0
    rank2 = u @ torch.diag_embed(sig) @ vh
    c = torch.randn(200, 3, 3, generator=g, dtype=torch.float64)
    cc = c @ c.transpose(1, 2) + 0.1 * torch.eye(3, dtype=torch.float64)
    axes = torch.randn(200, 3, generator=g, dtype=torch.float64)
    r180 = torch.stack([rot(a, math.pi) for a in axes])
    half = cc @ r180.transpose(1, 2)                            # S = C R^T: the rotation is R, at 180 degrees
    for name, S in (("det<0", m), ("rank 2", rank2), ("180 deg", half)):
        assert float(torch.det(m).max()) < 0
        h, s = O.horn_rotation(S), O.svd_rotation(S)
        assert (h - s).abs().max() < 1e-10, (name, float((h - s).abs().max()))
        assert (torch.det(h) - 1).abs().max() < 1e-12
    assert (O.svd_rotation(half) - r180).abs().max() < 1e-10
    # the reference's own estimate_rotation on one node per S (edges e = S's rows as s, identity t is not needed: use
    # s = I, t = S so that sum_n s_n t_n^T = S)
    for S in (m[:20], rank2[:20], half[:20]):
        eye = torch.eye(3, dtype=torch.float64)
        for k in range(S.shape[0]):
            src = torch.cat([torch.zeros(1, 3, dtype=torch.float64), -eye])       # node 0 at the origin, nodes 1..3 at -e_n
            tgt = torch.cat([torch.zeros(1, 3, dtype=torch.float64), -S[k]])      # so e_n = p_0 - p_n = row n
            ii, jj, nn = torch.zeros(3, dtype=torch.long), torch.arange(1, 4), torch.arange(3)
            r = A.estimate_rotation(src, tgt, ii, jj, nn, 3, torch.ones(1, 3, dtype=torch.float64), torch.tensor([0]))
            assert (r[0] - O.svd_rotation(S[k:k + 1])[0]).abs().max() < 1e-10


def test_harness_within_bounds(harness):
    """The kernel's arithmetic on the CPU passes every bound of every GPU case (unfused multiply-adds here, fused on the
    device: the bounds count each rounding, so they hold for both)."""
    for name, case in arap_cases():
        e, g = run_harness(harness, case)
        res, st = verdicts(case, e, g, deterministic=False, what=name)
        print("\n" + line(name, res, st))


def test_harness_mesh_within_bounds(harness):
    v, rp, col, V0 = mesh_csr(level=6)
    nodes = mesh_nodes(v)
    case = dict(nodes=nodes, nbr=mesh_sample_cpu(rp, col, 3, 1), weight=None, sample=mesh_sample_idx(v.shape[0], V0))
    assert int((case["nbr"] < 0).sum()) > 0
    e, g = run_harness(harness, case)
    res, st = verdicts(case, e, g, deterministic=False, what="mesh")
    assert st["rank1_family"] > 0, st                          # the degree-1 vertices reach the rank-1 derivation
    print("\n" + line("mesh", res, st))


def test_rank1_cases_use_the_family():
    for case in (line_case(), small_case(K=1, n=300, seed=50)):
        st = O.Arap(case["nodes"], case["nbr"]).stats()
        assert st["rank1_family"] > 0.9 * st["node_frames"], st


# ------------------------------------------------------------------------------------------------ negative controls
def emulate(case, variant=None):
    """A float64 ARAP with a deliberate defect (`variant`), on the fp32 edges of the case: (err [1], grad [Nt, Nv, 3])."""
    nodes, nbr, weight, sample = case["nodes"], case["nbr"].long(), case["weight"], case["sample"]
    Nt, Nv, _ = nodes.shape
    K = nbr.shape[1]
    idx = torch.arange(Nv) if sample is None else sample.long()
    if variant == "repeat_once":
        idx = torch.unique(idx)
    ok = (idx >= 0) & (idx < Nv)
    i = idx.clamp(0, Nv - 1)
    j = nbr[i]
    valid = ok[:, None] & (j >= 0) & (j < Nv)
    if variant == "minus1_as_node0":
        valid = ok[:, None] & (j < Nv)
        j = j.clamp(min=0)
    j = j.clamp(max=Nv - 1)
    w = valid.double() if weight is None else weight.double()[i] * valid
    if variant == "ignore_slot_weight":
        w[:, 0] = valid[:, 0].double()
    grad = torch.zeros(Nt, Nv, 3, dtype=torch.float64)
    err = torch.zeros(1, dtype=torch.float64)
    s = torch.where(valid[..., None], nodes[0][i][:, None] - nodes[0][j], torch.zeros(())).double()
    for t in range(1, Nt):
        tt = torch.where(valid[..., None], nodes[t][i][:, None] - nodes[t][j], torch.zeros(())).double()
        S = torch.einsum("mk,mka,mkb->mab", w, s, tt)
        same = (s == tt).all(1).any(-1)
        if variant != "no_same_axis":
            S[same] = 0
        u, sig, vh = torch.linalg.svd(S)
        R = vh.transpose(1, 2) @ u.transpose(1, 2)
        if variant != "no_reflection_fix":
            R = O.svd_rotation(S)
        R = torch.where((S == 0).flatten(1).all(1)[:, None, None], torch.eye(3, dtype=torch.float64), R)
        if variant == "R_transposed":
            R = R.transpose(1, 2)
        d = tt - torch.einsum("mab,mkb->mka", R, s)
        err += (w * (d * d).sum(-1)).sum()
        gt = 2 * w[..., None] * d
        g0 = -torch.einsum("mba,mkb->mka", R, gt) if variant != "g0_without_RT" else -gt
        m = valid.reshape(-1)
        ii = i[:, None].expand_as(j).reshape(-1)[m]
        jj = j.reshape(-1)[m]
        grad[t].index_add_(0, ii, gt.reshape(-1, 3)[m])
        grad[t].index_add_(0, jj, -gt.reshape(-1, 3)[m])
        if not (variant == "frame0_missing_one" and t == Nt - 1):
            grad[0].index_add_(0, ii, g0.reshape(-1, 3)[m])
            grad[0].index_add_(0, jj, -g0.reshape(-1, 3)[m])
    return err, grad


def _rotating_graph():
    c = graph_case(seed=60)
    x = c["nodes"][0].double()
    c["nodes"] = motion(x, 4, "smooth", 61).float()
    return c


CONTROLS = {
    "R_transposed": _rotating_graph,
    "no_reflection_fix": lambda: small_case("mirror", seed=62, spread=(1.0, 1.0, 0.2)),
    "no_same_axis": lambda: small_case("axis", seed=63),
    "ignore_slot_weight": _rotating_graph,
    "minus1_as_node0": _rotating_graph,
    "repeat_once": _rotating_graph,
    "frame0_missing_one": _rotating_graph,
    "g0_without_RT": _rotating_graph,
}


def test_emulator_passes_and_controls_fail():
    margins = {}
    cache = {}
    for variant, make in CONTROLS.items():
        key = make.__name__ if make is _rotating_graph else variant
        if key not in cache:
            cache[key] = make()
        case = cache[key]
        o = O.Arap(case["nodes"], case["nbr"], case["weight"], case["sample"])
        refs = {"err": o.err(True).ref, "grad": o.grad().ref}
        e0, g0 = emulate(case)
        for n, got in (("err", e0), ("grad", g0)):
            O.assert_within(got, refs[n], f"emulator {variant} case {n}")
        e, g = emulate(case, variant)
        margins[variant] = max(O.check(e, refs["err"]).ratio, O.check(g, refs["grad"]).ratio)
    print("\nARAP negative controls, |err| / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in margins.items()))
    print(f"smallest margin {min(margins.values()):.3g}")
    for k, v in margins.items():
        assert v >= 10, (k, v)


# ------------------------------------------------------------------------------------------------ KNN
def knn_emulate(p: torch.Tensor, K: int, variant=None):
    """The kernel's algorithm in numpy float32 (unfused): stable (d32, index) order, first dropped."""
    x = p.numpy().astype(np.float32)
    d = ((x[:, None, :] - x[None, :, :]) ** 2).sum(-1, dtype=np.float32)
    n = x.shape[0]
    if variant == "ties_by_higher_index":
        o = n - 1 - np.argsort(d[:, ::-1], axis=1, kind="stable")
    else:
        o = np.argsort(d, axis=1, kind="stable")
    take = o[:, 0:K] if variant == "self_not_dropped" else o[:, 1:K + 1]
    take = take.copy()
    if variant == "kth_missing":
        take[:, K - 1] = o[:, min(K + 3, n - 1)]
    dd = np.take_along_axis(d, take, 1)
    return torch.from_numpy(take.astype(np.int32)), torch.from_numpy(dd)


def lattice(m, spacing=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    ar = torch.arange(m ** 3)
    p = torch.stack([ar % m, (ar // m) % m, ar // (m * m)], 1).float() * spacing
    return p[torch.randperm(p.shape[0], generator=g)].contiguous()


def coincident(n=400, seed=1):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(n, 3, generator=g)
    p[100:140] = p[10]                       # 40 copies of point 10, later in index order
    p[5] = p[300]                            # a copy of a later point earlier in index order
    p[200:203] = p[201]
    return p


def knn_cases():
    g = torch.Generator().manual_seed(5)
    c = [("integer lattice 10^3, exact ties", lattice(10), 10),
         ("lattice spacing 0.1", lattice(9, 0.1), 6),
         ("coincident points", coincident(), 3),
         ("coincident points K=12", coincident(), 12)]
    for n in (127, 128, 129, 257):
        c.append((f"n={n}", torch.rand(n, 3, generator=g), 3))
    c.append(("n=K+1 (K=12)", torch.rand(13, 3, generator=g), 12))
    c.append(("n=K+1 (K=3)", torch.rand(4, 3, generator=g), 3))
    c.append(("K=n-1 (n=8)", torch.rand(8, 3, generator=g), 7))
    c.append(("K=1", torch.rand(500, 3, generator=g), 1))
    c.append(("K=12 random", torch.rand(3000, 3, generator=g), 12))
    return c


def test_knn_emulation_within_contract():
    for name, p, K in knn_cases():
        nbr, d2 = knn_emulate(p, K)
        v = O.knn_check(p, K, nbr, d2)
        print(f"\nknn {name}: worst {v.ratio:.3g}, unambiguous ranks {v.unambiguous:.3f}, dist2 bound/value median {v.median_rel:.2g}")
        assert v.ratio <= 1, (name, v)


def test_knn_coincident_rule():
    """Point i with a coincident lower-index point j: the lowest-index copy is the dropped first candidate, and i itself
    follows in (distance, index) order -- unless K lower-index copies come first."""
    p = coincident()
    nbr, _ = knn_emulate(p, 3)
    assert nbr[300].tolist()[0] == 300 and 5 not in nbr[300].tolist()     # one earlier copy (5): 300 lists itself
    assert nbr[202].tolist()[:2] == [201, 202]                            # copies 200 < 201 < 202: 200 dropped
    assert nbr[10].tolist() == [100, 101, 102]          # 10 is the lowest copy: its own dropped candidate
    assert nbr[120].tolist() == [100, 101, 102]         # 10 dropped, 120 not reached: 20 lower-index copies come first
    assert O.knn_order(p, 3)[2][120] == 10 and O.knn_order(p, 3)[2][300] == 5


def test_knn_controls_fail():
    margins = {}
    for variant, (p, K) in {"self_not_dropped": (torch.rand(300, 3, generator=torch.Generator().manual_seed(2)), 3),
                            "ties_by_higher_index": (lattice(8), 6),
                            "kth_missing": (torch.rand(300, 3, generator=torch.Generator().manual_seed(3)), 3)}.items():
        nbr, d2 = knn_emulate(p, K, variant)
        margins[variant] = O.knn_check(p, K, nbr, d2).ratio
    print("\nKNN negative controls, violation / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in margins.items()))
    for k, v in margins.items():
        assert v >= 10, (k, v)
