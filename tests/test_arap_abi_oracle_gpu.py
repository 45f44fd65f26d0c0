"""a3d_arap and a3d_knn_graph against the float64 oracle (oracle/arap_abi_oracle.py), element by element, through the C ABI
(so that null weight / sample / grad pointers are reachable).  Every ARAP case runs on the atomic and on the fixed-order
path into a grad buffer prefilled with NaN (both paths must overwrite it), checks err and the whole [Nt, Nv, 3] grad span,
runs the fixed-order path twice (torch.equal) and both paths once more with grad NULL.  The inputs are the CPU file's, where
the kernel's own arithmetic already passed the same bounds serially."""
import ctypes as C
import os
import sys
import time

import pytest
import torch

from oracle import arap_abi_oracle as O
from oracle import arap_oracle as A

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_arap_abi_oracle_cpu as S  # noqa: E402

pytestmark = pytest.mark.gpu


def _lib():
    from animate3d_b200 import _lib as L
    return L, L.load()


def _ptr(t):
    return C.c_void_p(None if t is None else t.data_ptr())


def _arap(case, det, with_grad=True):
    L, lib = _lib()
    nodes = case["nodes"].cuda().float().contiguous()
    nbr = case["nbr"].cuda().to(torch.int32).contiguous()
    w = None if case["weight"] is None else case["weight"].cuda().float().contiguous()
    s = None if case["sample"] is None else case["sample"].cuda().to(torch.int32).contiguous()
    Nt, Nv, _ = nodes.shape
    K = nbr.shape[1]
    Ns = Nv if s is None else s.numel()
    err = torch.full((1,), float("nan"), device="cuda")
    grad = torch.full_like(nodes, float("nan")) if with_grad else None
    nbytes = lib.a3d_arap_scratch_bytes(Nt, Nv, K, Ns, det)
    assert (nbytes > 0) == bool(det)
    scratch = L.scratch(nbytes, "cuda")
    L.check(lib.a3d_arap(_ptr(nodes), Nt, Nv, _ptr(nbr), K, _ptr(w), _ptr(s), Ns, det, _ptr(err), _ptr(grad), _ptr(scratch),
                         C.c_size_t(nbytes), L.stream_ptr()))
    torch.cuda.synchronize()
    return err, grad


def run_case(name, case):
    t0 = time.perf_counter()
    cuda = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in case.items()}
    o = O.Arap(cuda["nodes"], cuda["nbr"], cuda["weight"], cuda["sample"])
    gref = o.grad()
    lines = []
    outs = {}
    for det in (0, 1):
        path = "fixed-order" if det else "atomic"
        eref = o.err(bool(det))
        err, grad = _arap(case, det)
        outs[det] = (err, grad)
        for n, got, ref in (("err", err, eref), ("grad", grad, gref)):
            v = O.assert_within(got, ref.ref, f"{name} [{path}] {n}")
            t = O.tightness(ref)
            assert t.vacuous == 0, f"{name} [{path}] {n}: {t.vacuous} vacuous bounds (worst bound / magnitude {t.worst_mag:.3g})"
            lines.append(f"{path}/{n} |err|/bound {v.ratio:.3g} (bound/|value| median {t.median_rel:.2g}, bound/magnitude worst "
                         f"{t.worst_mag:.2g})")
        e2, _ = _arap(case, det, with_grad=False)
        O.assert_within(e2, eref.ref, f"{name} [{path}] err with grad NULL")
    e1, g1 = _arap(case, 1)
    assert torch.equal(e1, outs[1][0]) and torch.equal(g1, outs[1][1]), f"{name}: fixed-order path not reproducible"
    print(f"\n{name} {o.stats()} ({time.perf_counter() - t0:.2f} s): " + "; ".join(lines))


ARAP = S.arap_cases()


@pytest.mark.parametrize("name", [n for n, _ in ARAP])
def test_arap(name):
    run_case(name, dict(ARAP)[name])


def test_arap_mesh_mode():
    """The mesh-animation shape: a MeshGraph.sample(3) table on a 163 842-vertex icosphere plus 96 dangling vertices of
    degree 1 or 2 (trailing -1 slots; one-edge rank-1 fits), 17 frames, 512 samples plus every dangling vertex."""
    from animate3d_b200.mesh import MeshGraph
    v, rp, col, V0 = S.mesh_csr(level=7)
    nbr = MeshGraph(torch.from_numpy(rp).cuda(), torch.from_numpy(col).cuda()).sample(3, seed=11)
    assert int((nbr < 0).sum()) > 0
    case = dict(nodes=S.mesh_nodes(v), nbr=nbr.cpu(), weight=None, sample=S.mesh_sample_idx(v.shape[0], V0))
    run_case("mesh K=3, 163 938 vertices x 17", case)


# ------------------------------------------------------------------------------------------------ KNN
def _knn(p, K):
    from animate3d_b200 import arap
    return arap.knn_graph(p.cuda(), K)


def _knn_case(name, p, K):
    t0 = time.perf_counter()
    nbr, d2 = _knn(p, K)
    torch.cuda.synchronize()
    v = O.knn_check(p.cuda(), K, nbr, d2)
    print(f"\nknn {name} (n={p.shape[0]}, K={K}, {time.perf_counter() - t0:.2f} s): worst violation/bound {v.ratio:.3g}, "
          f"unambiguous ranks {v.unambiguous:.3f}, dist2 bound/value median {v.median_rel:.2g}")
    assert v.ratio <= 1, (name, v.where)
    return nbr, d2, v


@pytest.mark.parametrize("K", [3, 10])
def test_knn_50k(K):
    g = torch.Generator().manual_seed(K)
    _knn_case("50k random", torch.rand(50000, 3, generator=g), K)


@pytest.mark.parametrize("idx", range(len(S.knn_cases())))
def test_knn_cases(idx):
    name, p, K = S.knn_cases()[idx]
    _knn_case(name, p, K)


def test_knn_coincident_rule():
    """The a3d.h contract for coincident points, on the kernel: the lowest-index copy is dropped, i follows it."""
    p = S.coincident()
    nbr, _, _ = _knn_case("coincident", p, 3)
    nbr = nbr.cpu()
    assert nbr[300].tolist()[0] == 300 and 5 not in nbr[300].tolist()
    assert nbr[202].tolist()[:2] == [201, 202]
    assert nbr[10].tolist() == [100, 101, 102]
    assert nbr[120].tolist() == [100, 101, 102]
    ref, _ = S.knn_emulate(p, 3)
    assert torch.equal(nbr, ref)


@pytest.mark.parametrize("n,K,radius", [(3000, 3, 0.01), (800, 10, 0.1)])
def test_connectivity(n, K, radius):
    """cal_connectivity_from_points against arap_oracle.connectivity_from_points at float64: indices equal at every
    unambiguous rank, -1 on the same far edges, weights within their bound (where they are finite)."""
    from animate3d_b200 import arap
    g = torch.Generator().manual_seed(n)
    p = torch.rand(n, 3, generator=g) * (0.3 if K == 10 else 1.0)
    ii, jj, nn, w = arap.cal_connectivity_from_points(p[None].cuda(), radius=radius, K=K)
    oi, oj, on, ow = A.connectivity_from_points(p[None].double(), radius=radius, K=K)
    nbr, d2, v = _knn_case("connectivity", p, K)
    dense = torch.full((n, K), -1, dtype=torch.long)
    dense[ii.cpu(), nn.cpu()] = jj.cpu()
    odense = torch.full((n, K), -1, dtype=torch.long)
    odense[oi, on] = oj
    # the far-edge decision d >= radius^2 on fp32 dist2: ambiguous within the distance bound
    pairs = ((p.double()[:, None] - p.double()[nbr.cpu().long()]) ** 2).sum(-1)
    band = (pairs - radius ** 2).abs() <= O.knn_pair_bound(pairs, False)
    sure = v.checked.cpu() & ~band
    assert torch.equal(dense[sure], odense[sure])
    if K == 3:
        wb = O.connectivity_weight_bound(pairs, n * K)
        e = (w.cpu().double() - ow).abs()
        assert bool((e <= wb).all()), float((e / wb).max())
        print(f"\nconnectivity n={n} K={K}: weights worst |err|/bound {float((e / wb).max()):.3g}, "
              f"bound/value median {float((wb / ow).median()):.2g}; {int(sure.sum())} of {n * K} indices checked")
    else:
        assert torch.equal(torch.isnan(w.cpu()), torch.isnan(ow))
        print(f"\nconnectivity n={n} K={K}: {int(sure.sum())} of {n * K} indices checked, {int((odense < 0).sum())} far edges")
