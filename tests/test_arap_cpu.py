"""The ARAP arithmetic shared with the CUDA kernel (animate3d_b200/csrc/a3d_arap_math.h), driven serially on the CPU through
tests/cpu_harness/arap_cpu.cpp, against the reference goldens (ref_arap.pt: outputs of systems/util.py's own functions) and the
oracle.  CPU-only; the harness runs the kernels' own edge gather (arap_gather) and arap_node, and the GPU wrapper (a3d_arap.cu)
adds only the sample indexing and the gradient scatter around them."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("h") / "arap_cpu.so")
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", os.path.join(ROOT, "tests", "cpu_harness", "arap_cpu.cpp"), "-o", out])
    lib = C.CDLL(out)
    lib.arap_cpu.restype = C.c_double
    return lib


def fp(a):
    return a.ctypes.data_as(C.c_void_p)


def dense_graph(ii, jj, nn, nv, K):
    nbr = np.full((nv, K), -1, np.int32)
    nbr[ii.numpy(), nn.numpy()] = jj.numpy().astype(np.int32)
    return nbr


def test_energy_and_gradient_match_reference(harness, golden_dir):
    d = torch.load(os.path.join(golden_dir, "ref_arap.pt"), weights_only=False)
    nodes = np.ascontiguousarray(d["nodes"].numpy().astype(np.float32))
    nt, nv, _ = nodes.shape
    K = d["K"]
    nbr = dense_graph(d["ii"], d["jj"], d["nn"], nv, K)
    w = (nbr >= 0).astype(np.float32)                        # weight=None in the reference call: 1 on existing edges
    for key, idx in (("all", np.arange(nv, dtype=np.int32)), ("sub", d["sample_idx"].numpy().astype(np.int32))):
        grad = np.zeros_like(nodes)
        e = harness.arap_cpu(fp(nodes), nt, nv, fp(nbr), K, fp(np.ascontiguousarray(w)), fp(np.ascontiguousarray(idx)), len(idx),
                             fp(grad))
        want_e, want_g = float(d[f"err_{key}"]), d[f"grad_{key}"].numpy()
        assert abs(e - want_e) <= 2e-4 * abs(want_e) + 1e-7, (key, e, want_e)
        assert np.abs(grad - want_g).max() <= 2e-3 * np.abs(want_g).max() + 1e-7, key


def test_rotation_matches_reference_estimate(harness, golden_dir):
    """R from Horn's quaternion form == the reference's SVD form (incl. the reflection fix) on the golden's per-node
    covariances, and on random covariances with negative determinant."""
    from oracle import arap_oracle as A
    d = torch.load(os.path.join(golden_dir, "ref_arap.pt"), weights_only=False)
    nodes, K = d["nodes"], d["K"]
    nv = nodes.shape[1]
    se = A.edge_matrix(nodes[0], nv, K, d["ii"], d["jj"], d["nn"])
    te = A.edge_matrix(nodes[2], nv, K, d["ii"], d["jj"], d["nn"])
    S = torch.bmm(se.permute(0, 2, 1), torch.bmm(torch.diag_embed(d["weight"]), te))
    moved = ~((se == te).all(dim=1).any(dim=1))
    for i in torch.nonzero(moved).flatten().tolist()[:60]:
        s9 = np.ascontiguousarray(S[i].numpy().astype(np.float32).reshape(9))
        r9 = np.zeros(9, np.float32)
        harness.arap_rotation_cpu(fp(s9), fp(r9))
        np.testing.assert_allclose(r9.reshape(3, 3), d["rot_0_2"][i].numpy(), rtol=0, atol=3e-4)
    g = torch.Generator().manual_seed(8)
    for _ in range(40):
        m = torch.randn(3, 3, generator=g)
        if torch.det(m) > 0:
            m[:, 0] = -m[:, 0]                                # force the reflection branch of the reference
        u, sig, v = torch.svd(m[None])
        r = torch.bmm(v, u.permute(0, 2, 1))
        um = u.clone()
        um[0, :, torch.argmin(sig[0])] *= -1
        r = torch.bmm(v, um.permute(0, 2, 1))[0]
        r9 = np.zeros(9, np.float32)
        harness.arap_rotation_cpu(fp(np.ascontiguousarray(m.numpy().reshape(9))), fp(r9))
        np.testing.assert_allclose(r9.reshape(3, 3), r.numpy(), rtol=0, atol=5e-4)
    r9 = np.zeros(9, np.float32)
    harness.arap_rotation_cpu(fp(np.zeros(9, np.float32)), fp(r9))
    np.testing.assert_array_equal(r9.reshape(3, 3), np.eye(3, dtype=np.float32))
