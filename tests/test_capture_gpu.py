"""Motion-reconstruction and mesh-animation steps replayed from CUDA graphs (animate3d_b200/capture.py) against the eager
step.  Under torch.use_deterministic_algorithms(True) a replay must leave every parameter and Adam state bit-identical to an
eager step that is fed the same random draws (the gradient mask and the ARAP node sample, read back from the graph's
tensors).  That a capture succeeds at all shows the step makes no synchronising call.

Each case runs in a fresh interpreter: PyTorch needs CUBLAS_WORKSPACE_CONFIG set before CUDA initialises for its
deterministic cuBLAS calls (the MLPs of the global motion branch)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

N_VIEW, N_FRAME, RES = 4, 16, 256


def _run(case):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), case], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0 and f"CASE {case} OK" in r.stdout, (r.stdout[-3000:], r.stderr[-6000:])
    print(r.stdout[-2000:])


# ---------------------------------------------------------------------------------------------------------------- fixtures
def _model(xyz=None, P=20000, seed=11):
    import torch
    from animate3d_b200.gaussian4d import Gaussian4DModel
    from oracle import raster_oracle as R
    pts, s, q, o, sh = R.synthetic_scene(P if xyz is None else xyz.shape[0], seed)
    if xyz is not None:
        pts = torch.as_tensor(xyz, dtype=torch.float32) * 0.5
    model = Gaussian4DModel(pts, torch.log(s), q, o, sh[:, 0], grid_size=((20, 18, 22, 6), (40, 36, 44, 12)), seed=3,
                            use_global_trans=True)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name in ("delta_xyz_network", "delta_rot_network", "delta_scaling_network", "global_rot_network", "global_trans_network"):
            net = getattr(model, name)
            net[1].copy_((torch.randn(net[1].shape, generator=g) * 0.08).cuda())
        for pl in model.grids:
            for p in pl:
                p.copy_((torch.rand(p.shape, generator=g) * 0.8 + 0.3).cuda())
    return model


def _optimizer(model):
    """The recon config's groups (grid / deformation MLPs / global motion) with tensor learning rates, fused Adam."""
    import torch
    lr = lambda v: torch.tensor(v, device="cuda")
    groups = [{"params": [p for pl in model.grids for p in pl], "lr": lr(0.01)},
              {"params": [p for n in ("delta_xyz_network", "delta_rot_network", "delta_scaling_network")
                          for p in getattr(model, n)], "lr": lr(1e-4)},
              {"params": [p for n in ("global_rot_network", "global_trans_network") for p in getattr(model, n)], "lr": lr(1e-3)}]
    return torch.optim.Adam(groups, eps=1e-15, fused=True, capturable=True)


class _Setup:
    """One model + renderer + optimizer and the step body of systems/animate3d.py:120-244 (recon: do_guidance False)."""

    def __init__(self, mesh_graph=None, xyz=None):
        import torch
        from animate3d_b200.renderer import camera_rows, make_renderer
        from tools.splat_bench import cameras
        self.model = _model(xyz)
        self.rend = make_renderer(self.model).train()
        self.opt = _optimizer(self.model)
        self.mesh_graph = mesh_graph
        c2w, fovy, ts = cameras(n_views=N_VIEW, n_frames=N_FRAME)
        self.rows, self.ts = camera_rows(c2w, fovy), ts
        g = torch.Generator(device="cuda").manual_seed(1)
        n = N_VIEW * N_FRAME
        self.mask = (torch.rand(n, RES, RES, 1, device="cuda", generator=g) > 0.3).float()
        self.rgb = torch.rand(n, RES, RES, 3, device="cuda", generator=g)
        self.last = {}          # layout key -> the tensors that step's draws live in (a replay rewrites them)

    def inputs(self, start_index):
        """(layout key, static inputs) of the "normal" strategy: frames 1 .. start_index + 1 of every view."""
        from animate3d_b200.renderer import timestamp_layout
        idx = [v * N_FRAME + f for v in range(N_VIEW) for f in range(1, start_index + 2)]
        layout = timestamp_layout(self.ts.cpu()[idx].numpy())
        return (start_index, layout), {"ts": self.ts[idx], "rows": self.rows[idx], "rgb": self.rgb[idx], "mask": self.mask[idx]}

    def step_fn(self, key, grad_mask=None, sample_idx=None, nbr=None):
        import torch
        import torch.nn.functional as F
        from animate3d_b200 import arap as AP
        from animate3d_b200.mesh import edge_list
        start_index, layout = key

        def fn(inp):
            batch = {"camera_rows": inp["rows"], "timestamps": inp["ts"], "timestamp_layout": layout, "width": RES, "height": RES,
                     "do_guidance": False, "do_reconstruction": True}
            if grad_mask is not None:
                batch["grad_mask"] = grad_mask
            out = self.rend.batch_forward(batch)
            gt = inp["rgb"] * inp["mask"] + 0.5 * (1 - inp["mask"])
            loss = 100.0 * F.mse_loss(gt, out["comp_rgb"]) + 100.0 * F.mse_loss(inp["mask"], out["comp_mask"])
            nodes = torch.stack([self.model._xyz] + out["means3D"][:start_index + 1])
            if self.mesh_graph is not None:
                table = self.mesh_graph.sample(3) if nbr is None else nbr
                ii, jj, nn = edge_list(table)
                self.last.setdefault(key, {})["nbr"] = table
            else:
                ii, jj, nn, _ = AP.cal_connectivity_from_points(nodes[:1], radius=0.01, K=3)
            loss = loss + 12.0 * AP.cal_arap_error(nodes, ii, jj, nn, K=3, sample_num=512, sample_idx=sample_idx)
            loss.backward()
            self.last.setdefault(key, {}).update(mask=out["grad_mask"], sample=AP.last_sample_idx)
        return fn

    def state(self):
        out = [p.detach().clone() for p in self.model.parameters()]
        for p in self.model.parameters():
            st = self.opt.state.get(p, {})
            out += [st[k].clone() for k in ("step", "exp_avg", "exp_avg_sq") if k in st]
        return out


def _equal(a, b, what):
    import torch
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"{what}: tensor {i} differs (max |diff| {float((x.float() - y.float()).abs().max()):.3e})"


def _eager_like(ref, graph_setup, key, inp):
    """The eager step on `ref`, fed the draws the graph's last step used."""
    last = graph_setup.last[key]
    draws = dict(grad_mask=last["mask"].clone(), sample_idx=last["sample"].clone())
    if "nbr" in last:
        draws["nbr"] = last["nbr"].clone()
    ref.opt.zero_grad(set_to_none=True)
    ref.step_fn(key, **draws)(inp)
    ref.opt.step()


def _paired_run(keys, mesh_graph=None, xyz=None):
    """Graph steps on one model, eager steps fed the same draws on a twin; compared after every step."""
    import torch
    from animate3d_b200.capture import StepGraphs
    torch.use_deterministic_algorithms(True)
    A, B = _Setup(mesh_graph, xyz), _Setup(mesh_graph, xyz)
    graphs = StepGraphs(None, A.opt)
    replays = 0
    for start_index in keys:
        key, inp = A.inputs(start_index)
        graphs.step_fn = A.step_fn(key)
        replays += graphs.step(key, inp)
        _eager_like(B, A, key, inp)
        _equal(A.state(), B.state(), f"step at start_index {start_index}")
    return A, B, graphs, replays


def _mesh():
    """A jittered UV sphere of ~20 k vertices and its CSR graph."""
    import numpy as np
    import torch
    from animate3d_b200.mesh import MeshGraph
    from oracle import mesh_oracle as MO
    verts, _, polys, _ = MO.fixture_mesh(seed=2, n_lat=100, n_lon=200)
    faces = np.asarray([[p[0][0], p[k][0], p[k + 1][0]] for p in polys for k in range(1, len(p) - 1)], np.int64)
    row_ptr, col = MO.csr_from_faces(faces, verts.shape[0])
    return MeshGraph(torch.from_numpy(np.asarray(row_ptr, np.int32)).cuda(), torch.from_numpy(np.asarray(col, np.int32)).cuda()), verts


# ---------------------------------------------------------------------------------------------------------------- cases
def case_recon():
    """4 views x 4 frames (start_index 3): one eager warm-up, then 5 replays, each equal to the eager step."""
    A, _, graphs, replays = _paired_run([3] * 6)
    assert replays == 5 and len(graphs.graphs) == 1
    print(f"RECON {replays} replays bit-identical to eager, {graphs.recaptures} recaptures")


def case_mesh():
    """Mesh-edge ARAP: replay k draws the table of the eager sample(K, seed, offset0 + k); consecutive replays differ."""
    import torch
    torch.manual_seed(0)
    from animate3d_b200.capture import StepGraphs
    seed, offset0 = 1234567, 40
    mesh_graph, verts = _mesh()
    mesh_graph.set_sample_state(seed, offset0)
    torch.use_deterministic_algorithms(True)
    A = _Setup(mesh_graph, verts)
    graphs = StepGraphs(None, A.opt)
    key, inp = A.inputs(1)
    graphs.step_fn = A.step_fn(key)
    assert not graphs.step(key, inp)                   # eager warm-up: a host-seeded draw
    prev = None
    for k in range(4):
        assert graphs.step(key, inp)
        table = A.last[key]["nbr"].clone()
        want = mesh_graph.sample(3, seed=seed, offset=offset0 + k)
        assert torch.equal(table, want), f"replay {k}: neighbour table differs from sample(seed, {offset0 + k})"
        if prev is not None:
            assert not torch.equal(table, prev), f"replay {k} drew the same neighbours as replay {k - 1}"
        prev = table
    assert mesh_graph.sample_offset() == offset0 + 4
    _paired_run([1] * 4, mesh_graph, verts)            # full-step parity with the mesh-edge ARAP
    print("MESH 4 replays equal sample(seed, offset0 + k), and the mesh step matches eager")


def case_overflow():
    """A captured capacity below the need: the replay sets the flag and changes nothing; the helper then captures again
    and the step equals the eager step."""
    import torch
    from animate3d_b200 import rasterizer as RZ
    from animate3d_b200.capture import StepGraphs
    torch.use_deterministic_algorithms(True)
    A, B = _Setup(), _Setup()
    graphs = StepGraphs(None, A.opt)
    key, inp = A.inputs(2)
    graphs.step_fn = A.step_fn(key)
    graphs.step(key, inp)                              # eager warm-up
    _eager_like(B, A, key, inp)
    rkey = next(k for k in RZ._cap_hint if k[3] == inp["rows"].shape[0])
    need = RZ._cap_hint[rkey]
    RZ._cap_hint[rkey] = 1 << 12
    graphs.capture(key, inp)
    before = A.state()
    assert graphs.replay(key, inp), "the replay did not report the overflow"
    assert float(graphs.found_inf) == 1.0
    _equal(A.state(), before, "state after an overflowed replay")
    assert RZ._cap_hint[rkey] >= need * 0.9, (RZ._cap_hint[rkey], need)
    assert graphs.step(key, inp)
    assert graphs.recaptures >= 1
    _eager_like(B, A, key, inp)
    _equal(A.state(), B.state(), "step after the recapture")
    print(f"OVERFLOW flagged and skipped; hint grown to {RZ._cap_hint[rkey]} pairs; {graphs.recaptures} recaptures")


def case_layouts():
    """start_index 0 and 1 captured in turn; replaying the first afterwards still matches eager."""
    _, _, graphs, replays = _paired_run([0, 1, 0, 1, 0, 0])
    assert len(graphs.graphs) == 2 and replays == 4
    print("LAYOUTS two graphs in one pool, interleaved replays bit-identical to eager")


CASES = {"recon": case_recon, "mesh": case_mesh, "overflow": case_overflow, "layouts": case_layouts}


# ---------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.gpu
def test_recon_replay_matches_eager():
    _run("recon")


@pytest.mark.gpu
def test_mesh_replays_draw_fresh_neighbours():
    _run("mesh")


@pytest.mark.gpu
def test_overflow_skips_update_and_recaptures():
    _run("overflow")


@pytest.mark.gpu
def test_two_layouts_share_a_pool():
    _run("layouts")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    CASES[sys.argv[1]]()
    print(f"CASE {sys.argv[1]} OK")
