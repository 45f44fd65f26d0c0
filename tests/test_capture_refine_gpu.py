"""The 4D-SDS refine step replayed from CUDA graphs (animate3d_b200/capture.py) with the UNet, the CLIP tower and the VAE
recorded inside it, against the eager step.  Under torch.use_deterministic_algorithms(True) a replay must leave every
parameter and Adam state bit-identical to an eager twin that runs the same body with the same draws: the CUDA generator
state is restored before both (the timestep, the VAE posterior and the guidance noise come from it), and the ARAP node
sample is read back from the graph (its eager draw is numpy).  The twin shares the frozen networks with the graph.

Geometry: 2 views x 4 frames, a random-init SD1.5-geometry UNet and VAE, a 2-layer ViT-H-width CLIP tower, 20 000
gaussians, reconstruction renders at 512^2 (2 views x frames 1-3) and random cameras at 256^2.

Each case runs in a fresh interpreter: PyTorch needs CUBLAS_WORKSPACE_CONFIG set before CUDA initialises for its
deterministic cuBLAS calls (the matmul form of the bilinear resize, the global motion MLPs)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

N_VIEW, N_FRAME, REC, RND = 2, 4, 512, 256
VIT_H2 = dict(hidden_size=1280, intermediate_size=5120, num_attention_heads=16, num_hidden_layers=2, image_size=224,
              patch_size=14, projection_dim=1024, layer_norm_eps=1e-5, hidden_act="gelu")


def _run(case):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), case], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0 and f"CASE {case} OK" in r.stdout, (r.stdout[-3000:], r.stderr[-6000:])
    print(r.stdout[-2000:])


# ---------------------------------------------------------------------------------------------------------------- fixtures
def _nets():
    """(unet, vae, ip image processor, guidance): the frozen networks of the refine step, shared by the graph and its twin."""
    import torch
    from animate3d_b200.clip import CLIPImageProcessor, CLIPVisionModelWithProjection, IPAdapterImageProcessor
    from animate3d_b200.guidance import AnimateMVDiffusionGuidance
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from animate3d_b200.vae import AutoencoderKL
    from animate3d_b200.weights import random_state_dict
    from oracle import clip_oracle as CO
    from oracle import vae_oracle as VO
    cfg = UNetConfig(num_views=N_VIEW, num_frames=N_FRAME)
    unet = MVUNetMotionModel(cfg)
    unet.load_state_dict(random_state_dict(cfg, seed=5))
    vae = AutoencoderKL()
    vae.load_state_dict(VO.make_state_dict(VO.VAEConfig(), 0))
    enc = CLIPVisionModelWithProjection(VIT_H2, "cuda").load_state_dict(CO.random_state_dict(VIT_H2, 0))
    ip = IPAdapterImageProcessor(CLIPImageProcessor("cuda"), enc)
    guide = AnimateMVDiffusionGuidance({"n_view": N_VIEW, "n_frame": N_FRAME, "guidance_scale": 5.0, "recon_std_rescale": 0.5,
                                        "min_step_percent": 0.02, "max_step_percent": 0.98},
                                       unet=unet, vae=vae, ip_image_processor=ip)
    return unet, vae, ip, guide


class _Refine:
    """One gaussian model + renderer + fused Adam and the refine body of systems/animate3d.py:120-244 (do_guidance): the
    reconstruction batch, closed over with its targets, the random-camera batch, the SDS loss and the ARAP."""

    def __init__(self, guide):
        import torch
        from animate3d_b200.renderer import camera_rows, make_renderer, timestamp_layout
        from animate3d_b200.guidance import PrecomputedPromptUtils
        from tools.splat_bench import cameras, synthetic_model
        self.guide = guide
        self.model = synthetic_model(20000, seed=3)
        self.rend = make_renderer(self.model).train()
        params = [p for p in self.model.parameters() if p.requires_grad]
        self.opt = torch.optim.Adam([{"params": params, "lr": torch.tensor(1e-3, device="cuda")}], eps=1e-15, fused=True,
                                    capturable=True)
        c2w, fovy, ts = cameras(n_views=N_VIEW, n_frames=N_FRAME, seed=100)
        idx = [v * N_FRAME + f for v in range(N_VIEW) for f in range(1, N_FRAME)]
        self.rec_rows, self.rec_ts = camera_rows(c2w[idx], fovy[idx]), ts[idx]
        self.rec_layout = timestamp_layout(ts.cpu()[idx].numpy())
        g = torch.Generator(device="cuda").manual_seed(1)
        self.mask = (torch.rand(len(idx), REC, REC, 1, device="cuda", generator=g) > 0.3).float()
        self.rgb = torch.rand(len(idx), REC, REC, 3, device="cuda", generator=g)
        self.ts = ts
        self.layout = timestamp_layout(ts.cpu().numpy())
        self.pu = PrecomputedPromptUtils(torch.randn(77, 768, device="cuda", generator=g),
                                         torch.randn(77, 768, device="cuda", generator=g))
        self.z = torch.zeros(N_VIEW * N_FRAME, device="cuda")
        self.last = {}

    def body(self, sample_idx=None):
        import torch
        import torch.nn.functional as F
        from animate3d_b200 import arap as AP

        def fn(inp):
            rec = self.rend.batch_forward({"camera_rows": self.rec_rows, "timestamps": self.rec_ts,
                                           "timestamp_layout": self.rec_layout, "width": REC, "height": REC,
                                           "do_guidance": True, "do_reconstruction": True})
            gt = self.rgb * self.mask + 0.5 * (1 - self.mask)
            loss = 100.0 * F.mse_loss(gt, rec["comp_rgb"]) + 100.0 * F.mse_loss(self.mask, rec["comp_mask"])
            out = self.rend.batch_forward({"camera_rows": inp["rows"], "timestamps": self.ts, "timestamp_layout": self.layout,
                                           "width": RND, "height": RND, "do_guidance": True, "do_reconstruction": True})
            t = self.guide.draw_timestep(1)
            go = self.guide(out["comp_rgb"], self.pu, self.z, self.z, self.z, inp["c2w"], timestep=t)
            loss = loss + 0.1 * go["loss_sds"]
            nodes = torch.stack([self.model._xyz] + out["means3D"][:N_FRAME - 1])     # SURVEY 8c: the reference's [:15]
            ii, jj, nn, _ = AP.cal_connectivity_from_points(nodes[:1], radius=0.01, K=3)
            loss = loss + 12.0 * AP.cal_arap_error(nodes, ii, jj, nn, K=3, sample_num=512, sample_idx=sample_idx)
            loss.backward()
            self.last = {"t": self.guide.last_timestep, "sample": AP.last_sample_idx}
        return fn

    def state(self):
        out = [p.detach().clone() for p in self.model.parameters()]
        for p in self.model.parameters():
            st = self.opt.state.get(p, {})
            out += [st[k].clone() for k in ("step", "exp_avg", "exp_avg_sq") if k in st]
        return out


def _inputs(seed):
    from animate3d_b200.renderer import camera_rows
    from tools.splat_bench import cameras
    c2w, fovy, _ = cameras(n_views=N_VIEW, n_frames=N_FRAME, seed=seed)
    return {"rows": camera_rows(c2w, fovy), "c2w": c2w}


def _equal(a, b, what):
    import torch
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"{what}: tensor {i} differs (max |diff| {float((x.float() - y.float()).abs().max()):.3e})"


class _Pair:
    """Graph steps on A, eager steps with the same draws on its twin B, compared after every step."""

    KEY = "refine"

    def __init__(self):
        import numpy as np
        import torch
        from animate3d_b200.capture import StepGraphs
        torch.use_deterministic_algorithms(True)
        np.random.seed(0)
        self.unet, self.vae, self.ip, self.guide = _nets()
        self.A, self.B = _Refine(self.guide), _Refine(self.guide)
        self.graphs = StepGraphs(self.A.body(), self.A.opt)
        self.rng = None
        replay = self.graphs.replay

        def replay_noting_rng(key, inputs):           # the generator state the step's last replay starts from
            self.rng = torch.cuda.get_rng_state()
            return replay(key, inputs)
        self.graphs.replay = replay_noting_rng

    def step(self, inp, what):
        import torch
        self.rng = torch.cuda.get_rng_state()
        replayed = self.graphs.step(self.KEY, inp)
        torch.cuda.set_rng_state(self.rng)
        self.twin(inp)
        _equal(self.A.state(), self.B.state(), what)
        assert torch.equal(self.A.last["t"], self.B.last["t"]), (what, self.A.last["t"], self.B.last["t"])
        return replayed

    def twin(self, inp):
        self.B.opt.zero_grad(set_to_none=True)
        self.B.body(sample_idx=self.A.last["sample"].clone())(inp)
        self.B.opt.step()


# ---------------------------------------------------------------------------------------------------------------- cases
def case_refine():
    """One eager warm-up, 5 replays with fresh random cameras, each equal to the eager twin; then a single-value timestep
    range set between replays is drawn exactly by the next replay, without a recapture."""
    p = _Pair()
    assert not p.step(_inputs(0), "eager warm-up")
    ts = []
    for k in range(1, 6):
        assert p.step(_inputs(k), f"replay {k}")
        ts.append(int(p.A.last["t"]))
    assert len(set(ts)) > 1, f"every replay drew t = {ts[0]}"
    g0 = p.graphs.graphs[p.KEY][0]
    over = p.graphs.recaptures
    last = _inputs(5)                                  # the pair count of a replay that fitted: no overflow recapture
    for pct, want in ((0.5, 500), (0.25, 250)):
        p.guide.set_min_max_steps(pct, pct)
        assert p.step(last, f"annealed to {want}")
        assert int(p.A.last["t"]) == want, (int(p.A.last["t"]), want)
    p.guide.cfg.min_step_percent = p.guide.cfg.max_step_percent = 0.7
    p.guide.update_step(0, 100)
    assert p.step(last, "update_step") and int(p.A.last["t"]) == 700
    assert p.graphs.graphs[p.KEY][0] is g0 and p.graphs.recaptures == over and p.graphs.pointer_recaptures == 0
    print(f"REFINE 5 replays bit-identical to eager (t = {ts}), annealed draws 500 / 250 / 700 from one graph; "
          f"{over} overflow recaptures")


def case_overflow():
    """The 512^2 reconstruction render captured below its need: the replay sets the flag and changes nothing; the helper
    then captures again and the step equals the eager twin."""
    import torch
    from animate3d_b200 import rasterizer as RZ
    p = _Pair()
    inp = _inputs(0)
    p.step(inp, "eager warm-up")
    rkey = next(k for k in RZ._cap_hint if k[1] == REC)
    other = {k: v for k, v in RZ._cap_hint.items() if k != rkey}
    need = RZ._cap_hint[rkey]
    RZ._cap_hint[rkey] = 1 << 12
    p.graphs.capture(p.KEY, inp)
    before = p.A.state()
    assert p.graphs.replay(p.KEY, inp), "the replay did not report the overflow"
    assert float(p.graphs.found_inf) == 1.0
    _equal(p.A.state(), before, "state after an overflowed replay")
    assert RZ._cap_hint[rkey] >= need * 0.9, (RZ._cap_hint[rkey], need)
    assert all(RZ._cap_hint[k] == v for k, v in other.items()), "the 256^2 render's hint changed"
    assert p.step(inp, "step after the recapture")
    assert p.graphs.recaptures >= 1 and p.graphs.pointer_recaptures == 0
    assert torch.equal(p.graphs.found_inf, torch.zeros_like(p.graphs.found_inf))
    print(f"OVERFLOW of the {REC}^2 render flagged and skipped; hint grown to {RZ._cap_hint[rkey]} pairs; "
          f"{p.graphs.recaptures} recaptures")


def case_pointers():
    """Moved buffers or weights recapture before the next replay (UNet buffer growth, VAE reload); an eager guidance_eval
    between replays moves nothing and the replays stay bit-identical."""
    import torch
    from oracle import vae_oracle as VO
    p = _Pair()
    p.step(_inputs(0), "eager warm-up")
    assert p.step(_inputs(1), "replay 1")
    assert {type(m).__name__ for m, _ in p.graphs.modules[p.KEY]} == {"MVUNetMotionModel", "CLIPVisionModelWithProjection",
                                                                        "AutoencoderKL"}
    # an eager UNet call at twice the batch grows its buffers
    v0 = p.unet.capture_version
    bn = 4 * N_VIEW
    g = torch.Generator(device="cuda").manual_seed(3)
    p.unet(torch.randn(bn, 4, N_FRAME, 32, 32, device="cuda", generator=g), torch.full((bn,), 300.0, device="cuda"),
           torch.randn(bn, 77, 768, device="cuda", generator=g), camera=torch.randn(bn, 16, device="cuda", generator=g),
           added_cond_kwargs={"image_embeds": torch.randn(bn, 1024, device="cuda", generator=g)}, num_views=N_VIEW)
    assert p.unet.capture_version > v0
    assert p.step(_inputs(2), "after UNet buffer growth") and p.graphs.pointer_recaptures == 1
    assert p.step(_inputs(3), "replay after the recapture") and p.graphs.pointer_recaptures == 1
    # new VAE weights
    p.vae.load_state_dict(VO.make_state_dict(VO.VAEConfig(), 1))
    assert p.step(_inputs(4), "after a VAE load_state_dict") and p.graphs.pointer_recaptures == 2
    # an eager guidance_eval (25 more UNet evaluations, a VAE decode, host reads) between replays
    rgb = torch.rand(N_VIEW * N_FRAME, RND, RND, 3, device="cuda", generator=g)
    c2w = _inputs(9)["c2w"]
    ev = p.guide(rgb, p.A.pu, p.A.z, p.A.z, p.A.z, c2w, guidance_eval=True)["eval"]
    assert torch.isfinite(ev["latents_final"]).all()
    for k in (5, 6):
        assert p.step(_inputs(k), f"replay {k} after guidance_eval")
    assert p.graphs.pointer_recaptures == 2
    print(f"POINTERS 2 pointer recaptures (UNet growth, VAE reload), {p.graphs.recaptures} overflow recaptures; replays "
          "after guidance_eval bit-identical")


def case_nested():
    """The UNet and encode_image recorded in a plain torch.cuda.graph after an eager call equal their eager outputs; before
    it they raise ValueError and record nothing; guidance_eval under capture raises."""
    import torch
    torch.use_deterministic_algorithms(True)
    unet, vae, ip, guide = _nets()
    g = torch.Generator(device="cuda").manual_seed(4)
    bn = 2 * N_VIEW
    args = (torch.randn(bn, 4, N_FRAME, 32, 32, device="cuda", generator=g), torch.full((bn,), 421.0, device="cuda"),
            torch.randn(bn, 77, 768, device="cuda", generator=g))
    kw = dict(camera=torch.randn(bn, 16, device="cuda", generator=g), num_views=N_VIEW,
              added_cond_kwargs={"image_embeds": torch.randn(bn, 1024, device="cuda", generator=g)})
    imgs = torch.rand(N_VIEW, 3, RND, RND, device="cuda", generator=g)

    def refused(fn, match):
        """fn (whose inputs are all on the device already) raises ValueError under capture."""
        graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(graph):
                fn()
        except ValueError as e:
            assert match in str(e), str(e)
            return
        raise AssertionError(f"no ValueError ({match})")

    # before any eager call: nothing packed, no buffers, no resize tables
    versions = unet.capture_version, ip.image_encoder.capture_version
    refused(lambda: unet(*args, **kw), "one eager call")
    refused(lambda: ip.encode_image(imgs), "one eager call")
    assert not unet._prepared and not unet._static and not unet._bufs
    assert not ip.image_encoder._static and not ip.feature_extractor.tables._cache
    assert (unet.capture_version, ip.image_encoder.capture_version) == versions
    # eager, then recorded into a plain graph
    want_u = unet(*args, **kw).sample
    want_c = ip.encode_image(imgs)
    bufs = {k: v.data_ptr() for k, v in unet._bufs.items()}
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got_u = unet(*args, **kw).sample
        got_c = ip.encode_image(imgs)
    for _ in range(2):
        got_u.zero_(); got_c.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(got_u, want_u) and torch.equal(got_c, want_c)
    assert {k: v.data_ptr() for k, v in unet._bufs.items()} == bufs
    # shapes without an eager call raise (another batch size; another image size for the resize tables)
    refused(lambda: unet(*(a[:N_VIEW] for a in args), **dict(kw, camera=kw["camera"][:N_VIEW], added_cond_kwargs={
        "image_embeds": kw["added_cond_kwargs"]["image_embeds"][:N_VIEW]})), "one eager call")
    refused(lambda: ip.encode_image(imgs[:1]), "one eager call")
    small = torch.rand(N_VIEW, 3, 128, 128, device="cuda")
    refused(lambda: ip.encode_image(small), "one eager call")
    assert {k: v.data_ptr() for k, v in unet._bufs.items()} == bufs and 1 not in ip.image_encoder._static
    # guidance_eval cannot be captured
    rgb = torch.rand(N_VIEW * N_FRAME, RND, RND, 3, device="cuda")
    z = torch.zeros(N_VIEW * N_FRAME, device="cuda")
    from animate3d_b200.guidance import PrecomputedPromptUtils
    pu = PrecomputedPromptUtils(torch.randn(77, 768, device="cuda"), torch.randn(77, 768, device="cuda"))
    c2w = _inputs(0)["c2w"]
    refused(lambda: guide(rgb, pu, z, z, z, c2w, guidance_eval=True), "guidance_eval")
    print("NESTED UNet and encode_image replays bit-identical to eager; unwarmed shapes and guidance_eval refused")


CASES = {"refine": case_refine, "overflow": case_overflow, "pointers": case_pointers, "nested": case_nested}


# ---------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.gpu
def test_refine_replay_matches_eager_and_follows_annealing():
    _run("refine")


@pytest.mark.gpu
def test_refine_overflow_skips_update_and_recaptures():
    _run("overflow")


@pytest.mark.gpu
def test_moved_module_buffers_recapture():
    _run("pointers")


@pytest.mark.gpu
def test_nested_modules_record_into_the_callers_graph():
    _run("nested")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    CASES[sys.argv[1]]()
    print(f"CASE {sys.argv[1]} OK")
