"""Generate golden vectors by RUNNING THE REFERENCE'S OWN SOURCE (read from /root/reference at generation time, never
copied) with its absent third-party dependencies stubbed.  Run in the build container only:

    python tests/golden/gen_reference_goldens.py        ->  tests/golden/ref_processors_c{64,80,96}.pt, ref_embeddings.pt, ref_camera.pt

What is real and what is stubbed
  real   : animatediff/models/attention_processor.py (all processors + SoftmaxAlphaBlender), animatediff/models/embeddings.py,
           pipeline.py::get_camera/generate_c2w/normalize_camera (exec'd from the file's AST, the module itself cannot
           be imported because diffusers is missing)
  stubbed: `diffusers` (Attention container with to_q/to_k/to_v/to_out, head_to_batch_dim, batch_to_head_dim,
           get_attention_scores per diffusers 0.28.0; AlphaBlender; SinusoidalPositionalEmbedding; LabelEmbedding) and
           `xformers.ops.memory_efficient_attention` (softmax(q k^T scale) v in fp32 -- xformers 0.0.16 is CUDA-only).
The GPU box has no /root/reference; only the emitted .pt fixtures travel.
"""
import ast
import math
import os
import sys
import types
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))


# --------------------------------------------------------------------------------------------- stubs
class Attention(nn.Module):
    """diffusers 0.28.0 models/attention_processor.py::Attention, the subset the reference processors touch."""

    def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=8):
        super().__init__()
        inner = heads * dim_head
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(cross_attention_dim or query_dim, inner, bias=False)
        self.to_v = nn.Linear(cross_attention_dim or query_dim, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim, bias=True), nn.Dropout(0.0)])
        self.spatial_norm = None
        self.group_norm = None
        self.norm_cross = None
        self.residual_connection = False
        self.rescale_output_factor = 1.0

    def prepare_attention_mask(self, attention_mask, target_length, batch_size, out_dim=3):
        assert attention_mask is None
        return None

    def head_to_batch_dim(self, tensor, out_dim=3):
        head_size = self.heads
        if tensor.ndim == 3:
            batch_size, seq_len, dim = tensor.shape
            extra_dim = 1
        else:
            batch_size, extra_dim, seq_len, dim = tensor.shape
        tensor = tensor.reshape(batch_size, seq_len * extra_dim, head_size, dim // head_size)
        tensor = tensor.permute(0, 2, 1, 3)
        if out_dim == 3:
            tensor = tensor.reshape(batch_size * head_size, seq_len * extra_dim, dim // head_size)
        return tensor

    def batch_to_head_dim(self, tensor):
        head_size = self.heads
        batch_size, seq_len, dim = tensor.shape
        tensor = tensor.reshape(batch_size // head_size, head_size, seq_len, dim)
        return tensor.permute(0, 2, 1, 3).reshape(batch_size // head_size, seq_len, dim * head_size)

    def get_attention_scores(self, query, key, attention_mask=None):
        assert attention_mask is None
        baddbmm_input = torch.empty(query.shape[0], query.shape[1], key.shape[1], dtype=query.dtype)
        scores = torch.baddbmm(baddbmm_input, query, key.transpose(-1, -2), beta=0, alpha=self.scale)
        return scores.softmax(dim=-1).to(query.dtype)


class AlphaBlender(nn.Module):
    """diffusers 0.28.0 models/resnet.py::AlphaBlender, merge_strategy='learned' (2-D/3-D input path)."""

    def __init__(self, alpha, merge_strategy="learned", switch_spatial_to_temporal_mix=False):
        super().__init__()
        assert merge_strategy == "learned"
        self.register_parameter("mix_factor", nn.Parameter(torch.Tensor([alpha])))

    def forward(self, x_spatial, x_temporal, image_only_indicator=None):
        alpha = torch.sigmoid(self.mix_factor).to(x_spatial.dtype)
        return alpha * x_spatial + (1.0 - alpha) * x_temporal


class SinusoidalPositionalEmbedding(nn.Module):
    """diffusers 0.28.0 models/embeddings.py::SinusoidalPositionalEmbedding."""

    def __init__(self, embed_dim, max_seq_length=32):
        super().__init__()
        position = torch.arange(max_seq_length).unsqueeze(1)
        div_term = torch.exp(torch.arange(0, embed_dim, 2) * (-math.log(10000.0) / embed_dim))
        pe = torch.zeros(1, max_seq_length, embed_dim)
        pe[0, :, 0::2] = torch.sin(position * div_term)
        pe[0, :, 1::2] = torch.cos(position * div_term)
        self.register_buffer("pe", pe)

    def forward(self, x):
        _, seq_length, _ = x.shape
        return x + self.pe[:, :seq_length]


class LabelEmbedding(nn.Module):
    def __init__(self, num_classes, hidden_size, dropout_prob):
        super().__init__()
        self.embedding_table = nn.Embedding(num_classes + (dropout_prob > 0), hidden_size)

    def forward(self, labels):
        return self.embedding_table(labels)


def memory_efficient_attention(query, key, value, attn_bias=None, op=None, scale=None, p=0.0):
    """xformers.ops.memory_efficient_attention on 3-D [B*H, L, d] inputs."""
    assert attn_bias is None
    scale = scale if scale is not None else query.shape[-1] ** -0.5
    s = torch.bmm(query.float(), key.float().transpose(1, 2)) * scale
    return torch.bmm(s.softmax(-1), value.float()).to(query.dtype)


def install_stubs():
    def mod(name):
        m = types.ModuleType(name)
        sys.modules[name] = m
        return m
    d = mod("diffusers"); du = mod("diffusers.utils"); dm = mod("diffusers.models")
    dap = mod("diffusers.models.attention_processor"); de = mod("diffusers.models.embeddings")
    dr = mod("diffusers.models.resnet")
    du.USE_PEFT_BACKEND = False
    dap.Attention = Attention
    de.LabelEmbedding = LabelEmbedding
    de.SinusoidalPositionalEmbedding = SinusoidalPositionalEmbedding
    dr.AlphaBlender = AlphaBlender
    d.utils = du; d.models = dm; dm.attention_processor = dap; dm.embeddings = de; dm.resnet = dr
    x = mod("xformers"); xo = mod("xformers.ops")
    xo.memory_efficient_attention = memory_efficient_attention
    x.ops = xo


def load_camera_fns():
    """exec the three camera helpers out of pipeline.py without importing the module (it needs diffusers)."""
    src = open(os.path.join(REF, "animatediff/pipelines/pipeline.py")).read()
    tree = ast.parse(src)
    want = {"get_camera", "generate_c2w", "normalize_camera"}
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in want]
    import numpy as np
    ns = {"np": np, "torch": torch, "F": F, "math": math}
    exec(compile(ast.Module(body=body, type_ignores=[]), "pipeline_camera", "exec"), ns)
    return ns["get_camera"]


def load_kplanes_fns():
    """exec grid_sample_wrapper and Gaussian4DModel.interpolate_ms_features out of gaussian_4d.py (the module imports
    threestudio / simple_knn / the un-vendored threestudio-3dgs package and cannot be imported here)."""
    import itertools
    from typing import Collection, Iterable, Optional
    src = open(os.path.join(REF, "custom/threestudio-animate3d/geometry/gaussian_4d.py")).read()
    tree = ast.parse(src)
    fns = []
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name == "grid_sample_wrapper":
            fns.append(node)
        if isinstance(node, ast.ClassDef) and node.name == "Gaussian4DModel":
            for sub in node.body:
                if isinstance(sub, ast.FunctionDef) and sub.name == "interpolate_ms_features":
                    fns.append(sub)
    ns = {"torch": torch, "F": F, "nn": nn, "itertools": itertools, "Collection": Collection, "Iterable": Iterable,
          "Optional": Optional}
    exec(compile(ast.Module(body=fns, type_ignores=[]), "gaussian_4d_kplanes", "exec"), ns)
    return ns["interpolate_ms_features"]


def load_rotation_fns():
    """exec build_rotation / extract_rotation_torch / euler_angles_to_rotation_matrix out of geometry/utils.py (the module
    imports scipy's Rotation at top level for an unrelated helper; only these three functions are needed)."""
    src = open(os.path.join(REF, "custom/threestudio-animate3d/geometry/utils.py")).read()
    tree = ast.parse(src)
    want = {"build_rotation", "extract_rotation_torch", "euler_angles_to_rotation_matrix"}
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in want]
    ns = {"torch": torch, "math": math}
    exec(compile(ast.Module(body=body, type_ignores=[]), "geometry_utils_rot", "exec"), ns)
    return ns["build_rotation"], ns["extract_rotation_torch"], ns["euler_angles_to_rotation_matrix"]


def run_reference_load_ply(path, rot_x, rot_z, scale):
    """exec Gaussian4DModel.load_ply (gaussian_4d.py:177-306) out of the file against a fake `self` on the CPU.  `plyfile` is
    not installed: PlyData.read is stubbed by a thin adapter over the repo's own header parser, so the golden pins the
    loader's MATH (rotate / scale / quaternion re-orientation, buffer shapes), not the byte parsing -- that is checked
    separately against struct.unpack in tests/test_io.py."""
    import types
    import numpy as np
    sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))
    from animate3d_b200.io import read_ply_vertices
    usrc = open(os.path.join(REF, "custom/threestudio-animate3d/geometry/utils.py")).read()
    utree = ast.parse(usrc)
    ubody = [n for n in utree.body if isinstance(n, ast.FunctionDef) and n.name in {"build_rotation_np", "extract_rotation_scipy"}]
    from scipy.spatial.transform import Rotation
    uns = {"np": np, "R": Rotation}
    exec(compile(ast.Module(body=ubody, type_ignores=[]), "geometry_utils_np", "exec"), uns)

    class _Prop:
        def __init__(self, name): self.name = name

    class _Element:
        def __init__(self, cols): self.cols = cols; self.properties = [_Prop(k) for k in cols]
        def __getitem__(self, k): return self.cols[k]

    class PlyData:
        @staticmethod
        def read(pth):
            o = types.SimpleNamespace(); o.elements = [_Element(read_ply_vertices(pth))]; return o

    class _TorchCpu:          # torch with device="cuda" dropped
        float = torch.float
        @staticmethod
        def tensor(x, dtype=None, device=None): return torch.tensor(x, dtype=dtype)
        @staticmethod
        def zeros(shape, device=None): return torch.zeros(shape)

    src = open(os.path.join(REF, "custom/threestudio-animate3d/geometry/gaussian_4d.py")).read()
    fn = None
    for node in ast.parse(src).body:
        if isinstance(node, ast.ClassDef) and node.name == "Gaussian4DModel":
            for sub in node.body:
                if isinstance(sub, ast.FunctionDef) and sub.name == "load_ply":
                    fn = sub
    ns = {"np": np, "torch": _TorchCpu, "nn": nn, "PlyData": PlyData, "build_rotation_np": uns["build_rotation_np"],
          "extract_rotation_scipy": uns["extract_rotation_scipy"]}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "gaussian_4d_load_ply", "exec"), ns)

    class FakeSelf:
        def __init__(self):
            self.cfg = types.SimpleNamespace(load_ply_cfg=types.SimpleNamespace(rot_x_degree=rot_x, rot_z_degree=rot_z, scale_factor=scale))
            self.max_sh_degree = 0
            for k in ("_xyz", "_features_dc", "_features_rest", "_opacity"):
                setattr(self, k, None)
        def register_buffer(self, name, t): setattr(self, name, t)
    me = FakeSelf()
    ns["load_ply"](me, path)
    return {k: getattr(me, k).detach().clone() for k in ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")}


def fake_unet_eps(lat, ts, ehs, cam, img):
    """Deterministic stand-in for the UNet in the guidance golden (depends on every conditioning input).  tests/test_guidance.py
    carries the same function."""
    v = lambda x: x.reshape(-1, 1, 1, 1, 1)
    return (0.1 * lat * v(torch.cos(ts.float() / 1000.0)) + 0.01 * v(ehs.float().mean((1, 2))) + 0.02 * v(cam.float().sum(1))
            + 0.03 * v(img.float().mean(1)) + 0.05 * torch.sin(3.0 * lat))


def run_reference_recon_loss():
    """exec AnimateMVDiffusionGuidance.compute_mvdream_recon_loss + get_camera_cond + normalize_camera out of
    animatemv_guidance.py (391-513, 347-363, 40-52) against a fake `self`: the UNet is `fake_unet_eps`, the scheduler a
    minimal restatement of diffusers' DDIMScheduler.add_noise / step(...).pred_original_sample (not installed)."""
    import numpy as np
    from einops import rearrange
    src = open(os.path.join(REF, "custom/threestudio-animate3d/guidance/animatemv_guidance.py")).read()
    tree = ast.parse(src)
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "normalize_camera"]
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name == "AnimateMVDiffusionGuidance":
            for sub in node.body:
                if isinstance(sub, ast.FunctionDef) and sub.name in ("compute_mvdream_recon_loss", "get_camera_cond"):
                    sub.decorator_list = []
                    sub.returns = None
                    for a in sub.args.args + sub.args.kwonlyargs:
                        a.annotation = None
                    body.append(sub)
    ns = {"torch": torch, "np": np, "F": F, "rearrange": rearrange}
    exec(compile(ast.Module(body=body, type_ignores=[]), "animatemv_guidance_recon", "exec"), ns)

    betas = torch.linspace(0.00085, 0.012, 1000, dtype=torch.float32)
    acp = torch.cumprod(1.0 - betas, 0)

    class Sched:
        def add_noise(self, x, noise, t):
            a = acp[t]
            sa, sb = a.sqrt().flatten(), (1 - a).sqrt().flatten()
            while sa.ndim < x.ndim:
                sa, sb = sa.unsqueeze(-1), sb.unsqueeze(-1)
            return sa * x + sb * noise
        def step(self, eps, t, x):
            a = acp[t]
            return SimpleNamespace(pred_original_sample=(x - (1 - a) ** 0.5 * eps) / a ** 0.5)

    B, n, f = 1, 2, 3
    g = torch.Generator().manual_seed(123)
    latents = torch.randn(B * n * f, 4, 6, 6, generator=g)
    t = torch.tensor([137])
    text = torch.randn(2 * B * n, 77, 16, generator=g)
    c2w = torch.randn(B * n * f, 4, 4, generator=g)
    img = torch.randn(B * n, 32, generator=g)
    out = {}
    for rescale in (0.5, 0.0):
        me = SimpleNamespace(cfg=SimpleNamespace(n_view=n, n_frame=f, guidance_scale=5.0, recon_std_rescale=rescale,
                                                 i2v_cond_time_zero=False, view_dependent_prompting=False,
                                                 camera_condition_type="rotation"),
                             scheduler=Sched())
        me.get_camera_cond = lambda cam, fovy=None, _me=me: ns["get_camera_cond"](_me, cam, fovy)
        me.forward_unet = lambda lat, ts, encoder_hidden_states, camera, i2v_cond_time_zero, added_cond_kwargs: fake_unet_eps(
            lat, ts, encoder_hidden_states, camera, added_cond_kwargs["image_embeds"])
        prompt = SimpleNamespace(get_text_embeddings=lambda *a, **k: text, use_perp_neg=False)
        zeros = torch.zeros(B * n * f)
        torch.manual_seed(777)
        lat_in = latents.clone().requires_grad_(True)
        loss, aux = ns["compute_mvdream_recon_loss"](me, lat_in, t, prompt, zeros, zeros, zeros, camera=c2w.clone(),
                                                     image_embeds=img.clone())
        loss.backward()
        out[rescale] = {"loss": loss.detach(), "grad": lat_in.grad.clone(), "latents_noisy": aux["latents_noisy"].clone(),
                        "noise_pred": aux["noise_pred"].clone(), "latents_recon": aux["latents_recon"].detach().clone()}
    torch.save({"latents": latents, "t": t, "text": text, "c2w": c2w, "img": img, "n": n, "f": f, "seed": 777, "out": out},
               os.path.join(OUT, "ref_guidance.pt"))


def run_reference_cam_info():
    """exec convert_pose / get_projection_matrix_gaussian / get_cam_info_gaussian (threestudio/utils/ops.py:305-359) on the
    CPU: `.cuda()` calls are dropped and the `device="cuda"` default becomes "cpu" in the AST, nothing else changes."""
    src = open(os.path.join(REF, "threestudio/utils/ops.py")).read()
    want = {"convert_pose", "get_projection_matrix_gaussian", "get_cam_info_gaussian"}
    body = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in want]

    class NoCuda(ast.NodeTransformer):
        def visit_Call(self, node):
            self.generic_visit(node)
            if isinstance(node.func, ast.Attribute) and node.func.attr == "cuda" and not node.args:
                return node.func.value
            return node

        def visit_FunctionDef(self, node):
            self.generic_visit(node)
            node.args.defaults = [ast.Constant("cpu") if isinstance(d, ast.Constant) and d.value == "cuda" else d
                                  for d in node.args.defaults]
            return node
    mod = ast.fix_missing_locations(NoCuda().visit(ast.Module(body=body, type_ignores=[])))
    ns = {"torch": torch, "math": math}
    exec(compile(mod, "threestudio_ops_cam", "exec"), ns)
    g = torch.Generator().manual_seed(17)
    cams = []
    for i in range(6):
        q = torch.randn(4, generator=g)
        q = q / q.norm()
        r, x, y, z = q.tolist()
        rot = torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                            [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                            [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])
        c2w = torch.eye(4)
        c2w[:3, :3] = rot
        c2w[:3, 3] = torch.randn(3, generator=g) * 2
        fovx, fovy = 0.6 + 0.1 * i, 0.5 + 0.07 * i
        wv, full, center = ns["get_cam_info_gaussian"](c2w.clone(), fovx, fovy, 0.1, 100.0)
        cams.append({"c2w": c2w, "fovx": fovx, "fovy": fovy, "wv": wv.clone(), "full": full.clone(), "center": center.clone()})
    torch.save(cams, os.path.join(OUT, "ref_cam_info.pt"))


def run_reference_arap():
    """exec produce_edge_matrix_nfmt / cal_connectivity_from_points / estimate_rotation / cal_arap_error out of
    systems/util.py on the CPU: `.cuda()` / `.to(device)` dropped in the AST, pytorch3d.ops served by a brute-force KNN with
    the published knn_points contract, np.random.choice replaced by a recorded index draw."""
    import numpy as np
    src = open(os.path.join(REF, "custom/threestudio-animate3d/systems/util.py")).read()
    want = {"produce_edge_matrix_nfmt", "cal_connectivity_from_points", "estimate_rotation", "cal_arap_error"}
    body = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in want]
    for fn in body:
        fn.decorator_list = []

    class NoCuda(ast.NodeTransformer):
        def visit_Call(self, node):
            self.generic_visit(node)
            if isinstance(node.func, ast.Attribute) and node.func.attr == "cuda" and not node.args:
                return node.func.value
            if isinstance(node.func, ast.Attribute) and node.func.attr == "to" and len(node.args) == 1 and \
                    isinstance(node.args[0], ast.Name) and node.args[0].id == "device":
                return node.func.value
            return node
    mod = ast.fix_missing_locations(NoCuda().visit(ast.Module(body=body, type_ignores=[])))

    def knn_points(p1, p2, l1, l2, K):
        d2 = ((p1[:, :, None, :] - p2[:, None, :, :]) ** 2).sum(-1)
        dist, idx = torch.sort(d2, dim=2, stable=True)
        return SimpleNamespace(dists=dist[:, :, :K], idx=idx[:, :, :K])

    def knn_gather(x, idx):
        return torch.stack([x[b][idx[b]] for b in range(x.shape[0])])
    drawn = {}

    class FakeRandom:
        @staticmethod
        def choice(n, k):
            r = np.random.RandomState(99).choice(n, k)
            drawn["idx"] = torch.from_numpy(r).long()
            return r
    fake_np = SimpleNamespace(random=FakeRandom)
    ns = {"torch": torch, "np": fake_np, "svd": torch.svd,
          "pytorch3d": SimpleNamespace(ops=SimpleNamespace(knn_points=knn_points, knn_gather=knn_gather))}
    exec(compile(mod, "systems_util_arap", "exec"), ns)
    g = torch.Generator().manual_seed(41)
    nt, nv, K = 4, 120, 3                        # arap_K = 3 = least_edge_num in every shipped config
    base = torch.rand(nv, 3, generator=g)
    seq = [base]
    for t in range(1, nt):                       # smooth non-rigid motion: rotation about z growing with height + noise
        ang = 0.15 * t * (0.5 + base[:, 2])
        rot = torch.stack([torch.cos(ang) * base[:, 0] - torch.sin(ang) * base[:, 1],
                           torch.sin(ang) * base[:, 0] + torch.cos(ang) * base[:, 1], base[:, 2]], 1)
        seq.append(rot + 0.01 * torch.randn(nv, 3, generator=g))
    nodes = torch.stack(seq)
    nodes[:, :5] = nodes[0:1, :5]                # a few nodes that never move (the S = 0 branch)
    # as called by systems/animate3d.py:236-241: graph from frame 0 only, error with weight=None (indicator weights)
    ii, jj, nn, weight = ns["cal_connectivity_from_points"](nodes[:1].clone(), radius=0.01, K=K)
    rot = ns["estimate_rotation"](nodes[0], nodes[2], ii, jj, nn, K=K, weight=weight)
    lat = nodes.clone().requires_grad_(True)
    err_all = ns["cal_arap_error"](lat, ii, jj, nn, K=K, sample_num=512)
    err_all.backward()
    lat2 = nodes.clone().requires_grad_(True)
    err_sub = ns["cal_arap_error"](lat2, ii, jj, nn, K=K, sample_num=50)
    err_sub.backward()
    torch.save({"nodes": nodes, "K": K, "radius": 0.01, "ii": ii, "jj": jj, "nn": nn, "weight": weight, "rot_0_2": rot,
                "err_all": err_all.detach(), "grad_all": lat.grad.clone(), "sample_idx": drawn["idx"],
                "err_sub": err_sub.detach(), "grad_sub": lat2.grad.clone()}, os.path.join(OUT, "ref_arap.pt"))


def attn_weights(attn, prefix):
    return {f"{prefix}.to_q.weight": attn.to_q.weight.detach().clone(),
            f"{prefix}.to_k.weight": attn.to_k.weight.detach().clone(),
            f"{prefix}.to_v.weight": attn.to_v.weight.detach().clone(),
            f"{prefix}.to_out.0.weight": attn.to_out[0].weight.detach().clone(),
            f"{prefix}.to_out.0.bias": attn.to_out[0].bias.detach().clone()}


def main():
    install_stubs()
    sys.path.insert(0, REF)
    from animatediff.models import attention_processor as ap  # the reference's own file
    from animatediff.models.embeddings import SinePositionalEncoding2D

    torch.manual_seed(1234)
    cases = []
    for (c, heads, nv, nf, fs, b) in [(64, 8, 2, 3, 4, 1), (80, 8, 4, 4, 2, 2), (96, 8, 1, 4, 4, 1)]:
        l = fs * fs
        dh = c // heads
        cd = 48
        # ---- MVDreamI2V (attn1 of the spatial transformers)
        attn = Attention(c, None, heads, dh)
        proc = ap.MVDreamI2VXFormersAttnProcessor(hidden_size=c, num_views=nv, num_frames=nf)
        nn.init.normal_(proc.to_out_i2v.weight, std=0.1); nn.init.normal_(proc.to_out_i2v.bias, std=0.1)
        x = torch.randn(b * nv * nf, l, c)
        with torch.no_grad():
            y = proc(attn, x)
        w = attn_weights(attn, "a.attn1")
        w["a.attn1.processor.to_q_i2v.weight"] = proc.to_q_i2v.weight.detach().clone()
        w["a.attn1.processor.to_out_i2v.weight"] = proc.to_out_i2v.weight.detach().clone()
        w["a.attn1.processor.to_out_i2v.bias"] = proc.to_out_i2v.bias.detach().clone()
        cases.append(dict(kind="mv_i2v", c=c, heads=heads, nv=nv, nf=nf, fs=fs, b=b, x=x, y=y, w=w))
        # ---- plain MVDream (same regroup, no I2V branch)
        proc0 = ap.MVDreamXFormersAttnProcessor(num_views=nv, num_frames=nf)
        with torch.no_grad():
            y0 = proc0(attn, x)
        cases.append(dict(kind="mv", c=c, heads=heads, nv=nv, nf=nf, fs=fs, b=b, x=x, y=y0, w=w))
        # ---- IP adapter (attn2 of the spatial transformers)
        attn2 = Attention(c, cd, heads, dh)
        procip = ap.IPAdapterXFormersAttnProcessor(hidden_size=c, cross_attention_dim=cd, num_tokens=(4,), scale=0.7)
        text = torch.randn(b * nv * nf, 7, cd)
        ipt = torch.randn(b * nv * nf, 1, 4, cd)
        with torch.no_grad():
            yip = procip(attn2, x, encoder_hidden_states=(text, [ipt]))
        w2 = attn_weights(attn2, "a.attn2")
        w2["a.attn2.processor.to_k_ip.0.weight"] = procip.to_k_ip[0].weight.detach().clone()
        w2["a.attn2.processor.to_v_ip.0.weight"] = procip.to_v_ip[0].weight.detach().clone()
        cases.append(dict(kind="ip", c=c, heads=heads, nv=nv, nf=nf, fs=fs, b=b, x=x, text=text, ip=ipt[:, 0], y=yip,
                          w=w2, ip_scale=0.7))
        # ---- SpatioTemporal (attn1/attn2 of the motion modules), released config
        attn3 = Attention(c, None, heads, dh)
        spatial_cfg = SimpleNamespace(enabled=True, attn_cfg=SimpleNamespace(
            use_spatial_encoding=True, spatial_encoding_type="sinusoid", use_camera_encoding=False,
            camera_encoding_type="sinusoid"))
        image_cfg = SimpleNamespace(enabled=False)
        procst = ap.SpatioTemporalI2VXFormersAttnProcessor(
            hidden_size=c, feature_size=fs, num_views=nv, num_frames=nf, spatial_attn=spatial_cfg,
            image_attn=image_cfg, use_alpha_blender=True)
        with torch.no_grad():
            procst.alpha_blender.mix_factor.fill_(0.3)
        xt = torch.randn(b * nv * l, nf, c)
        with torch.no_grad():
            yst = procst(attn3, xt)
        w3 = attn_weights(attn3, "m.attn1")
        for n in ("to_q_sp", "to_k_sp", "to_v_sp", "to_out_sp"):
            w3[f"m.attn1.processor.{n}.weight"] = getattr(procst, n).weight.detach().clone()
        w3["m.attn1.processor.to_out_sp.bias"] = procst.to_out_sp.bias.detach().clone()
        w3["m.attn1.processor.time_pos_embed.pe"] = procst.time_pos_embed.pe.detach().clone()
        w3["m.attn1.processor.alpha_blender.mix_factor"] = procst.alpha_blender.mix_factor.detach().clone()
        cases.append(dict(kind="st", c=c, heads=heads, nv=nv, nf=nf, fs=fs, b=b, x=xt, y=yst, w=w3,
                          state_keys=sorted(procst.state_dict().keys())))
    for c in sorted({cs["c"] for cs in cases}):      # one file per channel width keeps every fixture under 1 MB
        torch.save([cs for cs in cases if cs["c"] == c], os.path.join(OUT, f"ref_processors_c{c}.pt"))

    emb = {}
    for (nfeat, h, w) in [(16, 4, 4), (160, 32, 32), (320, 16, 16), (640, 8, 8), (640, 4, 4)]:
        m = SinePositionalEncoding2D(nfeat, normalize=True)
        enc = m._forward(torch.zeros(1, h, w))[0]
        full = enc.reshape(-1)
        # a fixed, seeded sample of at most 8192 entries (the full 160 x 32 x 32 table alone would be 1.3 MB)
        idx = torch.arange(full.numel()) if full.numel() <= 8192 else \
            torch.randperm(full.numel(), generator=torch.Generator().manual_seed(0))[:8192].sort().values
        emb[(nfeat, h, w)] = {"shape": tuple(enc.shape), "idx": idx.to(torch.int32), "val": full[idx].clone()}
    torch.save(emb, os.path.join(OUT, "ref_embeddings.pt"))

    # k-planes lookup of the 4D gaussians (gaussian_4d.py:39-64, 450-484)
    interp = load_kplanes_fns()
    import itertools
    g = torch.Generator().manual_seed(77)
    grids = []
    for reso in ([6, 5, 7, 4], [12, 10, 14, 8]):
        planes = nn.ParameterList()
        for comb in itertools.combinations(range(4), 2):
            planes.append(nn.Parameter(torch.rand([1, 8] + [reso[cc] for cc in comb[::-1]], generator=g)))
        grids.append(planes)
    pts = torch.rand(200, 4, generator=g) * 2.4 - 1.2          # some points outside [-1,1] -> border padding
    with torch.no_grad():
        feats = interp(None, pts, grids)
    torch.save({"grids": [[p.detach().clone() for p in pl] for pl in grids], "pts": pts, "feats": feats},
               os.path.join(OUT, "ref_kplanes.pt"))

    # global rotation helpers of the use_global_trans branch (geometry/utils.py:33-62, 73-133, 135-167); the quaternions are
    # chosen so that all four branches of the matrix -> quaternion conversion are exercised
    build_rotation, extract_rotation, euler_to_matrix = load_rotation_fns()
    g = torch.Generator().manual_seed(91)
    quats = torch.randn(400, 4, generator=g)
    quats[:40, 0] *= 0.01          # small real part -> negative trace branches
    angles = torch.rand(6, 3, generator=g) * 2 * math.pi - math.pi
    with torch.no_grad():
        mats = build_rotation(quats)
        rmats = torch.stack([euler_to_matrix(a) for a in angles])
        rotated = torch.stack([extract_rotation(r @ mats) for r in rmats])
        tr = (rmats[:, None] @ mats[None]).diagonal(dim1=-2, dim2=-1).sum(-1)
    assert (tr <= 0).sum() > 20 and (tr > 0).sum() > 20
    torch.save({"quats": quats, "angles": angles, "mats": mats, "rmats": rmats, "rotated": rotated},
               os.path.join(OUT, "ref_rotation.pt"))

    # 3DGS PLY + the loader's rotate / scale step (gaussian_4d.py:177-306); the PLY itself is committed as a fixture
    import numpy as np
    sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))
    from animate3d_b200.io import write_gaussian_ply
    rng = np.random.default_rng(5)
    n = 300
    ply = os.path.join(OUT, "ref_gaussians.ply")
    write_gaussian_ply(ply, rng.normal(size=(n, 3)), rng.normal(size=(n, 3)), rng.normal(size=(n, 1)),
                       rng.normal(size=(n, 3)) * 0.5 - 3.0, rng.normal(size=(n, 4)))
    ply_out = {}
    for cfg in ((0.0, 0.0, 1.0), (-90.0, 30.0, 1.7), (45.0, -120.0, 0.4)):
        ply_out[cfg] = run_reference_load_ply(ply, *cfg)
    torch.save(ply_out, os.path.join(OUT, "ref_ply.pt"))

    run_reference_recon_loss()
    run_reference_cam_info()
    run_reference_arap()

    get_camera = load_camera_fns()
    cam = {n: get_camera(n) for n in (1, 4, 8)}
    torch.save(cam, os.path.join(OUT, "ref_camera.pt"))
    print("wrote", [f for f in os.listdir(OUT) if f.endswith(".pt")])


if __name__ == "__main__":
    main()
