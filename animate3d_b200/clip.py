"""The IP-Adapter image encoder on the engine: CLIP ViT-H/14 (transformers' CLIPVisionModelWithProjection) and the CLIP
processor in front of it, as drop-ins for the objects the reference's `load_ip_adapter(...)` returns
(animatediff/utils/util.py:49, 268-287).

* `CLIPVisionModelWithProjection`: packs the transformers state dict at load and runs the tower as
  patch GEMM (+ position / class row-bias table) -> pre_layrnorm -> layers of
  [LN1 -> fused QKV GEMM -> attention (257 queries and keys per image) -> out-proj GEMM + residual -> LN2 -> fc1 GEMM + GELU
  -> fc2 GEMM + residual] -> post_layernorm -> visual_projection (fp32 out), captured in one CUDA graph per batch size.
* `CLIPImageProcessor`: `__call__(images, return_tensors="pt").pixel_values` through `a3d_clip_preprocess`.
* `IPAdapterImageProcessor`: `encode_image(images)`; images go from their raw form (float renders in [0, 1] on the device,
  uint8 [n, H, W, 3], PIL) straight into the patch GEMM's operand in one launch.  A float device tensor never leaves the
  device, so the guidance's per-step call (animatemv_guidance.py:546-555) needs no host sync.

The processor reproduces the reference's host path -- (x*255).astype(np.uint8), PIL bicubic resize, centre crop,
normalise -- bit for bit up to the fp32 normalisation (include/a3d.h, a3d_clip_preprocess)."""
from __future__ import annotations

import json
import os
from types import SimpleNamespace
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib as L
from . import ops

HALF = torch.float16
TOKENS, PATCH_K, PATCH_K_PAD, CROP, PATCH = 257, 588, 640, 224, 14
HEAD_DIMS = (40, 80, 160)


def _pad16(x: int) -> int:
    return (x + 15) // 16 * 16


def check_config(cfg) -> SimpleNamespace:
    """The vision config as a namespace; raises on anything the IP-Adapter ViT-H/14 path does not implement."""
    get = (lambda k, d=None: cfg.get(k, d)) if isinstance(cfg, dict) else (lambda k, d=None: getattr(cfg, k, d))
    c = SimpleNamespace(hidden_size=get("hidden_size"), intermediate_size=get("intermediate_size"),
                        num_attention_heads=get("num_attention_heads"), num_hidden_layers=get("num_hidden_layers"),
                        image_size=get("image_size", CROP), patch_size=get("patch_size", PATCH),
                        projection_dim=get("projection_dim"), layer_norm_eps=get("layer_norm_eps", 1e-5),
                        hidden_act=get("hidden_act", "gelu"), num_channels=get("num_channels", 3))
    if c.hidden_act != "gelu":
        raise NotImplementedError(f"hidden_act={c.hidden_act!r}: only the erf GELU of the IP-Adapter ViT-H/14 is implemented")
    if c.image_size != CROP or c.patch_size != PATCH or c.num_channels != 3:
        raise NotImplementedError(f"image_size {c.image_size}, patch {c.patch_size}, {c.num_channels} channels: only 224 px, "
                                  "patch 14, RGB is implemented")
    if c.hidden_size % c.num_attention_heads or c.hidden_size // c.num_attention_heads not in HEAD_DIMS:
        raise NotImplementedError(f"head dim {c.hidden_size / c.num_attention_heads} not in {HEAD_DIMS}")
    if c.hidden_size % 8 or c.hidden_size > 1280 or c.intermediate_size % 8 or c.projection_dim % 8:
        raise NotImplementedError("hidden, intermediate and projection sizes must be multiples of 8, hidden <= 1280")
    return c


class CLIPVisionModelWithProjection:
    """Drop-in for transformers' CLIPVisionModelWithProjection at inference: `model(pixel_values).image_embeds`."""

    def __init__(self, config, device="cuda"):
        self.config = config
        self.cfg = check_config(config)
        self.device = torch.device(device)
        self.dtype = HALF
        self.w: Dict[str, torch.Tensor] = {}
        self.layers = []
        self._static: Dict[int, dict] = {}
        self._graphs: Dict[int, torch.cuda.CUDAGraph] = {}
        self.launches_per_forward = 0
        self.use_cuda_graph = True          # off for per-launch checks that synchronise between launches

    # -------------------------------------------------------------------------------------------- loading
    @classmethod
    def from_transformers(cls, model, device="cuda"):
        m = cls(model.config, device)
        m.load_state_dict(model.state_dict())
        return m

    @classmethod
    def from_pretrained(cls, local_dir: str, device="cuda"):
        """A local transformers checkpoint directory: config.json + model.safetensors (no hub access)."""
        from safetensors.torch import load_file
        with open(os.path.join(local_dir, "config.json")) as f:
            cfg = json.load(f)
        cfg = cfg.get("vision_config", cfg) if "hidden_size" not in cfg else cfg
        m = cls(cfg, device)
        m.load_state_dict(load_file(os.path.join(local_dir, "model.safetensors")))
        return m

    def parameters(self):
        return iter(self.w.values())

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def load_state_dict(self, sd: dict, strict: bool = True):
        c = self.cfg
        H, I, nh = c.hidden_size, c.intermediate_size, c.num_attention_heads
        d = H // nh
        dqk, dv = _pad16(d), _pad16(d + 1)
        dev = self.device
        used = set()

        def get(k):
            used.add(k)
            return sd[k].detach().to(dev, torch.float32)

        f16 = lambda t: t.to(HALF).contiguous()
        f32 = lambda t: t.to(torch.float32).contiguous()
        e = "vision_model.embeddings."
        pw = get(e + "patch_embedding.weight").reshape(H, PATCH_K)
        w = {"patch": f16(torch.nn.functional.pad(pw, (0, PATCH_K_PAD - PATCH_K)))}
        rb = get(e + "position_embedding.weight").clone()
        rb[0] += get(e + "class_embedding")
        w["rowbias"] = f32(rb)
        for n, k in (("pre", "vision_model.pre_layrnorm"), ("post", "vision_model.post_layernorm")):
            w[n + "_g"], w[n + "_b"] = f32(get(k + ".weight")), f32(get(k + ".bias"))
        w["proj"] = f16(get("visual_projection.weight"))
        n_qkv = 2 * nh * dqk + nh * dv
        layers = []
        for i in range(c.num_hidden_layers):
            p = f"vision_model.encoder.layers.{i}."
            wq = torch.zeros(n_qkv, H, device=dev)
            bq = torch.zeros(n_qkv, device=dev)
            for j, s in enumerate("qk"):
                wt, bt = get(p + f"self_attn.{s}_proj.weight"), get(p + f"self_attn.{s}_proj.bias")
                for h in range(nh):
                    wq[j * nh * dqk + h * dqk:j * nh * dqk + h * dqk + d] = wt[h * d:(h + 1) * d]
                    bq[j * nh * dqk + h * dqk:j * nh * dqk + h * dqk + d] = bt[h * d:(h + 1) * d]
            wt, bt = get(p + "self_attn.v_proj.weight"), get(p + "self_attn.v_proj.bias")
            for h in range(nh):
                o = 2 * nh * dqk + h * dv
                wq[o:o + d], bq[o:o + d] = wt[h * d:(h + 1) * d], bt[h * d:(h + 1) * d]
                bq[o + d] = 1.0                  # the ones column: the attention kernel's row sum (include/a3d.h)
            lw = {"qkv": f16(wq), "qkv_b": f32(bq)}
            for n, k in (("o", "self_attn.out_proj"), ("fc1", "mlp.fc1"), ("fc2", "mlp.fc2")):
                lw[n], lw[n + "_b"] = f16(get(p + k + ".weight")), f32(get(p + k + ".bias"))
            for n, k in (("ln1", "layer_norm1"), ("ln2", "layer_norm2")):
                lw[n + "_g"], lw[n + "_b"] = f32(get(p + k + ".weight")), f32(get(p + k + ".bias"))
            layers.append(lw)
            w.update({f"layer{i}.{k}": v for k, v in lw.items()})
        if strict:
            extra = [k for k in sd if k not in used and not k.endswith("position_ids")]
            if extra:
                raise KeyError(f"unexpected keys for the vision tower: {extra[:8]}")
        self.w, self.layers = w, layers
        self._static.clear(); self._graphs.clear()
        return self

    # -------------------------------------------------------------------------------------------- forward
    def _buffers(self, n: int) -> dict:
        st = self._static.get(n)
        if st is None:
            c, T = self.cfg, n * TOKENS
            H, nh = c.hidden_size, c.num_attention_heads
            d = H // nh
            n_qkv = 2 * nh * _pad16(d) + nh * _pad16(d + 1)
            z = lambda *s, dt=HALF: torch.zeros(*s, device=self.device, dtype=dt)
            st = {"patches": z(T, PATCH_K_PAD), "x": z(T, H), "h": z(T, H), "qkv": z(T, n_qkv), "attn": z(T, H),
                  "mlp": z(T, c.intermediate_size), "out": z(n, c.projection_dim, dt=torch.float32), "calls": 0}
            self._static[n] = st
        return st

    def patch_buffer(self, n: int) -> torch.Tensor:
        """The fp16 [n * 257, 640] patch-GEMM operand of batch size n (what a3d_clip_preprocess writes)."""
        return self._buffers(n)["patches"]

    def _run(self, n: int, st: dict) -> None:
        c, T = self.cfg, n * TOKENS
        H, I, nh = c.hidden_size, c.intermediate_size, c.num_attention_heads
        d = H // nh
        dqk = _pad16(d)
        w, eps = self.w, c.layer_norm_eps
        x, h, qkv, attn, mlp = st["x"], st["h"], st["qkv"], st["attn"], st["mlp"]
        nq = qkv.shape[1]
        ops.gemm(st["patches"], w["patch"], x, M=T, N=H, K=PATCH_K_PAD, rowbias=w["rowbias"], rb_mod=TOKENS)
        ops.layer_norm(x, w["pre_g"], w["pre_b"], h, T, H, eps)
        # Q / K / V of one image: 257 rows of the fused projection (i1), images along i3
        rows = (nq, TOKENS * nq, TOKENS * nq, n * TOKENS * nq)
        ext = (TOKENS, 1, n, 1)
        q = ops.view5(qkv, 0, nq, rows, ext)
        k = ops.view5(qkv, nh * dqk, nq - nh * dqk, rows, ext)
        v = ops.view5(qkv, 2 * nh * dqk, nq - 2 * nh * dqk, rows, ext)
        ostr = (H, TOKENS * H, TOKENS * H, n * TOKENS * H)
        for lw in self.layers:
            ops.layer_norm(h, lw["ln1_g"], lw["ln1_b"], x, T, H, eps)
            ops.gemm(x, lw["qkv"], qkv, M=T, N=nq, K=H, bias=lw["qkv_b"])
            ops.attention(q, k, v, attn, ostr, heads=nh, d=d, scale=d ** -0.5)
            ops.gemm(attn, lw["o"], h, M=T, N=H, K=H, bias=lw["o_b"], R2=h)
            ops.layer_norm(h, lw["ln2_g"], lw["ln2_b"], x, T, H, eps)
            ops.gemm(x, lw["fc1"], mlp, M=T, N=I, K=H, bias=lw["fc1_b"], gelu=True)
            ops.gemm(mlp, lw["fc2"], h, M=T, N=H, K=I, bias=lw["fc2_b"], R2=h)
        ops.layer_norm(h, w["post_g"], w["post_b"], x, T, H, eps)
        # the class row of every image: A rows 257 * H apart
        ops.gemm(x, w["proj"], st["out"], M=n, N=c.projection_dim, K=H, lda=TOKENS * H, out_f32=True)

    def run_patches(self, n: int) -> torch.Tensor:
        """The tower on the operand already in patch_buffer(n): image_embeds fp32 [n, projection_dim].  The first call per
        batch size runs eagerly, the second is captured, later ones replay the graph."""
        st = self._buffers(n)
        graph = self._graphs.get(n)
        if graph is not None:
            graph.replay()
        else:
            n0 = ops.launches
            self._run(n, st)
            self.launches_per_forward = ops.launches - n0
            st["calls"] += 1
            if self.use_cuda_graph and st["calls"] == 1:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._run(n, st)
                self._graphs[n] = g
        return st["out"].clone()

    def __call__(self, pixel_values: torch.Tensor, output_hidden_states: Optional[bool] = None, output_attentions: Optional[bool] = None,
                 return_dict: Optional[bool] = None, **kwargs):
        return self.forward(pixel_values, output_hidden_states, output_attentions, return_dict, **kwargs)

    def forward(self, pixel_values: torch.Tensor, output_hidden_states: Optional[bool] = None, output_attentions: Optional[bool] = None,
                return_dict: Optional[bool] = None, **kwargs):
        """Normalised pixel values [n, 3, 224, 224] (the processor's output) -> an object with `.image_embeds` (fp32)."""
        if output_hidden_states or output_attentions or kwargs.get("interpolate_pos_encoding"):
            raise NotImplementedError("only image_embeds are produced (no hidden states, attentions or interpolated positions)")
        if return_dict is False:
            raise NotImplementedError("return_dict=False is not supported: read .image_embeds")
        if pixel_values.dim() != 4 or tuple(pixel_values.shape[1:]) != (3, CROP, CROP):
            raise ValueError(f"pixel_values must be [n, 3, {CROP}, {CROP}], got {tuple(pixel_values.shape)}")
        n = pixel_values.shape[0]
        px = pixel_values.to(self.device, torch.float32).contiguous()
        ops.clip_preprocess(px, L.CLIP_SRC_PIXELS, self.patch_buffer(n))
        return SimpleNamespace(image_embeds=self.run_patches(n))


# ------------------------------------------------------------------------------------------------ processors
class _Tables:
    """Device copies of the resize tables, one set per input size (built on the host once)."""

    def __init__(self):
        self._cache = {}

    def get(self, h: int, w: int, device) -> tuple:
        key = (h, w, str(device))
        t = self._cache.get(key)
        if t is None:
            rh, rw, (by, cy, ky), (bx, cx, kx) = ops.clip_resize_tables(h, w)
            t = (rh, rw, (by.to(device), cy.to(device), ky), (bx.to(device), cx.to(device), kx))
            self._cache[key] = t
        return t


def _count(images) -> int:
    if isinstance(images, torch.Tensor):
        return images.shape[0] if images.dim() == 4 else 1
    return len(images) if isinstance(images, (list, tuple)) else 1


def _sources(images, device):
    """-> list of (source tensor on the device, CLIP_SRC_* format) with one image size per entry."""
    if isinstance(images, torch.Tensor):
        if images.dtype == torch.uint8:
            if images.dim() == 3:
                images = images[None]
            if images.dim() != 4 or images.shape[-1] != 3:
                raise ValueError(f"uint8 images must be [n, H, W, 3], got {tuple(images.shape)}")
            return [(images.to(device).contiguous(), L.CLIP_SRC_U8_NHWC)]
        if not images.is_floating_point():
            raise ValueError(f"images must be fp32 [n, 3, H, W] in [0, 1] or uint8 [n, H, W, 3], got {images.dtype}")
        if images.dim() == 3:
            images = images[None]
        if images.dim() != 4 or images.shape[1] != 3:
            raise ValueError(f"float images must be [n, 3, H, W], got {tuple(images.shape)}")
        return [(images.detach().to(device, torch.float32).contiguous(), L.CLIP_SRC_F32_NCHW)]
    if isinstance(images, (list, tuple)) and images and isinstance(images[0], torch.Tensor):
        return _sources(torch.stack(list(images)), device)
    if not isinstance(images, (list, tuple)):
        images = [images]
    out = []
    for im in images:                         # PIL: RGB on the host, one launch per size run
        a = torch.from_numpy(np.asarray(im.convert("RGB")).copy())[None]
        if out and out[-1][0].shape[1:] == a.shape[1:]:
            out[-1] = (torch.cat([out[-1][0], a]), L.CLIP_SRC_U8_NHWC)
        else:
            out.append((a, L.CLIP_SRC_U8_NHWC))
    return [(t.to(device), f) for t, f in out]


class CLIPImageProcessor:
    """Drop-in for transformers' CLIPImageProcessor of the IP-Adapter encoder (224 px, OpenAI mean / std): `__call__(images,
    return_tensors="pt").pixel_values` is fp32 [n, 3, 224, 224] on `device`.  images: PIL images, uint8 [n, H, W, 3] or fp32
    [n, 3, H, W] in [0, 1] (quantised by truncation like the reference's (x*255).astype(np.uint8))."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)
        self.tables = _Tables()

    def write(self, images, patches: Optional[torch.Tensor], pixel_values: Optional[torch.Tensor] = None) -> int:
        """Preprocess into the patch-GEMM operand and / or pixel_values; returns the image count."""
        n0 = 0
        for src, fmt in _sources(images, self.device):
            n = src.shape[0]
            h, w = (src.shape[1], src.shape[2]) if fmt == L.CLIP_SRC_U8_NHWC else (src.shape[2], src.shape[3])
            ops.clip_preprocess(src, fmt, None if patches is None else patches[n0 * TOKENS:(n0 + n) * TOKENS],
                                None if pixel_values is None else pixel_values[n0:n0 + n], self.tables.get(h, w, self.device))
            n0 += n
        return n0

    def __call__(self, images, return_tensors: str = "pt", **kwargs):
        if return_tensors != "pt":
            raise NotImplementedError("return_tensors='pt' only")
        if kwargs:
            raise NotImplementedError(f"processor options are fixed to the IP-Adapter configuration (got {sorted(kwargs)})")
        pv = torch.empty(_count(images), 3, CROP, CROP, device=self.device, dtype=torch.float32)
        self.write(images, None, pv)
        return SimpleNamespace(pixel_values=pv)


class IPAdapterImageProcessor:
    """Drop-in for animatediff/utils/util.py:268-287 with the engine's processor and encoder: `encode_image(images)` ->
    image_embeds fp32 [n, projection_dim], the raw images going straight into the patch-GEMM operand in one launch."""

    def __init__(self, feature_extractor: CLIPImageProcessor, image_encoder: CLIPVisionModelWithProjection, device="cuda"):
        if not isinstance(feature_extractor, CLIPImageProcessor) or not isinstance(image_encoder, CLIPVisionModelWithProjection):
            raise TypeError("IPAdapterImageProcessor takes the engine's CLIPImageProcessor and CLIPVisionModelWithProjection "
                            "(animate3d_b200.clip); wrap transformers' own modules with the reference's class instead")
        self.feature_extractor, self.image_encoder = feature_extractor, image_encoder

    def encode_image(self, images) -> torch.Tensor:
        n = _count(images)
        patches = self.image_encoder.patch_buffer(n)
        got = self.feature_extractor.write(images, patches)
        assert got == n, (got, n)
        return self.image_encoder.run_patches(n)
