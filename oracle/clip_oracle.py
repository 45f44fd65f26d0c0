"""fp32 torch restatement of the IP-Adapter image conditioning: the CLIP processor the reference runs on the host and the
CLIP vision tower (transformers' CLIPVisionModelWithProjection), generic over the vision config.

Processor (custom/threestudio-animate3d/guidance/animatemv_guidance.py:546-555, transformers 4.25-4.28):
  float renders -> (x * 255).astype(np.uint8) (truncation) -> PIL -> resize (short edge 224, long edge int(224 long / short),
  Image.resize(BICUBIC)) -> centre crop 224 at floor((size - 224) / 2) -> x / 255 -> (x - mean) / std, fp32.
The resize restates Pillow's Resample.c for 8-bit images: bicubic a = -0.5, support 2 max(scale, 1), weights in double,
normalised per output sample, 22-bit fixed point rounded half away from zero, horizontal pass then vertical, each pass
adding 2^21 and clamping to uint8.  Written here with vectorised integer tensors, independently of the C header the kernel
and the CPU harness share.  tests/golden/ref_clip.pt pins it against Pillow itself."""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
CROP = 224
PREC = 22


# ------------------------------------------------------------------------------------------------ processor
def quantise(x: torch.Tensor) -> torch.Tensor:
    """(x * 255).astype(np.uint8) of fp32 x in [0, 1]: truncation (clamped outside [0, 255], NaN -> 0)."""
    v = x.float() * 255
    return torch.nan_to_num(v, nan=0.0).clamp(0, 255).trunc().to(torch.uint8)


def resize_shape(h: int, w: int, size: int = CROP):
    if w <= h:
        return int(size * h / w), size
    return size, int(size * w / h)


def _bicubic(x):
    a = -0.5
    x = np.abs(x)
    return np.where(x < 1, ((a + 2) * x - (a + 3)) * x * x + 1, np.where(x < 2, (((x - 5) * x + 8) * x - 4) * a, 0.0))


def resize_coeffs(n_in: int, n_out: int, round_half: bool = True):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc -> (first [n_out], taps [n_out], fixed-point weights [n_out, ksize])."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(n_out) + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)          # C (int) truncation of a positive value
    xmax = np.minimum((center + support + 0.5).astype(np.int64), n_in) - xmin
    i = np.arange(ksize)
    w = _bicubic((i[None, :] + xmin[:, None] - center[:, None] + 0.5) / fs)
    w = np.where(i[None, :] < xmax[:, None], w, 0.0)
    ww = w.sum(1, keepdims=True)
    w = np.where(ww != 0, w / np.where(ww != 0, ww, 1), w)
    s = w * (1 << PREC)
    half = 0.5 if round_half else 0.0
    k = np.trunc(np.where(w < 0, s - half, s + half)).astype(np.int64)          # C (int) casts truncate toward zero
    return torch.from_numpy(xmin), torch.from_numpy(xmax), torch.from_numpy(k)


def _pass(img: torch.Tensor, n_out: int, dim: int, round_half: bool = True) -> torch.Tensor:
    """One Pillow pass along `dim` of an int64 image."""
    n_in = img.shape[dim]
    first, taps, k = resize_coeffs(n_in, n_out, round_half)
    idx = (first[:, None] + torch.arange(k.shape[1])[None, :]).clamp(max=n_in - 1)     # [n_out, ksize]; k = 0 past the taps
    x = img.movedim(dim, -1)
    g = x[..., idx]                                                                       # [..., n_out, ksize]
    ss = (g * k).sum(-1) + (1 << (PREC - 1))
    out = (ss >> PREC).clamp(0, 255)
    return out.movedim(-1, dim)


def pil_resize(u8: torch.Tensor, out_h: int, out_w: int, vertical_first: bool = False, round_half: bool = True) -> torch.Tensor:
    """Image.resize((out_w, out_h), BICUBIC) of uint8 [..., H, W] (channels independent).  A pass whose size does not change
    is the identity in Pillow's arithmetic as well, so both passes always run."""
    x = u8.to(torch.int64)
    if vertical_first:
        x = _pass(_pass(x, out_h, -2, round_half), out_w, -1, round_half)
    else:
        x = _pass(_pass(x, out_w, -1, round_half), out_h, -2, round_half)
    return x.to(torch.uint8)


def preprocess_u8(u8_chw: torch.Tensor) -> torch.Tensor:
    """uint8 [n, 3, H, W] -> the resized, centre-cropped uint8 [n, 3, 224, 224]."""
    h, w = u8_chw.shape[-2:]
    rh, rw = resize_shape(h, w)
    r = pil_resize(u8_chw, rh, rw)
    top, left = (rh - CROP) // 2, (rw - CROP) // 2
    return r[..., top:top + CROP, left:left + CROP]


def normalise(u8: torch.Tensor) -> torch.Tensor:
    mean = torch.tensor(CLIP_MEAN, dtype=torch.float32).view(3, 1, 1)
    std = torch.tensor(CLIP_STD, dtype=torch.float32).view(3, 1, 1)
    return (u8.to(torch.float32) / 255.0 - mean) / std


def pixel_values(images) -> torch.Tensor:
    """The reference's processor output: `images` is fp32 [n, 3, H, W] in [0, 1] (renders), uint8 [n, H, W, 3], or a list of
    PIL images (converted to RGB)."""
    if isinstance(images, torch.Tensor):
        t = images.detach().cpu()
        u8 = t.permute(0, 3, 1, 2) if t.dtype == torch.uint8 else quantise(t)
        return normalise(preprocess_u8(u8))
    return torch.cat([normalise(preprocess_u8(torch.from_numpy(np.array(im.convert("RGB"))).permute(2, 0, 1)[None]))
                      for im in images])


# ------------------------------------------------------------------------------------------------ vision tower
def config_of(cfg) -> SimpleNamespace:
    """The fields the tower uses, from a transformers CLIPVisionConfig, a dict or a namespace."""
    get = (lambda k, d=None: cfg.get(k, d)) if isinstance(cfg, dict) else (lambda k, d=None: getattr(cfg, k, d))
    return SimpleNamespace(hidden_size=get("hidden_size"), intermediate_size=get("intermediate_size"),
                           num_attention_heads=get("num_attention_heads"), num_hidden_layers=get("num_hidden_layers"),
                           image_size=get("image_size", 224), patch_size=get("patch_size", 14),
                           projection_dim=get("projection_dim"), layer_norm_eps=get("layer_norm_eps", 1e-5),
                           hidden_act=get("hidden_act", "gelu"), num_channels=get("num_channels", 3))


def random_state_dict(cfg, seed: int = 0, std: float = 0.02) -> dict:
    """A random CLIPVisionModelWithProjection state dict (fp32) with transformers' key names."""
    c = config_of(cfg)
    g = torch.Generator().manual_seed(seed)
    H, I, P = c.hidden_size, c.intermediate_size, c.patch_size
    T = (c.image_size // P) ** 2 + 1
    r = lambda *s: torch.randn(*s, generator=g) * std
    ln = lambda: (1 + 0.1 * torch.randn(H, generator=g), 0.1 * torch.randn(H, generator=g))
    sd = {"vision_model.embeddings.class_embedding": torch.randn(H, generator=g) * 0.5,
          "vision_model.embeddings.patch_embedding.weight": r(H, c.num_channels, P, P) * 5,
          "vision_model.embeddings.position_embedding.weight": torch.randn(T, H, generator=g) * 0.1}
    for name in ("vision_model.pre_layrnorm", "vision_model.post_layernorm"):
        sd[name + ".weight"], sd[name + ".bias"] = ln()
    for i in range(c.num_hidden_layers):
        p = f"vision_model.encoder.layers.{i}."
        for proj in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{proj}.weight"], sd[p + f"self_attn.{proj}.bias"] = r(H, H), r(H)
        for n in ("layer_norm1", "layer_norm2"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = ln()
        sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"] = r(I, H), r(I)
        sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"] = r(H, I), r(H)
    sd["visual_projection.weight"] = r(c.projection_dim, H)
    return sd


def vision_forward(sd: dict, cfg, pixel_values: torch.Tensor) -> torch.Tensor:
    """CLIPVisionModelWithProjection(pixel_values).image_embeds in fp32: [n, projection_dim]."""
    c = config_of(cfg)
    f = lambda k: sd[k].float()
    H, nh = c.hidden_size, c.num_attention_heads
    hd = H // nh
    x = F.conv2d(pixel_values.float(), f("vision_model.embeddings.patch_embedding.weight"), stride=c.patch_size)
    x = x.flatten(2).transpose(1, 2)
    n = x.shape[0]
    cls = f("vision_model.embeddings.class_embedding").expand(n, 1, H)
    x = torch.cat([cls, x], 1) + f("vision_model.embeddings.position_embedding.weight")[None]
    lnorm = lambda t, p: F.layer_norm(t, (H,), f(p + ".weight"), f(p + ".bias"), c.layer_norm_eps)
    lin = lambda t, p: F.linear(t, f(p + ".weight"), f(p + ".bias"))
    x = lnorm(x, "vision_model.pre_layrnorm")
    L = x.shape[1]
    for i in range(c.num_hidden_layers):
        p = f"vision_model.encoder.layers.{i}."
        h = lnorm(x, p + "layer_norm1")
        q, k, v = (lin(h, p + f"self_attn.{s}_proj").view(n, L, nh, hd).transpose(1, 2) for s in "qkv")
        a = torch.softmax((q * hd ** -0.5) @ k.transpose(-1, -2), -1) @ v
        x = x + lin(a.transpose(1, 2).reshape(n, L, H), p + "self_attn.out_proj")
        h = lnorm(x, p + "layer_norm2")
        x = x + lin(F.gelu(lin(h, p + "mlp.fc1")), p + "mlp.fc2")
    pooled = lnorm(x[:, 0], "vision_model.post_layernorm")
    return pooled @ f("visual_projection.weight").t()
