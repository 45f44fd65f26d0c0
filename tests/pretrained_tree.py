"""Writes a checkpoint tree in the published layout (mvdream-sd1.5-diffusers, animatediff-motion-adapter-v1-5-2,
IP-Adapter, the Animate3D motion-module checkpoint) from seeded random weights, and builds the same model by hand from the
same tensors (INTEGRATION §1), for the from_pretrained tests."""
from __future__ import annotations

import json
import os
from types import SimpleNamespace

import torch

from animate3d_b200.unet_config import UNetConfig
from animate3d_b200.weights import random_state_dict

IP = "encoder_hid_proj.image_projection_layers.0"


def is_motion(k: str) -> bool:
    """The keys the released motion-module checkpoint holds (train.py's trainable subset)."""
    return "motion_modules." in k or "i2v." in k


def attn2_processors(cfg: UNetConfig):
    """Spatial attn2 processor names in `attn_processors` order (the IP-Adapter file numbers them 1, 3, 5, ...)."""
    from animate3d_b200.unet import MVUNetMotionModel
    names = list(MVUNetMotionModel(cfg, device="meta").attn_processors)
    return [n for n in names if n.endswith("attn2.processor") and ".attentions." in n]


def split(cfg: UNetConfig, seed: int, dtype=torch.float32, device="cpu"):
    """-> dict of the published files' contents: unet, adapter, ip (image_proj / ip_adapter), ckpt (motion modules).
    The adapter's motion-module weights differ from the checkpoint's, which must win."""
    full = {k: v.to("cpu", dtype) for k, v in random_state_dict(cfg, seed, device=device).items()}
    other = {k: v.to("cpu", dtype) for k, v in random_state_dict(cfg, seed + 1, device=device).items()}
    unet = {k: v for k, v in full.items() if not is_motion(k) and not k.startswith(IP) and "_ip." not in k}
    adapter = {k: other[k] for k in full if "motion_modules." in k and ".processor." not in k}
    for k in [k for k in adapter if k.endswith("attn1.to_q.weight")]:      # diffusers' MotionAdapter also holds these
        adapter[k.replace("attn1.to_q.weight", "pos_embed.pe")] = torch.zeros(1, 32, adapter[k].shape[0], dtype=dtype)
    ip = {"image_proj": {"proj.weight": full[f"{IP}.image_embeds.weight"], "proj.bias": full[f"{IP}.image_embeds.bias"],
                         "norm.weight": full[f"{IP}.norm.weight"], "norm.bias": full[f"{IP}.norm.bias"]},
          "ip_adapter": {}}
    for i, n in enumerate(attn2_processors(cfg)):
        ip["ip_adapter"][f"{2 * i + 1}.to_k_ip.weight"] = full[f"{n}.to_k_ip.0.weight"]
        ip["ip_adapter"][f"{2 * i + 1}.to_v_ip.weight"] = full[f"{n}.to_v_ip.0.weight"]
    ckpt = {k: v for k, v in full.items() if is_motion(k)}
    return SimpleNamespace(full=full, unet=unet, adapter=adapter, ip=ip, ckpt=ckpt)


def unet_config_json(cfg: UNetConfig) -> dict:
    return {"_class_name": "MVUNet2DConditionModel", "in_channels": cfg.in_channels, "out_channels": cfg.out_channels,
            "block_out_channels": list(cfg.block_out_channels), "layers_per_block": cfg.layers_per_block,
            "norm_num_groups": cfg.norm_num_groups, "norm_eps": cfg.norm_eps, "cross_attention_dim": cfg.cross_attention_dim,
            "attention_head_dim": cfg.num_attention_heads, "sample_size": 32,
            "down_block_types": ["CrossAttnDownBlock2D" if a else "DownBlock2D" for a in cfg.down_has_attn],
            "up_block_types": ["CrossAttnUpBlock2D" if a else "UpBlock2D" for a in reversed(cfg.down_has_attn)]}


def adapter_config_json(cfg: UNetConfig) -> dict:
    return {"_class_name": "MotionAdapter", "block_out_channels": list(cfg.block_out_channels), "motion_layers_per_block": 2,
            "motion_mid_block_layers_per_block": 1, "motion_num_attention_heads": cfg.motion_num_attention_heads,
            "motion_norm_num_groups": 32, "motion_max_seq_length": cfg.motion_max_seq_length, "use_motion_mid_block": True,
            "conv_in_channels": None}


def write_json(path, obj):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        json.dump(obj, f)


def write_tree(root, cfg: UNetConfig, parts, vae_config: dict, vae_sd: dict):
    """root/base/{unet,vae}, root/adapter, root/ip/models/ip-adapter_sd15.{bin,safetensors}, root/motion.ckpt."""
    from safetensors.torch import save_file
    root = str(root)
    base, adapter, ip = os.path.join(root, "base"), os.path.join(root, "adapter"), os.path.join(root, "ip")
    write_json(os.path.join(base, "unet", "config.json"), unet_config_json(cfg))
    save_file({k: v.contiguous() for k, v in parts.unet.items()}, os.path.join(base, "unet", "diffusion_pytorch_model.safetensors"))
    write_json(os.path.join(base, "vae", "config.json"), {"_class_name": "AutoencoderKL", "act_fn": "silu",
                                                          "down_block_types": ["DownEncoderBlock2D"] * 4,
                                                          "up_block_types": ["UpDecoderBlock2D"] * 4, **vae_config})
    torch.save(vae_sd, os.path.join(base, "vae", "diffusion_pytorch_model.bin"))
    write_json(os.path.join(adapter, "config.json"), adapter_config_json(cfg))
    save_file({k: v.contiguous() for k, v in parts.adapter.items()}, os.path.join(adapter, "diffusion_pytorch_model.safetensors"))
    os.makedirs(os.path.join(ip, "models"), exist_ok=True)
    torch.save(parts.ip, os.path.join(ip, "models", "ip-adapter_sd15.bin"))
    save_file({f"{p}.{k}": v.contiguous() for p, d in parts.ip.items() for k, v in d.items()},
              os.path.join(ip, "models", "ip-adapter_sd15.safetensors"))
    torch.save({"state_dict": parts.ckpt, "epoch": 3}, os.path.join(root, "motion.ckpt"))
    return SimpleNamespace(root=root, base=base, adapter=adapter, ip=ip, ckpt=os.path.join(root, "motion.ckpt"))


def hand_assembled_unet(cfg: UNetConfig, parts, device, **kwargs):
    """INTEGRATION §1: from_unet2d on the two source models, the IP-Adapter state dict, then the motion-module checkpoint
    with strict=False and 726 keys missing."""
    from animate3d_b200.unet import MVUNetMotionModel
    mvunet = SimpleNamespace(config=unet_config_json(cfg), state_dict=lambda: parts.unet)
    motion_adapter = SimpleNamespace(config=adapter_config_json(cfg), state_dict=lambda: parts.adapter)
    unet = MVUNetMotionModel.from_unet2d(mvunet, motion_adapter, device=device, **kwargs)
    unet._load_ip_adapter_weights(parts.ip)
    missing, unexpected = unet.load_state_dict(parts.ckpt, strict=False)
    assert len(missing) == 726 and not unexpected
    return unet
