"""Checkpoint files on disk -> the tensors and configs the engine's loaders take, as the reference's loading code reads
them (inference.py:60-245, animatemv_guidance.py:115-160, animatediff/utils/util.py:49-170).

Local only: a checkpoint is a directory, or a Hugging Face id already in the hub cache on disk.  Nothing here downloads or
opens a connection; a checkpoint that is not on disk is a FileNotFoundError naming every place that was searched."""
from __future__ import annotations

import json
import os
from types import SimpleNamespace
from typing import Dict, List, Optional

import torch

WEIGHTS_NAME = "diffusion_pytorch_model"
IP_ADAPTER_WEIGHTS = ("ip-adapter_sd15.bin", "ip-adapter_sd15.safetensors")      # util.py:49 weight_name, then its twin


def hub_cache_dir() -> str:
    """$HF_HUB_CACHE, else $HF_HOME/hub, else ~/.cache/huggingface/hub (huggingface_hub's lookup order)."""
    if os.environ.get("HF_HUB_CACHE"):
        return os.environ["HF_HUB_CACHE"]
    if os.environ.get("HF_HOME"):
        return os.path.join(os.environ["HF_HOME"], "hub")
    return os.path.join(os.path.expanduser("~"), ".cache", "huggingface", "hub")


def resolve(name_or_path: Optional[str], subfolder: Optional[str] = None) -> str:
    """A checkpoint directory, or a hub id ("org/name"), plus an optional subfolder -> an existing local directory.

    A directory is used as is.  An id is looked up in the hub cache (`hub_cache_dir`): the snapshot named by
    `models--{org}--{name}/refs/main`.  A miss raises FileNotFoundError listing every place it looked."""
    if not name_or_path:
        raise FileNotFoundError(f"no checkpoint path or hub id given (got {name_or_path!r})")
    name_or_path = os.fspath(name_or_path)
    looked: List[str] = []
    if os.path.isdir(name_or_path):
        path = os.path.join(name_or_path, subfolder) if subfolder else name_or_path
        if os.path.isdir(path):
            return path
        looked.append(path)
    else:
        looked.append(name_or_path)
        if name_or_path.count("/") == 1 and not name_or_path.startswith((".", "/")):
            repo = os.path.join(hub_cache_dir(), "models--" + name_or_path.replace("/", "--"))
            ref = os.path.join(repo, "refs", "main")
            if os.path.isfile(ref):
                with open(ref) as f:
                    snap = os.path.join(repo, "snapshots", f.read().strip())
                path = os.path.join(snap, subfolder) if subfolder else snap
                if os.path.isdir(path):
                    return path
                looked.append(path)
            else:
                looked.append(ref)
    raise FileNotFoundError(f"checkpoint {name_or_path!r}{f' (subfolder {subfolder!r})' if subfolder else ''} is not on "
                            f"disk; looked in: {', '.join(looked)}.  Nothing is downloaded: fetch it into the hub cache "
                            "or pass a local directory")


def read_config(directory: str) -> dict:
    path = os.path.join(directory, "config.json")
    if not os.path.isfile(path):
        raise FileNotFoundError(f"no config.json in {directory}")
    with open(path) as f:
        return json.load(f)


def load_weights(directory: str, name: str = WEIGHTS_NAME) -> Dict[str, torch.Tensor]:
    """`{name}.safetensors`, else `{name}.bin` (torch.load with weights_only=True), on the CPU.  Sharded checkpoints (an
    index file) are not read."""
    for ext in (".safetensors", ".bin"):
        index = os.path.join(directory, f"{name}{ext}.index.json")
        if os.path.isfile(index):
            raise NotImplementedError(f"sharded checkpoint {index}: only single-file weights are read")
    st, pt = os.path.join(directory, f"{name}.safetensors"), os.path.join(directory, f"{name}.bin")
    if os.path.isfile(st):
        from safetensors.torch import load_file
        return load_file(st)
    if os.path.isfile(pt):
        return torch.load(pt, map_location="cpu", weights_only=True)
    raise FileNotFoundError(f"no weights in {directory}: looked for {st} and {pt}")


def load_model(name_or_path: str, subfolder: Optional[str] = None) -> SimpleNamespace:
    """config.json + weights of a diffusers model directory as an object with `.config` and `.state_dict()`: what
    `MVUNetMotionModel.from_unet2d` reads from the reference's MVUNet2DConditionModel and MotionAdapter."""
    directory = resolve(name_or_path, subfolder)
    config, sd = read_config(directory), load_weights(directory)
    return SimpleNamespace(config=config, state_dict=lambda: sd, path=directory)


def ip_adapter_file(ip_adapter_path: str) -> str:
    """`<ip_adapter_path>/models/ip-adapter_sd15.bin`, else its `.safetensors` twin."""
    directory = resolve(ip_adapter_path, "models")
    for n in IP_ADAPTER_WEIGHTS:
        if os.path.isfile(os.path.join(directory, n)):
            return os.path.join(directory, n)
    raise FileNotFoundError(f"no IP-Adapter weights in {directory}: looked for {', '.join(IP_ADAPTER_WEIGHTS)}")


def load_ip_adapter(path: str) -> Dict[str, Dict[str, torch.Tensor]]:
    """One IP-Adapter weight file -> {"image_proj": {...}, "ip_adapter": {...}} (util.py:124-142): a .safetensors file is
    split by its `image_proj.` / `ip_adapter.` key prefixes, a .bin file already holds the two dicts."""
    if not os.path.isfile(path):
        raise FileNotFoundError(f"no IP-Adapter weights at {path}")
    if path.endswith(".safetensors"):
        from safetensors import safe_open
        sd: Dict[str, Dict[str, torch.Tensor]] = {"image_proj": {}, "ip_adapter": {}}
        with safe_open(path, framework="pt", device="cpu") as f:
            for key in f.keys():
                for prefix in sd:
                    if key.startswith(prefix + "."):
                        sd[prefix][key[len(prefix) + 1:]] = f.get_tensor(key)
    else:
        sd = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(sd, dict) or list(sd.keys()) != ["image_proj", "ip_adapter"]:
        raise ValueError(f"{path}: required keys (`image_proj` and `ip_adapter`) missing from the state dict")
    return sd


# inference.yaml:9-24 and refine_frame_16.yaml:133-149: the attention wiring the released weights were trained with
RELEASED_ATTN_CFG = {
    "mvdream_attn_cfg": {"image_attn": {"enabled": True}},
    "motion_module_attn_cfg": {"enabled": True,
                               "spatial_attn": {"enabled": True,
                                                "attn_cfg": {"use_spatial_encoding": True, "spatial_encoding_type": "sinusoid",
                                                             "use_camera_encoding": False}},
                               "image_attn": {"enabled": False},
                               "use_alpha_blender": True},
}


def check_model_config(model_config: Optional[dict]) -> None:
    """Raises NotImplementedError naming the first entry of `mvdream_attn_cfg` / `motion_module_attn_cfg` that differs
    from the released wiring (the engine builds that wiring only).  Entries left out take the released value;
    `camera_encoding_type` is not read while camera encoding is off, and `i2v_cond_time_zero` is a sampling option the
    UNet forward takes either way."""
    def walk(want, got, path):
        if got is None:
            return
        if isinstance(want, dict):
            if not hasattr(got, "get"):
                raise NotImplementedError(f"model_config.{path} must be a mapping, got {got!r}")
            for k, v in want.items():
                walk(v, got.get(k), f"{path}.{k}")
        elif got != want:
            raise NotImplementedError(f"model_config.{path} = {got!r}: the engine implements the released wiring only "
                                      f"({path} = {want!r})")
    if model_config is None:
        return
    for k, v in RELEASED_ATTN_CFG.items():
        walk(v, model_config.get(k), k)
    flag = model_config.get("i2v_cond_time_zero", False)
    if not isinstance(flag, bool):
        raise ValueError(f"model_config.i2v_cond_time_zero must be true or false, got {flag!r}")
