"""nn.Module surface of the MV motion UNet (SURVEY 8b "UNet module" and "diffusers attention-processor protocol").

The engine never executes these modules: it repacks their parameters into fused fp16 operands (`unet.py::_prepare`, and
`processor_exec.pack_*` for the attention processors).  They exist so that code written against the reference keeps working
unchanged:

  * `state_dict()` / `load_state_dict()` with the reference's key names (diffusers 0.28 naming, processors' parameters under
    `<attn>.processor.*`), the 726-missing rule of inference.py:219-223
  * attribute paths the reference's scripts poke: `unet.down_blocks[i].motion_modules[j].transformer_blocks[0].pos_embed`
    (inference.py:183-192), `attn_module.to_q.weight`, `attn_module.to_out[0].out_features` (inference.py:152-160)
  * `unet.attn_processors` / `unet.set_attn_processor(dict)` (unet_motion_mv_model.py:441-497) with processor classes of the
    reference's names and constructor arguments (attention_processor.py:129-167, 302-323, 448-539)

Only the released wiring is executable (inference.py:107-174: SpatioTemporalI2V on every motion-module attention,
MVDreamI2V on attn1 and IPAdapter on attn2 of every spatial transformer); anything else is rejected loudly."""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, Optional

import torch
from torch import nn

from .unet_config import UNetConfig, key_plan, sinusoidal_pe


class Node(nn.Module):
    """Generic container: children are addressed by attribute or, for numeric names, by index (ModuleList behaviour)."""

    def __getitem__(self, i: int) -> nn.Module:
        return self._modules[str(i if i >= 0 else len(self) + i)]

    def __len__(self) -> int:
        return sum(1 for k in self._modules if k.isdigit())

    def __iter__(self):
        return (self._modules[str(i)] for i in range(len(self)))

    @property
    def out_features(self) -> int:
        return self.weight.shape[0]

    @property
    def in_features(self) -> int:
        return self.weight.shape[1]

    def forward(self, *a, **k):
        raise RuntimeError("animate3d_b200 modules hold parameters for the sm_90a engine; they are not executed one by one "
                           "-- call MVUNetMotionModel.forward")


def _linear(cout: int, cin: int, bias: bool, device) -> Node:
    n = Node()
    n.weight = nn.Parameter(torch.zeros(cout, cin, device=device), requires_grad=False)
    if bias:
        n.bias = nn.Parameter(torch.zeros(cout, device=device), requires_grad=False)
    return n


# ------------------------------------------------------------------------------------------------ processors
class _Processor(Node):
    kind = ""

    def signature(self) -> tuple:
        raise NotImplementedError

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, *args, **kwargs):
        """diffusers attention-processor protocol (attention_processor.py:39-48, 169-178, 325-334, 541-550).  Runs the packer and
        launch stages of `animate3d_b200.processor_exec` that `MVUNetMotionModel.forward` runs for every attention layer, on
        fresh tensors instead of the UNet's activation arena."""
        from . import processor_exec
        return processor_exec.run(self, attn, hidden_states, encoder_hidden_states, attention_mask, temb, **kwargs)


class MVDreamI2VXFormersAttnProcessor(_Processor):
    """attention_processor.py:302-445.  Parameters: to_q_i2v (no bias), to_out_i2v (bias)."""
    kind = "MVDreamI2VXFormersAttnProcessor"

    def __init__(self, attention_op=None, hidden_size: int = 128, num_views: int = 4, num_frames: int = 8, device=None):
        super().__init__()
        self.attention_op, self.hidden_size, self.num_views, self.num_frames = attention_op, hidden_size, num_views, num_frames
        self.to_q_i2v = _linear(hidden_size, hidden_size, False, device)
        self.to_out_i2v = _linear(hidden_size, hidden_size, True, device)

    def signature(self):
        return (self.kind, self.hidden_size, self.num_views, self.num_frames)


class IPAdapterXFormersAttnProcessor(_Processor):
    """attention_processor.py:129-298.  Parameters: to_k_ip[i], to_v_ip[i] (no bias), one pair per image-token group."""
    kind = "IPAdapterXFormersAttnProcessor"

    def __init__(self, hidden_size: int, cross_attention_dim: Optional[int] = None, num_tokens=(4,), scale=1.0, attention_op=None,
                 device=None):
        super().__init__()
        if not isinstance(num_tokens, (tuple, list)):
            num_tokens = [num_tokens]
        if not isinstance(scale, list):
            scale = [scale] * len(num_tokens)
        if len(scale) != len(num_tokens):
            raise ValueError("`scale` should be a list of integers with the same length as `num_tokens`.")
        self.hidden_size, self.cross_attention_dim, self.num_tokens, self.scale = hidden_size, cross_attention_dim, list(num_tokens), scale
        self.attention_op = attention_op
        self.to_k_ip, self.to_v_ip = Node(), Node()
        for i in range(len(num_tokens)):
            self.to_k_ip.add_module(str(i), _linear(hidden_size, cross_attention_dim, False, device))
            self.to_v_ip.add_module(str(i), _linear(hidden_size, cross_attention_dim, False, device))

    def signature(self):
        return (self.kind, self.hidden_size, self.cross_attention_dim, tuple(self.num_tokens), tuple(float(s) for s in self.scale))


def released_attn_cfg():
    """configs/inference/inference.yaml:9-24 as the attribute bags the reference passes to the processor constructor."""
    spatial = SimpleNamespace(enabled=True, attn_cfg=SimpleNamespace(use_spatial_encoding=True, use_camera_encoding=False,
                                                                     spatial_encoding_type="sinusoid", camera_encoding_type="sinusoid"))
    return spatial, SimpleNamespace(enabled=False)


class SpatioTemporalI2VXFormersAttnProcessor(_Processor):
    """attention_processor.py:448-723 in the released configuration: spatial (cross-view) attention on with the 2-D sinusoid
    encoding, image attention off, learned alpha blender.  Parameters: to_{q,k,v}_sp (no bias), to_out_sp (bias),
    time_pos_embed.pe (buffer), alpha_blender.mix_factor."""
    kind = "SpatioTemporalI2VXFormersAttnProcessor"

    def __init__(self, attention_op=None, hidden_size: int = 128, feature_size: int = 64, num_views: int = 4, num_frames: int = 16,
                 spatial_attn=None, image_attn=None, use_alpha_blender: bool = False, device=None, max_seq_length: int = 32):
        super().__init__()
        if spatial_attn is None or image_attn is None:
            spatial_attn, image_attn = released_attn_cfg()
        ac = spatial_attn.attn_cfg
        if not (spatial_attn.enabled and ac.use_spatial_encoding and not ac.use_camera_encoding and ac.spatial_encoding_type == "sinusoid"
                and not image_attn.enabled and use_alpha_blender):
            raise NotImplementedError("only the released motion-module attention configuration is built for the engine: spatial "
                                      "attention with sinusoid 2-D encoding, no camera encoding, no image attention, alpha blender "
                                      "(configs/inference/inference.yaml:9-24)")
        self.attention_op, self.hidden_size, self.feature_size = attention_op, hidden_size, feature_size
        self.num_views, self.num_frames = num_views, num_frames
        self.use_spatial_attn, self.use_spatial_encoding, self.use_camera_encoding = True, True, False
        self.spatial_encoding_type, self.use_image_attn, self.use_alpha_blender = "sinusoid", False, True
        for n in ("to_q_sp", "to_k_sp", "to_v_sp"):
            setattr(self, n, _linear(hidden_size, hidden_size, False, device))
        self.to_out_sp = _linear(hidden_size, hidden_size, True, device)
        self.time_pos_embed = Node()
        self.time_pos_embed.register_buffer("pe", sinusoidal_pe(hidden_size, max_seq_length).to(device))
        self.alpha_blender = Node()
        self.alpha_blender.mix_factor = nn.Parameter(torch.zeros(1, device=device), requires_grad=False)   # AlphaBlender(alpha=0.0)

    def signature(self):
        return (self.kind, self.hidden_size, self.feature_size, self.num_views, self.num_frames)


PROCESSOR_CLASSES = {c.kind: c for c in (MVDreamI2VXFormersAttnProcessor, IPAdapterXFormersAttnProcessor, SpatioTemporalI2VXFormersAttnProcessor)}


class AttentionNode(Node):
    """The part of diffusers `Attention` the reference's processors and scripts touch: to_q / to_k / to_v / to_out[0],
    heads, scale, get_processor / set_processor."""

    def __init__(self, heads: int, dim_head: int):
        super().__init__()
        self.heads, self.scale = heads, dim_head ** -0.5
        self.inner_dim = heads * dim_head
        self.residual_connection, self.rescale_output_factor = False, 1.0
        self.spatial_norm = self.group_norm = self.norm_cross = None

    def get_processor(self, return_deprecated_lora: bool = False):
        return self.processor

    def set_processor(self, processor) -> None:
        """Accepts a processor of the SAME kind and hyper-parameters as the slot's (the released wiring); its parameters are
        copied.  Instances of the reference's own classes qualify (matched by class name and attributes)."""
        cur: _Processor = self.processor
        kind = type(processor).__name__
        if kind != cur.kind:
            raise ValueError(f"this attention slot runs {cur.kind} in the released model (inference.py:107-174); got {kind}. "
                             "The H100 engine implements the released wiring only.")
        want = cur.signature()
        got = _foreign_signature(processor)
        if got != want:
            raise ValueError(f"{kind}: constructor arguments {got[1:]} do not match the model geometry {want[1:]}")
        sd = processor.state_dict()
        missing = [k for k in cur.state_dict() if k not in sd]
        extra = [k for k in sd if k not in cur.state_dict()]
        if missing or extra:
            raise ValueError(f"{kind}: parameter names differ from the released layout (missing {missing}, unexpected {extra})")
        with torch.no_grad():
            for k, v in cur.state_dict().items():
                v.copy_(sd[k].to(v.device, v.dtype))


def _foreign_signature(p) -> tuple:
    kind = type(p).__name__
    if kind == "MVDreamI2VXFormersAttnProcessor":
        return (kind, p.hidden_size, p.num_views, p.num_frames)
    if kind == "IPAdapterXFormersAttnProcessor":
        return (kind, p.hidden_size, p.cross_attention_dim, tuple(p.num_tokens), tuple(float(s) for s in p.scale))
    if kind == "SpatioTemporalI2VXFormersAttnProcessor":
        ok = (getattr(p, "use_spatial_attn", False) and getattr(p, "use_spatial_encoding", False) and not getattr(p, "use_camera_encoding", True)
              and getattr(p, "spatial_encoding_type", "") == "sinusoid" and not getattr(p, "use_image_attn", True)
              and getattr(p, "use_alpha_blender", False))
        if not ok:
            raise ValueError("SpatioTemporalI2VXFormersAttnProcessor: only the released configuration (spatial sinusoid encoding, "
                             "no camera encoding, no image attention, alpha blender) runs on the engine")
        return (kind, p.hidden_size, p.feature_size, p.num_views, p.num_frames)
    raise ValueError(f"unknown attention processor class {kind}")


# ------------------------------------------------------------------------------------------------ tree builder
def _processor_for(path: str, cfg: UNetConfig, c: int, level_feature: int, device) -> _Processor:
    if ".motion_modules." in path:
        return SpatioTemporalI2VXFormersAttnProcessor(hidden_size=c, feature_size=level_feature, num_views=cfg.num_views,
                                                      num_frames=cfg.num_frames, use_alpha_blender=True, device=device,
                                                      max_seq_length=cfg.motion_max_seq_length)
    if path.endswith("attn1.processor"):
        return MVDreamI2VXFormersAttnProcessor(hidden_size=c, num_views=cfg.num_views, num_frames=cfg.num_frames, device=device)
    return IPAdapterXFormersAttnProcessor(hidden_size=c, cross_attention_dim=cfg.cross_attention_dim, num_tokens=(cfg.ip_num_tokens,),
                                          scale=cfg.ip_scale, device=device)


def _level_of(path: str, cfg: UNetConfig) -> int:
    n = len(cfg.block_out_channels)
    if path.startswith("down_blocks."):
        return int(path.split(".")[1])
    if path.startswith("up_blocks."):
        return n - 1 - int(path.split(".")[1])
    return n - 1


def build_tree(root: nn.Module, cfg: UNetConfig, device) -> None:
    """Attach one parameter (or buffer) per entry of `key_plan(cfg)` under `root`, creating the module path on the way."""
    plan = key_plan(cfg)
    for key, shape in plan.items():
        parts = key.split(".")
        node = root
        for depth, name in enumerate(parts[:-1]):
            child = node._modules.get(name)
            if child is None:
                path = ".".join(parts[:depth + 1])
                lvl = _level_of(path, cfg)
                c = cfg.block_out_channels[lvl]
                if name == "processor":
                    child = _processor_for(path, cfg, c, cfg.feature_size(lvl), device)
                elif name in ("attn1", "attn2"):
                    heads = cfg.motion_num_attention_heads if ".motion_modules." in path else cfg.num_attention_heads
                    child = AttentionNode(heads, c // heads)
                else:
                    child = Node()
                    if name == "0" and parts[depth - 1] == "transformer_blocks":
                        child.pos_embed = None        # inference.py:183-192 sets it to None; the engine never had one
                node.add_module(name, child)
            node = child
        leaf = parts[-1]
        if leaf in node._parameters or leaf in node._buffers:
            if tuple(getattr(node, leaf).shape) != tuple(shape):
                raise AssertionError(f"{key}: processor built {tuple(getattr(node, leaf).shape)}, key plan says {shape}")
            continue
        if leaf == "pe":
            node.register_buffer("pe", sinusoidal_pe(shape[2], shape[1]).to(device))
        else:
            init = torch.ones if (leaf == "weight" and len(shape) == 1) else torch.zeros      # norm scales start at 1
            node.register_parameter(leaf, nn.Parameter(init(shape, device=device), requires_grad=False))


def attn_processors_of(root: nn.Module) -> Dict[str, _Processor]:
    """unet_motion_mv_model.py:441-462."""
    out: Dict[str, _Processor] = {}

    def rec(name, module):
        if hasattr(module, "get_processor"):
            out[f"{name}.processor"] = module.get_processor(return_deprecated_lora=True)
        for sub, child in module.named_children():
            rec(f"{name}.{sub}", child)

    for name, module in root.named_children():
        rec(name, module)
    return out
