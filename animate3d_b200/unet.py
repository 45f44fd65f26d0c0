"""Host-side mirror of the reference's `MVUNetMotionModel` (animatediff/models/unet_motion_mv_model.py:55-867) whose forward
runs entirely on the sm_90a kernels of liba3d.so.

Same constructor geometry, same state-dict keys (incl. the processors' `<attn>.processor.*` parameters installed by
inference.py:107-174), same `forward(sample, timestep, encoder_hidden_states, ..., camera, num_views, i2v_cond_time_zero)`
signature and `UNet3DConditionOutput(sample=...)` result.  What differs is everything underneath:

  * activations are token-major (NHWC) fp16 end to end: the reference's two whole-tensor layout copies (lines 767, 862)
    fold into conv_in / conv_out, and every "(b n f) l c -> (b f) (n l) c" / "(b l) f c -> (b f) l c" regroup and the
    frame-0 K/V broadcast of the processors (attention_processor.py:340, 389-397, 557, 669) become strides of a rank-5 TMA
    view read in place by the attention kernel -- nothing is ever rearranged or cloned
  * every Linear/Conv is one wgmma GEMM (implicit im2col for 3x3) with bias / time-embedding / residual / GEGLU /
    alpha-blend / row-permute fused into its epilogue; q,k,v(,q_i2v) projections are one GEMM per attention
  * positional encodings are folded into the projections: (x + pe) W = x W + (pe W), the second term is a per-position
    row-bias table computed once at load
  * text / IP-adapter K,V are computed once per (view) instead of once per frame (unet_motion_mv_model.py:754, 763 repeat
    them F times)
  * the whole forward is captured in one CUDA graph after the first call; inside a caller's capture (a captured refine step,
    capture.StepGraphs) it records its kernels into that graph instead, on the buffers of an earlier eager call
Torch is used for device memory and the stream only; there is no fallback path.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

from . import _lib as L
from . import ops
from . import processor_exec as P
from .capture import capturing, note_module
from .modules import attn_processors_of, build_tree
from .processor_exec import HALF, _Lin, linear
from .unet_config import UNetConfig, key_plan, up_plan


@dataclass
class UNet3DConditionOutput:
    sample: torch.Tensor


def _geglu_interleave(w: torch.Tensor) -> torch.Tensor:
    """rows [u(4C) | g(4C)] -> blocks of 32: [u0..31 | g0..31 | u32..63 | g32..63 ...] (GEMM GEGLU epilogue layout)."""
    half = w.shape[0] // 2
    u, g = w[:half], w[half:]
    rest = w.shape[1:]
    return torch.stack([u.reshape(half // 32, 32, *rest), g.reshape(half // 32, 32, *rest)], dim=1).reshape(w.shape)


class MVUNetMotionModel(torch.nn.Module):
    """Drop-in for the reference class on the inference path (eval mode, no grad -- the reference never back-propagates
    through the UNet: animatemv_guidance.py:422, pipeline.py:758).

    It IS an nn.Module: its parameter tree carries the reference's state-dict keys (fp32 masters on the device, see
    modules.py), `attn_processors` / `set_attn_processor` / `from_unet2d` / `.to()` / `.config` behave like the reference's.
    The forward does not execute those modules one by one: `_prepare()` repacks them into fused fp16 operands once."""

    def __init__(self, config: Optional[UNetConfig] = None, device: str = "cuda", view_group=None, **kwargs):
        """view_group: a torch.distributed process group whose ranks each hold ONE view of the same prompts (SURVEY 8e,
        "views span ranks").  Everything stays local except the cross-view attentions, whose K/V are all-gathered over the
        group (NCCL over NVLink); forward() is then called with the local view only and num_views=1."""
        super().__init__()
        self.cfg = config or UNetConfig(**kwargs)
        self.view_group = view_group
        self.view_world = 1
        if view_group is not None:
            import torch.distributed as dist
            self.view_world = dist.get_world_size(view_group)
        self.config = self.cfg        # diffusers-style attribute used by the pipeline (`unet.config.in_channels`)
        self._device = torch.device(device)
        build_tree(self, self.cfg, self._device)          # parameters / buffers under the reference's key names
        self._loaded = set()                              # keys that received weights (the engine refuses to run on defaults)
        self._masters_dropped = False
        self._prepared = False
        self._bufs: Dict[str, torch.Tensor] = {}
        self._graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self._static: Dict[tuple, dict] = {}
        # bumped whenever a tensor the recorded kernels read or write may have moved (capture.StepGraphs recaptures then)
        self.capture_version = 0
        # View-sharded forwards run eagerly: capturing the asynchronous NCCL all-gathers of torch 2.11 / NCCL 2.28 in a CUDA graph
        # deadlocks on this stack; the kernels between two gathers are long enough for the launch stream to stay ahead.
        self.use_cuda_graph = view_group is None
        self.launches_per_forward = 0   # kernels enqueued by the last eager run (bench's gpu_launches claim)
        self.collectives = 0         # view-sharded mode: K|V all-gathers issued by the last eager run and their payload
        self.collective_bytes = 0
        self.comm_enabled = True     # False = skip the all-gathers (timing only: measures the compute of the sharded forward)
        self.eval()
        self.requires_grad_(False)

    # ------------------------------------------------------------------------------------------------ module surface
    @property
    def device(self) -> torch.device:
        return self._device

    @property
    def dtype(self) -> torch.dtype:
        return HALF                   # compute dtype of the engine (fp16 operands, fp32 accumulation)

    def to(self, *args, **kwargs):
        """Device moves relocate the fp32 masters and invalidate the packed operands; dtype requests are accepted and ignored
        (the reference calls `.to(torch.float16)`, animatemv_guidance.py:275 -- that IS the engine's operand type)."""
        device = kwargs.get("device")
        for a in args:
            if isinstance(a, (str, torch.device)):
                device = a
            elif isinstance(a, torch.Tensor):
                device = a.device
        if device is not None and torch.device(device) != self._device:
            if torch.device(device).type != "cuda":
                raise RuntimeError("MVUNetMotionModel runs on an sm_90a device only; there is no CPU path")
            super().to(device)
            self._device = torch.device(device)
            self._prepared = False
            self._bufs.clear(); self._graphs.clear(); self._static.clear()
            self.capture_version += 1
        return self

    def half(self):
        return self

    def float(self):
        return self

    @property
    def attn_processors(self):
        """unet_motion_mv_model.py:441-462: {"<path>.processor": processor module} for all 74 attention layers."""
        return attn_processors_of(self)

    def set_attn_processor(self, processor):
        """unet_motion_mv_model.py:465-497.  Only the released wiring runs on the engine: a dict with one processor per layer,
        each of the kind and geometry the released model uses there (modules.AttentionNode.set_processor checks both)."""
        cur = self.attn_processors
        if not isinstance(processor, dict):
            raise ValueError("a single processor for all layers cannot express the released wiring (three processor kinds, "
                             "inference.py:107-174); pass the dict built from `unet.attn_processors`")
        if len(processor) != len(cur):
            raise ValueError(f"A dict of processors was passed, but the number of processors {len(processor)} does not match the"
                             f" number of attention layers: {len(cur)}. Please make sure to pass {len(cur)} processor classes.")
        unknown = [k for k in processor if k not in cur]
        if unknown:
            raise ValueError(f"unknown attention layers: {unknown[:3]}")
        for name, module in self.named_modules():
            if hasattr(module, "set_processor"):
                key = f"{name}.processor"
                new = processor[key]
                if new is not cur[key]:
                    module.set_processor(new)
                    self._loaded.update(f"{key}.{k}" for k in cur[key].state_dict())
        self._prepared = False
        self.capture_version += 1

    @classmethod
    def from_unet2d(cls, unet, motion_adapter=None, load_weights: bool = True, device: str = "cuda", **kwargs):
        """unet_motion_mv_model.py:275-368: geometry from the 2-D multi-view UNet's config, its weights copied, motion modules
        taken from the adapter.  Unlike the reference the result already carries the released processors (inference.py:107-174
        installs them right afterwards): to_q_i2v starts as a copy of to_q and to_out_i2v at zero (inference.py:161-165)."""
        src = unet.config
        get = (lambda k, d=None: src.get(k, d)) if hasattr(src, "get") else (lambda k, d=None: getattr(src, k, d))
        heads = get("num_attention_heads") or get("attention_head_dim")
        heads = heads[0] if isinstance(heads, (tuple, list)) else heads
        cfg_kw = dict(in_channels=get("in_channels", 4), out_channels=get("out_channels", 4),
                      block_out_channels=tuple(get("block_out_channels")), layers_per_block=get("layers_per_block", 2),
                      norm_num_groups=get("norm_num_groups", 32), norm_eps=get("norm_eps", 1e-5),
                      cross_attention_dim=get("cross_attention_dim", 768), num_attention_heads=heads,
                      down_has_attn=tuple("CrossAttn" in t for t in get("down_block_types")))
        if motion_adapter is not None:
            mc = motion_adapter.config
            mget = (lambda k, d=None: mc.get(k, d)) if hasattr(mc, "get") else (lambda k, d=None: getattr(mc, k, d))
            cfg_kw.update(motion_num_attention_heads=mget("motion_num_attention_heads", 8),
                          motion_max_seq_length=mget("motion_max_seq_length", 32))
            if mget("conv_in_channels"):
                raise NotImplementedError("PIA adapters (conv_in_channels) are not part of Animate3D")
        cfg_kw.update(kwargs)
        model = cls(UNetConfig(**cfg_kw), device=device)
        if not load_weights:
            return model
        sd = {k: v for k, v in unet.state_dict().items() if k in key_plan(model.cfg)}
        if motion_adapter is not None:     # load_motion_modules: same "<block>.motion_modules.*" key names
            sd.update({k: v for k, v in motion_adapter.state_dict().items() if k in key_plan(model.cfg)})
        for k in list(sd):                  # the I2V branch of every spatial attn1 starts from to_q (inference.py:161-165)
            if k.endswith("attn1.to_q.weight") and ".attentions." in k:
                sd.setdefault(k.replace("attn1.to_q.weight", "attn1.processor.to_q_i2v.weight"), sd[k])
        model.load_state_dict(sd, strict=False)
        for k in key_plan(model.cfg):        # zero-initialised branches count as initialised
            if k.endswith(("to_out_i2v.weight", "to_out_i2v.bias", "time_pos_embed.pe", "mix_factor")):
                model._loaded.add(k)
        return model

    def _load_ip_adapter_weights(self, state_dict):
        """diffusers' loader hook used by animatediff/utils/util.py::load_ip_adapter: {"image_proj": {...}, "ip_adapter": {...}}
        -> encoder_hid_proj.image_projection_layers.0.* and the 16 attn2 processors' to_k_ip / to_v_ip."""
        sds = state_dict if isinstance(state_dict, (list, tuple)) else [state_dict]
        if len(sds) != 1:
            raise NotImplementedError("one IP-Adapter (the released model's) is supported")
        sd = sds[0]
        ip = "encoder_hid_proj.image_projection_layers.0"
        new = {f"{ip}.image_embeds.weight": sd["image_proj"]["proj.weight"], f"{ip}.image_embeds.bias": sd["image_proj"]["proj.bias"],
               f"{ip}.norm.weight": sd["image_proj"]["norm.weight"], f"{ip}.norm.bias": sd["image_proj"]["norm.bias"]}
        names = [n for n in self.attn_processors if n.endswith("attn2.processor") and ".attentions." in n]
        # diffusers numbers the adapter's layers over ALL attn processors in definition order: attn2 slots are the odd ones
        for i, n in enumerate(names):
            new[f"{n}.to_k_ip.0.weight"] = sd["ip_adapter"][f"{2 * i + 1}.to_k_ip.weight"]
            new[f"{n}.to_v_ip.0.weight"] = sd["ip_adapter"][f"{2 * i + 1}.to_v_ip.weight"]
        self.load_state_dict(new, strict=False)

    # ------------------------------------------------------------------------------------------------ weights
    @staticmethod
    def expected_keys(cfg: Optional[UNetConfig] = None) -> List[str]:
        return list(key_plan(cfg or UNetConfig()).keys())

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True, assign: bool = False):
        """Returns torch's (missing_keys, unexpected_keys) pair.  With strict=False a partial (motion-module-only) checkpoint
        updates what it holds (inference.py:219-223)."""
        if self._masters_dropped:
            raise RuntimeError("the fp32 masters were released (drop_reference_weights); build a new model to load weights")
        res = super().load_state_dict({k: v for k, v in sd.items()}, strict=strict)
        plan = key_plan(self.cfg)
        self._loaded.update(k for k in sd if k in plan)
        self._prepared = False
        self.capture_version += 1
        return res

    def share_packed_weights(self, other: "MVUNetMotionModel"):
        """Use `other`'s packed fp16 operands (same geometry, same device) instead of packing a second copy -- e.g. a
        view-sharded engine next to a whole-batch one in the same process (bench.py)."""
        if not other._prepared:
            other._prepare()
        if other.cfg != self.cfg or other.device != self.device:
            raise ValueError("share_packed_weights: geometry / device differ")
        self.W, self._kv_off = other.W, other._kv_off
        self._prepared = True
        self._masters_dropped = True
        for p_ in list(self.parameters()) + list(self.buffers()):
            p_.data = torch.empty(0, device=p_.device, dtype=p_.dtype)
        self._graphs.clear(); self._static.clear()
        self.capture_version += 1

    def drop_reference_weights(self):
        """Free the fp32 master copies (6 GB for the released geometry) once the packed operands exist; `state_dict()` is then
        unavailable.  bench.py uses it to keep the working set to what a serving process would hold."""
        if not self._prepared:
            self._prepare()
        for p in list(self.parameters()) + list(self.buffers()):
            p.data = torch.empty(0, device=p.device, dtype=p.dtype)
        self._masters_dropped = True

    def state_dict(self, *args, **kwargs):
        if self._masters_dropped:
            raise RuntimeError("the fp32 masters were released (drop_reference_weights)")
        return super().state_dict(*args, **kwargs)

    def _prepare(self):
        """Repack the reference-layout fp32 weights into the fused fp16 operands the kernels consume."""
        if capturing(self.device):
            raise ValueError("MVUNetMotionModel: the packed weights cannot be (re)built inside a CUDA-graph capture; one eager "
                             "call of this shape must come first")
        L.load()
        if self._masters_dropped:
            raise RuntimeError("the fp32 masters were released; the packed operands cannot be rebuilt")
        cfg, dev = self.cfg, self.device
        miss = [k for k in key_plan(cfg) if k not in self._loaded]
        if miss:
            raise KeyError(f"cannot run: {len(miss)} weights missing, e.g. {miss[:3]}")
        sd = {k: v.detach() for k, v in torch.nn.Module.state_dict(self).items()}
        W: Dict[str, object] = {}
        f32 = lambda k: sd[k].to(dev, torch.float32).contiguous()

        def conv3(p):
            w = sd[f"{p}.weight"]
            return _Lin(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1), sd[f"{p}.bias"], dev)

        def conv1(p):
            w = sd[f"{p}.weight"]
            return _Lin(w.reshape(w.shape[0], -1), sd[f"{p}.bias"], dev)

        def lin(p, bias=True):
            return _Lin(sd[f"{p}.weight"], sd[f"{p}.bias"] if bias else None, dev)

        temb_w, temb_b, temb_off = [], [], {}
        off = 0

        def resnet(p, c1, c2):
            nonlocal off
            r = {"norm1": (f32(f"{p}.norm1.weight"), f32(f"{p}.norm1.bias")),
                 "norm2": (f32(f"{p}.norm2.weight"), f32(f"{p}.norm2.bias")),
                 "conv1": conv3(f"{p}.conv1"), "conv2": conv3(f"{p}.conv2"), "c1": c1, "c2": c2}
            cout = r["conv1"].n
            # time_emb_proj of all resnets is one GEMM; conv1's bias is folded into its bias
            temb_w.append(sd[f"{p}.time_emb_proj.weight"])
            temb_b.append(sd[f"{p}.time_emb_proj.bias"] + sd[f"{p}.conv1.bias"])
            r["temb_off"] = off
            off += cout
            r["conv1"].b = None
            if f"{p}.conv_shortcut.weight" in sd:
                ws = sd[f"{p}.conv_shortcut.weight"].reshape(cout, -1)
                r["sc_a"] = _Lin(ws[:, :c1], sd[f"{p}.conv_shortcut.bias"], dev)
                r["sc_b"] = _Lin(ws[:, c1:], None, dev) if c2 else None
            return r

        kv_w, kv_b, ip_w, ip_b = [], [], [], []
        self._kv_off = 0

        def transformer2d(p, c):
            tb = f"{p}.transformer_blocks.0"
            node = self.get_submodule(tb)
            t = {"c": c, "norm": (f32(f"{p}.norm.weight"), f32(f"{p}.norm.bias")),
                 "proj_in": conv1(f"{p}.proj_in"), "proj_out": conv1(f"{p}.proj_out"),
                 "attn1": P.pack_mv_i2v(node.attn1.processor, node.attn1, dev),
                 "attn2": P.pack_ip_adapter(node.attn2.processor, node.attn2, dev)}
            for i in (1, 2, 3):
                t[f"ln{i}"] = (f32(f"{tb}.norm{i}.weight"), f32(f"{tb}.norm{i}.bias"))
            # text / ip K,V projections of all spatial transformers are two GEMMs (one per token source): the layers' packed
            # operands side by side, this layer's at column kv_off
            kv, ip = t["attn2"].pop("kv"), t["attn2"].pop("ip")
            t["kv_off"] = self._kv_off
            self._kv_off += kv.n
            kv_w.append(kv.w); kv_b.append(kv.b); ip_w.append(ip.w); ip_b.append(ip.b)
            t["ff1"] = _Lin(_geglu_interleave(sd[f"{tb}.ff.net.0.proj.weight"]), _geglu_interleave(sd[f"{tb}.ff.net.0.proj.bias"]), dev)
            t["ff2"] = lin(f"{tb}.ff.net.2")
            return t

        def motion(p, c):
            tb = f"{p}.transformer_blocks.0"
            node = self.get_submodule(tb)
            m = {"c": c, "norm": (f32(f"{p}.norm.weight"), f32(f"{p}.norm.bias")),
                 "proj_in": lin(f"{p}.proj_in"), "proj_out": lin(f"{p}.proj_out")}
            for i in (1, 2, 3):
                m[f"ln{i}"] = (f32(f"{tb}.norm{i}.weight"), f32(f"{tb}.norm{i}.bias"))
            for a in ("attn1", "attn2"):
                m[a] = P.pack_spatiotemporal(getattr(node, a).processor, getattr(node, a), dev)
            m["ff1"] = _Lin(_geglu_interleave(sd[f"{tb}.ff.net.0.proj.weight"]), _geglu_interleave(sd[f"{tb}.ff.net.0.proj.bias"]), dev)
            m["ff2"] = lin(f"{tb}.ff.net.2")
            return m

        ch = cfg.block_out_channels
        W["conv_in"] = (f32("conv_in.weight"), f32("conv_in.bias"))
        W["conv_out"] = (f32("conv_out.weight"), f32("conv_out.bias"))
        W["norm_out"] = (f32("conv_norm_out.weight"), f32("conv_norm_out.bias"))
        for n in ("time_embedding", "camera_embedding"):
            W[n] = tuple(f32(f"{n}.linear_{i}.{s}") for i in (1, 2) for s in ("weight", "bias"))
        ipp = "encoder_hid_proj.image_projection_layers.0"
        W["ip_proj"] = (f32(f"{ipp}.image_embeds.weight"), f32(f"{ipp}.image_embeds.bias"), f32(f"{ipp}.norm.weight"), f32(f"{ipp}.norm.bias"))
        down = []
        cout = ch[0]
        for i, c in enumerate(ch):
            cin, cout = cout, c
            layers = []
            for j in range(cfg.layers_per_block):
                lay = {"res": resnet(f"down_blocks.{i}.resnets.{j}", cin if j == 0 else cout, 0)}
                if cfg.down_has_attn[i]:
                    lay["attn"] = transformer2d(f"down_blocks.{i}.attentions.{j}", cout)
                lay["motion"] = motion(f"down_blocks.{i}.motion_modules.{j}", cout)
                layers.append(lay)
            down.append({"layers": layers, "down": conv3(f"down_blocks.{i}.downsamplers.0.conv") if i != len(ch) - 1 else None})
        W["down"] = down
        c = ch[-1]
        W["mid"] = {"res0": resnet("mid_block.resnets.0", c, 0), "attn": transformer2d("mid_block.attentions.0", c),
                    "motion": motion("mid_block.motion_modules.0", c),
                    "res1": resnet("mid_block.resnets.1", c, 0)}
        up = []
        skips = []
        from .unet_config import skip_channels
        sk = skip_channels(cfg)
        prev = ch[-1]
        for i, (cins, cout, has_attn, has_up) in enumerate(up_plan(cfg)):
            layers = []
            for j, cin in enumerate(cins):
                c2 = sk.pop()
                lay = {"res": resnet(f"up_blocks.{i}.resnets.{j}", cin - c2, c2)}
                if has_attn:
                    lay["attn"] = transformer2d(f"up_blocks.{i}.attentions.{j}", cout)
                lay["motion"] = motion(f"up_blocks.{i}.motion_modules.{j}", cout)
                layers.append(lay)
            up.append({"layers": layers, "up": conv3(f"up_blocks.{i}.upsamplers.0.conv") if has_up else None, "cout": cout})
        W["up"] = up
        W["temb"] = _Lin(torch.cat(temb_w, 0), torch.cat(temb_b, 0), dev)
        W["kv_text"] = _Lin(torch.cat(kv_w, 0), torch.cat(kv_b, 0), dev)
        W["kv_ip"] = _Lin(torch.cat(ip_w, 0), torch.cat(ip_b, 0), dev)
        self.W = W
        self._prepared = True
        self._graphs.clear()
        self._static.clear()
        self.capture_version += 1

    # ------------------------------------------------------------------------------------------------ buffers
    def _buf(self, name: str, shape, dtype=HALF) -> torch.Tensor:
        key = name
        t = self._bufs.get(key)
        numel = 1
        for s in shape:
            numel *= s
        if t is None or t.numel() < numel or t.dtype != dtype:
            if capturing(self.device):
                raise ValueError(f"MVUNetMotionModel: buffer {name!r} would have to grow inside a CUDA-graph capture; one eager "
                                 "call of this shape must come first")
            if t is not None and self._graphs:
                # graphs captured for other shape keys hold the old pointer: drop them, every key recaptures lazily
                self._graphs.clear()
                for st in self._static.values():
                    st["calls"] = 0
            t = torch.empty(numel, dtype=dtype, device=self.device)
            self._bufs[key] = t
            self.capture_version += 1
        return t[:numel].view(*shape)

    # ------------------------------------------------------------------------------------------------ building blocks
    def _gn(self, x1, c1, x2, c2, gb, y, samples, rps, eps, silu, perm=(0, 0)):
        ws = self._buf("gn_stats", (ops.group_norm_ws_floats(samples, rps, c1 + (c2 if x2 is not None else 0),
                                                             self.cfg.norm_num_groups),), torch.float32)
        return ops.group_norm(x1, c1, x2, c2, gb[0], gb[1], y, samples, rps, self.cfg.norm_num_groups, eps, silu, ws, perm)

    def _ln(self, x, gb, y, rows, c):
        return ops.layer_norm(x, gb[0], gb[1], y, rows, c, 1e-5)

    def _resnet(self, r, x, skip, out, n_img, h, w, lvl):
        """ResnetBlock2D: out = shortcut(cat(x, skip)) + conv2(silu(GN(conv1(silu(GN(cat))) + temb)))."""
        M = n_img * h * w
        c1, c2 = r["c1"], r["c2"]
        cin = c1 + c2
        cout = r["conv1"].n
        g = self._buf(f"gn{lvl}", (M, max(cin, cout)))
        gin = g.view(-1)[: M * cin].view(M, cin)
        self._gn(x, c1, skip, c2, r["norm1"], gin, n_img, h * w, self.cfg.norm_eps, 1)
        h1 = self._buf(f"h1_{lvl}", (M, cout))
        temb = self._temb_table
        linear(gin, r["conv1"], h1, M, conv=(n_img, h, w, cin, 1), rowbias=temb[:, r["temb_off"]:], rb_div=h * w,
               rb_mod=1 << 40)
        gout = g.view(-1)[: M * cout].view(M, cout)
        self._gn(h1, cout, None, 0, r["norm2"], gout, n_img, h * w, self.cfg.norm_eps, 1)
        if "sc_a" in r:
            sc = self._buf(f"sc{lvl}", (M, cout))
            linear(x, r["sc_a"], sc, M)
            if r["sc_b"] is not None:
                linear(skip, r["sc_b"], sc, M, R2=sc, ldr2=cout)
            res = sc
        else:
            res = x
        linear(gout, r["conv2"], out, M, conv=(n_img, h, w, cout, 1), R2=res, ldr2=cout)
        return out

    def _ff(self, t, ln_gb, ff1, ff2, M, c, lvl):
        ln = self._buf(f"ln{lvl}", (M, c))
        self._ln(t, ln_gb, ln, M, c)
        mid = self._buf(f"ff{lvl}", (M, 4 * c))
        linear(ln, ff1, mid, M, geglu=True)
        linear(mid, ff2, t, M, R2=t, ldr2=c)

    def _kv_gather_start(self, ln, lin, n_q, M, lvl, table, rb_div, rb_mod):
        """View-parallel projection, first half: the K|V rows of the fused [q.. | k | v] projection are computed FIRST and their
        all-gather over the view group is started asynchronously (NCCL runs it on its own stream over NVLink); the caller keeps
        issuing work that does not need the remote views (the query projection, the whole temporal branch of a motion module)
        and calls `_kv_gather_finish` right before the cross-view attention.  Returns a token for `_kv_gather_finish`."""
        import torch.distributed as dist
        V = self.view_world
        n_kv = lin.n - n_q
        kv_loc = self._buf(f"kvloc{lvl}", (M, n_kv))
        kv_all = self._buf(f"kvall{lvl}", (V, M, n_kv))
        rb = {} if table is None else {"rb_div": rb_div, "rb_mod": rb_mod}
        linear(ln, lin.rows(n_q, lin.n), kv_loc, M, rowbias=None if table is None else table[:, n_q:], **rb)
        work = None
        if self.comm_enabled:
            work = dist.all_gather_into_tensor(kv_all.view(-1), kv_loc.view(-1), group=self.view_group, async_op=True)
            self.collectives += 1
            self.collective_bytes += kv_loc.numel() * 2 * (V - 1)
        return work, kv_all

    def _q_project(self, ln, lin, n_q, M, lvl, table, rb_div, rb_mod):
        qb = self._buf(f"qkv{lvl}", (M, n_q))
        rb = {} if table is None else {"rb_div": rb_div, "rb_mod": rb_mod}
        linear(ln, lin.rows(0, n_q), qb, M, rowbias=None if table is None else table[:, :n_q], **rb)
        return qb

    def _kv_gather_finish(self, token, p, qb, hw, F, B):
        """-> the processor's views over the local queries and the K|V gathered from every view."""
        work, kv_all = token
        if work is not None:
            work.wait()            # the compute stream waits for the gathered K|V (no host sync)
        return P.qkv_views(p, qb, kv_all, hw, F, B, 1, kv_view_rows=qb.shape[0])

    def _transformer2d(self, t, x, n_img, h, w, lvl, B, Nv, F):
        """Transformer2DModel + BasicTransformerBlock with the MVDreamI2V (attn1) and IPAdapter (attn2) processors."""
        a1, a2 = t["attn1"], t["attn2"]
        c = t["c"]
        hw = h * w
        M = n_img * hw
        g = self._buf(f"gn{lvl}", (M, c))
        self._gn(x, c, None, 0, t["norm"], g, n_img, hw, 1e-6, 0)
        tok = self._buf(f"tok{lvl}", (M, c))
        linear(g, t["proj_in"], tok, M)
        ln = self._buf(f"ln{lvl}", (M, c))
        # ---- attn1: cross-view self attention over the Nv views of a frame + I2V attention against frame 0
        self._ln(tok, t["ln1"], ln, M, c)
        qkv = self._buf(f"qkv{lvl}", (M, a1["qkv"].n))
        if self.view_group is None:
            linear(ln, a1["qkv"], qkv, M)
            views = P.qkv_views(a1, qkv, qkv, hw, F, B, Nv)
        else:
            # views span ranks: local rows are (b f p) of ONE view; K|V of every view are all-gathered while the two query
            # projections run
            tok_kv = self._kv_gather_start(ln, a1["qkv"], 2 * a1["hq"], M, lvl, None, 0, 0)
            qb = self._q_project(ln, a1["qkv"], 2 * a1["hq"], M, lvl, None, 0, 0)
            views = self._kv_gather_finish(tok_kv, a1, qb, hw, F, B)
        o12 = self._buf(f"ao{lvl}", (M, 2 * c))                                  # [O1 | O2], rows of 2C
        P.mv_i2v_attend(a1, views, o12, tok, residual=tok)
        # ---- attn2: text (77) + image (4) cross attention, K/V shared by the F frames of a view
        self._ln(tok, t["ln2"], ln, M, c)
        q2 = qkv.view(-1)[: M * a2["hq"]].view(M, a2["hq"])
        linear(ln, a2["q"], q2, M)
        o1 = o12.view(-1)[: M * c].view(M, c)
        for kv, image in ((self._kv_text, False), (self._kv_ip, True)):
            P.ip_adapter_attend(a2, q2, kv, t["kv_off"], o1, hw, F, image)
        linear(o1, a2["out"], tok, M, residual=tok)
        # ---- feed forward
        self._ff(tok, t["ln3"], t["ff1"], t["ff2"], M, c, lvl)
        linear(tok, t["proj_out"], x, M, R2=x, ldr2=c)
        return x

    def _motion(self, m, x, n_img, h, w, lvl, B, Nv, F):
        """TransformerTemporalModel with the SpatioTemporalI2V processor on attn1 and attn2 (released configuration)."""
        c = m["c"]
        hw = h * w
        M = n_img * hw
        g = self._buf(f"gn{lvl}", (M, c))
        # GroupNorm statistics pooled over the F frames of a sample; rows re-ordered (bn f p) -> (bn p f) on the way out
        self._gn(x, c, None, 0, m["norm"], g, B * Nv, F * hw, 1e-6, 0, perm=(F, hw))
        tok = self._buf(f"tok{lvl}", (M, c))
        linear(g, m["proj_in"], tok, M)
        ln = self._buf(f"ln{lvl}", (M, c))
        tq = self._buf(f"tqkv{lvl}", (M, 3 * c))
        st2 = self._buf(f"ao{lvl}", (M, 2 * c))                                  # [S | T]: cross-view branch | temporal branch
        for a, lnk in (("attn1", "ln1"), ("attn2", "ln2")):
            p = m[a]
            self._ln(tok, m[lnk], ln, M, c)
            if self.view_group is not None:
                # spatial (cross-view) K|V first: their all-gather overlaps the query projection and the WHOLE temporal branch
                tok_kv = self._kv_gather_start(ln, p["s_qkv"], p["hq"], M, lvl, p["s_table"], F, hw)
                qb = self._q_project(ln, p["s_qkv"], p["hq"], M, lvl, p["s_table"], F, hw)
            P.spatiotemporal_temporal(p, ln, tq, st2, F)
            if self.view_group is None:
                views = P.spatiotemporal_project(p, ln, self._buf(f"qkv{lvl}", (M, p["s_qkv"].n)), hw, F, B, Nv)
            else:
                views = self._kv_gather_finish(tok_kv, p, qb, hw, F, B)
            # cross-view attention, then the AlphaBlender of both branches' output projections + the block residual
            P.spatiotemporal_attend(p, views, st2, tok, residual=tok)
        self._ff(tok, m["ln3"], m["ff1"], m["ff2"], M, c, lvl)
        # proj_out, rows back to (bn f p), + residual
        linear(tok, m["proj_out"], x, M, perm=(hw, F), R2=x, ldr2=c)
        return x

    # ------------------------------------------------------------------------------------------------ forward
    def _run(self, sig, st):
        cfg = self.cfg
        BN, F, h0, w0, Nv, cond_zero = sig
        B = BN // Nv
        N = BN * F
        W = self.W
        ch = cfg.block_out_channels
        # ---- embeddings (fp32, tiny)
        tproj = self._buf("tproj", (BN, ch[0]), torch.float32)
        ops.timestep_proj(st["t"], tproj, BN, ch[0] // 2)
        e1 = self._buf("e1", (BN, cfg.time_embed_dim), torch.float32)
        emb = self._buf("emb", (BN, cfg.time_embed_dim), torch.float32)
        te = W["time_embedding"]
        ops.linear_f32(tproj, te[0], te[1], e1, BN, cfg.time_embed_dim, ch[0])
        ops.linear_f32(e1, te[2], te[3], emb, BN, cfg.time_embed_dim, cfg.time_embed_dim, act_in=1)
        ce = W["camera_embedding"]
        c1 = self._buf("c1", (BN, cfg.time_embed_dim), torch.float32)
        ops.linear_f32(st["camera"], ce[0], ce[1], c1, BN, cfg.time_embed_dim, cfg.camera_embedding_dim)
        ops.linear_f32(c1, ce[2], ce[3], emb, BN, cfg.time_embed_dim, cfg.time_embed_dim, act_in=1, accumulate=True)
        semb = self._buf("semb", (N, cfg.time_embed_dim))
        if cond_zero:
            # frame-0 rows use the t=0 embedding (unet_motion_mv_model.py:732-752); rare path, assembled with torch indexing
            t0 = self._buf("t0", (BN,), torch.float32).zero_()
            ops.timestep_proj(t0, tproj, BN, ch[0] // 2)
            emb0 = self._buf("emb0", (BN, cfg.time_embed_dim), torch.float32)
            ops.linear_f32(tproj, te[0], te[1], e1, BN, cfg.time_embed_dim, ch[0])
            ops.linear_f32(e1, te[2], te[3], emb0, BN, cfg.time_embed_dim, cfg.time_embed_dim, act_in=1)
            ops.linear_f32(c1, ce[2], ce[3], emb0, BN, cfg.time_embed_dim, cfg.time_embed_dim, act_in=1, accumulate=True)
            rows = self._buf("emb_rows", (BN, F, cfg.time_embed_dim), torch.float32)
            rows.copy_(emb[:, None, :].expand(BN, F, -1))
            rows[:, 0] = emb0
            ops.silu_rows(rows, semb, N, cfg.time_embed_dim, 1)
        else:
            ops.silu_rows(emb, semb, N, cfg.time_embed_dim, F)
        self._temb_table = self._buf("temb_table", (N, W["temb"].n), torch.float32)
        linear(semb, W["temb"], self._temb_table, N, out_f32=True)
        # ---- text / ip tokens -> K,V of all 16 spatial transformers (once per view, not per frame)
        n_text = st["text"].shape[1]
        self._n_text = n_text
        text16 = self._buf("text16", (BN * n_text, cfg.cross_attention_dim))
        ops.cast_f32_f16(st["text"], text16)
        self._kv_text = self._buf("kv_text", (BN * n_text, W["kv_text"].n))
        linear(text16, W["kv_text"], self._kv_text, BN * n_text)
        ipw = W["ip_proj"]
        ipt = self._buf("ipt", (BN, cfg.ip_num_tokens * cfg.cross_attention_dim), torch.float32)
        ops.linear_f32(st["image_embeds"], ipw[0], ipw[1], ipt, BN, cfg.ip_num_tokens * cfg.cross_attention_dim, cfg.ip_image_embed_dim)
        ip16 = self._buf("ip16", (BN * cfg.ip_num_tokens, cfg.cross_attention_dim))
        ops.cast_f32_f16(ipt, ip16)
        ipn = self._buf("ipn", (BN * cfg.ip_num_tokens, cfg.cross_attention_dim))
        ops.layer_norm(ip16, ipw[2], ipw[3], ipn, BN * cfg.ip_num_tokens, cfg.cross_attention_dim, 1e-5)
        self._kv_ip = self._buf("kv_ip", (BN * cfg.ip_num_tokens, W["kv_ip"].n))
        linear(ipn, W["kv_ip"], self._kv_ip, BN * cfg.ip_num_tokens)
        # ---- conv_in (+ layout change of line 767)
        hs = [h0 >> i for i in range(len(ch))]
        ws = [w0 >> i for i in range(len(ch))]
        skips = []
        x = self._buf("skip0", (N * hs[0] * ws[0], ch[0]))
        ops.conv_in(st["sample"], W["conv_in"][0], W["conv_in"][1], x, BN, cfg.in_channels, F, hs[0], ws[0], ch[0])
        skips.append(x)
        si = 1
        for i, blk in enumerate(W["down"]):
            h, w = hs[i], ws[i]
            for lay in blk["layers"]:
                out = self._buf(f"skip{si}", (N * h * w, lay["res"]["conv1"].n)); si += 1
                self._resnet(lay["res"], x, None, out, N, h, w, i)
                x = out
                if "attn" in lay:
                    self._transformer2d(lay["attn"], x, N, h, w, i, B, Nv, F)
                self._motion(lay["motion"], x, N, h, w, i, B, Nv, F)
                skips.append(x)
            if blk["down"] is not None:
                c = blk["down"].n
                out = self._buf(f"skip{si}", (N * hs[i + 1] * ws[i + 1], c)); si += 1
                linear(x, blk["down"], out, N * hs[i + 1] * ws[i + 1], conv=(N, h, w, c, 2))
                x = out
                skips.append(x)
        lv = len(ch) - 1
        h, w = hs[lv], ws[lv]
        mid = W["mid"]
        xm = self._buf("xmid", (N * h * w, ch[-1]))
        self._resnet(mid["res0"], x, None, xm, N, h, w, lv)
        self._transformer2d(mid["attn"], xm, N, h, w, lv, B, Nv, F)
        self._motion(mid["motion"], xm, N, h, w, lv, B, Nv, F)
        xm2 = self._buf("xmid2", (N * h * w, ch[-1]))
        self._resnet(mid["res1"], xm, None, xm2, N, h, w, lv)
        x = xm2
        for i, blk in enumerate(W["up"]):
            lv = len(ch) - 1 - i
            h, w = hs[lv], ws[lv]
            for j, lay in enumerate(blk["layers"]):
                skip = skips.pop()
                out = self._buf(f"xup{lv}_{j % 2}", (N * h * w, blk["cout"]))
                self._resnet(lay["res"], x, skip, out, N, h, w, lv)
                x = out
                if "attn" in lay:
                    self._transformer2d(lay["attn"], x, N, h, w, lv, B, Nv, F)
                self._motion(lay["motion"], x, N, h, w, lv, B, Nv, F)
            if blk["up"] is not None:
                c = blk["cout"]
                upb = self._buf(f"upsampled{lv}", (N * 4 * h * w, c))
                ops.upsample2x(x, upb, N, h, w, c)
                out = self._buf(f"xup{lv - 1}_up", (N * 4 * h * w, c))
                linear(upb, blk["up"], out, N * 4 * h * w, conv=(N, 2 * h, 2 * w, c, 1))
                x = out
        # ---- out: GroupNorm + SiLU + conv_out (+ layout change of line 862)
        h, w = hs[0], ws[0]
        g = self._buf("gn0", (N * h * w, ch[0]))
        self._gn(x, ch[0], None, 0, W["norm_out"], g, N, h * w, cfg.norm_eps, 1)
        ops.conv_out(g, W["conv_out"][0], W["conv_out"][1], st["out"], BN, ch[0], F, h, w, cfg.out_channels)

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, timestep_cond=None, attention_mask=None,
                cross_attention_kwargs=None, added_cond_kwargs=None, down_block_additional_residuals=None,
                mid_block_additional_residual=None, return_dict: bool = True, camera=None, num_views: int = 4,
                i2v_cond_time_zero: bool = False):
        """Signature of unet_motion_mv_model.py:633-649.  sample [B*Nv, 4, F, h, w]; returns `.sample` of the same shape.

        Inside a caller's CUDA-graph capture the kernels are recorded into the caller's graph (no inner capture, replay or
        synchronise).  That allocates nothing, so an eager call of the same shape must have come first; otherwise, and for a
        view-sharded model (its NCCL gathers cannot be captured), it raises ValueError before recording anything."""
        in_capture = capturing(self.device)
        if in_capture and self.view_group is not None:
            raise ValueError("a view-sharded MVUNetMotionModel cannot be recorded into a CUDA graph: its K|V all-gathers run "
                             "eagerly")
        if in_capture and not self._prepared:
            raise ValueError("MVUNetMotionModel: no packed weights inside a CUDA-graph capture; one eager call of this shape "
                             "must come first")
        if not self._prepared:
            self._prepare()
        if attention_mask is not None or timestep_cond is not None or down_block_additional_residuals is not None \
                or mid_block_additional_residual is not None:
            raise NotImplementedError("attention_mask / timestep_cond / additional residuals are never used by the "
                                      "reference's call sites (pipeline.py:1012, animatemv_guidance.py:339)")
        if added_cond_kwargs is None or "image_embeds" not in added_cond_kwargs:
            raise ValueError("added_cond_kwargs['image_embeds'] is required (unet_motion_mv_model.py:757-760)")
        if camera is None:
            raise ValueError("camera is required by the MV-VDM UNet")
        BN, cin, F, h0, w0 = sample.shape
        assert BN % num_views == 0, "[UNet] input batch size must be dividable by num_views!"   # line 684
        fs = self.cfg.sample_size
        if h0 != fs or w0 != fs:
            raise ValueError(f"latent size {h0}x{w0} != {fs}: the processors' feature_size is wired to one resolution "
                             "(inference.py:93; SURVEY Appendix A)")
        sig = (BN, F, h0, w0, num_views, bool(i2v_cond_time_zero))
        dev = self.device
        n_text = encoder_hidden_states.shape[1]
        key = sig + (n_text,)
        st = self._static.get(key)
        if in_capture and st is None:
            raise ValueError(f"MVUNetMotionModel: no buffers for shape {key} inside a CUDA-graph capture; one eager call of "
                             "this shape must come first")
        if st is None:
            st = {"sample": torch.empty(BN, cin, F, h0, w0, device=dev, dtype=torch.float32),
                  "t": torch.empty(BN, device=dev, dtype=torch.float32),
                  "text": torch.empty(BN, n_text, self.cfg.cross_attention_dim, device=dev, dtype=torch.float32),
                  "camera": torch.empty(BN, self.cfg.camera_embedding_dim, device=dev, dtype=torch.float32),
                  "image_embeds": torch.empty(BN, self.cfg.ip_image_embed_dim, device=dev, dtype=torch.float32),
                  "out": torch.empty(BN, self.cfg.out_channels, F, h0, w0, device=dev, dtype=torch.float32), "calls": 0}
            self._static[key] = st
        st["sample"].copy_(sample)
        if in_capture and not isinstance(timestep, torch.Tensor):
            st["t"].fill_(float(timestep))                  # an upload of a host scalar cannot be captured
        else:
            t = torch.as_tensor(timestep, dtype=torch.float32, device=dev)
            st["t"].copy_(t.reshape(-1).expand(BN) if t.numel() in (1, BN) else t)
        st["text"].copy_(encoder_hidden_states)
        st["camera"].copy_(camera.reshape(BN, -1))
        st["image_embeds"].copy_(added_cond_kwargs["image_embeds"])
        graph = self._graphs.get(key)
        if in_capture:
            note_module(self)
            self._run(sig, st)
        elif graph is not None:
            graph.replay()
        else:
            self.collectives = self.collective_bytes = 0
            n0 = ops.launches
            self._run(sig, st)
            self.launches_per_forward = ops.launches - n0
            st["calls"] += 1
            if self.use_cuda_graph and st["calls"] == 1:
                # second pass under capture: same launches, same buffers
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._run(sig, st)
                self._graphs[key] = g
        out = st["out"].clone()
        return UNet3DConditionOutput(sample=out) if return_dict else (out,)

