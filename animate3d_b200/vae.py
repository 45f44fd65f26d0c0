"""SD-1.5 `AutoencoderKL` on the sm_90a engine (SURVEY 8f-1): the module that sits immediately either side of the UNet.

  * `encode(x).latent_dist.sample()` -- with INPUT GRADIENT: in the 4D-SDS step the encoder runs on the 64 rendered 256^2 views
    and is the only autograd path from `loss_sds` back to the rasterizer (animatemv_guidance.py:365-373, 533-542; the VAE
    parameters are frozen, 301-302, so only d/d input is needed: ~17 TFLOP forward + ~17 TFLOP dgrad per step)
  * `decode(z).sample` -- forward only (pipeline.py:554-567 `decode_latents`, guidance_eval)

Same layout and kernels as the UNet: activations NHWC fp16, every 3x3 convolution is the implicit-GEMM wgmma kernel
(`a3d_gemm`, A3D_A_CONV3) -- the input gradient of a convolution is the same kernel with the flipped / transposed weights (the
stride-2 downsampler's through a zero-inserted copy of the output gradient) --, GroupNorm(+SiLU) forward / backward are
`a3d_group_norm` / `a3d_group_norm_backward`, the 3- / 4- / 8-channel edge convolutions are `a3d_conv_in` / `a3d_conv_out`.
torch supplies memory, the stream and the autograd tape that strings the per-layer Functions together; the single-head
mid-block attention core (softmax(QK^T)V on 1024 tokens, 0.5 % of the FLOPs) and the 8-channel 1x1 quant convolutions are
torch ops.  State-dict keys are diffusers' (`vae/diffusion_pytorch_model.safetensors` loads unchanged).  Oracle:
oracle/vae_oracle.py."""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from . import _lib as L
from . import ops
from .capture import capturing, note_module

HALF = torch.float16
GROUPS = 32


def _pack_conv(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """[Cout, Cin, 3, 3] -> (forward operand [Cout, (ky, kx, cin)], input-gradient operand [Cin, (ky', kx', cout)] with the taps
    flipped: dX = conv(dY, flip(W)^T))."""
    fwd = w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)
    bwd = w.flip(2, 3).permute(1, 2, 3, 0).reshape(w.shape[1], -1)
    return fwd.to(HALF).contiguous(), bwd.to(HALF).contiguous()


def vae_key_plan(cfg) -> Dict[str, tuple]:
    """Every tensor of diffusers' AutoencoderKL state dict (encoder / decoder of DownEncoderBlock2D / UpDecoderBlock2D,
    UNetMidBlock2D with one single-head attention, quant / post_quant 1x1 convolutions) -> shape."""
    ch = cfg.block_out_channels
    lc = cfg.latent_channels
    ks: Dict[str, tuple] = {}

    def res(p, cin, cout):
        ks.update({f"{p}.norm1.weight": (cin,), f"{p}.norm1.bias": (cin,), f"{p}.conv1.weight": (cout, cin, 3, 3), f"{p}.conv1.bias": (cout,),
                   f"{p}.norm2.weight": (cout,), f"{p}.norm2.bias": (cout,), f"{p}.conv2.weight": (cout, cout, 3, 3),
                   f"{p}.conv2.bias": (cout,)})
        if cin != cout:
            ks[f"{p}.conv_shortcut.weight"] = (cout, cin, 1, 1)
            ks[f"{p}.conv_shortcut.bias"] = (cout,)

    def mid(p, c):
        res(f"{p}.resnets.0", c, c)
        a = f"{p}.attentions.0"
        ks[f"{a}.group_norm.weight"] = (c,)
        ks[f"{a}.group_norm.bias"] = (c,)
        for n in ("to_q", "to_k", "to_v", "to_out.0"):
            ks[f"{a}.{n}.weight"] = (c, c)
            ks[f"{a}.{n}.bias"] = (c,)
        res(f"{p}.resnets.1", c, c)

    ks["encoder.conv_in.weight"] = (ch[0], cfg.in_channels, 3, 3)
    ks["encoder.conv_in.bias"] = (ch[0],)
    cout = ch[0]
    for i, c in enumerate(ch):
        cin, cout = cout, c
        for j in range(cfg.layers_per_block):
            res(f"encoder.down_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i != len(ch) - 1:
            ks[f"encoder.down_blocks.{i}.downsamplers.0.conv.weight"] = (cout, cout, 3, 3)
            ks[f"encoder.down_blocks.{i}.downsamplers.0.conv.bias"] = (cout,)
    mid("encoder.mid_block", ch[-1])
    ks.update({"encoder.conv_norm_out.weight": (ch[-1],), "encoder.conv_norm_out.bias": (ch[-1],),
               "encoder.conv_out.weight": (2 * lc, ch[-1], 3, 3), "encoder.conv_out.bias": (2 * lc,),
               "quant_conv.weight": (2 * lc, 2 * lc, 1, 1), "quant_conv.bias": (2 * lc,),
               "post_quant_conv.weight": (lc, lc, 1, 1), "post_quant_conv.bias": (lc,),
               "decoder.conv_in.weight": (ch[-1], lc, 3, 3), "decoder.conv_in.bias": (ch[-1],)})
    mid("decoder.mid_block", ch[-1])
    rev = list(reversed(ch))
    cout = rev[0]
    for i, c in enumerate(rev):
        cin, cout = cout, c
        for j in range(cfg.layers_per_block + 1):
            res(f"decoder.up_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i != len(ch) - 1:
            ks[f"decoder.up_blocks.{i}.upsamplers.0.conv.weight"] = (cout, cout, 3, 3)
            ks[f"decoder.up_blocks.{i}.upsamplers.0.conv.bias"] = (cout,)
    ks.update({"decoder.conv_norm_out.weight": (ch[0],), "decoder.conv_norm_out.bias": (ch[0],),
               "decoder.conv_out.weight": (cfg.out_channels, ch[0], 3, 3), "decoder.conv_out.bias": (cfg.out_channels,)})
    return ks


class _Conv3(torch.autograd.Function):
    """3x3 convolution, NHWC fp16, stride 1 (padding 1) or the VAE downsampler (stride 2, padding (0,1,0,1)); optional fused
    residual add."""

    @staticmethod
    def forward(ctx, x, res, lay, n, h, w, stride):
        cin, cout = lay["cin"], lay["cout"]
        oh, ow = h // stride, w // stride
        out = torch.empty(n * oh * ow, cout, device=x.device, dtype=HALF)
        ops.gemm(x, lay["w"], out, M=n * oh * ow, N=cout, K=9 * cin, conv=(n, h, w, cin, stride), bias=lay["b"], R2=res,
                 ldr2=cout, conv_nopad_lo=stride == 2)
        ctx.lay, ctx.geom, ctx.has_res = lay, (n, h, w, stride), res is not None
        return out

    @staticmethod
    def backward(ctx, g):
        lay = ctx.lay
        n, h, w, stride = ctx.geom
        cin, cout = lay["cin"], lay["cout"]
        g = g.contiguous()
        if stride == 2:     # dY sits at the odd positions of a zero image of the input size (see module docstring)
            u = torch.zeros(n, h, w, cout, device=g.device, dtype=HALF)
            u[:, 1::2, 1::2] = g.view(n, h // 2, w // 2, cout)
            src = u.view(n * h * w, cout)
        else:
            src = g
        dx = torch.empty(n * h * w, cin, device=g.device, dtype=HALF)
        ops.gemm(src, lay["wt"], dx, M=n * h * w, N=cin, K=9 * cout, conv=(n, h, w, cout, 1))
        return dx, (g if ctx.has_res else None), None, None, None, None, None


class _Lin(torch.autograd.Function):
    """1x1 convolution / Linear on tokens [M, K] -> [M, N] (+ residual)."""

    @staticmethod
    def forward(ctx, x, res, lay):
        m = x.shape[0]
        out = torch.empty(m, lay["cout"], device=x.device, dtype=HALF)
        ops.gemm(x, lay["w"], out, M=m, N=lay["cout"], K=lay["cin"], bias=lay["b"], R2=res, ldr2=lay["cout"])
        ctx.lay, ctx.has_res = lay, res is not None
        return out

    @staticmethod
    def backward(ctx, g):
        lay = ctx.lay
        g = g.contiguous()
        dx = torch.empty(g.shape[0], lay["cin"], device=g.device, dtype=HALF)
        ops.gemm(g, lay["wt"], dx, M=g.shape[0], N=lay["cin"], K=lay["cout"])
        return dx, (g if ctx.has_res else None), None


class _GroupNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gb, n, rows, silu, eps):
        c = x.shape[1]
        y = torch.empty_like(x)
        ws = torch.empty(ops.group_norm_ws_floats(n, rows, c, GROUPS), device=x.device, dtype=torch.float32)
        ops.group_norm(x, c, None, 0, gb[0], gb[1], y, n, rows, GROUPS, eps, silu, ws)
        ctx.save_for_backward(x, ws[: 2 * GROUPS * n].clone())
        ctx.meta = (gb, n, rows, silu)
        return y

    @staticmethod
    def backward(ctx, g):
        x, stats = ctx.saved_tensors
        gb, n, rows, silu = ctx.meta
        c = x.shape[1]
        dx = torch.empty_like(x)
        ws = torch.empty(ops.group_norm_ws_floats(n, rows, c, GROUPS), device=x.device, dtype=torch.float32)
        ops.group_norm_backward(x, c, gb[0], gb[1], stats, g.contiguous(), dx, n, rows, GROUPS, silu, ws)
        return dx, None, None, None, None, None


class _ConvIn(torch.autograd.Function):
    """[N, cin <= 8, H, W] fp32 (NCHW) -> NHWC fp16 [N*H*W, cout]; backward back to NCHW fp32."""

    @staticmethod
    def forward(ctx, x, lay):
        n, cin, h, w = x.shape
        y = torch.empty(n * h * w, lay["cout"], device=x.device, dtype=HALF)
        ops.conv_in(x.contiguous().float(), lay["w32"], lay["b"], y, n, cin, 1, h, w, lay["cout"])
        ctx.lay, ctx.geom = lay, (n, cin, h, w)
        return y

    @staticmethod
    def backward(ctx, g):
        lay = ctx.lay
        n, cin, h, w = ctx.geom
        dx = torch.empty(n, cin, 1, h, w, device=g.device, dtype=torch.float32)
        zero = lay["zero_b"]
        for c0 in range(0, cin, 4):          # a3d_conv_out writes <= 4 output channels per call
            c1 = min(c0 + 4, cin)
            part = torch.empty(n, c1 - c0, 1, h, w, device=g.device, dtype=torch.float32)
            ops.conv_out(g.contiguous(), lay["wt32"][c0:c1].contiguous(), zero, part, n, lay["cout"], 1, h, w, c1 - c0)
            dx[:, c0:c1] = part
        return dx.reshape(n, cin, h, w), None


class _ConvOut(torch.autograd.Function):
    """NHWC fp16 [N*H*W, cin] -> [N, cout <= 8, H, W] fp32 (NCHW); backward back to NHWC fp16."""

    @staticmethod
    def forward(ctx, x, lay, n, h, w):
        cout = lay["cout"]
        y = torch.empty(n, cout, 1, h, w, device=x.device, dtype=torch.float32)
        for c0 in range(0, cout, 4):
            c1 = min(c0 + 4, cout)
            part = torch.empty(n, c1 - c0, 1, h, w, device=x.device, dtype=torch.float32)
            ops.conv_out(x, lay["w32"][c0:c1].contiguous(), lay["b"][c0:c1].contiguous(), part, n, lay["cin"], 1, h, w, c1 - c0)
            y[:, c0:c1] = part
        ctx.lay, ctx.geom = lay, (n, h, w)
        return y.reshape(n, cout, h, w)

    @staticmethod
    def backward(ctx, g):
        lay = ctx.lay
        n, h, w = ctx.geom
        dx = torch.empty(n * h * w, lay["cin"], device=g.device, dtype=HALF)
        ops.conv_in(g.contiguous().float(), lay["wt32"], lay["zero_b"], dx, n, lay["cout"], 1, h, w, lay["cin"])
        return dx, None, None, None, None


class DiagonalGaussianDistribution:
    """diffusers.models.autoencoders.vae.DiagonalGaussianDistribution on [N, 2*latent, h, w] moments."""

    def __init__(self, parameters: torch.Tensor):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        noise = torch.randn(self.mean.shape, generator=generator, device=self.parameters.device, dtype=self.parameters.dtype)
        return self.mean + self.std * noise

    def mode(self) -> torch.Tensor:
        return self.mean


class AutoencoderKL(torch.nn.Module):
    def __init__(self, in_channels: int = 3, out_channels: int = 3, latent_channels: int = 4,
                 block_out_channels: Tuple[int, ...] = (128, 256, 512, 512), layers_per_block: int = 2, norm_num_groups: int = 32,
                 scaling_factor: float = 0.18215, sample_size: int = 512, device: str = "cuda"):
        super().__init__()
        if norm_num_groups != GROUPS:
            raise NotImplementedError("the SD VAE uses 32 groups")
        self.config = SimpleNamespace(in_channels=in_channels, out_channels=out_channels, latent_channels=latent_channels,
                                      block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                      norm_num_groups=norm_num_groups, scaling_factor=scaling_factor, sample_size=sample_size)
        self._device = torch.device(device)
        self.eps = 1e-6
        self.W: Optional[Dict[str, dict]] = None
        # bumped when the packed weights are replaced: a CUDA graph that recorded the VAE reads them by address
        self.capture_version = 0

    @property
    def device(self):
        return self._device

    @property
    def dtype(self):
        return HALF

    def to(self, *a, **k):
        return self

    def enable_slicing(self):
        pass

    # ------------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True, assign: bool = False):
        """diffusers key names; returns (missing_keys, unexpected_keys).  The weights are repacked into the kernels' operand
        layouts right away (there is no per-parameter module tree: the VAE is frozen everywhere in the reference)."""
        return self._load(sd, vae_key_plan(self.config), strict)

    def _load(self, sd: Dict[str, torch.Tensor], plan: Dict[str, tuple], strict: bool):
        L.load(require_gpu=False)
        missing = [k for k in plan if k not in sd]
        unexpected = [k for k in sd if k not in plan]
        if strict and (missing or unexpected):
            raise KeyError(f"VAE state dict mismatch: {len(missing)} missing, {len(unexpected)} unexpected")
        for k, shape in plan.items():
            if k in sd and tuple(sd[k].shape) != tuple(shape):
                raise ValueError(f"{k}: shape {tuple(sd[k].shape)} != {tuple(shape)}")
        dev = self._device
        f32 = lambda k: sd[k].detach().to(dev, torch.float32).contiguous()
        W: Dict[str, dict] = {}

        def conv3(p):
            w = f32(f"{p}.weight")
            fw, bw = _pack_conv(w)
            return {"w": fw, "wt": bw, "b": f32(f"{p}.bias"), "cin": w.shape[1], "cout": w.shape[0]}

        def lin(p, scale=1.0):
            w = f32(f"{p}.weight").reshape(sd[f"{p}.weight"].shape[0], -1) * scale
            return {"w": w.to(HALF).contiguous(), "wt": w.t().to(HALF).contiguous(), "b": f32(f"{p}.bias") * scale, "cin": w.shape[1],
                    "cout": w.shape[0]}

        def edge(p):            # 3 / 4 / 8-channel edge convolutions: fp32 weights for the SIMT edge kernels
            w = f32(f"{p}.weight")
            return {"w32": w.reshape(w.shape[0], -1).contiguous(),                                  # [cout, cin*9] (ci, tap)
                    "wt32": w.flip(2, 3).permute(1, 0, 2, 3).reshape(w.shape[1], -1).contiguous(),  # [cin, cout*9] flipped taps
                    "b": f32(f"{p}.bias"), "zero_b": torch.zeros(max(w.shape[0], w.shape[1]), device=dev), "cin": w.shape[1],
                    "cout": w.shape[0]}

        def gn(p):
            return (f32(f"{p}.weight"), f32(f"{p}.bias"))

        def res(p):
            r = {"norm1": gn(f"{p}.norm1"), "conv1": conv3(f"{p}.conv1"), "norm2": gn(f"{p}.norm2"), "conv2": conv3(f"{p}.conv2")}
            if f"{p}.conv_shortcut.weight" in sd:
                r["sc"] = lin(f"{p}.conv_shortcut")
            return r

        def mid(p):
            a = f"{p}.attentions.0"
            c = sd[f"{a}.to_q.weight"].shape[0]
            qkv_w = torch.cat([f32(f"{a}.to_q.weight"), f32(f"{a}.to_k.weight"), f32(f"{a}.to_v.weight")], 0)
            qkv_b = torch.cat([f32(f"{a}.to_q.bias"), f32(f"{a}.to_k.bias"), f32(f"{a}.to_v.bias")], 0)
            return {"res0": res(f"{p}.resnets.0"), "res1": res(f"{p}.resnets.1"), "gn": gn(f"{a}.group_norm"),
                    "qkv": {"w": qkv_w.to(HALF).contiguous(), "wt": qkv_w.t().to(HALF).contiguous(), "b": qkv_b, "cin": c, "cout": 3 * c},
                    "out": lin(f"{a}.to_out.0"), "c": c}

        cfg = self.config
        ch = cfg.block_out_channels
        W["enc_in"] = edge("encoder.conv_in")
        W["enc_down"] = []
        for i in range(len(ch)):
            W["enc_down"].append({"res": [res(f"encoder.down_blocks.{i}.resnets.{j}") for j in range(cfg.layers_per_block)],
                                  "down": conv3(f"encoder.down_blocks.{i}.downsamplers.0.conv") if i != len(ch) - 1 else None})
        W["enc_mid"] = mid("encoder.mid_block")
        W["enc_norm"] = gn("encoder.conv_norm_out")
        W["enc_out"] = edge("encoder.conv_out")
        W["quant"] = (f32("quant_conv.weight"), f32("quant_conv.bias"))
        W["post_quant"] = (f32("post_quant_conv.weight"), f32("post_quant_conv.bias"))
        W["dec_in"] = edge("decoder.conv_in")
        W["dec_mid"] = mid("decoder.mid_block")
        W["dec_up"] = []
        for i in range(len(ch)):
            W["dec_up"].append({"res": [res(f"decoder.up_blocks.{i}.resnets.{j}") for j in range(cfg.layers_per_block + 1)],
                                "up": conv3(f"decoder.up_blocks.{i}.upsamplers.0.conv") if i != len(ch) - 1 else None})
        W["dec_norm"] = gn("decoder.conv_norm_out")
        W["dec_out"] = edge("decoder.conv_out")
        self.W = W
        self.capture_version += 1
        return missing, unexpected

    # ------------------------------------------------------------------------------------------------ blocks
    def _res(self, r, x, n, h, w):
        hw = h * w
        t = _GroupNorm.apply(x, r["norm1"], n, hw, 1, self.eps)
        t = _Conv3.apply(t, None, r["conv1"], n, h, w, 1)
        t = _GroupNorm.apply(t, r["norm2"], n, hw, 1, self.eps)
        skip = _Lin.apply(x, None, r["sc"]) if "sc" in r else x
        return _Conv3.apply(t, skip, r["conv2"], n, h, w, 1)

    def _mid(self, m, x, n, h, w):
        hw, c = h * w, m["c"]
        x = self._res(m["res0"], x, n, h, w)
        t = _GroupNorm.apply(x, m["gn"], n, hw, 0, self.eps)
        qkv = _Lin.apply(t, None, m["qkv"]).view(n, 1, hw, 3 * c)
        q, k, v = qkv[..., :c], qkv[..., c:2 * c], qkv[..., 2 * c:]
        a = F.scaled_dot_product_attention(q, k, v, scale=c ** -0.5).reshape(n * hw, c).contiguous()
        x = _Lin.apply(a, x, m["out"])                                  # residual_connection=True
        return self._res(m["res1"], x, n, h, w)

    # ------------------------------------------------------------------------------------------------ encode / decode
    def encode_moments(self, x: torch.Tensor) -> torch.Tensor:
        """x [N, 3, H, W] in [-1, 1] (fp32, may require grad) -> moments [N, 8, H/8, W/8] fp32."""
        if self.W is None:
            raise RuntimeError("AutoencoderKL: load_state_dict first")
        if capturing(self._device):
            note_module(self)
        W = self.W
        n, _, h, w = x.shape
        if h % 8 or w % 8 or (w > 128 and w % 128) or (w <= 128 and 128 % w):
            raise ValueError(f"image size {h}x{w}: widths must be powers of two >= 32 (the reference renders 256^2 / 512^2 views)")
        t = _ConvIn.apply(x.to(self._device, torch.float32), W["enc_in"])
        for blk in W["enc_down"]:
            for r in blk["res"]:
                t = self._res(r, t, n, h, w)
            if blk["down"] is not None:
                t = _Conv3.apply(t, None, blk["down"], n, h, w, 2)
                h, w = h // 2, w // 2
        t = self._mid(W["enc_mid"], t, n, h, w)
        t = _GroupNorm.apply(t, W["enc_norm"], n, h * w, 1, self.eps)
        m = _ConvOut.apply(t, W["enc_out"], n, h, w)
        return F.conv2d(m, W["quant"][0], W["quant"][1])

    def encode(self, x: torch.Tensor, return_dict: bool = True):
        dist = DiagonalGaussianDistribution(self.encode_moments(x))
        return SimpleNamespace(latent_dist=dist) if return_dict else (dist,)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True):
        """z [N, 4, h, w] (latents / scaling_factor) -> `.sample` [N, 3, 8h, 8w] fp32.  Forward only."""
        if self.W is None:
            raise RuntimeError("AutoencoderKL: load_state_dict first")
        if capturing(self._device):
            note_module(self)
        W = self.W
        n, _, h, w = z.shape
        t = F.conv2d(z.to(self._device, torch.float32), W["post_quant"][0], W["post_quant"][1])
        t = _ConvIn.apply(t, W["dec_in"])
        t = self._mid(W["dec_mid"], t, n, h, w)
        for blk in W["dec_up"]:
            for r in blk["res"]:
                t = self._res(r, t, n, h, w)
            if blk["up"] is not None:
                c = t.shape[1]
                up = torch.empty(n * 4 * h * w, c, device=t.device, dtype=HALF)
                ops.upsample2x(t, up, n, h, w, c)
                h, w = 2 * h, 2 * w
                t = _Conv3.apply(up, None, blk["up"], n, h, w, 1)
        t = _GroupNorm.apply(t, W["dec_norm"], n, h * w, 1, self.eps)
        img = _ConvOut.apply(t, W["dec_out"], n, h, w)
        return SimpleNamespace(sample=img) if return_dict else (img,)

    def forward(self, x):
        return self.decode(self.encode(x).latent_dist.sample()).sample
