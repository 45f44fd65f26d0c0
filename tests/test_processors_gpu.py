"""diffusers attention-processor protocol (SURVEY 8b): each released processor class, driven stand-alone as
`processor(attn, hidden_states, encoder_hidden_states=...)`, against the oracle restatements that are pinned to the reference's own
processor source (tests/test_oracle_vs_reference.py).  Also the module surface: attn_processors / set_attn_processor."""
import pytest
import torch

pytestmark = pytest.mark.gpu
HEADS = 8


def _attn_and_sd(c, kv_dim, seed, proc):
    """An AttentionNode with random weights + the matching oracle state dict under the prefix 'a'."""
    from animate3d_b200.modules import AttentionNode, _linear
    g = torch.Generator().manual_seed(seed)
    attn = AttentionNode(HEADS, c // HEADS)
    attn.to_q, attn.to_k, attn.to_v = _linear(c, c, False, "cuda"), _linear(c, kv_dim, False, "cuda"), _linear(c, kv_dim, False, "cuda")
    from animate3d_b200.modules import Node
    attn.to_out = Node()
    attn.to_out.add_module("0", _linear(c, c, True, "cuda"))
    attn.processor = proc
    sd = {}
    with torch.no_grad():
        for name, p in list(attn.named_parameters()) + list(attn.named_buffers()):
            if name.endswith("pe"):
                sd[f"a.{name}"] = p.detach().cpu().clone()
                continue
            v = torch.randn(p.shape, generator=g) * (0.3 if name.endswith("mix_factor") else 0.05)
            p.copy_(v.cuda())
            sd[f"a.{name}"] = v
    return attn, sd


def _close(got, ref, what):
    rel = ((got.float().cpu() - ref).norm() / ref.norm()).item()
    print(f"{what}: rel-l2 {rel:.3e}")
    assert rel < 5e-3, (what, rel)


@pytest.mark.parametrize("c,l", [(320, 256), (640, 64), (1280, 16)])
def test_mvdream_i2v_processor_protocol(c, l):
    from animate3d_b200.modules import MVDreamI2VXFormersAttnProcessor
    from oracle import unet_oracle as O
    nv, nf, b = 4, 3, 2
    proc = MVDreamI2VXFormersAttnProcessor(hidden_size=c, num_views=nv, num_frames=nf, device="cuda")
    attn, sd = _attn_and_sd(c, c, c, proc)
    x = torch.randn(b * nv * nf, l, c, generator=torch.Generator().manual_seed(1))
    got = proc(attn, x.cuda())
    assert got.shape == x.shape and got.dtype == x.dtype
    _close(got, O.proc_mv_i2v(sd, "a", x, HEADS, nv, nf), f"MVDreamI2V c={c}")


@pytest.mark.parametrize("c,l", [(320, 256), (1280, 16)])
def test_ip_adapter_processor_protocol(c, l):
    from animate3d_b200.modules import IPAdapterXFormersAttnProcessor
    from oracle import unet_oracle as O
    n = 6
    proc = IPAdapterXFormersAttnProcessor(hidden_size=c, cross_attention_dim=768, num_tokens=(4,), scale=0.7, device="cuda")
    attn, sd = _attn_and_sd(c, 768, c + 1, proc)
    g = torch.Generator().manual_seed(2)
    x, text, ip = torch.randn(n, l, c, generator=g), torch.randn(n, 77, 768, generator=g), torch.randn(n, 4, 768, generator=g)
    got = proc(attn, x.cuda(), encoder_hidden_states=(text.cuda(), [ip.cuda()]))
    _close(got, O.proc_ip_adapter(sd, "a", x, text, ip, HEADS, 0.7), f"IPAdapter c={c}")
    with pytest.raises(ValueError):
        proc(attn, x.cuda(), encoder_hidden_states=text.cuda())


def test_ip_adapter_processor_scale_zero():
    """scale = 0 switches the image branch off: the processor equals its text-only attention."""
    from animate3d_b200.modules import IPAdapterXFormersAttnProcessor
    from oracle import unet_oracle as O
    c, l, n = 320, 256, 6
    proc = IPAdapterXFormersAttnProcessor(hidden_size=c, cross_attention_dim=768, num_tokens=(4,), scale=0.0, device="cuda")
    attn, sd = _attn_and_sd(c, 768, c + 5, proc)
    g = torch.Generator().manual_seed(7)
    x, text, ip = torch.randn(n, l, c, generator=g), torch.randn(n, 77, 768, generator=g), torch.randn(n, 4, 768, generator=g)
    got = proc(attn, x.cuda(), encoder_hidden_states=(text.cuda(), [ip.cuda()]))
    ref = O.proc_ip_adapter(sd, "a", x, text, ip, HEADS, 0.0)
    _close(got, ref, "IPAdapter scale=0")
    assert ((O.proc_ip_adapter(sd, "a", x, text, ip, HEADS, 1.0) - ref).norm() / ref.norm()).item() > 1e-2


@pytest.mark.parametrize("c,fs", [(320, 16), (1280, 4)])
def test_spatiotemporal_processor_protocol(c, fs):
    from animate3d_b200.modules import SpatioTemporalI2VXFormersAttnProcessor
    from oracle import unet_oracle as O
    nv, nf, b = 4, 16, 1
    proc = SpatioTemporalI2VXFormersAttnProcessor(hidden_size=c, feature_size=fs, num_views=nv, num_frames=nf, use_alpha_blender=True,
                                                  device="cuda")
    attn, sd = _attn_and_sd(c, c, c + 2, proc)
    x = torch.randn(b * nv * fs * fs, nf, c, generator=torch.Generator().manual_seed(3))
    got = proc(attn, x.cuda())
    _close(got, O.proc_spatiotemporal(sd, "a", x, HEADS, nv, nf, fs), f"SpatioTemporalI2V c={c}")


def test_module_surface_attn_processors_roundtrip():
    """unet.attn_processors -> rebuild every processor the way inference.py:107-174 does -> unet.set_attn_processor: accepted;
    wrong kinds / geometry / counts: rejected loudly.  Paths the reference scripts poke exist."""
    from animate3d_b200 import modules as Mo
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    cfg = UNetConfig(block_out_channels=(64, 128, 256, 256), cross_attention_dim=64, ip_image_embed_dim=32, num_views=2, num_frames=3)
    unet = MVUNetMotionModel(cfg, device="cuda")
    procs = unet.attn_processors
    assert len(procs) == 74 and sum(".motion_modules." in k for k in procs) == 42
    assert isinstance(unet, torch.nn.Module) and len(unet.state_dict()) == len(MVUNetMotionModel.expected_keys(cfg))
    assert unet.down_blocks[0].motion_modules[1].transformer_blocks[0].pos_embed is None        # inference.py:183-192
    a1 = unet.down_blocks[0].attentions[0].transformer_blocks[0].attn1
    assert a1.to_out[0].out_features == 64 and a1.to_q.weight.shape == (64, 64) and a1.heads == 8
    new = {}
    for name, p in procs.items():
        if ".motion_modules." in name:
            q = Mo.SpatioTemporalI2VXFormersAttnProcessor(hidden_size=p.hidden_size, feature_size=p.feature_size, num_views=2, num_frames=3,
                                                          use_alpha_blender=True, device="cuda")
        elif name.endswith("attn1.processor"):
            q = Mo.MVDreamI2VXFormersAttnProcessor(hidden_size=p.hidden_size, num_views=2, num_frames=3, device="cuda")
        else:
            q = Mo.IPAdapterXFormersAttnProcessor(hidden_size=p.hidden_size, cross_attention_dim=64, num_tokens=(4,), scale=1.0, device="cuda")
        with torch.no_grad():
            for t in q.parameters():
                t.fill_(0.25)
        new[name] = q
    unet.set_attn_processor(new)
    assert float(unet.down_blocks[1].attentions[0].transformer_blocks[0].attn1.processor.to_q_i2v.weight.mean()) == 0.25
    bad = dict(new)
    k_motion = next(k for k in bad if ".motion_modules." in k)
    bad[k_motion] = Mo.MVDreamI2VXFormersAttnProcessor(hidden_size=64, num_views=2, num_frames=3, device="cuda")
    with pytest.raises(ValueError, match="SpatioTemporal"):
        unet.set_attn_processor(bad)
    bad = dict(new)
    k1 = next(k for k in bad if k.endswith("attn1.processor") and ".attentions." in k)
    bad[k1] = Mo.MVDreamI2VXFormersAttnProcessor(hidden_size=new[k1].hidden_size, num_views=4, num_frames=3, device="cuda")
    with pytest.raises(ValueError, match="geometry"):
        unet.set_attn_processor(bad)
    with pytest.raises(ValueError, match="number of processors"):
        unet.set_attn_processor({k: v for k, v in list(new.items())[:10]})
    assert unet.to("cuda") is unet and unet.to(torch.float16) is unet and unet.dtype == torch.float16
