"""The IP-Adapter image encoder on the engine (animate3d_b200/clip.py): the preprocessing kernel against the Pillow-exact
oracle (oracle/clip_oracle.py), the GELU GEMM epilogue and ragged query tiles against the float64 ABI oracle, the full
ViT-H/14 geometry against the fp32 tower, graph replay, a shadow-checked pass and the guidance's per-step call."""
import numpy as np
import pytest
import torch

from oracle import abi_gelu as G
from oracle import abi_oracle as A
from oracle import clip_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
VIT_H = dict(hidden_size=1280, intermediate_size=5120, num_attention_heads=16, num_hidden_layers=32, image_size=224,
             patch_size=14, projection_dim=1024, layer_norm_eps=1e-5, hidden_act="gelu")
SMALL = dict(VIT_H, hidden_size=160, intermediate_size=640, num_attention_heads=2, num_hidden_layers=2, projection_dim=64)


@pytest.fixture(scope="module", autouse=True)
def _no_tf32():
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _encoder(cfg, seed=0):
    from animate3d_b200.clip import CLIPVisionModelWithProjection
    sd = O.random_state_dict(cfg, seed)
    return CLIPVisionModelWithProjection(cfg, DEV).load_state_dict(sd), sd


def _engine(cfg, seed=0):
    from animate3d_b200.clip import CLIPImageProcessor, IPAdapterImageProcessor
    enc, sd = _encoder(cfg, seed)
    fe = CLIPImageProcessor(DEV)
    return IPAdapterImageProcessor(fe, enc), enc, fe, sd


def _patches_of(pv):
    """The patch-GEMM operand a3d_clip_preprocess must write for normalised pixel values [n, 3, 224, 224]."""
    n = pv.shape[0]
    p = pv.reshape(n, 3, 16, 14, 16, 14).permute(0, 2, 4, 1, 3, 5).reshape(n, 256, 588)
    out = torch.zeros(n, 257, 640, dtype=torch.float16)
    out[:, 1:, :588] = p.half()
    return out.reshape(n * 257, 640)


def _ulps(a, b):
    ia = a.float().contiguous().view(torch.int32).long()
    ib = b.float().contiguous().view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int((ia - ib).abs().max())


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item(), ((a - b).abs().max() / b.abs().max()).item()


# ------------------------------------------------------------------------------------------------ preprocessing kernel
CASES = [("f32", 256, 256), ("f32", 1024, 1024), ("f32", 384, 512), ("u8", 256, 256), ("u8", 199, 257), ("u8", 100, 100)]


@pytest.mark.parametrize("kind,h,w", CASES, ids=[f"{k}_{h}x{w}" for k, h, w in CASES])
def test_preprocess_matches_pillow_oracle(kind, h, w):
    from animate3d_b200 import _lib as L
    from animate3d_b200 import ops
    from animate3d_b200.clip import CLIPImageProcessor
    g = _g(h * w)
    n = 3
    if kind == "f32":
        x = torch.rand(n, 3, h, w, generator=g)
        x[0, 0, 0, :8] = torch.tensor([k / 255 for k in range(248, 256)])       # the k/255 boundaries
        x[1, 1, :8, 0] = torch.tensor([k / 255 for k in range(8)])
        src, fmt, u8 = x.to(DEV), L.CLIP_SRC_F32_NCHW, O.quantise(x)
    else:
        x = torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8)
        src, fmt, u8 = x.to(DEV), L.CLIP_SRC_U8_NHWC, x.permute(0, 3, 1, 2)
    want_u8 = O.preprocess_u8(u8)
    want_pv = O.normalise(want_u8)
    patches = torch.full((n * 257, 640), float("nan"), device=DEV, dtype=torch.float16)
    pv = torch.full((n, 3, 224, 224), float("nan"), device=DEV)
    ops.clip_preprocess(src, fmt, patches, pv, CLIPImageProcessor(DEV).tables.get(h, w, DEV))
    pv = pv.cpu()
    mean = torch.tensor(O.CLIP_MEAN).view(3, 1, 1).double()
    std = torch.tensor(O.CLIP_STD).view(3, 1, 1).double()
    got_u8 = torch.round((pv.double() * std + mean) * 255).to(torch.uint8)
    assert torch.equal(got_u8, want_u8), int((got_u8 != want_u8).sum())
    assert _ulps(pv, want_pv) <= 1
    assert torch.equal(patches.cpu(), _patches_of(pv))


def test_float_render_path_equals_pil_path():
    """encode_image on float device renders == on the reference's uint8 PIL list: same pixel values, same embeddings."""
    from PIL import Image
    ipp, enc, fe, _ = _engine(SMALL)
    x = torch.rand(2, 3, 256, 256, generator=_g(7), device="cpu").to(DEV)
    pil = [Image.fromarray((im.permute(1, 2, 0).cpu().numpy() * 255).astype(np.uint8)) for im in x]
    assert torch.equal(fe(x, return_tensors="pt").pixel_values, fe(pil, return_tensors="pt").pixel_values)
    e_float = ipp.encode_image(x)
    e_pil = ipp.encode_image(pil)
    assert torch.equal(e_float, e_pil)


# ------------------------------------------------------------------------------------------------ ragged query tiles
def _qkv(rows_total, heads, d, g):
    dqk, dv = (d + 15) // 16 * 16, (d + 16) // 16 * 16
    buf = torch.zeros(rows_total, heads * (2 * dqk + dv))
    q = buf[:, :heads * dqk].view(rows_total, heads, dqk)
    k = buf[:, heads * dqk:2 * heads * dqk].view(rows_total, heads, dqk)
    v = buf[:, 2 * heads * dqk:].view(rows_total, heads, dv)
    q[..., :d] = torch.randn(rows_total, heads, d, generator=g)
    k[..., :d] = torch.randn(rows_total, heads, d, generator=g)
    v[..., :d] = torch.randn(rows_total, heads, d, generator=g)
    v[..., d] = 1.0
    return buf.half().to(DEV), dqk


@pytest.mark.parametrize("lq", [257, 129, 383])
@pytest.mark.parametrize("d", [40, 80, 160])
def test_attention_ragged_query_tiles(lq, d):
    """e1 not a multiple of 128 with e2 == 1: the tensor-core path within the ABI-oracle bound on every element, rows between
    the images (past e1) untouched."""
    from animate3d_b200 import ops
    heads, n, gap = 3, 3, 5
    buf, dqk = _qkv(n * lq, heads, d, _g(lq * d))
    nq = buf.shape[1]
    rows, ext = (nq, lq * nq, lq * nq, n * lq * nq), (lq, 1, n, 1)
    C = heads * d
    ostr = (C, (lq + gap) * C, (lq + gap) * C, n * (lq + gap) * C)     # `gap` rows between images that must stay untouched
    q = ops.view5(buf, 0, nq, rows, ext)
    k = ops.view5(buf, heads * dqk, nq - heads * dqk, rows, ext)
    v = ops.view5(buf, 2 * heads * dqk, nq - 2 * heads * dqk, rows, ext)
    out = torch.randn(n * (lq + gap), C, generator=_g(1)).half().to(DEV)
    before = out.clone()
    V = lambda t, col: A.V5(buf, col, nq - col, rows, ext)
    ref = A.attention(V(q, 0), V(k, heads * dqk), V(v, 2 * heads * dqk), before, ostr, heads=heads, d=d, scale=d ** -0.5)
    kw = dict(heads=heads, d=d, scale=d ** -0.5)
    assert ops.attention_kernel(q, k, v, out, ostr, **kw) == "tc"
    ops.attention(q, k, v, out, ostr, **kw)
    torch.cuda.synchronize()
    A.assert_within(A.flat(out, ref.value.numel()), ref, f"lq={lq} d={d}")
    assert torch.equal(out[ref.value.numel() // C:], before[ref.value.numel() // C:])


def test_attention_ragged_queries_need_e2_one():
    from animate3d_b200 import _lib as L
    from animate3d_b200 import ops
    buf, dqk = _qkv(2 * 257, 1, 80, _g(3))
    nq = buf.shape[1]
    rows, ext = (nq, 257 * nq, 514 * nq, 514 * nq), (257, 2, 1, 1)
    q = ops.view5(buf, 0, nq, rows, ext)
    k = ops.view5(buf, dqk, nq - dqk, rows, ext)
    v = ops.view5(buf, 2 * dqk, nq - 2 * dqk, rows, ext)
    out = torch.zeros(514, 80, device=DEV, dtype=torch.float16)
    with pytest.raises(L.A3DError, match="e2 == 1"):
        ops.attention(q, k, v, out, (80, 257 * 80, 514 * 80, 514 * 80), heads=1, d=80, scale=0.1, impl=L.IMPL_TC)


# ------------------------------------------------------------------------------------------------ GELU epilogue
# A 257-row table leaves room for fewer than two stages of the 256-column tile (up to 64 table rows per warpgroup), so those
# calls run at 128 columns; CLIP's fc1 itself (bias only) takes the 256-column GELU instance.
@pytest.mark.parametrize("M,N,K,rowbias,bn", [(1028, 384, 128, True, 128), (300, 640, 1280, True, 160),
                                              (1028, 5120, 1280, True, 128), (77, 256, 64, True, 128),
                                              (1028, 5120, 1280, False, 256)])
def test_gemm_gelu_epilogue(M, N, K, rowbias, bn):
    from animate3d_b200 import ops
    g = _g(M + N + K)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(DEV)
    b = (torch.randn(N, K, generator=g) / K ** 0.5 * 2).half().to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    rb = dict(rowbias=torch.randn(257, N, generator=g).to(DEV), rb_mod=257) if rowbias else {}
    for impl in (0, 2):
        out = torch.zeros(M, N, device=DEV, dtype=torch.float16)
        kw = dict(M=M, N=N, K=K, bias=bias, gelu=True, impl=impl, **rb)
        ref = G.gemm(a, b, out.clone(), **kw)
        assert ops.gemm_kernel(a, b, out, **kw) == (f"tc BN{bn} gelu plain" if impl == 0 else "simt")
        ops.gemm(a, b, out, **kw)
        torch.cuda.synchronize()
        A.assert_within(out, ref, f"gelu M={M} N={N} K={K} impl={impl}")


# ------------------------------------------------------------------------------------------------ the encoder
def test_vit_h_against_fp32_oracle_and_graph_replay():
    """Random-init ViT-H/14 geometry (32 layers, 1280 wide), 4 images: fp16 engine vs the fp32 tower; the replayed graph is
    bit-identical to the eager pass."""
    ipp, enc, fe, sd = _engine(VIT_H, seed=1)
    x = torch.rand(4, 3, 256, 256, generator=_g(11)).to(DEV)
    e1 = ipp.encode_image(x)            # eager
    e2 = ipp.encode_image(x)            # eager + capture
    e3 = ipp.encode_image(x)            # replay
    assert torch.equal(e1, e3) and torch.equal(e1, e2)
    pv = O.pixel_values(x.cpu())
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        ref = O.vision_forward(sdd, VIT_H, pv.to(DEV).half().float())
    rel, mx = _rel(e1, ref)
    print(f"ViT-H 32 layers, 4 images: rel-L2 {rel:.3e}, max-abs/max-ref {mx:.3e}, launches {enc.launches_per_forward}")
    assert rel < 1e-2 and mx < 2e-2
    # forward(pixel_values) (pipeline.encode_image's route) agrees with the one-launch raw-image route
    pv_dev = fe(x, return_tensors="pt").pixel_values
    assert torch.equal(enc(pv_dev).image_embeds, e1)


def test_shadow_pass_covers_new_ops(monkeypatch):
    """One encoder pass at ViT-H width (2 layers, 2 images) with every launch checked against the ABI oracle; the
    preprocessing launch against the Pillow-exact oracle."""
    from animate3d_b200 import ops
    from shadow import Shadow
    cfg = dict(VIT_H, num_hidden_layers=2)
    ipp, enc, fe, _ = _engine(cfg, seed=2)
    enc.use_cuda_graph = False                  # the shadow synchronises around every launch
    x = torch.rand(2, 3, 320, 256, generator=_g(5)).to(DEV)
    sh = Shadow("clip")
    prep = []
    real_prep = ops.clip_preprocess

    def checked_prep(src, fmt, patches, pixel_values=None, tables=None):
        real_prep(src, fmt, patches, pixel_values, tables)
        torch.cuda.synchronize()
        want = _patches_of(O.pixel_values(src.cpu()))
        prep.append(torch.equal(patches.cpu(), want))

    ops.clip_preprocess = checked_prep
    gelu_checked = []

    def gemm_oracle(*a, **kw):                  # the shadow's GEMM oracle, with the GELU epilogue of oracle/abi_gelu.py
        gelu_checked.append(bool(kw.get("gelu")))
        return G.gemm(*a, **kw)

    monkeypatch.setattr(A, "gemm", gemm_oracle)
    try:
        with sh.active():
            ipp.encode_image(x)
    finally:
        ops.clip_preprocess = real_prep
    print(sh.summary())
    assert prep == [True]
    assert not sh.failures(), sh.table(sh.failures())
    geos = [r["geo"] for r in sh.records if r["op"] == "gemm"]
    assert len(gelu_checked) == len(geos) and sum(gelu_checked) == 2          # fc1 of both layers
    assert sum(1 for r in sh.records if r["op"] == "attention" and r["path"] == "tc" and "Lq=257" in r["geo"]) == 2
    assert len(geos) == 2 * 4 + 2 and sh.calls["layer_norm"] == 2 * 2 + 2


def test_guidance_call_is_sync_free_and_matches_reference_pil_path():
    """AnimateMVDiffusionGuidance.__call__ with the engine's IP-Adapter processor: no host sync after warm-up, and the image
    embeddings the UNet receives equal the reference's PIL path through the oracle (fp16 bar)."""
    from PIL import Image
    from types import SimpleNamespace
    from animate3d_b200.guidance import AnimateMVDiffusionGuidance, PrecomputedPromptUtils
    ipp, enc, fe, sd = _engine(SMALL, seed=3)
    seen = []

    class StubUNet:
        device = torch.device(DEV)

        def __call__(self, sample, timestep, encoder_hidden_states, camera=None, added_cond_kwargs=None, num_views=None,
                     i2v_cond_time_zero=False):
            seen.append(added_cond_kwargs["image_embeds"])
            return SimpleNamespace(sample=0.1 * sample + 0.01 * added_cond_kwargs["image_embeds"].mean())

    n, f, H = 2, 2, 256
    g = AnimateMVDiffusionGuidance({"n_view": n, "n_frame": f, "guidance_scale": 5.0}, unet=StubUNet(), ip_image_processor=ipp)
    gen = _g(9)
    rgb = torch.rand(n * f, H, H, 3, generator=gen).to(DEV)
    c2w = torch.eye(4).repeat(n * f, 1, 1)
    c2w[:, :3, 3] = torch.randn(n * f, 3, generator=gen)
    c2w = c2w.to(DEV)
    pu = PrecomputedPromptUtils(torch.randn(77, 768, generator=gen).to(DEV), torch.zeros(77, 768, device=DEV))
    z = torch.zeros(n * f, device=DEV)
    t = torch.tensor([300], device=DEV)
    for _ in range(3):                                          # warm-up: tables, eager pass, graph capture
        g(rgb, pu, z, z, z, c2w, rgb_as_latents=True, timestep=t)
    seen.clear()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        g(rgb, pu, z, z, z, c2w, rgb_as_latents=True, timestep=t)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    got = seen[0][:n]
    cond = rgb.reshape(n, f, H, H, 3)[:, 0]
    pil = [Image.fromarray((im.cpu().numpy() * 255).astype(np.uint8)) for im in cond]
    pv = O.pixel_values(pil)
    with torch.no_grad():
        ref = O.vision_forward({k: v.to(DEV) for k, v in sd.items()}, SMALL, pv.to(DEV).half().float())
    rel, mx = _rel(got, ref)
    assert rel < 1e-2 and mx < 2e-2, (rel, mx)
