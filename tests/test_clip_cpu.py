"""CLIP preprocessing and vision tower without a GPU: the arithmetic the kernel shares (animate3d_b200/csrc/a3d_resize_math.h,
driven through tests/cpu_harness/clip_resize_cpu.cpp) and the oracle (oracle/clip_oracle.py) against Pillow and transformers;
negative controls for the three easy mistakes of the resize; config checks and weight packing of animate3d_b200/clip.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import abi_gelu as G
from oracle import abi_oracle as A
from oracle import clip_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "ref_clip.pt"), weights_only=False)


@pytest.fixture(scope="module")
def gen():
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen_clip_goldens", os.path.join(ROOT, "tests", "golden", "gen_clip_goldens.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("h") / "clip_resize_cpu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(ROOT, "tests", "cpu_harness", "clip_resize_cpu.cpp"), "-o", out])
    return C.CDLL(out)


def _resize(harness, img, oh, ow, variant=0):
    h, w = img.shape[:2]
    out = np.empty((oh, ow, 3), np.uint8)
    img = np.ascontiguousarray(img)
    harness.clip_resize_u8(img.ctypes.data_as(C.c_void_p), h, w, oh, ow, variant, out.ctypes.data_as(C.c_void_p))
    return out


def _prep(harness, x, variant=0):
    h, w = x.shape[1:]
    u8 = np.empty((3, 224, 224), np.uint8)
    pv = np.empty((3, 224, 224), np.float32)
    x = np.ascontiguousarray(x, dtype=np.float32)
    harness.clip_prep_f32(x.ctypes.data_as(C.c_void_p), h, w, variant, u8.ctypes.data_as(C.c_void_p), pv.ctypes.data_as(C.c_void_p))
    return u8, pv


# ------------------------------------------------------------------------------------------------ resize vs Pillow
def test_harness_and_oracle_match_pillow_bit_for_bit(harness, golden, gen):
    for case in golden["resize"]:
        img = gen.resize_input(case["seed"], *case["in"])
        oh, ow = case["out"]
        got = _resize(harness, img, oh, ow)
        assert gen.digest(got) == case["sha256"], case["in"]
        ora = O.pil_resize(torch.from_numpy(img).permute(2, 0, 1), oh, ow).permute(1, 2, 0).numpy()
        assert gen.digest(ora) == case["sha256"], case["in"]
        if case["pixels"] is not None:
            assert np.array_equal(got, case["pixels"].numpy())


def test_harness_matches_installed_pillow_on_random_images(harness):
    from PIL import Image
    rng = np.random.default_rng(5)
    for (h, w), (oh, ow) in [((256, 256), (224, 224)), ((384, 512), (224, 298)), ((100, 100), (224, 224)), ((257, 199), (289, 224)),
                             ((31, 700), (224, 5057))]:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        want = np.asarray(Image.fromarray(img).resize((ow, oh), Image.BICUBIC))
        assert int((_resize(harness, img, oh, ow) != want).sum()) == 0, (h, w)


@pytest.mark.parametrize("variant,what", [(2, "vertical pass first"), (3, "no +-0.5 in the fixed-point coefficients")])
def test_resize_negative_controls(harness, golden, gen, variant, what):
    for case in golden["resize"]:
        if case["pixels"] is None:
            continue
        img = gen.resize_input(case["seed"], *case["in"])
        got = _resize(harness, img, *case["out"], variant=variant)
        assert int((got != case["pixels"].numpy()).sum()) > 0, what


def test_float_input_truncates_on_k_over_255_boundaries(harness):
    """fp32 renders on and next to the k/255 boundaries: truncation like (x*255).astype(np.uint8), not rounding."""
    from PIL import Image
    g = torch.Generator().manual_seed(3)
    k = torch.randint(0, 256, (3, 256, 256), generator=g).float()
    x = (k / 255 + torch.randint(-1, 2, k.shape, generator=g) * 0.4 / 255).clamp(0, 1).numpy().astype(np.float32)
    pil = Image.fromarray((x.transpose(1, 2, 0) * 255).astype(np.uint8))
    want = np.asarray(pil.resize((224, 224), Image.BICUBIC)).transpose(2, 0, 1)
    u8, pv = _prep(harness, x)
    assert np.array_equal(u8, want)
    assert torch.equal(torch.from_numpy(pv), O.normalise(torch.from_numpy(want)))
    assert torch.equal(O.pixel_values(torch.from_numpy(x)[None])[0], torch.from_numpy(pv))
    u8_round, _ = _prep(harness, x, variant=1)
    assert int((u8_round != want).sum()) > 0


def test_processor_shapes_and_crop():
    for (h, w) in [(256, 256), (384, 512), (1024, 600), (224, 300)]:
        x = torch.rand(1, 3, h, w)
        rh, rw = O.resize_shape(h, w)
        assert min(rh, rw) == 224 and max(rh, rw) == int(224 * max(h, w) / min(h, w))
        assert O.pixel_values(x).shape == (1, 3, 224, 224)


# ------------------------------------------------------------------------------------------------ vision tower
def test_oracle_matches_transformers_golden(golden, gen):
    v = golden["vision"]
    sd = gen.vision_state_dict(v["sd_seed"])
    x = gen.vision_inputs(v["x_seed"])
    assert gen.digest(sd) == v["sd_sha256"] and gen.digest(x.numpy()) == v["x_sha256"]
    got = O.vision_forward(sd, v["config"], x)
    want = v["image_embeds"]
    assert ((got - want).norm() / want.norm()).item() < 1e-5


@pytest.mark.parametrize("width", ["small", "vit_h_1_layer"])
def test_oracle_matches_transformers_directly(width):
    transformers = pytest.importorskip("transformers")
    cfg = dict(hidden_size=160, intermediate_size=640, num_attention_heads=2, num_hidden_layers=2, projection_dim=64)
    if width == "vit_h_1_layer":
        cfg = dict(hidden_size=1280, intermediate_size=5120, num_attention_heads=16, num_hidden_layers=1, projection_dim=1024)
    cfg.update(image_size=224, patch_size=14, hidden_act="gelu", layer_norm_eps=1e-5)
    sd = O.random_state_dict(cfg, 4)
    model = transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**cfg)).eval()
    model.load_state_dict(sd, strict=False)
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        want = model(pixel_values=x).image_embeds
        got = O.vision_forward(sd, cfg, x)
    assert ((got - want).norm() / want.norm()).item() < 1e-5


# ------------------------------------------------------------------------------------------------ GELU epilogue in the ABI oracle
def test_gemm_gelu_oracle_and_negative_control():
    g = torch.Generator().manual_seed(8)
    M, N, K = 40, 64, 96
    a = torch.randn(M, K, generator=g).half()
    b = (torch.randn(N, K, generator=g) * 0.2).half()
    bias = torch.randn(N, generator=g)
    rb = torch.randn(3, N, generator=g)
    out = torch.zeros(M, N, dtype=torch.float16)
    ref = G.gemm(a, b, out, M=M, N=N, K=K, bias=bias, rowbias=rb, rb_mod=3, gelu=True)
    v = a.double() @ b.double().t() + bias.double() + rb.double()[torch.arange(M) % 3]
    want = torch.nn.functional.gelu(v)
    assert ((ref.value - want.reshape(-1)).abs().max() / want.abs().max()).item() < 1e-10
    assert A.check(ref.value.half(), ref).ratio <= 1.0
    bad = ref.value.half().view(M, N).clone()
    bad[7, 16:24] = v[7, 16:24].half()                       # GELU dropped on one 8-column group
    assert A.check(bad, ref).ratio > 1.0
    # without `gelu` it is the ABI oracle's plain GEMM
    plain = G.gemm(a, b, out, M=M, N=N, K=K, bias=bias, rowbias=rb, rb_mod=3)
    want_plain = A.gemm(a, b, out, M=M, N=N, K=K, bias=bias, rowbias=rb, rb_mod=3)
    assert torch.equal(plain.value, want_plain.value) and torch.equal(plain.bound, want_plain.bound)
    with pytest.raises(ValueError):
        G.gemm(a, b, out, M=M, N=N, K=K, R2=out, gelu=True)


# ------------------------------------------------------------------------------------------------ host module
def test_unsupported_configs_raise():
    from animate3d_b200.clip import check_config
    base = dict(hidden_size=1280, intermediate_size=5120, num_attention_heads=16, num_hidden_layers=32, projection_dim=1024)
    check_config(base)
    for bad in (dict(hidden_act="quick_gelu"), dict(num_attention_heads=20), dict(image_size=336), dict(patch_size=16),
                dict(hidden_size=1536, num_attention_heads=16, intermediate_size=6144)):
        with pytest.raises(NotImplementedError):
            check_config({**base, **bad})


def test_from_transformers_and_from_pretrained_pack_the_same(tmp_path):
    transformers = pytest.importorskip("transformers")
    from animate3d_b200.clip import CLIPVisionModelWithProjection
    cfg = dict(hidden_size=160, intermediate_size=320, num_attention_heads=2, num_hidden_layers=2, projection_dim=64,
               hidden_act="gelu", image_size=224, patch_size=14)
    model = transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**cfg))
    model.save_pretrained(str(tmp_path), safe_serialization=True)
    a = CLIPVisionModelWithProjection.from_transformers(model, device="cpu")
    b = CLIPVisionModelWithProjection.from_pretrained(str(tmp_path), device="cpu")
    assert a.w.keys() == b.w.keys() and all(torch.equal(a.w[k], b.w[k]) for k in a.w)
    assert next(a.parameters()).dtype == torch.float16
    # packed layout: [Q | K | V] per layer, V heads padded to 96 columns with 1.0 at column 80 (bias slot), K padded to 640
    sd = model.state_dict()
    qkv, bq = a.w["layer1.qkv"], a.w["layer1.qkv_b"]
    assert qkv.shape == (2 * 160 + 2 * 96, 160)
    assert torch.equal(qkv[160 + 80:160 + 160], sd["vision_model.encoder.layers.1.self_attn.k_proj.weight"][80:].half())
    assert torch.equal(qkv[320 + 96:320 + 96 + 80], sd["vision_model.encoder.layers.1.self_attn.v_proj.weight"][80:].half())
    assert bq[320 + 80] == 1 and bq[320 + 96 + 80] == 1 and qkv[320 + 80].abs().sum() == 0
    assert a.w["patch"].shape == (160, 640) and a.w["patch"][:, 588:].abs().sum() == 0
    e = "vision_model.embeddings."
    assert torch.allclose(a.w["rowbias"][0], sd[e + "position_embedding.weight"][0] + sd[e + "class_embedding"])
