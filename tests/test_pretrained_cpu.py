"""Loading the released model from checkpoint files on disk (MVUNetMotionModel.from_pretrained, AutoencoderKL.from_pretrained,
pretrained.resolve) and the inference command's GIF writer and flags, on a width-reduced tree of the published layout.
CPU-only."""
import os
import shutil
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pretrained_tree as T  # noqa: E402

from animate3d_b200 import pretrained as PT  # noqa: E402
from animate3d_b200.unet import MVUNetMotionModel  # noqa: E402
from animate3d_b200.unet_config import UNetConfig, key_plan  # noqa: E402

# the width-reduced geometry of test_state_dict_layout.py::test_load_unet_checkpoint_rules: the released key names
CFG = UNetConfig(block_out_channels=(32, 64, 128, 128), cross_attention_dim=16, ip_image_embed_dim=16, sample_size=8)
VAE_CFG = dict(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=[32, 32, 64, 64], layers_per_block=1,
               norm_num_groups=32, scaling_factor=0.13025, sample_size=64)


@pytest.fixture(autouse=True)
def offline(monkeypatch):
    monkeypatch.setenv("HF_HUB_OFFLINE", "1")
    monkeypatch.setenv("TRANSFORMERS_OFFLINE", "1")


def _vae_sd(seed=0):
    from types import SimpleNamespace

    from animate3d_b200.vae import vae_key_plan
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(s, generator=g) * 0.02 for k, s in vae_key_plan(SimpleNamespace(**VAE_CFG)).items()}


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    parts = T.split(CFG, seed=5)
    return T.write_tree(tmp_path_factory.mktemp("ckpt"), CFG, parts, VAE_CFG, _vae_sd()), parts


def _load(tree, **kw):
    args = dict(pretrained_model_path=tree.base, motion_adapter_path=tree.adapter, ip_adapter_path=tree.ip,
                pretrained_unet_path=tree.ckpt, device="cpu", sample_size=8)
    args.update(kw)
    return MVUNetMotionModel.from_pretrained(**args)


def _assert_same_model(a, b):
    sa, sb = torch.nn.Module.state_dict(a), torch.nn.Module.state_dict(b)
    assert sa.keys() == sb.keys() and set(sa) == set(key_plan(a.cfg))
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


def test_from_pretrained_equals_hand_assembly(tree):
    tree, parts = tree
    model = _load(tree)
    assert model.cfg == CFG                      # ip_image_embed_dim / ip_num_tokens read off the IP-Adapter projection
    hand = T.hand_assembled_unet(CFG, parts, "cpu", ip_image_embed_dim=16, sample_size=8)
    _assert_same_model(model, hand)
    # the checkpoint's motion-module weights won over the adapter's, to_q_i2v is the checkpoint's and not to_q's copy
    sd = torch.nn.Module.state_dict(model)
    k = "down_blocks.0.motion_modules.0.transformer_blocks.0.attn1.to_q.weight"
    assert torch.equal(sd[k], parts.ckpt[k]) and not torch.equal(sd[k], parts.adapter[k])
    for k, v in parts.full.items():
        assert torch.equal(sd[k], v), k
    assert not [k for k in key_plan(CFG) if k not in model._loaded]


def test_ip_adapter_bin_and_safetensors_load_identically(tree, tmp_path):
    tree, parts = tree
    a = PT.load_ip_adapter(os.path.join(tree.ip, "models", "ip-adapter_sd15.bin"))
    b = PT.load_ip_adapter(os.path.join(tree.ip, "models", "ip-adapter_sd15.safetensors"))
    assert list(a) == list(b) == ["image_proj", "ip_adapter"]
    for p in a:
        assert a[p].keys() == b[p].keys() == parts.ip[p].keys()
        for k in a[p]:
            assert torch.equal(a[p][k], b[p][k]), (p, k)
    # a tree with only the .safetensors twin gives the same model
    ip2 = tmp_path / "ip"
    shutil.copytree(tree.ip, ip2)
    os.remove(ip2 / "models" / "ip-adapter_sd15.bin")
    assert PT.ip_adapter_file(str(ip2)).endswith(".safetensors")
    _assert_same_model(_load(tree), _load(tree, ip_adapter_path=str(ip2)))


def test_hub_id_resolves_through_the_cache(tree, tmp_path, monkeypatch):
    tree, _ = tree
    cache = tmp_path / "hub"
    repo = cache / "models--someorg--mvdream-test"
    (repo / "refs").mkdir(parents=True)
    (repo / "refs" / "main").write_text("0123abcd\n")
    shutil.copytree(tree.base, repo / "snapshots" / "0123abcd")
    # a second, unreferenced snapshot must not be picked
    shutil.copytree(tree.base, repo / "snapshots" / "ffffffff")
    monkeypatch.setenv("HF_HUB_CACHE", str(cache))
    assert PT.resolve("someorg/mvdream-test", "unet") == str(repo / "snapshots" / "0123abcd" / "unet")
    monkeypatch.delenv("HF_HUB_CACHE")
    monkeypatch.setenv("HF_HOME", str(tmp_path))
    assert PT.resolve("someorg/mvdream-test") == str(repo / "snapshots" / "0123abcd")
    assert PT.resolve(tree.base, "vae") == os.path.join(tree.base, "vae")
    _assert_same_model(_load(tree), _load(tree, pretrained_model_path="someorg/mvdream-test"))
    with pytest.raises(FileNotFoundError) as e:
        PT.resolve("someorg/not-there", "unet")
    assert "someorg/not-there" in str(e.value) and str(tmp_path / "hub" / "models--someorg--not-there") in str(e.value)
    with pytest.raises(FileNotFoundError, match="text_encoder"):
        PT.resolve("someorg/mvdream-test", "text_encoder")


def test_vae_from_pretrained(tree):
    from animate3d_b200.vae import AutoencoderKL
    tree, _ = tree
    vae = AutoencoderKL.from_pretrained(tree.base, subfolder="vae", device="cpu")
    assert vae.config.scaling_factor == 0.13025 and vae.config.block_out_channels == (32, 32, 64, 64)
    assert vae.config.layers_per_block == 1


def test_errors_name_their_file_or_key(tree, tmp_path):
    tree, parts = tree
    with pytest.raises(FileNotFoundError, match="nowhere"):
        _load(tree, pretrained_model_path=str(tmp_path / "nowhere"))
    with pytest.raises(FileNotFoundError, match="org/absent"):
        _load(tree, motion_adapter_path="org/absent")
    with pytest.raises(FileNotFoundError, match="missing.ckpt"):
        _load(tree, pretrained_unet_path=str(tmp_path / "missing.ckpt"))
    torch.save({"state_dict": {**parts.ckpt, "bogus.weight": torch.zeros(1)}}, tmp_path / "stray.ckpt")
    with pytest.raises(ValueError, match="stray.ckpt.*unexpected"):
        _load(tree, pretrained_unet_path=str(tmp_path / "stray.ckpt"))
    torch.save({"state_dict": dict(list(parts.ckpt.items())[:-5])}, tmp_path / "partial.ckpt")
    with pytest.raises(ValueError, match="partial.ckpt.*missing"):
        _load(tree, pretrained_unet_path=str(tmp_path / "partial.ckpt"))
    # without the checkpoint, the processors' weights come from nowhere: refused at load time, naming the keys
    with pytest.raises(ValueError, match=r"in none of the files.*processor\.to_q_sp"):
        _load(tree, pretrained_unet_path=None)
    with pytest.raises(ValueError, match=r"in none of the files.*_ip\.0\.weight"):
        _load(tree, ip_adapter_path=None)
    sharded = tmp_path / "sharded"
    shutil.copytree(os.path.join(tree.base, "unet"), sharded / "unet")
    (sharded / "unet" / "diffusion_pytorch_model.safetensors.index.json").write_text("{}")
    with pytest.raises(NotImplementedError, match="diffusion_pytorch_model.safetensors.index.json"):
        _load(tree, pretrained_model_path=str(sharded))
    bad_ip = tmp_path / "badip" / "models"
    bad_ip.mkdir(parents=True)
    torch.save({"image_proj": {}}, bad_ip / "ip-adapter_sd15.bin")
    with pytest.raises(ValueError, match="ip-adapter_sd15.bin"):
        _load(tree, ip_adapter_path=str(bad_ip.parent))


@pytest.mark.parametrize("key,value", [
    ("mvdream_attn_cfg", {"image_attn": {"enabled": False}}),
    ("motion_module_attn_cfg", {"enabled": True, "spatial_attn": {"enabled": True, "attn_cfg": {"use_camera_encoding": True}}}),
    ("motion_module_attn_cfg", {"enabled": True, "image_attn": {"enabled": True}}),
    ("motion_module_attn_cfg", {"use_alpha_blender": False}),
])
def test_non_released_model_config_raises(tree, key, value):
    tree, _ = tree
    with pytest.raises(NotImplementedError, match=key):
        _load(tree, model_config={key: value})


def test_released_model_config_loads(tree):
    import yaml
    tree, _ = tree
    block = yaml.safe_load(REFINE_MODEL_CONFIG)
    PT.check_model_config(block)
    PT.check_model_config({**block, "i2v_cond_time_zero": True})        # a sampling option, not wiring
    with pytest.raises(ValueError, match="i2v_cond_time_zero"):
        PT.check_model_config({**block, "i2v_cond_time_zero": "yes"})
    _assert_same_model(_load(tree), _load(tree, model_config=block))


# refine_frame_16.yaml's guidance.model_config block
REFINE_MODEL_CONFIG = """
i2v_cond_time_zero: false
motion_module_attn_cfg:
  enabled: true
  spatial_attn:
    enabled: true
    attn_cfg:
      use_spatial_encoding: true
      spatial_encoding_type: "sinusoid"
      use_camera_encoding: false
      camera_encoding_type: "sinusoid"
  image_attn:
    enabled: false
  use_alpha_blender: true
mvdream_attn_cfg:
  image_attn:
    enabled: true
"""


def test_gif_writer_layout(tmp_path):
    from PIL import Image

    from animate3d_b200.inference import export_to_gif_mv
    L, N, W, H = 5, 3, 24, 16
    samples = [[Image.new("RGB", (W, H), (40 * v, 10 * f, 200)) for f in range(L)] for v in range(N)]
    path = export_to_gif_mv(samples, str(tmp_path / "sub" / "0-a-lion.gif"))
    with Image.open(path) as im:
        assert im.n_frames == L and im.size == (N * W, H)
        assert im.info["duration"] == 100 and im.info["loop"] == 0
        im.seek(2)
        rgb = im.convert("RGB")
        for v in range(N):                       # view v occupies columns [v W, (v + 1) W) of every frame
            assert rgb.getpixel((v * W + W // 2, H // 2)) == (40 * v, 20, 200)


def test_load_image_applies_exif_orientation(tmp_path):
    from PIL import Image

    from animate3d_b200.inference import load_image
    im = Image.new("RGBA", (4, 2), (1, 2, 3, 4))
    exif = Image.Exif()
    exif[0x0112] = 6                             # rotate 90 degrees clockwise on display
    im.convert("RGB").save(tmp_path / "x.jpg", exif=exif)
    got = load_image(str(tmp_path / "x.jpg"))
    assert got.mode == "RGB" and got.size == (2, 4)
    im.save(tmp_path / "y.png")
    assert load_image(str(tmp_path / "y.png")).mode == "RGB"


def test_cli_defaults_match_reference():
    from animate3d_b200.inference import parser
    p = parser()
    args = p.parse_args(["--pretrained_unet_path", "m.ckpt", "--config", "c.yaml", "--ip_image_name", "", "--prompt", "x"])
    assert vars(args) == {"pretrained_unet_path": "m.ckpt", "config": "c.yaml", "save_name": "debug", "L": 16, "W": 512,
                          "H": 512, "N": 4, "ip_image_root": "examples/images", "ip_image_name": "", "prompt": "x"}
    required = {a.dest for a in p._actions if a.required}
    assert required == {"pretrained_unet_path", "config", "ip_image_name", "prompt"}
    with pytest.raises(SystemExit):
        p.parse_args(["--config", "c.yaml", "--ip_image_name", "a", "--prompt", "x"])
