"""The released model built from checkpoint files on disk, on the H100: `pipeline.load_pipeline` against the hand-assembled
pipeline of INTEGRATION §1, the guidance built from the refine config's guidance block against the injected one, and
`python -m animate3d_b200.inference` end to end.  The tree is the released UNet geometry in fp16 with seeded random
weights, a small CLIP text tower and a small ViT image tower."""
import gc
import json
import os
import subprocess
import sys
import time

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pretrained_tree as T  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NV, NF = 4, 16
PROMPT = "a lion is idling"
SCHED = {"num_train_timesteps": 1000, "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "linear", "steps_offset": 1,
         "clip_sample": False}
ATTN = {"mvdream_attn_cfg": {"image_attn": {"enabled": True}},
        "motion_module_attn_cfg": {"enabled": True,
                                   "spatial_attn": {"enabled": True,
                                                    "attn_cfg": {"use_spatial_encoding": True, "spatial_encoding_type": "sinusoid",
                                                                 "use_camera_encoding": False, "camera_encoding_type": "sinusoid"}},
                                   "image_attn": {"enabled": False}, "use_alpha_blender": True}}
VIT = dict(hidden_size=80, intermediate_size=160, num_attention_heads=1, num_hidden_layers=2, image_size=224, patch_size=14,
           projection_dim=1024, layer_norm_eps=1e-5, hidden_act="gelu", num_channels=3)


@pytest.fixture(autouse=True)
def offline(monkeypatch):
    monkeypatch.setenv("HF_HUB_OFFLINE", "1")
    monkeypatch.setenv("TRANSFORMERS_OFFLINE", "1")


def _write_text_side(base):
    """tokenizer/ and text_encoder/: a character-level CLIP tokenizer and a one-layer 768-wide CLIP text tower."""
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTokenizer
    chars = "abcdefghijklmnopqrstuvwxyz"
    vocab = {"<|startoftext|>": 0, "<|endoftext|>": 1}
    for c in chars:
        vocab[c] = len(vocab)
        vocab[c + "</w>"] = len(vocab)
    tmp = os.path.join(base, "tok_src")
    os.makedirs(tmp)
    with open(os.path.join(tmp, "vocab.json"), "w") as f:
        json.dump(vocab, f)
    with open(os.path.join(tmp, "merges.txt"), "w") as f:
        f.write("#version: 0.2\n")
    CLIPTokenizer(os.path.join(tmp, "vocab.json"), os.path.join(tmp, "merges.txt"), model_max_length=77).save_pretrained(
        os.path.join(base, "tokenizer"))
    torch.manual_seed(0)
    cfg = CLIPTextConfig(vocab_size=len(vocab), hidden_size=768, intermediate_size=256, num_hidden_layers=1,
                         num_attention_heads=12, max_position_embeddings=77, bos_token_id=0, eos_token_id=1, pad_token_id=1)
    CLIPTextModel(cfg).save_pretrained(os.path.join(base, "text_encoder"))


def _write_image_encoder(ip):
    from transformers import CLIPVisionConfig
    from transformers import CLIPVisionModelWithProjection as HFVision
    torch.manual_seed(1)
    HFVision(CLIPVisionConfig(**VIT)).save_pretrained(os.path.join(ip, "models", "image_encoder"))


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    from animate3d_b200.unet_config import UNetConfig
    from oracle import vae_oracle as VO
    cfg = UNetConfig(num_views=NV, num_frames=NF)
    parts = T.split(cfg, seed=5, dtype=torch.float16, device="cuda")
    vae_sd = {k: v.half() for k, v in VO.make_state_dict(VO.VAEConfig(), 0).items()}
    vae_cfg = dict(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=[128, 256, 512, 512], layers_per_block=2,
                   norm_num_groups=32, scaling_factor=0.18215, sample_size=256)
    t = T.write_tree(tmp_path_factory.mktemp("ckpt"), cfg, parts, vae_cfg, vae_sd)
    _write_text_side(t.base)
    _write_image_encoder(t.ip)
    return t, cfg, parts, vae_sd


@pytest.fixture(scope="module")
def hand(tree):
    """INTEGRATION §1's hand assembly from the same tensors."""
    from transformers import CLIPTextModel, CLIPTokenizer

    from animate3d_b200.clip import CLIPImageProcessor, CLIPVisionModelWithProjection
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    from animate3d_b200.scheduler import DDIMScheduler
    from animate3d_b200.vae import AutoencoderKL
    t, cfg, parts, vae_sd = tree
    unet = T.hand_assembled_unet(cfg, parts, "cuda")
    vae = AutoencoderKL()
    vae.load_state_dict(vae_sd)
    tower = CLIPVisionModelWithProjection.from_pretrained(os.path.join(t.ip, "models", "image_encoder"))
    pipe = AnimateDiffMVI2VPipeline(vae=vae, text_encoder=CLIPTextModel.from_pretrained(
                                        os.path.join(t.base, "text_encoder"), local_files_only=True).to("cuda").eval(),
                                    tokenizer=CLIPTokenizer.from_pretrained(os.path.join(t.base, "tokenizer"), local_files_only=True),
                                    unet=unet, scheduler=DDIMScheduler(**SCHED), feature_extractor=CLIPImageProcessor(),
                                    image_encoder=tower)
    pipe.enable_free_init(method="butterworth", num_iters=2, use_fast_sampling=False)
    return pipe


def _images(n=NV, size=256):
    from PIL import Image
    g = torch.Generator().manual_seed(3)
    return [Image.fromarray(torch.randint(0, 256, (size, size, 3), generator=g, dtype=torch.uint8).numpy()) for _ in range(n)]


def _inference_config(t, out_dir, freeinit=True, iters=2, steps=2):
    return {"i2v_cond_time_zero": False, "output_dir": out_dir, "pretrained_model_path": t.base,
            "motion_adapter_path": t.adapter, "ip_adapter_path": t.ip, **ATTN, "freeinit_enabled": freeinit,
            "freeinit_num_iters": iters, "i2v_similarity_init": None, "noise_scheduler_kwargs": SCHED, "seed": [8673],
            "steps": steps, "guidance_scale": 7.5}


def test_load_pipeline_matches_hand_assembly(tree, hand, tmp_path):
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline, load_pipeline
    t = tree[0]
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    pipe = load_pipeline(_inference_config(t, str(tmp_path)), t.ckpt, device="cuda", num_views=NV, num_frames=NF)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"\nload_pipeline ({torch.cuda.get_device_name()}): {dt:.2f} s wall, peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB "
          f"allocated ({(torch.cuda.max_memory_allocated() - before) / 2**30:.2f} GiB above the {before / 2**30:.2f} GiB "
          f"held before), {(torch.cuda.memory_allocated() - before) / 2**30:.2f} GiB held after")
    assert isinstance(pipe, AnimateDiffMVI2VPipeline) and pipe.free_init_enabled and pipe._free_init_num_iters == 2
    assert pipe.vae.config.scaling_factor == 0.18215
    _assert_same_unet(pipe.unet, hand.unet)
    call = dict(negative_prompt="", num_inference_steps=2, guidance_scale=7.5, width=256, height=256, num_frames=NF,
                num_videos_per_prompt=NV, ip_adapter_image=_images(), output_type="latent")
    torch.manual_seed(8673)
    got = pipe(PROMPT, **call).frames
    torch.manual_seed(8673)
    want = hand(PROMPT, **call).frames
    assert got.shape == (NV, 4, NF, 32, 32) and torch.isfinite(got).all()
    assert torch.equal(got, want)
    del pipe, got
    gc.collect()
    torch.cuda.empty_cache()


def _assert_same_unet(a, b):
    sa, sb = torch.nn.Module.state_dict(a), torch.nn.Module.state_dict(b)
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


def test_guidance_from_refine_config_matches_injected(tree, hand, monkeypatch):
    from animate3d_b200.clip import CLIPImageProcessor, IPAdapterImageProcessor
    from animate3d_b200.guidance import AnimateMVDiffusionGuidance, PrecomputedPromptUtils
    t = tree[0]
    # refine_frame_16.yaml's guidance block, the paths pointing into the tree and n_view / n_frame resolved
    block = {"pretrained_model_name_or_path": t.base, "motion_adapter_path": t.adapter, "ip_adapter_path": t.ip,
             "pretrained_unet_path": t.ckpt, "noise_scheduler_kwargs": SCHED,
             "model_config": {"i2v_cond_time_zero": False, **ATTN}, "n_view": NV, "n_frame": NF, "guidance_scale": 5.0,
             "min_step_percent": 0.02, "max_step_percent": 0.2, "recon_std_rescale": 0.25}
    loaded = AnimateMVDiffusionGuidance(block)
    _assert_same_unet(loaded.unet, hand.unet)
    injected = AnimateMVDiffusionGuidance(block, unet=hand.unet, vae=hand.vae,
                                          ip_image_processor=IPAdapterImageProcessor(CLIPImageProcessor(), hand.image_encoder))
    assert injected.unet is hand.unet and injected.vae is hand.vae
    g = torch.Generator(device="cuda").manual_seed(11)
    B = NV * NF
    rgb0 = torch.rand(B, 256, 256, 3, device="cuda", generator=g)
    text = torch.randn(2, 77, 768, device="cuda", generator=g)
    prompt_utils = PrecomputedPromptUtils(text[0], text[1])
    ele, azi = torch.full((B,), 15.0, device="cuda"), torch.linspace(0, 270, NV, device="cuda").repeat_interleave(NF)
    dist = torch.full((B,), 2.0, device="cuda")
    c2w = torch.eye(4, device="cuda").repeat(B, 1, 1)
    c2w[:, :3, 3] = torch.stack([torch.cos(torch.deg2rad(azi)), torch.sin(torch.deg2rad(azi)), torch.full_like(azi, 0.5)], -1) * 2
    # The default CUDA backward of the bilinear resize in front of the VAE scatters with atomics, so rgb.grad is
    # bit-reproducible only in deterministic mode, where the guidance resizes with two matmuls instead.
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    was_deterministic = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    res = []
    try:
        for guide in (loaded, injected):
            rgb = rgb0.clone().requires_grad_(True)
            torch.manual_seed(4)
            out = guide(rgb, prompt_utils, ele, azi, dist, c2w, timestep=torch.tensor([300], device="cuda"))
            out["loss_sds"].backward()
            res.append((out["loss_sds"].detach(), rgb.grad))
    finally:
        torch.use_deterministic_algorithms(was_deterministic)
    assert torch.isfinite(res[0][0]) and res[0][1].abs().sum() > 0
    assert torch.equal(res[0][0], res[1][0])
    assert torch.equal(res[0][1], res[1][1])
    del loaded
    gc.collect()
    torch.cuda.empty_cache()


def test_inference_command_writes_gif_and_config(tree, tmp_path):
    import yaml
    from PIL import Image
    t = tree[0]
    cfg = _inference_config(t, str(tmp_path / "outputs"), freeinit=False)
    with open(tmp_path / "inference.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    img_dir = tmp_path / "images"
    img_dir.mkdir()
    for i, im in enumerate(_images()):
        im.save(img_dir / f"lion_{i}.png")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable, "-m", "animate3d_b200.inference", "--pretrained_unet_path", t.ckpt, "--config",
           str(tmp_path / "inference.yaml"), "--W", "256", "--H", "256", "--L", str(NF), "--N", str(NV), "--ip_image_root",
           str(img_dir), "--ip_image_name", "lion", "--prompt", PROMPT, "--save_name", "run"]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    gif = tmp_path / "outputs" / "run" / "0-a-lion-is-idling.gif"
    with Image.open(gif) as im:
        assert im.n_frames == NF and im.size == (NV * 256, 256)
        assert im.info["duration"] == 100 and im.info["loop"] == 0
    with open(tmp_path / "outputs" / "run" / "config.yaml") as f:
        assert yaml.safe_load(f) == cfg
