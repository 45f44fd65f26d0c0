"""MV-VDM sampling from the command line (README step 3; the reference's inference.sh -> inference.py), on the engine:

    python -m animate3d_b200.inference --config configs/inference/inference.yaml \\
        --pretrained_unet_path pretrained_models/animate3d_motion_modules.ckpt --W 256 --H 256 --L 16 --N 4 \\
        --ip_image_root examples/images --ip_image_name butterfly --prompt "a butterfly is flying"

Same flags and defaults as inference.py:290-303, and the same outputs: `{output_dir}/{save_name}/{idx}-{prompt words}.gif`
per seed of the config (an existing GIF is skipped) and the config as `config.yaml` beside them.  The checkpoints the config
names are read from local directories or the hub cache (`pretrained.resolve`); nothing is downloaded.  The released UNet
is wired for 256 x 256 (inference.sh passes --W 256 --H 256); the reference's default of 512 is kept and the UNet refuses
it with a ValueError that says so."""
from __future__ import annotations

import argparse
import os
from typing import List

import torch


def load_image(path: str):
    """diffusers' load_image for a local file: PIL open, EXIF orientation applied, converted to RGB."""
    import PIL.Image
    import PIL.ImageOps
    image = PIL.ImageOps.exif_transpose(PIL.Image.open(path))
    return image.convert("RGB")


def export_to_gif_mv(samples: List[list], save_path: str) -> str:
    """util.py:190-219: frame i of every view pasted side by side (left to right in view order) on an RGB canvas of the
    summed width and the largest height, then diffusers 0.28.0's export_to_gif with its defaults: 10 fps, so 100 ms per
    frame (`duration=1000 // fps`), `loop=0` (forever) and `optimize=False`."""
    from PIL import Image
    frames = []
    for i in range(len(samples[0])):
        views = [v[i] for v in samples if i < len(v)]
        canvas = Image.new("RGB", (sum(im.size[0] for im in views), max(im.size[1] for im in views)))
        x = 0
        for im in views:
            canvas.paste(im, (x, 0))
            x += im.size[0]
        frames.append(canvas)
    if os.path.dirname(save_path):
        os.makedirs(os.path.dirname(save_path), exist_ok=True)
    frames[0].save(save_path, save_all=True, append_images=frames[1:], optimize=False, duration=1000 // 10, loop=0)
    return save_path


def parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="Sample multi-view videos with the MV-VDM (inference.py on the engine)")
    p.add_argument("--pretrained_unet_path", type=str, default=None, required=True)
    p.add_argument("--config", type=str, required=True)
    p.add_argument("--save_name", type=str, default="debug")
    p.add_argument("--L", type=int, default=16)
    p.add_argument("--W", type=int, default=512)
    p.add_argument("--H", type=int, default=512)
    p.add_argument("--N", type=int, default=4)
    p.add_argument("--ip_image_root", type=str, default="examples/images")
    p.add_argument("--ip_image_name", type=str, default="", required=True)
    p.add_argument("--prompt", type=str, default="", required=True)
    return p


def main(args) -> List[str]:
    """inference.py:47-286.  Returns the GIF paths of all seeds, written now or found already there."""
    import yaml

    from .pipeline import load_pipeline, read_yaml
    config = read_yaml(args.config)
    savedir = f"{config['output_dir']}/{args.save_name}"
    os.makedirs(savedir, exist_ok=True)
    pipeline = load_pipeline(config, args.pretrained_unet_path, device="cuda", num_views=args.N, num_frames=args.L)
    seeds = config.get("seed", [-1])
    seeds = [seeds] if isinstance(seeds, int) else list(seeds)
    name = "-".join(args.prompt.replace("/", "").split(" ")[:10])
    if args.ip_image_name != "":
        files = [os.path.join(args.ip_image_root, f"{args.ip_image_name}_{i}.png") for i in range(args.N)]
    else:
        files = [os.path.join(args.ip_image_root, f"{i}.png") for i in range(args.N)]
    paths = []
    for idx, seed in enumerate(seeds):
        path = f"{savedir}/{idx}-{name}.gif"
        paths.append(path)
        if seed != -1:
            torch.manual_seed(seed)
        else:
            torch.seed()
        if os.path.exists(path):
            continue
        print(f"current seed: {torch.initial_seed()}\nsampling {args.prompt} ...")
        frames = pipeline(args.prompt, negative_prompt="", num_inference_steps=config["steps"],
                          guidance_scale=config["guidance_scale"], width=args.W, height=args.H, num_frames=args.L,
                          num_videos_per_prompt=args.N, ip_adapter_image=[load_image(f) for f in files],
                          i2v_cond_time_zero=config.get("i2v_cond_time_zero", False),
                          i2v_similarity_init=config.get("i2v_similarity_init")).frames
        export_to_gif_mv(frames, path)
        print(f"save to {path}")
    with open(f"{savedir}/config.yaml", "w") as f:
        yaml.safe_dump(config, f, sort_keys=False)
    return paths


if __name__ == "__main__":
    main(parser().parse_args())
