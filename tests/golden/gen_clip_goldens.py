"""Generate tests/golden/ref_clip.pt with Pillow and the installed transformers (not from the reference checkout):

    python tests/golden/gen_clip_goldens.py        ->  tests/golden/ref_clip.pt

* resize: Pillow's Image.resize(BICUBIC) of seeded random RGB images (numpy PCG64, `resize_input(seed, h, w)`) for the sizes the
  CLIP processor meets; the fixture keeps the sha256 of every output and the full output of the small cases.  The processor
  golden is Pillow's resize itself: transformers 5.x's CLIPImageProcessor no longer resizes through PIL and differs from
  the reference's 4.25-4.28 path by up to one uint8 level.
* vision: a small random CLIPVisionConfig (hidden 160, 2 heads of 80, 2 layers, 224 px, patch 14), its state dict
  (oracle.clip_oracle.random_state_dict(cfg, seed) rounded to fp16 values, regenerated from the seed by the test and pinned
  by a digest), seeded pixel values and the image_embeds of transformers' own CLIPVisionModelWithProjection in fp32.
"""
import hashlib
import os
import sys

import numpy as np
import torch

OUT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(OUT))
RESIZE_CASES = [((256, 256), (224, 224)), ((1024, 1024), (224, 224)), ((384, 512), (224, 298)), ((100, 100), (224, 224)),
                ((199, 257), (173, 224)), ((257, 199), (289, 224))]          # (h, w) -> (out_h, out_w)
FULL = ((100, 100), (199, 257))
VISION = dict(hidden_size=160, intermediate_size=320, num_attention_heads=2, num_hidden_layers=2, image_size=224, patch_size=14,
              projection_dim=64, layer_norm_eps=1e-5, hidden_act="gelu")


def resize_input(seed: int, h: int, w: int) -> np.ndarray:
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def vision_state_dict(seed: int = 0) -> dict:
    sys.path.insert(0, ROOT)
    from oracle import clip_oracle as O
    return {k: v.half().float() for k, v in O.random_state_dict(VISION, seed).items()}


def vision_inputs(seed: int = 1) -> torch.Tensor:
    return torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(seed))


def digest(t) -> str:
    if isinstance(t, dict):
        h = hashlib.sha256()
        for k in sorted(t):
            h.update(k.encode())
            h.update(t[k].contiguous().numpy().tobytes())
        return h.hexdigest()
    return hashlib.sha256(np.ascontiguousarray(t).tobytes()).hexdigest()


def main():
    import PIL
    import transformers
    from PIL import Image
    resize = []
    for i, ((h, w), (oh, ow)) in enumerate(RESIZE_CASES):
        out = np.asarray(Image.fromarray(resize_input(i, h, w)).resize((ow, oh), Image.BICUBIC))
        resize.append({"seed": i, "in": (h, w), "out": (oh, ow), "sha256": digest(out),
                       "pixels": torch.from_numpy(out.copy()) if (h, w) in FULL else None})
    sd = vision_state_dict()
    model = transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**VISION)).eval()
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.endswith("position_ids") for k in missing), (missing, unexpected)
    x = vision_inputs()
    with torch.no_grad():
        emb = model(pixel_values=x).image_embeds
    torch.save({"resize": resize, "vision": {"config": VISION, "sd_seed": 0, "sd_sha256": digest(sd), "x_seed": 1,
                                             "x_sha256": digest(x.numpy()), "image_embeds": emb.clone()},
                "versions": {"Pillow": PIL.__version__, "transformers": transformers.__version__}},
               os.path.join(OUT, "ref_clip.pt"))


if __name__ == "__main__":
    main()
