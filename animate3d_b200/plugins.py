"""Import this module from a threestudio application to register the H100 replacements of the reference's plugins
(the reference registers them by importing every directory under `custom/`, launch.py:70-102):

    import animate3d_b200.plugins            # -> threestudio.find("animatemv-diffusion-guidance"), ...

| registered name                         | class                         | reference                                              |
|-----------------------------------------|-------------------------------|--------------------------------------------------------|
| animatemv-diffusion-guidance            | guidance.AnimateMVDiffusionGuidance | guidance/animatemv_guidance.py:54                |
| diff-gaussian-rasterizer-advanced-4d    | renderer.DiffGaussian4D       | renderer/diff_gaussian_rasterizer_advanced_4d.py:23    |

The guidance's IP-Adapter image encoder runs on the engine when it gets the drop-ins of `animate3d_b200.clip` in place of
what the reference's `load_ip_adapter(...)` returns (INTEGRATION.md):

    from animate3d_b200.clip import CLIPImageProcessor, CLIPVisionModelWithProjection, IPAdapterImageProcessor
    ipp = IPAdapterImageProcessor(CLIPImageProcessor(), CLIPVisionModelWithProjection.from_pretrained(image_encoder_dir))
    AnimateMVDiffusionGuidance(cfg, unet=unet, vae=vae, ip_image_processor=ipp)
"""
from .guidance import AnimateMVDiffusionGuidance  # noqa: F401
from .renderer import DiffGaussian4D  # noqa: F401
from .registry import find, register  # noqa: F401
