"""Host logic of the captured 4D-SDS refine step: the device-side timestep draw of the guidance and its bounds, the pointer
recaptures of StepGraphs (a recorded module whose capture_version changed), and the capture_version counters of the three
engine networks."""
from types import SimpleNamespace

import torch

from animate3d_b200 import capture as CP
from animate3d_b200.capture import StepGraphs


class _StubUNet:
    device = torch.device("cpu")


def _guidance(**cfg):
    from animate3d_b200.guidance import AnimateMVDiffusionGuidance
    return AnimateMVDiffusionGuidance({"n_view": 2, "n_frame": 4, **cfg}, unet=_StubUNet())


def test_draw_timestep_covers_the_inclusive_range():
    g = _guidance()
    assert g.step_bounds.tolist() == [g.min_step, g.max_step] == [20, 980]
    g.set_min_max_steps(0.02, 0.025)                  # [20, 25]: six values
    torch.manual_seed(0)
    t = g.draw_timestep(6000)
    assert t.dtype == torch.int64 and t.shape == (6000,)
    assert int(t.min()) == 20 and int(t.max()) == 25
    counts = torch.bincount(t - 20, minlength=6)
    assert counts.numel() == 6 and int(counts.min()) > 800, counts.tolist()


def test_draw_timestep_follows_set_min_max_steps_in_place():
    g = _guidance()
    bounds = g.step_bounds
    g.set_min_max_steps(0.5, 0.5)
    assert g.step_bounds is bounds and bounds.tolist() == [500, 500]
    assert torch.equal(g.draw_timestep(64), torch.full((64,), 500))
    g.cfg.min_step_percent, g.cfg.max_step_percent = 0.3, 0.31       # update_step's schedule writes the same tensor
    g.update_step(0, 10)
    assert g.step_bounds is bounds and bounds.tolist() == [300, 310]
    t = g.draw_timestep(2000)
    assert int(t.min()) == 300 and int(t.max()) == 310


def test_eager_call_keeps_randint_draws():
    """Outside a capture the reference's torch.randint draw is unchanged, and last_timestep holds it."""
    from animate3d_b200.guidance import AnimateMVDiffusionGuidance, PrecomputedPromptUtils

    class Eps(_StubUNet):
        def __call__(self, sample, timestep, encoder_hidden_states, **kw):
            return SimpleNamespace(sample=0.1 * sample)

    n, f = 2, 4
    g = AnimateMVDiffusionGuidance({"n_view": n, "n_frame": f, "guidance_scale": 5.0}, unet=Eps())
    rgb = torch.rand(n * f, 32, 32, 4)[..., :3]
    pu = PrecomputedPromptUtils(torch.randn(77, 768), torch.randn(77, 768))
    z, img, c2w = torch.zeros(n * f), torch.randn(n, 1024), torch.eye(4).expand(n * f, 4, 4) + 0
    torch.manual_seed(5)
    g(rgb, pu, z, z, z, c2w, rgb_as_latents=True, image_embeds=img)
    torch.manual_seed(5)
    want = torch.randint(g.min_step, g.max_step + 1, [1], dtype=torch.long)
    assert torch.equal(g.last_timestep, want)


class _Module:
    def __init__(self):
        self.capture_version = 0


class _Opt:
    param_groups = [{"fused": True, "capturable": True, "params": []}]


class _Recorder(StepGraphs):
    """StepGraphs with its device work replaced by a log; each capture records `mods` through note_module."""

    def __init__(self, mods):
        super().__init__(lambda inp: None, _Opt())
        self.mods, self.log = mods, []

    def eager(self, inputs):
        self.log.append("eager")

    def capture(self, key, inputs):
        self.log.append("capture")
        with CP.collect_modules() as got:
            for m in self.mods + self.mods:           # a module recorded twice is registered once
                CP.note_module(m)
        self.graphs[key] = None
        self.modules[key] = list(got)

    def replay(self, key, inputs):
        self.log.append("replay")
        return False


def test_recaptures_on_a_changed_module_version_only():
    a, b = _Module(), _Module()
    p = _Recorder([a, b])
    p.step("k", {}); p.step("k", {})
    assert p.log == ["eager", "capture", "replay"] and len(p.modules["k"]) == 2
    for _ in range(3):
        p.step("k", {})
    assert p.log[3:] == ["replay"] * 3 and p.pointer_recaptures == 0
    b.capture_version += 1
    p.step("k", {})
    assert p.log[6:] == ["capture", "replay"] and p.pointer_recaptures == 1 and p.recaptures == 0
    p.step("k", {})
    assert p.log[8:] == ["replay"] and p.pointer_recaptures == 1
    unrelated = _Module()
    unrelated.capture_version += 5
    p.step("k", {})
    assert p.log[9:] == ["replay"]


def test_release_drops_graphs_and_captures_again():
    p = _Recorder([_Module()])
    p.step("k", {}); p.step("k", {})
    p.pool = object()
    p.release()
    assert p.graphs == {} and p.modules == {} and p.pool is None
    p.step("k", {})
    assert p.log[3:] == ["capture", "replay"] and p.recaptures == p.pointer_recaptures == 0


def test_note_module_outside_collect_is_a_no_op():
    CP.note_module(_Module())
    with CP.collect_modules() as outer:
        with CP.collect_modules() as inner:
            CP.note_module(m := _Module())
        assert inner == [(m, 0)] and outer == []


def test_load_state_dict_bumps_every_capture_version():
    from animate3d_b200.clip import CLIPVisionModelWithProjection
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig, key_plan
    from animate3d_b200.vae import AutoencoderKL, vae_key_plan
    from oracle import clip_oracle as CO

    vae = AutoencoderKL(block_out_channels=(32, 32), layers_per_block=1, device="cpu")
    sd = {k: torch.randn(s) * 0.1 for k, s in vae_key_plan(vae.config).items()}
    v0 = vae.capture_version
    vae.load_state_dict(sd)
    w0 = vae.W["enc_in"]["w32"]
    vae.load_state_dict(sd)
    assert vae.capture_version == v0 + 2 and vae.W["enc_in"]["w32"] is not w0

    cfg = dict(hidden_size=160, intermediate_size=640, num_attention_heads=2, num_hidden_layers=1, image_size=224,
               patch_size=14, projection_dim=64, layer_norm_eps=1e-5, hidden_act="gelu")
    enc = CLIPVisionModelWithProjection(cfg, "cpu")
    c0 = enc.capture_version
    enc.load_state_dict(CO.random_state_dict(cfg, 0))
    assert enc.capture_version == c0 + 1

    ucfg = UNetConfig(block_out_channels=(32, 64, 128, 128), cross_attention_dim=16, ip_image_embed_dim=16, sample_size=8)
    unet = MVUNetMotionModel(ucfg, device="cpu")
    u0 = unet.capture_version
    unet.load_state_dict({k: torch.zeros(s) for k, s in list(key_plan(ucfg).items())[:4]}, strict=False)
    assert unet.capture_version == u0 + 1
    unet.to("cpu")                                     # no move: nothing changes
    assert unet.capture_version == u0 + 1
