"""Pin the oracle (oracle/unet_oracle.py) against golden vectors produced by the reference's OWN source
(tests/golden/gen_reference_goldens.py: attention_processor.py, embeddings.py and pipeline.py camera helpers run with
diffusers/xformers stubbed).  CPU-only."""
import os

import pytest
import torch

from oracle import unet_oracle as O


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name), weights_only=False)


def _processor_cases(golden_dir):
    """The processor fixtures are stored one file per channel width (64 / 80 / 96) to keep each file small."""
    return [cs for c in (64, 80, 96) for cs in _load(golden_dir, f"ref_processors_c{c}.pt")]


def test_processors_match_reference_source(golden_dir):
    cases = _processor_cases(golden_dir)
    assert len(cases) == 12
    for cs in cases:
        kind, w = cs["kind"], cs["w"]
        if kind == "mv_i2v":
            y = O.proc_mv_i2v(w, "a.attn1", cs["x"], cs["heads"], cs["nv"], cs["nf"])
        elif kind == "mv":
            w0 = dict(w)
            w0["a.attn1.processor.to_out_i2v.weight"] = torch.zeros_like(w["a.attn1.processor.to_out_i2v.weight"])
            w0["a.attn1.processor.to_out_i2v.bias"] = torch.zeros_like(w["a.attn1.processor.to_out_i2v.bias"])
            y = O.proc_mv_i2v(w0, "a.attn1", cs["x"], cs["heads"], cs["nv"], cs["nf"])
        elif kind == "ip":
            y = O.proc_ip_adapter(w, "a.attn2", cs["x"], cs["text"], cs["ip"], cs["heads"], cs["ip_scale"])
        else:
            y = O.proc_spatiotemporal(w, "m.attn1", cs["x"], cs["heads"], cs["nv"], cs["nf"], cs["fs"])
        torch.testing.assert_close(y, cs["y"], rtol=2e-5, atol=2e-5, msg=lambda m: f"{kind} c={cs['c']}: {m}")


def test_spatiotemporal_state_keys_match_reference(golden_dir):
    """The processor's own parameter/buffer names are part of the checkpoint contract (SURVEY Appendix B.12)."""
    cases = [c for c in _processor_cases(golden_dir) if c["kind"] == "st"]
    want = {"to_q_sp.weight", "to_k_sp.weight", "to_v_sp.weight", "to_out_sp.weight", "to_out_sp.bias",
            "time_pos_embed.pe", "alpha_blender.mix_factor"}
    for cs in cases:
        assert set(cs["state_keys"]) == want
    plan = O.key_plan(O.UNetConfig())
    p = "down_blocks.0.motion_modules.0.transformer_blocks.0.attn1.processor."
    assert {k[len(p):] for k in plan if k.startswith(p)} == want


def test_sine_pos_enc_matches_reference(golden_dir):
    """The fixture holds the reference's full shape and a fixed, seeded sample of at most 8192 entries per encoding."""
    emb = _load(golden_dir, "ref_embeddings.pt")
    for (nfeat, h, w), ref in emb.items():
        ours = O.sine_pos_enc_2d(nfeat, h, w)
        assert tuple(ours.shape) == tuple(ref["shape"])
        torch.testing.assert_close(ours.reshape(-1)[ref["idx"].long()], ref["val"], rtol=1e-6, atol=1e-6)


def test_camera_matches_reference(golden_dir):
    cam = _load(golden_dir, "ref_camera.pt")
    for n, ref in cam.items():
        torch.testing.assert_close(O.get_camera(n), ref, rtol=1e-6, atol=1e-6)


def test_time_pos_embed_matches_reference_buffer(golden_dir):
    cs = [c for c in _processor_cases(golden_dir) if c["kind"] == "st"][0]
    pe = cs["w"]["m.attn1.processor.time_pos_embed.pe"]
    torch.testing.assert_close(O.sinusoidal_pe(pe.shape[2], pe.shape[1]), pe, rtol=1e-6, atol=1e-6)
