"""Sampler options without a GPU: the eta step oracle, the scheduler's step coefficients, the truncated schedule of
`i2v_similarity_init` and its initial latents (animate3d_b200/scheduler.py, pipeline.py) against tests/sampler_oracle.py."""
import math

import numpy as np
import pytest
import torch

from sampler_oracle import DDIMEtaOracle, similarity_init


def _inputs(seed=0, shape=(2, 4, 5, 6, 6)):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g), torch.randn(shape, generator=g), torch.randn(shape, generator=g)


def test_eta_oracle_at_eta_zero_is_the_deterministic_step():
    from oracle.scheduler_oracle import DDIMOracle
    o, e = DDIMOracle(), DDIMEtaOracle()
    x, eps, z = _inputs()
    for n in (25, 7):
        o.set_timesteps(n)
        e.set_timesteps(n)
        for t in e.timesteps.tolist():
            want, want_x0 = o.step(eps, t, x)
            got, got_x0 = e.step(eps, t, x)
            assert torch.equal(got, want) and torch.equal(got_x0, want_x0), t
            assert torch.equal(e.step(eps, t, x, 0.0, z)[0], want), t        # eta 0 never reads the noise


def test_step_coefficients_follow_the_eta_formula():
    """std_dev = eta sqrt((1 - a_p)/(1 - a_t) (1 - a_t/a_p)) and dir_coef = sqrt(1 - a_p - std_dev^2), fp32; at eta 0 they
    are exactly what a3d_ddim_cfg_step uses (std_dev 0, sqrtf(1 - a_prev))."""
    from animate3d_b200.scheduler import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(25)
    for t in s.timesteps.tolist():
        a_t, a_p = s.alphas_for(t)
        for eta in (0.0, 0.5, 1.0):
            ct, cp, dc, sd = s.step_coefficients(t, eta)
            assert (ct, cp) == (a_t, a_p)
            var = (1 - a_p) / (1 - a_t) * (1 - a_t / a_p)
            assert sd == pytest.approx(eta * math.sqrt(var), rel=1e-6, abs=1e-7)
            assert dc == pytest.approx(math.sqrt(max(1 - a_p - sd * sd, 0.0)), rel=1e-6, abs=1e-7)
            if eta == 0:
                assert sd == 0.0 and dc == float(np.sqrt(np.float32(1) - np.float32(a_p)))


def test_engine_step_arithmetic_matches_eta_oracle():
    """x' = sqrt(a_p) x0 + dir_coef eps + std_dev z with the scheduler's coefficients is the oracle's eta step."""
    from animate3d_b200.scheduler import DDIMScheduler
    s, o = DDIMScheduler(), DDIMEtaOracle()
    s.set_timesteps(25)
    o.set_timesteps(25)
    x, eps, z = _inputs(1)
    for t in (961, 481, 41, 1):
        for eta in (0.5, 1.0):
            a_t, a_p, dc, sd = s.step_coefficients(t, eta)
            x0 = (x.double() - math.sqrt(1 - a_t) * eps.double()) / math.sqrt(a_t)
            mine = math.sqrt(a_p) * x0 + dc * eps.double() + sd * z.double()
            want, _ = o.step(eps, t, x, eta, z)
            torch.testing.assert_close(mine.float(), want, rtol=1e-5, atol=1e-5)


def test_last_step_has_no_variance():
    """prev_t < 0 takes alpha_prev = 1 (set_alpha_to_one), so the variance and std_dev are 0 whatever eta."""
    from animate3d_b200.scheduler import DDIMScheduler
    s, o = DDIMScheduler(), DDIMEtaOracle()
    s.set_timesteps(25)
    o.set_timesteps(25)
    t = int(s.timesteps[-1])
    assert t - 1000 // 25 < 0
    for eta in (0.5, 1.0):
        _, a_p, dc, sd = s.step_coefficients(t, eta)
        assert a_p == 1.0 and sd == 0.0 and dc == 0.0
    x, eps, z = _inputs(2)
    assert torch.equal(o.step(eps, t, x, 1.0, z)[0], o.step(eps, t, x, 0.0)[0])


def test_get_timesteps_truncates_and_keeps_the_stride():
    from animate3d_b200.scheduler import DDIMScheduler
    s, o = DDIMScheduler(), DDIMEtaOracle()
    ts = s.get_timesteps(25, 0.5)
    assert ts.tolist() == o.get_timesteps(25, 0.5).tolist()
    assert len(ts) == 12 and ts[0] == 441 and ts[-1] == 1
    assert s.timesteps.tolist() == o.set_timesteps(25).tolist()      # the scheduler still holds the 25-step schedule
    for t in ts.tolist():
        a_t, a_p = s.alphas_for(t)
        assert a_p == (float(s.alphas_cumprod[t - 40]) if t >= 40 else 1.0)
    assert s.get_timesteps(10, 1.0).tolist() == s.set_timesteps(10).tolist()
    assert len(s.get_timesteps(10, 0.0)) == 0


def test_add_noise_matches_oracle():
    from animate3d_b200.scheduler import DDIMScheduler
    s, o = DDIMScheduler(), DDIMEtaOracle()
    o.alphas_cumprod = torch.from_numpy(s.alphas_cumprod.copy())    # constants are checked in test_host_logic
    x, n, _ = _inputs(3)
    t = torch.tensor([441, 801])
    assert torch.equal(s.add_noise(x, n, t), o.add_noise(x, n, t))
    assert torch.equal(s.add_noise(x, n, 441), o.add_noise(x, n, 441))


def test_similarity_init_matches_reference_restatement():
    """pipeline.similarity_init_latents draws the mask, then the noise, then blends, exactly as pipeline.py:707-724: the same
    seeded generator gives the same latents bit for bit (the oracle scheduler takes the engine's alphas so that only the
    draws and the blend are compared), and the generator is left at the same point of its stream."""
    from animate3d_b200.pipeline import similarity_init_latents
    from animate3d_b200.scheduler import DDIMScheduler
    s, o = DDIMScheduler(), DDIMEtaOracle()
    o.alphas_cumprod = torch.from_numpy(s.alphas_cumprod.copy())
    first = torch.randn(2, 4, 1, 6, 6, generator=torch.Generator().manual_seed(4))
    t0 = int(s.get_timesteps(25, 0.5)[0])
    for p in (0.0, 0.3, 1.0):
        g1, g2 = torch.Generator().manual_seed(11), torch.Generator().manual_seed(11)
        got = similarity_init_latents(first, 7, t0, p, s, g1)
        want = similarity_init(first, 7, torch.full((2,), t0), p, o, g2)
        assert got.shape == (2, 4, 7, 6, 6)
        assert torch.equal(got, want), p
        assert torch.equal(torch.randn(3, generator=g1), torch.randn(3, generator=g2))
    kept = similarity_init_latents(first, 7, t0, 1.0, s, torch.Generator().manual_seed(1))
    assert torch.equal(kept, first.expand(-1, -1, 7, -1, -1))        # origin_prob 1: every pixel is the first frame


def test_similarity_init_with_freeinit_is_rejected():
    """The reference reads an undefined `strength` there (NameError, pipeline.py:997): the engine refuses the pair."""
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    pipe = AnimateDiffMVI2VPipeline.__new__(AnimateDiffMVI2VPipeline)     # host logic only: no UNet, no device
    pipe.free_init_enabled = False
    pipe.enable_free_init(num_iters=2)
    with pytest.raises(ValueError, match="FreeInit"):
        pipe(i2v_similarity_init={"strength": 0.5, "origin_prob": 0.3}, output_type="latent")
