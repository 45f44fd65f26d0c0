"""FreeInit's filters and coarse-to-fine sampling, and per-view generator lists, without a GPU: the engine's filters
against diffusers' triple loop, the step count of every FreeInit iteration, `randn_tensor` against diffusers', and the
pipeline's sampling loop (float64 stand-ins for the step kernels, a cheap stand-in UNet) against the reference loop of
tests/freeinit_oracle.py for DDIM, DPM-Solver++, Euler-ancestral, PNDM with PRK and LMS, with negative controls that the
same comparators must reject."""
import math
from types import SimpleNamespace

import pytest
import torch

import freeinit_oracle as FO
from freeinit_oracle import free_init_freq_filter, free_init_num_steps, randn_tensor
import multistep_oracle as MO
import sampler_oracle as SO
import solver_oracle as SV

EPS32 = torch.finfo(torch.float32).eps


# ------------------------------------------------------------------------------------------------ filters
FILTER_SHAPES = [(15, 32, 32), (3, 8, 8), (5, 7, 9)]
STOPS = [(0.25, 0.25), (0.4, 0.2), (0.0, 0.25), (0.25, 0.0)]


def _engine_filter(shape, method, order, ds, dt):
    from animate3d_b200.pipeline import free_init_filter
    return free_init_filter((2, 4) + shape, method, order, ds, dt)


@pytest.mark.parametrize("shape", FILTER_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("stops", STOPS, ids=lambda s: f"ds{s[0]}-dt{s[1]}")
@pytest.mark.parametrize("method", ["gaussian", "ideal"])
def test_gaussian_and_ideal_filters_are_diffusers_bit_for_bit(shape, stops, method):
    got = _engine_filter(shape, method, 4, *stops)
    want = free_init_freq_filter((1, 4) + shape, method, 4, *stops)
    assert got.dtype == torch.float32 and got.shape == shape
    assert torch.equal(got.expand(want.shape), want)
    if 0.0 in stops:
        assert not got.any()


@pytest.mark.parametrize("shape", FILTER_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("stops", STOPS, ids=lambda s: f"ds{s[0]}-dt{s[1]}")
@pytest.mark.parametrize("order", [1, 4, 8])
def test_butterworth_filter_within_float32_rounding(shape, stops, order):
    """The butterworth filter keeps its float32 arithmetic: d² carries a few ulps of relative rounding, which the power
    multiplies by `order`, so it stays within (order + 2) float32 epsilons of diffusers' float64 entries."""
    got = _engine_filter(shape, "butterworth", order, *stops)
    want = free_init_freq_filter((1, 4) + shape, "butterworth", order, *stops)[0, 0]
    err = (got.double() - want.double()).abs().max().item()
    assert err <= (order + 2) * EPS32, err
    if 0.0 in stops:
        assert not got.any()


def test_ideal_filter_compares_with_twice_the_stop_frequency():
    """At d_s = d_t = 0.5 on (2, 4, 4) the squared distances take the values 0, 0.25, ..., 3 and several equal 2 d_s = 1
    exactly: those are inside.  The same filter against d_s (0.5) -- a tempting "fix" -- is rejected."""
    shape = (2, 4, 4)
    want = free_init_freq_filter((1, 1) + shape, "ideal", 4, 0.5, 0.5)[0, 0]
    got = _engine_filter(shape, "ideal", 4, 0.5, 0.5)
    assert torch.equal(got, want)
    t = torch.arange(2.0)[:, None, None]
    h = torch.arange(4.0)[None, :, None]
    w = torch.arange(4.0)[None, None, :]
    d2 = (2 * t / 2 - 1) ** 2 + (2 * h / 4 - 1) ** 2 + (2 * w / 4 - 1) ** 2
    assert (d2 == 1.0).any() and got[d2 == 1.0].eq(1).all() and got[d2 > 1.0].eq(0).all() and (d2 > 1.0).any()
    against_ds = (d2 <= 0.5).float()                                                  # negative control
    assert not torch.equal(against_ds, want)


def test_filter_rejects_unknown_method():
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline, free_init_filter
    with pytest.raises(NotImplementedError, match="gaussian, butterworth or ideal"):
        free_init_filter((3, 8, 8), "box")
    with pytest.raises(NotImplementedError, match="gaussian, butterworth or ideal"):
        free_init_freq_filter((1, 1, 3, 8, 8), "box")
    pipe = AnimateDiffMVI2VPipeline.__new__(AnimateDiffMVI2VPipeline)
    with pytest.raises(NotImplementedError, match="gaussian, butterworth or ideal"):
        pipe.enable_free_init(method="box")


def test_enable_free_init_stores_every_argument():
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    pipe = AnimateDiffMVI2VPipeline.__new__(AnimateDiffMVI2VPipeline)
    assert (pipe._free_init_method, pipe._free_init_use_fast_sampling) == ("butterworth", False)
    pipe.enable_free_init(num_iters=5, use_fast_sampling=True, method="gaussian", order=2, spatial_stop_frequency=0.3,
                          temporal_stop_frequency=0.1)
    assert pipe.free_init_enabled and pipe._free_init_num_iters == 5
    assert (pipe._free_init_method, pipe._free_init_use_fast_sampling, pipe._fi) == ("gaussian", True, (2, 0.3, 0.1))
    pipe.disable_free_init()
    assert not pipe.free_init_enabled


# ------------------------------------------------------------------------------------------------ coarse-to-fine counts
def _engine_steps(n, iters, fast):
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    pipe = AnimateDiffMVI2VPipeline.__new__(AnimateDiffMVI2VPipeline)
    pipe.enable_free_init(num_iters=iters, use_fast_sampling=fast)
    return [pipe._free_init_steps(it, n) for it in range(iters)]


def test_fast_sampling_counts_pinned():
    assert _engine_steps(25, 3, True) == [8, 16, 25]
    assert _engine_steps(50, 3, True) == [16, 33, 50]
    assert _engine_steps(25, 3, False) == [25, 25, 25]
    assert sum(_engine_steps(25, 3, True)) == 49


@pytest.mark.parametrize("n", [1, 2, 4, 10, 25, 50])
@pytest.mark.parametrize("iters", [1, 2, 3, 5])
def test_fast_sampling_schedule_of_every_iteration(n, iters):
    """Each iteration's schedule, as `_apply_free_init` leaves it, is a fresh set_timesteps of diffusers' count, and the
    scheduler's step arithmetic (alphas_for, the stride) follows that count."""
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    from animate3d_b200.scheduler import DDIMScheduler
    pipe = AnimateDiffMVI2VPipeline.__new__(AnimateDiffMVI2VPipeline)
    pipe.scheduler = DDIMScheduler()
    pipe.enable_free_init(num_iters=iters, use_fast_sampling=True)
    x = torch.randn(2, 4, 3, 4, 4, generator=torch.Generator().manual_seed(n))
    assert _engine_steps(n, iters, True) == [free_init_num_steps(n, iters, it, True) for it in range(iters)]
    for it in range(iters):
        k = free_init_num_steps(n, iters, it, True)
        x, ts = pipe._apply_free_init(x, it, n, torch.Generator().manual_seed(it))
        fresh = DDIMScheduler()
        assert ts.tolist() == fresh.set_timesteps(k).tolist() and len(ts) == k
        assert pipe.scheduler.num_inference_steps == k
        assert [pipe.scheduler.alphas_for(int(t)) for t in ts] == [fresh.alphas_for(int(t)) for t in ts]


# ------------------------------------------------------------------------------------------------ randn_tensor
def _gens(seeds):
    return [torch.Generator().manual_seed(s) for s in seeds]


@pytest.mark.parametrize("case", ["none", "one", "list of one", "list"])
def test_randn_tensor_matches_diffusers(case):
    from animate3d_b200.pipeline import randn_tensor as engine_randn
    shape = (4, 3, 5, 6, 6)
    make = {"none": lambda: None, "one": lambda: torch.Generator().manual_seed(5),
            "list of one": lambda: _gens([5]), "list": lambda: _gens([3, 1, 4, 1])}[case]
    if case == "none":
        torch.manual_seed(9)
        got = engine_randn(shape, None, "cpu")
        torch.manual_seed(9)
        want = randn_tensor(shape, None, torch.device("cpu"), torch.float32)
    else:
        got = engine_randn(shape, make(), torch.device("cpu"))
        want = randn_tensor(shape, make(), torch.device("cpu"), torch.float32)
    assert torch.equal(got, want) and got.dtype == torch.float32
    if case == "list":
        for i, s in enumerate([3, 1, 4, 1]):                        # item i is generator i's first draw of one item
            assert torch.equal(got[i:i + 1], torch.randn((1,) + shape[1:], generator=torch.Generator().manual_seed(s)))
        assert torch.equal(got[1], got[3]) and not torch.equal(got[0], got[1])


def test_randn_tensor_list_draws_each_view_from_its_generator():
    """A list is not one batch from its first generator (negative control)."""
    from animate3d_b200.pipeline import randn_tensor as engine_randn
    shape = (2, 4, 3, 4, 4)
    got = engine_randn(shape, _gens([7, 8]), "cpu")
    one_batch = torch.randn(shape, generator=torch.Generator().manual_seed(7))
    assert torch.equal(got[0], one_batch[0]) and not torch.equal(got, one_batch)


def test_list_length_must_be_the_view_count(monkeypatch):
    with pytest.raises(ValueError, match="one generator per view"):
        _run_pipeline(monkeypatch, _sched("DDIMScheduler"), 4, gens=3)
    with pytest.raises(ValueError, match="one generator per view"):
        _run_pipeline(monkeypatch, _sched("DDIMScheduler"), 4, gens=1)
    with pytest.raises(IndexError):                                  # diffusers indexes past a short list
        randn_tensor((3, 2), _gens([1, 2]), torch.device("cpu"))


def test_similarity_init_rejects_a_generator_list():
    from animate3d_b200.pipeline import similarity_init_latents
    from animate3d_b200.scheduler import DDIMScheduler
    first = torch.randn(2, 4, 1, 4, 4)
    with pytest.raises(ValueError, match="single torch.Generator"):
        similarity_init_latents(first, 3, 961, 0.3, DDIMScheduler(), _gens([1, 2]))


# ------------------------------------------------------------------------------------------------ the sampling loop
NV, NF, H = 2, 4, 4


def _model(x, t, *rest):
    """Stand-in UNet: elementwise in x, depends on t and on the batch half (so CFG and the input scaling matter)."""
    b = torch.arange(x.shape[0], dtype=x.dtype).view(-1, 1, 1, 1, 1)
    return torch.tanh(0.7 * x + float(t) / 700.0) + 0.05 * b - 0.2 * x


class _UNet:
    config = SimpleNamespace(in_channels=4)

    def __init__(self):
        self.calls = 0

    def __call__(self, x, t, pe, camera=None, added_cond_kwargs=None, num_views=4, i2v_cond_time_zero=False):
        self.calls += 1
        return SimpleNamespace(sample=_model(x, t))


def _write(buf, ref):
    buf.view(-1).copy_(torch.where(torch.isinf(ref.bound), buf.view(-1).double(), ref.value).float())


def _ddim_cfg_step(lat, eps, first, bn, c, f, hw, guidance, a_t, a_p, uncond_first=True):
    _write(lat, SO.ddim_step(lat.clone(), eps, first, None, bn, c, f, hw, 1 if uncond_first else 2, guidance, a_t, a_p,
                             math.sqrt(1 - a_p), 0.0))
    return lat


def _ddim_step(lat, eps, first, z, bn, c, f, hw, cfg_mode, guidance, a_t, a_p, dir_coef, std_dev):
    _write(lat, SO.ddim_step(lat.clone(), eps, first, z if std_dev else None, bn, c, f, hw, cfg_mode, guidance, a_t, a_p,
                             dir_coef, std_dev))
    return lat


def _sampler_step(lat, eps, first, bn, c, f, hw, cfg_mode, guidance, step, noise=None, history_out=None, history_in=None):
    ref, m0 = SV.sampler_step(lat.clone(), eps, first, noise, history_out, history_in, bn, c, f, hw, cfg_mode, guidance, step)
    if m0 is not None:
        _write(history_out, m0)
    _write(lat, ref)
    return lat


def _multistep_step(lat, eps, first, bn, c, f, hw, cfg_mode, guidance, step, ring, sample=None, accum=None):
    out_buf = ring[step.out_slot] if step.out_slot is not None else None
    refs = MO.multistep_step(lat.clone(), eps, first, out_buf, [ring[s] for s in step.in_slots], sample, accum, bn, c, f, hw,
                             cfg_mode, guidance, step)
    for key, buf in (("history_out", out_buf), ("sample", sample), ("accum", accum), ("latents", lat)):
        if key in refs:
            _write(buf, refs[key])
    return lat


def _sched(name, **kw):
    from animate3d_b200 import scheduler as S
    return getattr(S, name)(**kw)


def _run_pipeline(monkeypatch, sched, steps, free_init=None, eta=0.0, gens=None, kernels=None):
    """The engine's `__call__` on the CPU with the stand-ins (or `kernels`, by ops name); `gens` is None (one generator)
    or the length of a list of per-view generators.  Returns the latents, the generator(s), a copy at the same stream
    point, the conditioning and the UNet-call count."""
    from animate3d_b200 import ops
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    stand_ins = dict(ddim_cfg_step=_ddim_cfg_step, ddim_step=_ddim_step, sampler_step=_sampler_step,
                     multistep_step=_multistep_step)
    for name, fn in dict(stand_ins, **(kernels or {})).items():
        monkeypatch.setattr(ops, name, fn)
    pipe = AnimateDiffMVI2VPipeline.__new__(AnimateDiffMVI2VPipeline)
    pipe.unet, pipe.scheduler, pipe.device = _UNet(), sched, torch.device("cpu")
    pipe.free_init_enabled, pipe._free_init_num_iters = False, 1
    if free_init is not None:
        pipe.enable_free_init(**free_init)
    g = torch.Generator().manual_seed(77) if gens is None else _gens(range(70, 70 + gens))
    g_ref = [torch.Generator() for _ in (g if gens is not None else [g])]
    for a, b in zip(g_ref, g if gens is not None else [g]):
        a.set_state(b.get_state())
    g_ref = g_ref if gens is not None else g_ref[0]
    gc = torch.Generator().manual_seed(3)
    first = torch.randn(NV, 4, 1, H, H, generator=gc)
    cond = torch.randn(NV, 77, 768, generator=gc), torch.randn(NV, 77, 768, generator=gc), torch.randn(NV, 1024, generator=gc)
    out = pipe(num_frames=NF, height=8 * H, width=8 * H, num_inference_steps=steps, guidance_scale=7.5,
               num_videos_per_prompt=NV, eta=eta, generator=g, prompt_embeds=cond[0], negative_prompt_embeds=cond[1],
               ip_adapter_image_embeds=cond[2], output_type="latent", first_frame_latents=first).frames
    return out, first, g, g_ref, cond, pipe.unet.calls


ORACLES = {"DDIMScheduler": FO.DDIMLoop, "DPMSolverMultistepScheduler": SV.DPMSolverOracle,
           "EulerAncestralDiscreteScheduler": FO.EulerAncestralLists, "PNDMScheduler": MO.PNDMOracle,
           "LMSDiscreteScheduler": MO.LMSOracle}


def _compare(monkeypatch, name, kw, steps, free_init=None, eta=0.0, gens=None):
    """(ok, rel-L2, UNet calls of the engine, of the reference loop) for one configuration."""
    sched = _sched(name, **kw)
    got, first, g, g_ref, (pos, neg, img), calls = _run_pipeline(monkeypatch, sched, steps, free_init, eta, gens)
    oracle = ORACLES[name](eta=eta, **kw) if name == "DDIMScheduler" else ORACLES[name](**kw)
    want, want_calls = FO.sampler(first, pos, neg, img, NF, steps, 7.5, oracle, g_ref, _model, free_init)
    rel = ((got - want).norm() / want.norm()).item()
    pairs = zip(g, g_ref) if gens is not None else [(g, g_ref)]
    same_stream = all(torch.equal(torch.randn(4, generator=a), torch.randn(4, generator=b)) for a, b in pairs)
    ok = rel < 1e-5 and torch.equal(got[:, :, :1], first) and same_stream and calls == want_calls
    return ok, rel, calls, want_calls, same_stream


SCHEDULERS = [
    ("DDIMScheduler", {}, 10),
    ("DPMSolverMultistepScheduler", {}, 10),
    ("EulerAncestralDiscreteScheduler", dict(timestep_spacing="linspace"), 10),
    ("PNDMScheduler", dict(steps_offset=1), 12),
    ("LMSDiscreteScheduler", {}, 10),
]
FREE_INIT = [dict(method=m, use_fast_sampling=f) for m in ("butterworth", "gaussian", "ideal") for f in (False, True)]


@pytest.mark.parametrize("fi", FREE_INIT, ids=lambda f: f"{f['method']}-{'fast' if f['use_fast_sampling'] else 'full'}")
@pytest.mark.parametrize("case", SCHEDULERS, ids=lambda c: c[0])
def test_pipeline_loop_matches_reference_loop(monkeypatch, case, fi):
    name, kw, steps = case
    ok, rel, calls, want_calls, same = _compare(monkeypatch, name, kw, steps, dict(fi, num_iters=3))
    assert ok, (rel, calls, want_calls, same)
    extra = 9 if name == "PNDMScheduler" else 0                      # PRK: n + 9 UNet calls for n steps
    counts = [free_init_num_steps(steps, 3, it, fi["use_fast_sampling"]) for it in range(3)]
    assert calls == sum(k + extra for k in counts), calls


def test_non_default_filter_options(monkeypatch):
    fi = dict(num_iters=2, method="gaussian", order=2, spatial_stop_frequency=0.4, temporal_stop_frequency=0.2,
              use_fast_sampling=True)
    ok, rel, calls, _, _ = _compare(monkeypatch, "DDIMScheduler", {}, 10, fi)
    assert ok and calls == 5 + 10, (rel, calls)


def test_pndm_prk_needs_four_steps_in_every_iteration(monkeypatch):
    """10 steps over 3 coarse-to-fine iterations start with 3: too few for the PRK steps."""
    with pytest.raises(ValueError, match="skip_prk_steps"):
        _run_pipeline(monkeypatch, _sched("PNDMScheduler"), 10, dict(num_iters=3, use_fast_sampling=True))


@pytest.mark.parametrize("case", [("DDIMScheduler", 0.5), ("EulerAncestralDiscreteScheduler", 0.0)], ids=lambda c: c[0])
@pytest.mark.parametrize("free_init", [None, dict(num_iters=2, method="gaussian", use_fast_sampling=True)],
                         ids=["plain", "freeinit"])
def test_generator_list_matches_reference_loop(monkeypatch, case, free_init):
    """One CPU generator per view: the initial noise, FreeInit's z_rand and every per-step draw come view by view."""
    name, eta = case
    kw = dict(timestep_spacing="linspace") if name != "DDIMScheduler" else {}
    ok, rel, calls, want_calls, same = _compare(monkeypatch, name, kw, 10, free_init, eta=eta, gens=NV)
    assert ok, (rel, calls, want_calls, same)


def test_single_generator_freeinit_on_ddim(monkeypatch):
    """A CPU generator with FreeInit on the DDIM path (z_rand drawn on the generator's device)."""
    ok, rel, _, _, _ = _compare(monkeypatch, "DDIMScheduler", {}, 10, dict(num_iters=3), eta=0.5)
    assert ok, rel


# ------------------------------------------------------------------------------------------------ negative controls
def _keep_history(monkeypatch, cls_name):
    """set_timesteps that keeps the past model outputs of the previous schedule.  (PLMS is where stale entries change
    the result: DPM-Solver++'s first step has no earlier sigma, so its second-order term vanishes, and LMS pairs only as
    many entries as the schedule has written.)"""
    from animate3d_b200 import scheduler as S
    cls = getattr(S, cls_name)
    orig = cls.set_timesteps

    def kept(self, n, device=None):
        saved = {k: getattr(self, k) for k in ("lower_order_nums", "_slots", "_pushed", "_ring") if hasattr(self, k)}
        out = orig(self, n, device)
        if self.__dict__.get("_started"):
            for k, v in saved.items():
                setattr(self, k, v)
        self._started = True
        return out
    monkeypatch.setattr(cls, "set_timesteps", kept)


@pytest.mark.parametrize("control", ["fast sampling not on iteration 0", "PLMS history kept across iterations",
                                     "list drawn as one batch"])
def test_negative_controls_are_rejected(monkeypatch, control):
    from animate3d_b200 import pipeline as P
    fi, name, kw, eta, gens = dict(num_iters=3, use_fast_sampling=True), "DDIMScheduler", {}, 0.0, None
    if control == "fast sampling not on iteration 0":
        orig = P.AnimateDiffMVI2VPipeline._free_init_steps
        monkeypatch.setattr(P.AnimateDiffMVI2VPipeline, "_free_init_steps",
                            lambda self, it, n: n if it == 0 else orig(self, it, n))
    elif control == "PLMS history kept across iterations":
        name, kw = "PNDMScheduler", dict(skip_prk_steps=True, steps_offset=1)
        _keep_history(monkeypatch, name)
    else:
        real = P.randn_tensor
        monkeypatch.setattr(P, "randn_tensor", lambda shape, generator, device: real(
            shape, generator[0] if isinstance(generator, list) else generator, device))
        fi, eta, gens = dict(num_iters=2), 0.5, NV
    ok, rel, calls, want_calls, same = _compare(monkeypatch, name, kw, 10, fi, eta=eta, gens=gens)
    assert not ok, (control, rel, calls, want_calls, same)
    print(f"{control}: rel-L2 {rel:.2e}, UNet calls {calls} vs {want_calls}, same stream {same}")


def test_history_buffers_are_written_before_read(monkeypatch):
    """With coarse-to-fine FreeInit, every a3d_sampler_step m1 read and every a3d_multistep_step ring, sample and
    accumulator read in an iteration comes after a write of that buffer in the same iteration (the buffers are allocated
    once per call)."""
    from animate3d_b200 import ops
    log = []

    def dpm(lat, eps, first, bn, c, f, hw, cfg_mode, guidance, step, noise=None, history_out=None, history_in=None):
        log.append(("r", id(history_in)) if history_in is not None else ("-",))
        log.append(("w", id(history_out)))
        return _sampler_step(lat, eps, first, bn, c, f, hw, cfg_mode, guidance, step, noise, history_out, history_in)

    def multi(lat, eps, first, bn, c, f, hw, cfg_mode, guidance, step, ring, sample=None, accum=None):
        log.extend(("r", id(ring[s])) for s in step.in_slots)
        if step.from_sample:
            log.append(("r", id(sample)))
        if step.prk in (2, 3):
            log.append(("r", id(accum)))
        if step.out_slot is not None:
            log.append(("w", id(ring[step.out_slot])))
        if step.save_sample:
            log.append(("w", id(sample)))
        if step.prk in (1, 2):
            log.append(("w", id(accum)))
        return _multistep_step(lat, eps, first, bn, c, f, hw, cfg_mode, guidance, step, ring, sample, accum)

    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline
    orig = AnimateDiffMVI2VPipeline._apply_free_init

    def marked(self, *a, **k):
        log.append(("iteration",))
        return orig(self, *a, **k)
    monkeypatch.setattr(AnimateDiffMVI2VPipeline, "_apply_free_init", marked)
    for name, kw, steps in SCHEDULERS[1:]:
        log.clear()
        _run_pipeline(monkeypatch, _sched(name, **kw), steps, dict(num_iters=3, use_fast_sampling=True),
                      kernels=dict(sampler_step=dpm, multistep_step=multi))
        written, reads = set(), 0
        assert log.count(("iteration",)) == 3, name
        for entry in log:
            if entry[0] == "iteration":
                written = set()
            elif entry[0] == "w":
                written.add(entry[1])
            elif entry[0] == "r":
                assert entry[1] in written, (name, entry)
                reads += 1
        assert reads > 0 or name == "EulerAncestralDiscreteScheduler", name
