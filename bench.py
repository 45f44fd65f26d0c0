#!/usr/bin/env python
"""bench.py -- MV-VDM denoise-steps/s at 4 views x 16 frames x 256^2 (BASELINE.json metric) on N H100s of one node.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl native|reference] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

A "step" = one denoise step of the reference sampler (animatediff/pipelines/pipeline.py:1006-1031): classifier-free-guided
UNet evaluation on 2 x 4 views x 16 frames = 128 latent images of 4x32x32, CFG combine, DDIM update, frame-0 re-injection.
Weights are seeded random of the released SD1.5 + motion-module geometry, inputs synthetic (no network).
N > 1: every rank denoises its own prompt (the (prompt x view-group) batch is partitioned, no data-path collective) ->
"scaling": "weak"; value = N * steps / max-over-ranks device time.

JSON line keys beyond the base contract:
  roofline     the fused cross-view attention kernel at level 0 (L = 4 views * 32*32 = 4096 tokens, head_dim 40, 8 heads,
               2*16 (CFG x frame) batches) timed alone with CUDA events; achieved = 4*L^2*C*batches FLOP / duration against
               the fp16 tensor peak (MEASURED_PEAKS.json when present, else the H100 SXM data sheet's dense figure)
  cpu_baseline the oracle port (oracle/unet_oracle.py) on the host cores for a bounded sample, extrapolated by FLOPs
  e2e          the same step through pipeline.denoise_step_host with pinned HOST buffers (H2D of the step inputs + D2H of
               the updated latents inside the timed region)
  roofline_gemm  the worst short-K projection (HBM-bound: bytes / time against the measured copy bandwidth) and the best long-K
               implicit-GEMM convolution (tensor-bound) of the step, timed alone
  splat        the second half of the BASELINE metric: Mpix/s of the batched 4D-gaussian renderer at BASELINE configs[2]
               (50k gaussians, 4 views x 16 timestamps = 64 cameras at 512^2), forward and forward+backward, with per-stage
               times from CUDA events inside liba3d.so and the stage rooflines of SURVEY 8(d); for N > 1 the cameras are
               sharded r::N and the deformation-field gradients all-reduced (one flat bucket)
  sds_step     (N = 1) one whole 4D-SDS refine step of BASELINE configs[2] on the engine: render -> VAE encoder (with grad) -> CFG
               UNet -> loss -> backward to the deformation field
  view_sharded (N > 1) ONE prompt spread over the N ranks -- CFG branches over 2 ranks and / or the 4 views over 4 ranks with
               the cross-view K|V all-gather over NCCL -- as a strong-scaling number next to the weak-scaling `value`, with the
               exposed communication time (same forward with the collectives skipped)
--dump-outputs DIR (native) writes the latents the last timed step returned as DIR/latents.npy (float32); the inputs are seeded,
so two builds run with the same arguments can be compared output for output.
--impl reference times the oracle port (the reference's diffusers CPU path is not installable here: SURVEY section 8c) on a
BOUNDED sample per step (one forward of 4 views x 1 frame: the real L = 4096 cross-view attention shape); `ms_per_step` is the
measured time of that sample, `value` the steps/s extrapolated by FLOPs -- flagged `extrapolated` / `same_config: false`.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "MV-VDM denoise-steps/sec @ 4view x 16frame x 256^2"
UNIT = "denoise-steps/s"
NV, NF, LAT = 4, 16, 32
STEP_TFLOP = None  # filled from animate3d_b200.flops


def step_flops():
    from animate3d_b200.flops import unet_forward_flops
    from animate3d_b200.unet_config import UNetConfig
    return unet_forward_flops(UNetConfig(), 2, NV, NF)["total"]


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d.get("bf16_tflops", 989.0), d.get("hbm_gbs", 3350.0), "measured (MEASURED_PEAKS.json, burst)"
    # NVIDIA H100 SXM data sheet: 989 TFLOP/s dense fp16 / bf16, 3.35 TB/s HBM3 (a 700 W card; a lower power limit lowers both)
    return 989.0, 3350.0, "H100 SXM data sheet (not measured)"


class ClockSampler:
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.proc, self.path = index, None, f"/tmp/a3d_clocks_{os.getpid()}.csv"

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i",
                                          str(self.index), "-lms", "100"], stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        self.proc.wait()
        sm, mx, reasons = [], 0, set()
        for line in open(self.path):
            f = [x.strip() for x in line.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx = max(mx, float(f[1]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        hot = [s for s in sm if s > 0.5 * mx] or sm
        return {"sm_mhz": statistics.median(hot) if hot else None, "sm_max_mhz": mx or None, "reasons": sorted(reasons),
                "samples": len(sm)}


def best_cpu_threads(sd):
    """Pick the torch thread count that runs the oracle fastest on this host (on a 128-core box all-cores is ~15x SLOWER
    than 16-32 threads for these layer sizes); the baseline is reported at its best setting.  Probes 8 / 16 / 32 threads on
    a single-frame forward (about a second each) -- never the all-cores setting, which alone can take minutes."""
    import torch
    from oracle import unet_oracle as O
    ocfg = O.UNetConfig(num_views=1, num_frames=1)
    sample, text, camera, img = O.synthetic_inputs(ocfg, 1, 1, 1, 0)
    ncpu = os.cpu_count() or 1
    best, best_t = 1, float("inf")
    for n in sorted({min(ncpu, c) for c in (8, 16, 32)}):
        torch.set_num_threads(n)
        with torch.no_grad():
            t0 = time.perf_counter()
            O.unet_forward(sd, ocfg, sample, 500, text, camera, img, 1)
            dt = time.perf_counter() - t0
        if dt < best_t:
            best, best_t = n, dt
        if dt > 1.5 * best_t:
            break
    torch.set_num_threads(best)
    return best


def cpu_oracle_sample(repeats=1):
    """Time the oracle port on a bounded sample (one forward of 4 views x 1 frame: cross-view attention at its real
    L = 4096) and extrapolate by FLOPs."""
    import torch
    from animate3d_b200.flops import unet_forward_flops
    from animate3d_b200.unet_config import UNetConfig
    from oracle import unet_oracle as O
    nv, nf = 4, 1
    ocfg = O.UNetConfig(num_views=nv, num_frames=nf)
    torch.set_num_threads(min(16, os.cpu_count() or 1))   # never run the oracle (or build its weights) on all cores
    sd = O.make_state_dict(ocfg, 0)
    cores = best_cpu_threads(sd)
    sample, text, camera, img = O.synthetic_inputs(ocfg, 1, nv, nf, 0)
    times = []
    with torch.no_grad():
        for _ in range(repeats):
            t0 = time.perf_counter()
            O.unet_forward(sd, ocfg, sample, 500, text, camera, img, nv)
            times.append(time.perf_counter() - t0)
    fl = unet_forward_flops(UNetConfig(), 1, nv, nf)["total"]
    return times, fl, cores


def run_reference(args, rank, world):
    if rank != 0:
        return
    sf = step_flops()
    import torch
    from oracle import unet_oracle as O
    from animate3d_b200.flops import unet_forward_flops
    from animate3d_b200.unet_config import UNetConfig
    tiny = bool(os.environ.get("A3D_BENCH_TINY"))
    nv, nf = (1, 1) if tiny else (4, 1)
    ocfg = O.UNetConfig(num_views=nv, num_frames=nf)
    torch.set_num_threads(min(16, os.cpu_count() or 1))   # never run the oracle (or build its weights) on all cores
    sd = O.make_state_dict(ocfg, 0)
    cores = best_cpu_threads(sd)
    sample, text, camera, img = O.synthetic_inputs(ocfg, 1, nv, nf, 0)
    fl = unet_forward_flops(UNetConfig(), 1, nv, nf)["total"]
    with torch.no_grad():
        for _ in range(args.warmup):
            O.unet_forward(sd, ocfg, sample, 500, text, camera, img, nv)
        t0 = time.perf_counter()
        for _ in range(args.steps):
            O.unet_forward(sd, ocfg, sample, 500, text, camera, img, nv)
        dt = (time.perf_counter() - t0) / args.steps
    val = (fl / dt) / sf
    factor = sf / fl
    sample_desc = (f"each step = one fp32 oracle forward of {nv} view(s) x {nf} frame(s) x 32x32x4 ({fl / 1e12:.2f} TFLOP of the "
                   f"{sf / 1e12:.2f} TFLOP CFG step, cross-view attention at its real L = {nv * 1024}); steps/s extrapolated by "
                   f"FLOPs (x{factor:.1f}); ms_per_step is the measured time of the sample")
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": 1000.0 * dt, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic", "extrapolated": True, "same_config": False,
        "config": {"workload": "MV-VDM CFG denoise step, 1 prompt x 2 CFG x 4 views x 16 frames x 32x32x4 latents",
                   "sample": sample_desc, "sample_tflop": fl / 1e12, "step_tflop": sf / 1e12, "extrapolation_factor": factor,
                   "note": "reference's diffusers CPU path is not installable here; oracle port (oracle/unet_oracle.py) timed"},
        "cpu_baseline": {"value": val, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample_desc},
        "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0}))


def sm_count():
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def mufu_note(att_flops, att_ms, clocks):
    """Lower bound of this kernel at head_dim 40 from its exponentials: one ex2 per score on the MUFU pipe, which retires 16
    results per clock per SM (one warp instruction every 8 cycles per SM sub-partition)."""
    try:
        scores = att_flops / (4.0 * 40.0)                       # 4 * d FLOP per (query, key) pair
        cycles = (scores / 32.0 * 8.0) / (sm_count() * 4)
        mhz = float(clocks.get("sm_mhz") or 1980.0)
        floor_ms = cycles / (mhz * 1e3)
        return {"floor_ms": floor_ms, "frac_of_floor": floor_ms / att_ms, "sm_mhz_used": mhz}
    except Exception as e:                                      # never let a diagnostic field break the bench line
        return {"error": str(e)}


def time_attention_l0(torch, iters=10):
    """The dominant kernel alone: level-0 cross-view attention launch of the CFG step (32 batches x 8 heads, L=4096, d=40)."""
    from animate3d_b200 import ops
    B, heads, d, hw = 2, 8, 40, LAT * LAT
    dqk = dv = 48
    M = B * NV * NF * hw
    nq = 4 * heads * dqk
    qkv = (torch.randn(M, nq, device="cuda", dtype=torch.float16))
    vcol = 3 * heads * dqk
    qkv[:, vcol:].view(M, heads, dv)[:, :, d] = 1.0
    qkv[:, vcol:].view(M, heads, dv)[:, :, d + 1:] = 0.0
    out = torch.empty(M, heads * d, device="cuda", dtype=torch.float16)
    st = (nq, NF * hw * nq, hw * nq, NV * NF * hw * nq)
    ext = (hw, NV, NF, B)
    c = heads * d
    ostr = (c, NF * hw * c, hw * c, NV * NF * hw * c)
    vq = ops.view5(qkv, 0, nq, st, ext)
    vk = ops.view5(qkv, 2 * heads * dqk, nq - 2 * heads * dqk, st, ext)
    vv = ops.view5(qkv, vcol, nq - vcol, st, ext)
    for _ in range(3):
        ops.attention(vq, vk, vv, out, ostr, heads=heads, d=d, scale=d ** -0.5)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.attention(vq, vk, vv, out, ostr, heads=heads, d=d, scale=d ** -0.5)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    flops = B * NF * 4.0 * (NV * hw) ** 2 * c
    return ms, flops


def _time_cuda(torch, fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def gemm_rooflines(torch, peak_tf, peak_hbm):
    """Two GEMM shapes of the step timed alone (operands >> L2 are re-read every launch at level 0):
    worst short-K  : the merged attention output projection at level 0, M=131072 N=320 K=640 + residual  -> HBM-bound
    best long-K    : ResnetBlock2D conv3x3 1280->1280 at level 2, implicit GEMM M=8192 N=1280 K=11520 -> tensor-bound."""
    from animate3d_b200 import ops
    out = {}
    M, N, K = 131072, 320, 640
    A = torch.randn(M, K, device="cuda").half()
    B = (torch.randn(N, K, device="cuda") * 0.05).half()
    R2 = torch.randn(M, N, device="cuda").half()
    bias = torch.randn(N, device="cuda")
    C_ = torch.empty(M, N, device="cuda", dtype=torch.float16)
    ms = _time_cuda(torch, lambda: ops.gemm(A, B, C_, M=M, N=N, K=K, bias=bias, R2=R2, ldr2=N))
    nbytes = 2.0 * (M * K + N * K + 2 * M * N)
    gbs = nbytes / (ms * 1e-3) / 1e9
    out["short_k"] = {"shape": f"M={M} N={N} K={K} +bias +residual (to_out([O1|O2]) at level 0)", "bound": "hbm", "us": ms * 1e3,
                      "bytes": nbytes, "achieved": gbs, "peak": peak_hbm, "unit": "GB/s", "frac": gbs / peak_hbm,
                      "tflops": 2.0 * M * N * K / (ms * 1e-3) / 1e12}
    n_img, h, w, c = 128, 8, 8, 1280
    M, N, K = n_img * h * w, 1280, 9 * c
    A = torch.randn(M, c, device="cuda").half()
    B = (torch.randn(N, K, device="cuda") * 0.02).half()
    R2 = torch.randn(M, N, device="cuda").half()
    C_ = torch.empty(M, N, device="cuda", dtype=torch.float16)
    bias2 = torch.zeros(N, device="cuda")
    ms = _time_cuda(torch, lambda: ops.gemm(A, B, C_, M=M, N=N, K=K, conv=(n_img, h, w, c, 1), bias=bias2, R2=R2, ldr2=N))
    tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
    out["long_k"] = {"shape": f"conv3x3 {c}->{N} on {n_img}x{h}x{w} (implicit GEMM M={M} N={N} K={K}) +residual", "bound": "tensor",
                     "us": ms * 1e3, "achieved": tf, "peak": peak_tf, "unit": "TFLOP/s", "frac": tf / peak_tf}
    return out


def splat_bench(torch, rank, world, peak_hbm, sm_mhz, iters=5):
    """BASELINE configs[2] geometry: 50k gaussians, 4 views x 16 timestamps at 512^2 (SURVEY 8d config 3).  world > 1: rank r
    renders cameras r::world, the deformation-field gradients are summed with one flat all-reduce per step."""
    import ctypes as C
    import torch.distributed as dist
    from animate3d_b200 import _lib as L
    from animate3d_b200.parallel import allreduce_gradients, shard_cameras
    from animate3d_b200.renderer import make_renderer
    from tools.splat_bench import cameras, synthetic_model
    P, H, W = 50000, 512, 512
    lib = L.load()
    model = synthetic_model(P)
    rend = make_renderer(model)
    c2w, fovy, ts = cameras()
    full = {"c2w": c2w, "fovy": fovy, "width": W, "height": H, "timestamps": ts, "do_guidance": True, "do_reconstruction": True}
    batch = shard_cameras(full, rank, world) if world > 1 else full
    ncam_total, ncam = int(c2w.shape[0]), int(batch["c2w"].shape[0])
    target = torch.rand(ncam, H, W, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    params = [p for p in model.parameters() if p.requires_grad]

    def fwd():
        return rend.batch_forward(batch)

    def fwd_bwd():
        for p_ in params:
            p_.grad = None
        out = rend.batch_forward(batch)
        (0.5 * ((out["comp_rgb"] - target) ** 2).sum()).backward()
        allreduce_gradients(params, world)

    res = {}
    for name, fn in (("fwd", fwd), ("fwd_bwd", fwd_bwd)):
        fn(); fn()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        ms = _time_cuda(torch, fn, iters=iters, warm=0)
        if world > 1:
            t = torch.tensor([ms], device="cuda")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = t.item()
        res[name] = ms
    # one instrumented fwd+bwd on this rank: per-stage times from events inside liba3d.so
    L.check(lib.a3d_debug_raster_timing(1))
    fwd_bwd()
    stage = (C.c_float * 8)()
    L.check(lib.a3d_debug_raster_stage_ms(stage))
    L.check(lib.a3d_debug_raster_timing(0))
    st = {k: float(stage[i]) for i, k in enumerate(("preprocess", "scan_duplicate", "radix_sort", "ranges", "render_fwd",
                                                    "render_bwd", "preprocess_bwd"))}
    with torch.no_grad():
        out = rend.batch_forward(batch)
        radii = torch.stack(out["radii"])
    from animate3d_b200 import rasterizer as RZ
    pairs = int(RZ.last_num_rendered)                             # (tile, gaussian) pairs of this rank's cameras
    tiles = (H // 16) * (W // 16)
    passes = -(-(32 + max(1, (ncam * tiles).bit_length())) // 8)
    # SURVEY 8(d) algorithmic bytes: preprocess 44 + 12 read, 72 written per (camera, gaussian); binning 12 B per pair written
    # once + 2 x 12 B per pair per radix pass; render 44 B per pair + 28 B per pixel
    b_pre = ncam * P * (44 + 12 + 72.0)
    b_bin = pairs * 12.0 + passes * 2 * 12.0 * pairs
    t_bin = (st["scan_duplicate"] + st["radix_sort"] + st["ranges"]) * 1e-3
    evals = float(pairs) * 256.0                                   # pixel-gaussian evaluations (upper bound: early exit at T < 1e-4)
    mufu_evals_s = sm_count() * 16 * sm_mhz * 1e6                   # one ex2 per evaluation, 16 per clock per SM
    out = {"config": {"gaussians": P, "cameras": ncam_total, "cameras_per_rank": ncam, "H": H, "W": W,
                      "scene": "SURVEY 8(d) config 3 (seeded synthetic), k-planes + 3 MLPs deformation per timestamp",
                      "parallelism": "single GPU" if world == 1 else f"cameras r::{world}, 1 flat all-reduce of the deformation-field gradients"},
           "fwd_mpix_s": ncam_total * H * W / res["fwd"] / 1e3, "fwd_bwd_mpix_s": ncam_total * H * W / res["fwd_bwd"] / 1e3,
           "fwd_ms": res["fwd"], "fwd_bwd_ms": res["fwd_bwd"], "pairs_per_rank": pairs, "radix_passes": passes, "stages_ms": st,
           "roofline": {
               "preprocess": {"bound": "hbm", "bytes": b_pre, "achieved": b_pre / (st["preprocess"] * 1e-3) / 1e9 if st["preprocess"] else None,
                              "peak": peak_hbm, "unit": "GB/s"},
               "binning": {"bound": "hbm", "bytes": b_bin, "achieved": b_bin / t_bin / 1e9 if t_bin else None, "peak": peak_hbm,
                           "unit": "GB/s"},
               "render_fwd": {"bound": "xu (one ex2 per pixel-gaussian evaluation)", "evals": evals,
                              "achieved": evals / (st["render_fwd"] * 1e-3) / 1e9 if st["render_fwd"] else None,
                              "peak": mufu_evals_s / 1e9, "unit": "G eval/s"}}}
    for v in out["roofline"].values():
        if v.get("achieved"):
            v["frac"] = v["achieved"] / v["peak"]
    return out


def sds_step_bench(torch, unet, iters=3):
    """BASELINE configs[2] end to end: ONE 4D-SDS refine step on the engine -- 64 cameras (4 views x 16 timestamps) of 50k deformed
    gaussians rendered at 512^2, resized to 256^2, VAE-encoded WITH grad, one CFG UNet evaluation (no grad), x0-reconstruction
    loss, backward through the VAE encoder, the rasterizer and the deformation field (systems/animate3d.py:180-215;
    animatemv_guidance.py:515-600).  Random-init VAE / UNet weights, seeded synthetic scene."""
    from animate3d_b200.guidance import AnimateMVDiffusionGuidance, PrecomputedPromptUtils
    from animate3d_b200.renderer import make_renderer
    from animate3d_b200.vae import AutoencoderKL, vae_key_plan
    from tools.splat_bench import cameras, synthetic_model
    dev = unet.device
    g = torch.Generator(device=dev).manual_seed(7)
    vae = AutoencoderKL(device=dev)
    sd = {}
    for k, shape in vae_key_plan(vae.config).items():
        if "norm" in k.split(".")[-2]:
            sd[k] = torch.ones(shape, device=dev) if k.endswith("weight") else torch.zeros(shape, device=dev)
        elif k.endswith("bias"):
            sd[k] = torch.zeros(shape, device=dev)
        else:
            fan = 1
            for s_ in shape[1:]:
                fan *= s_
            sd[k] = torch.randn(shape, device=dev, generator=g) * fan ** -0.5
    vae.load_state_dict(sd)
    del sd
    model = synthetic_model(50000, device=dev)
    rend = make_renderer(model).train()
    c2w, fovy, ts = cameras(device=dev)
    batch = {"c2w": c2w, "fovy": fovy, "width": 512, "height": 512, "timestamps": ts, "do_guidance": True, "do_reconstruction": True}
    guide = AnimateMVDiffusionGuidance({"n_view": NV, "n_frame": NF, "guidance_scale": 5.0, "recon_std_rescale": 0.5,
                                        "min_step_percent": 0.02, "max_step_percent": 0.2}, unet=unet, vae=vae)
    guide.update_step(0, 0)
    pu = PrecomputedPromptUtils(torch.randn(77, 768, device=dev, generator=g), torch.randn(77, 768, device=dev, generator=g))
    img = torch.randn(NV, 1024, device=dev, generator=g)
    z = torch.zeros(NV * NF, device=dev)
    params = [p for p in model.parameters() if p.requires_grad]

    def step():
        for p_ in params:
            p_.grad = None
        out = rend.batch_forward(batch)
        go = guide(out["comp_rgb"], pu, z, z, z, c2w, image_embeds=img)
        go["loss_sds"].backward()
        return go["loss_sds"]

    loss = step()
    step()
    ms = _time_cuda(torch, step, iters=iters, warm=0)
    gn = float(sum(p_.grad.float().pow(2).sum() for p_ in params if p_.grad is not None).sqrt())
    return {"ms_per_step": ms, "steps_per_s": 1000.0 / ms, "loss": float(loss.detach()), "grad_norm_deformation_field": gn,
            "workload": "render 64 x 512^2 (50k gaussians, deformation field) -> 256^2 -> VAE encoder fwd+bwd (64 images) -> CFG UNet "
                        "(2 x 4 views x 16 frames) -> x0-recon loss -> rasterizer + deformation backward",
            "finite": bool(loss.isfinite()) and gn == gn}


def view_sharded_bench(torch, args, rank, world, local_rank, base_model, timesteps):
    """ONE prompt over all ranks (SURVEY 8e / BASELINE configs[3]): world 2 = the two CFG branches; world 4 = the 4 views (K|V
    all-gather per cross-view attention); world 8 = both.  Returns steps/s of that single prompt, the exposed communication
    (same sharded step with the all-gathers skipped) and the collective volume."""
    import torch.distributed as dist
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline, get_camera
    from animate3d_b200.scheduler import DDIMScheduler
    from animate3d_b200.unet import MVUNetMotionModel
    if world not in (2, 4, 8):
        return None
    cfg_world = 2 if world in (2, 8) else 1
    view_world = 4 if world in (4, 8) else 1
    cfg_idx, view_idx = rank // view_world, rank % view_world
    view_group = cfg_group = None
    for c in range(cfg_world):           # every rank creates every group, in the same order
        g = dist.new_group([c * view_world + v for v in range(view_world)])
        if c == cfg_idx and view_world > 1:
            view_group = g
    for v in range(view_world):
        g = dist.new_group([c * view_world + v for c in range(cfg_world)])
        if v == view_idx and cfg_world > 1:
            cfg_group = g
    dev = torch.device("cuda", local_rank)
    cfg = base_model.cfg
    model = MVUNetMotionModel(cfg, device=dev, view_group=view_group)
    model.share_packed_weights(base_model)
    sched = DDIMScheduler()
    sched.set_timesteps(25)
    pipe = AnimateDiffMVI2VPipeline(unet=model, scheduler=sched)
    g = torch.Generator(device=dev).manual_seed(4242)               # the SAME prompt on every rank
    lat = torch.randn(NV, 4, NF, LAT, LAT, device=dev, generator=g)
    pe = torch.randn(2 * NV, 77, cfg.cross_attention_dim, device=dev, generator=g)
    ie = torch.randn(2 * NV, cfg.ip_image_embed_dim, device=dev, generator=g)
    ie[:NV] = 0
    cam = get_camera(NV).to(dev)
    vs = slice(view_idx, view_idx + 1) if view_world > 1 else slice(0, NV)
    nloc = 1 if view_world > 1 else NV
    lat_loc = lat[vs].contiguous()
    first_loc = lat_loc[:, :, :1].clone()
    pick = lambda x: x.reshape(2, NV, *x.shape[1:])[:, vs]            # (branch, view, ...)
    if cfg_world > 1:
        pe_l, ie_l, cam_l = pick(pe)[cfg_idx], pick(ie)[cfg_idx], cam[vs]
    else:
        pe_l, ie_l = pick(pe).reshape(2 * nloc, *pe.shape[1:]), pick(ie).reshape(2 * nloc, *ie.shape[1:])
        cam_l = torch.cat([cam[vs], cam[vs]])

    def run(n, x):
        for i in range(n):
            pipe.denoise_step_sharded(x, timesteps[i % len(timesteps)], pe_l, cam_l, ie_l, first_loc, 7.5, cfg_group=cfg_group,
                                      num_views_local=nloc)

    def timed(comm):
        model.comm_enabled = comm
        model._graphs.clear()
        for st_ in model._static.values():
            st_["calls"] = 0
        x = lat_loc.clone()
        run(3, x)
        torch.cuda.synchronize()
        dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(args.steps, x)
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.item() / args.steps, x

    ms, x = timed(True)
    finite = bool(torch.isfinite(x).all())
    ncoll, nbytes = model.collectives, model.collective_bytes
    ms_nocomm = None
    if view_world > 1:
        ms_nocomm, _ = timed(False)
        model.comm_enabled = True
    return {"value": 1000.0 / ms, "unit": UNIT, "ms_per_step": ms, "scaling": "strong",
            "mode": f"1 prompt over {world} ranks = {cfg_world} CFG rank(s) x {view_world} view rank(s)",
            "collectives_per_forward": ncoll, "kv_bytes_received_per_rank_per_forward": nbytes,
            "cfg_allgather_bytes_per_step": (2 * nloc * 4 * NF * LAT * LAT * 4) if cfg_world > 1 else 0,
            "ms_per_step_collectives_skipped": ms_nocomm,
            "exposed_comm_ms_per_step": (ms - ms_nocomm) if ms_nocomm is not None else None,
            "overlap": "K|V all-gather issued async right after the K|V projection; query projection and the temporal branch run under it",
            "cuda_graph": bool(model._graphs), "finite": finite}


def dump_outputs(directory, arrays):
    """Save each tensor as directory/<name>.npy in float32."""
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    for name, t in arrays.items():
        np.save(os.path.join(directory, f"{name}.npy"), t.detach().float().cpu().numpy())


def run_native(args, rank, world, local_rank):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    from animate3d_b200.pipeline import AnimateDiffMVI2VPipeline, get_camera
    from animate3d_b200.scheduler import DDIMScheduler
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from animate3d_b200.weights import random_state_dict

    dev = torch.device("cuda", local_rank)
    cfg = UNetConfig()
    model = MVUNetMotionModel(cfg, device=dev)
    model.load_state_dict(random_state_dict(cfg, seed=0, device=dev))
    model._prepare()
    model.drop_reference_weights()          # free the fp32 masters (6 GB)
    torch.cuda.empty_cache()
    sched = DDIMScheduler()
    pipe = AnimateDiffMVI2VPipeline(unet=model, scheduler=sched)
    timesteps = [int(t) for t in sched.set_timesteps(25)]
    g = torch.Generator(device=dev).manual_seed(1000 + rank)     # every rank owns a different prompt
    lat = torch.randn(NV, 4, NF, LAT, LAT, device=dev, generator=g)
    first = lat[:, :, :1].clone()
    pe = torch.randn(2 * NV, 77, cfg.cross_attention_dim, device=dev, generator=g)
    ie = torch.randn(2 * NV, cfg.ip_image_embed_dim, device=dev, generator=g)
    ie[:NV] = 0
    cam = get_camera(NV).to(dev)
    cam2 = torch.cat([cam, cam])

    def step(i):
        pipe.denoise_step(lat, timesteps[i % len(timesteps)], pe, cam2, ie, first, 7.5, num_views=NV)

    for i in range(max(args.warmup, 3)):
        step(i)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        step(i)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {"latents": lat})
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = t.item()
    ms_step = ms / args.steps
    value = world * 1000.0 / ms_step
    assert torch.isfinite(lat).all(), "latents diverged"

    # ---- end-to-end through host buffers
    lat_h = lat.cpu().pin_memory(); pe_h = pe.cpu().pin_memory(); cam_h = cam2.cpu().pin_memory()
    ie_h = ie.cpu().pin_memory(); ff_h = first.cpu().pin_memory(); out_h = torch.empty_like(lat_h).pin_memory()
    for i in range(2):
        pipe.denoise_step_host(lat_h, timesteps[i], pe_h, cam_h, ie_h, ff_h, 7.5, out_host=out_h, num_views=NV)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0.record()
    for i in range(args.steps):
        pipe.denoise_step_host(lat_h, timesteps[i % len(timesteps)], pe_h, cam_h, ie_h, ff_h, 7.5, out_host=out_h, num_views=NV)
        lat_h, out_h = out_h, lat_h
    e1.record()
    torch.cuda.synchronize()
    ms_e2e = e0.elapsed_time(e1)
    if world > 1:
        t = torch.tensor([ms_e2e], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms_e2e = t.item()
    e2e_val = world * 1000.0 * args.steps / ms_e2e
    h2d = sum(x.numel() * x.element_size() for x in (lat_h, pe_h, cam_h, ie_h, ff_h))
    d2h = out_h.numel() * out_h.element_size()

    peak_tf, peak_hbm, peak_src = peaks()
    del lat_h, pe_h, cam_h, ie_h, ff_h, out_h
    splat = splat_bench(torch, rank, world, peak_hbm, float((clocks or {}).get("sm_mhz") or 1965.0))
    if rank != 0:
        # the one-prompt-over-all-ranks mode runs LAST, under a watchdog: a wedged collective must not cost the bench line
        guard = _Watchdog(180.0, None)
        if world > 1:
            try:
                view_sharded_bench(torch, args, rank, world, local_rank, model, timesteps)
            except Exception:
                pass
        guard.cancel()
        if world > 1:
            dist.destroy_process_group()
        return
    sf = step_flops()
    att_ms, att_flops = time_attention_l0(torch)
    att_tf = att_flops / (att_ms * 1e-3) / 1e12
    gemm_rf = gemm_rooflines(torch, peak_tf, peak_hbm)
    sds = None
    if world == 1:
        try:
            sds = sds_step_bench(torch, model)
        except Exception as e:                     # noqa: BLE001 -- an extra, must not cost the headline line
            sds = {"error": f"{type(e).__name__}: {e}"}
    cpu = None
    if world == 1:
        times, fl, cores = cpu_oracle_sample(1)
        cpu_val = (fl / min(times)) / sf
        cpu = {"value": cpu_val, "unit": UNIT, "cores": cores, "kind": "port",
               "extrapolated": True,
               "sample": f"one fp32 oracle forward of 4 views x 1 frame ({fl / 1e12:.2f} TFLOP, {min(times):.1f} s; cross-view "
                         f"attention at L = 4096) extrapolated by FLOPs (x{sf / fl:.1f}) to the {sf / 1e12:.2f} TFLOP CFG step"}
    out = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
        "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp16",
        "data": "synthetic",
        "config": {"workload": f"MV-VDM CFG denoise step, {world} prompt(s) x 2 CFG x 4 views x 16 frames x 32x32x4 latents "
                               "(BASELINE configs[1]); random-init SD1.5+motion-module weights (1.53 B params)",
                   "parallelism": f"prompt-sharded dp{world}, no data-path collective",
                   "step_tflop": sf / 1e12, "achieved_tflops_per_gpu": sf / 1e12 / (ms_step * 1e-3),
                   "l2": "working set (3.1 GB fp16 weights + activations) >> 50 MB L2; no flush needed",
                   "cuda_graph": bool(model.use_cuda_graph)},
        "roofline": {"bound": "tensor", "kernel": "a3d_attention head_dim 40 (fused cross-view attention, L=4096, 32 batches x 8 heads)",
                     "achieved": att_tf, "peak": peak_tf, "unit": "TFLOP/s", "frac": att_tf / peak_tf,
                     "ms_per_launch": att_ms, "flop_per_launch": att_flops, "peak_source": peak_src,
                     "mufu": mufu_note(att_flops, att_ms, clocks),
                     "note": "at head_dim 40 every score needs one exponential: the MUFU pipe floors the kernel at `mufu.floor_ms`, "
                             "well above the tensor-only bound; logits here are randn"},
        "roofline_gemm": gemm_rf,
        "splat": splat,
        "sds_step": sds,
        "view_sharded": None,
        "cpu_baseline": cpu,
        "e2e": {"value": e2e_val, "unit": UNIT, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h},
        "gpu_launches": (model.launches_per_forward + 1) * args.steps,
        "clocks": clocks,
    }
    if world > 1:
        # strong-scaling mode last, under a watchdog that prints the line without it if a collective wedges
        fallback = dict(out)
        fallback["view_sharded"] = {"error": "timed out after 180 s (collective did not complete); not measured in this run"}
        guard = _Watchdog(180.0, json.dumps(fallback))
        try:
            out["view_sharded"] = view_sharded_bench(torch, args, rank, world, local_rank, model, timesteps)
        except Exception as e:                     # noqa: BLE001 -- a diagnostic mode must not cost the headline line
            out["view_sharded"] = {"error": f"{type(e).__name__}: {e}"}
        guard.cancel()
    print(json.dumps(out), flush=True)
    if world > 1:
        dist.destroy_process_group()


class _Watchdog:
    """If not cancelled within `seconds`: print `line` (rank 0's complete JSON line without the wedged section) and leave the
    process with exit code 0 -- an in-flight NCCL call cannot be interrupted from Python."""

    def __init__(self, seconds, line):
        import threading
        self._t = threading.Timer(seconds, self._fire, args=(line,))
        self._t.daemon = True
        self._t.start()

    @staticmethod
    def _fire(line):
        if line is not None:
            print(line, flush=True)
        os._exit(0)

    def cancel(self):
        self._t.cancel()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="native", choices=["native", "reference"])
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step computed as DIR/<name>.npy (native only)")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus and world == 1 and args.gpus > 1:
        # launched without torchrun: re-exec under it
        port = os.environ.get("MASTER_PORT", "29517")
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={args.gpus}", "--master-addr",
               "127.0.0.1", "--master-port", port, os.path.abspath(__file__), "--gpus", str(args.gpus), "--steps", str(args.steps),
               "--warmup", str(args.warmup), "--impl", args.impl]
        if args.dump_outputs:
            cmd += ["--dump-outputs", args.dump_outputs]
        sys.exit(subprocess.call(cmd))
    if args.impl == "reference":
        run_reference(args, rank, world)
    else:
        run_native(args, rank, world, local_rank)


if __name__ == "__main__":
    main()
