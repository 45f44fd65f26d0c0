"""Cost of torch.use_deterministic_algorithms(True) on the 4D path, measured in one process with the two modes alternating:
splat forward+backward Mpix/s and rasterizer stage times (bench.py's `splat` leg, BASELINE config 3), the 4D-SDS step
(bench.py's `sds_step` leg), the rasterizer pair count and the deterministic scratch bytes, and the card's name and power
limit.  bench.py itself always measures the default (flag-off) kernels; this tool runs its two 4D legs under either setting.
Prints one JSON line; `python tools/deterministic_bench.py [--rounds R] [--out FILE]`."""
import argparse
import json
import os
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")     # before CUDA initialises (PyTorch's deterministic cuBLAS)
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": sm}
    except Exception as e:   # noqa: BLE001 -- the measurement stands without it, flagged
        return {"error": f"{type(e).__name__}: {e}"}


class deterministic:
    """torch.use_deterministic_algorithms(on) for the length of a block; the previous setting is restored."""

    def __init__(self, torch, on):
        self.torch, self.on = torch, bool(on)

    def __enter__(self):
        self.prev = self.torch.are_deterministic_algorithms_enabled()
        self.torch.use_deterministic_algorithms(self.on)

    def __exit__(self, *exc):
        self.torch.use_deterministic_algorithms(self.prev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import bench
    from animate3d_b200 import rasterizer as RZ
    from animate3d_b200.unet import MVUNetMotionModel
    from animate3d_b200.unet_config import UNetConfig
    from animate3d_b200.weights import random_state_dict
    _, peak_hbm, _ = bench.peaks()
    cfg = UNetConfig()
    unet = MVUNetMotionModel(cfg, device=torch.device("cuda"))
    unet.load_state_dict(random_state_dict(cfg, seed=0, device=torch.device("cuda")))
    unet._prepare()
    unet.drop_reference_weights()
    torch.cuda.empty_cache()
    runs = []
    for r in range(args.rounds):
        for det in ((False, True) if r % 2 == 0 else (True, False)):
            with deterministic(torch, det):
                splat = bench.splat_bench(torch, 0, 1, peak_hbm, 1980.0)
                scratch = int(RZ.last_backward_scratch_bytes)      # of splat_bench's last backward, taken in this mode
                sds = bench.sds_step_bench(torch, unet)
            runs.append({"deterministic": det, "splat_fwd_bwd_mpix_s": splat["fwd_bwd_mpix_s"], "splat_fwd_mpix_s": splat["fwd_mpix_s"],
                         "splat_fwd_bwd_ms": splat["fwd_bwd_ms"], "stages_ms": splat["stages_ms"], "pairs": splat["pairs_per_rank"],
                         "raster_backward_scratch_bytes": scratch, "sds_step_ms": sds["ms_per_step"],
                         "sds_loss": sds["loss"]})
            print(json.dumps(runs[-1]), file=sys.stderr, flush=True)
    summary = {}
    for det in (False, True):
        rs = [x for x in runs if x["deterministic"] == det]
        summary["on" if det else "off"] = {k: [x[k] for x in rs] for k in ("splat_fwd_bwd_mpix_s", "sds_step_ms")}
    out = {"card": card(), "torch": torch.__version__, "runs": runs, "summary": summary,
           "peak_memory_gib": torch.cuda.max_memory_allocated() / 2 ** 30}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
