"""Time the IP-Adapter image encoder: the engine's encode_image on 4 float renders at 256^2 (raw renders -> patch operand in
one launch, then the graph-replayed ViT-H/14), and, when transformers is importable, the reference's path in the same run
(.cpu() -> uint8 PIL -> CLIPImageProcessor -> fp16 CLIPVisionModelWithProjection).  Random-init weights of the ViT-H/14
geometry; CUDA events around each call.  Prints one JSON line with the card name and power limit.

    python tools/clip_bench.py [--iters 50] [--warmup 5] [--out clip_bench.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VIT_H = dict(hidden_size=1280, intermediate_size=5120, num_attention_heads=16, num_hidden_layers=32, image_size=224,
             patch_size=14, projection_dim=1024, layer_norm_eps=1e-5, hidden_act="gelu")


def vit_flops(cfg, n):
    """Multiply-adds x 2 of one forward from the shapes: patch GEMM, per layer QKV / scores / PV / out-proj / MLP, projection."""
    T, H, I, L = 257, cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
    per_layer = 2 * T * (4 * H * H + 2 * H * I) + 2 * 2 * T * T * H
    return n * (2 * 256 * 588 * H + L * per_layer + 2 * H * cfg["projection_dim"])


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(np.min(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clip_bench needs a CUDA device")
    from animate3d_b200.clip import CLIPImageProcessor, CLIPVisionModelWithProjection, IPAdapterImageProcessor
    from oracle import clip_oracle as O
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": q.stdout.strip(), "images": 4, "render": 256}
    sd = O.random_state_dict(VIT_H, 0)
    enc = CLIPVisionModelWithProjection(VIT_H, "cuda").load_state_dict(sd)
    ipp = IPAdapterImageProcessor(CLIPImageProcessor("cuda"), enc)
    x = torch.rand(4, 3, 256, 256, generator=torch.Generator().manual_seed(0)).cuda()
    with torch.no_grad():
        res["engine_ms_median"], res["engine_ms_min"] = timed(lambda: ipp.encode_image(x), args.iters, args.warmup)
    fl = vit_flops(VIT_H, 4)
    res["vit_h_gflop"] = fl / 1e9
    res["engine_tflops"] = fl / (res["engine_ms_median"] * 1e-3) / 1e12
    res["launches_per_forward"] = enc.launches_per_forward
    try:
        import transformers
        from PIL import Image
        cfg = transformers.CLIPVisionConfig(**VIT_H)
        ref = transformers.CLIPVisionModelWithProjection(cfg)
        ref.load_state_dict(sd, strict=False)
        ref = ref.half().cuda().eval()
        proc = transformers.CLIPImageProcessor()

        def reference():
            ims = [Image.fromarray((im.permute(1, 2, 0).cpu().numpy() * 255).astype(np.uint8)) for im in x]
            pv = proc(ims, return_tensors="pt").pixel_values.to("cuda", torch.float16)
            return ref(pv).image_embeds

        with torch.no_grad():
            res["reference_ms_median"], res["reference_ms_min"] = timed(reference, args.iters, args.warmup)
            e = ipp.encode_image(x).double()
            r = reference().double()
        res["transformers"] = transformers.__version__
        res["speedup_median"] = res["reference_ms_median"] / res["engine_ms_median"]
        res["rel_l2_vs_reference"] = ((e - r).norm() / r.norm()).item()
    except ImportError as exc:
        res["reference"] = f"not run: {exc}"
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
