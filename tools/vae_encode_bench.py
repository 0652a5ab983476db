#!/usr/bin/env python
"""Throughput of the SD-VAE encoder (`AutoencoderKLEncoder.encode_moments`, the work of extract_latent.py) on one GPU.

    python tools/vae_encode_bench.py [--iters 10] [--warmup 3] [--profile] [--out DIR]

Times encode_moments with CUDA events after warm-up at 256 px (batch 64) and 512 px (batch 16) on stand-in weights
(the arithmetic does not depend on their values) and prints one JSON line per size: images/s, the algorithmic work per
image computed from the layer shapes (convolutions + the AttnBlock's two batched products), and the achieved rate.
The card's name and power limit are read in the same run.  --profile adds a separate torch.profiler run per size
that splits the device time between the im2col kernel, the wgmma GEMM and everything else (written to DIR).
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from maskdit_b200.vae import AutoencoderKLEncoder  # noqa: E402

SIZES = ((256, 64), (512, 16))


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clk = (s.strip() for s in r.stdout.strip().split(","))
    except Exception:                                   # nvidia-smi missing: the name still comes from the runtime
        name, power, clk = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "sm_clock_max": clk}


def work_per_image(model, res):
    """(convolution GFLOP, attention GFLOP) of one res x res image: 2 * output pixels * C_out * C_in * kh * kw per
    convolution (conv_in on its 3 real channels) and 2 * 2 * T^2 * C for q k^T and softmax(.) v over T = (res/8)^2."""
    conv, H = 0.0, res
    for k, v in model.state_dict().items():
        shp = v.shape
        if not k.endswith(".weight") or len(shp) != 4:
            continue
        if ".downsample." in k:
            H //= 2
        co, ci, kh, kw = shp
        conv += 2.0 * H * H * co * ci * kh * kw
    T, c = (res // 8) ** 2, model.state_dict()["encoder.mid.attn_1.q.weight"].shape[0]
    return conv / 1e9, 4.0 * T * T * c / 1e9


def stand_in(model):
    g = torch.Generator().manual_seed(0)
    sd = {}
    for k, v in model.state_dict().items():
        if k.endswith("weight") and v.ndim == 4:
            sd[k] = torch.randn(v.shape, generator=g) * (v[0].numel()) ** -0.5
        elif k.endswith("weight"):
            sd[k] = 1 + 0.1 * torch.randn(v.shape, generator=g)
        else:
            sd[k] = 0.05 * torch.randn(v.shape, generator=g)
    model.load_state_dict(sd)
    return model.cuda().eval()


def kernel_split(model, x, out_dir, res):
    from torch.profiler import ProfilerActivity, profile
    model.encode_moments(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.encode_moments(x)
        torch.cuda.synchronize()
    split = {"im2col": 0.0, "gemm": 0.0, "other": 0.0}
    per_kernel = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t <= 0:
            continue
        name = ev.key
        per_kernel[name] = per_kernel.get(name, 0.0) + t / 1e3
        cat = "im2col" if "im2col" in name else "gemm" if "gemm" in name else "other"
        split[cat] += t / 1e3
    total = sum(split.values())
    rec = {"res": res, "batch": x.shape[0], "device_ms": round(total, 3),
           **{f"{k}_ms": round(v, 3) for k, v in split.items()},
           **{f"{k}_share": round(v / total, 4) for k, v in split.items()},
           "top_kernels_ms": dict(sorted(((k[:90], round(v, 3)) for k, v in per_kernel.items()),
                                         key=lambda kv: -kv[1])[:8])}
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, f"vae_encode_profile_{res}.json"), "w") as f:
            json.dump(rec, f, indent=1)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="also run the torch.profiler kernel split (separate run)")
    ap.add_argument("--out", default=None, help="directory for the profiler records")
    ap.add_argument("--sizes", default=",".join(f"{r}x{b}" for r, b in SIZES), help="res x batch list")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_encode_bench needs a CUDA device")
    info = card()
    model = stand_in(AutoencoderKLEncoder())
    for spec in args.sizes.split(","):
        res, batch = (int(v) for v in spec.split("x"))
        x = torch.rand(batch, 3, res, res, generator=torch.Generator().manual_seed(res)).mul_(2).sub_(1).cuda()
        for _ in range(args.warmup):
            model.encode_moments(x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            model.encode_moments(x)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        conv_gf, attn_gf = work_per_image(model, res)
        ips = batch * 1e3 / ms
        rec = {"metric": "vae_encode_moments", "res": res, "batch": batch, "iters": args.iters, "ms_per_batch": round(ms, 3),
               "images_per_s": round(ips, 2), "gflop_per_image_conv": round(conv_gf, 1),
               "gflop_per_image_attn": round(attn_gf, 2), "tflops": round(ips * (conv_gf + attn_gf) / 1e3, 1),
               "max_memory_gb": round(torch.cuda.max_memory_allocated() / 1e9, 1), **info}
        print(json.dumps(rec), flush=True)
        if args.profile:
            print(json.dumps({"metric": "vae_encode_kernel_split", **kernel_split(model, x, args.out, res), **info}),
                  flush=True)
        del x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
