#!/usr/bin/env python
"""Training-step throughput of MaskDiT against the decoder-less DiT, XL/2 at 256 px (32x32x4 latents), one GPU.

    python tools/variant_step_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--batch 256] [--dit-batch 0]

Variants (the reference README's "DiT" / "Ours" training-speed comparison, BASELINE.md):
    maskdit      use_decoder=True,  mask 0.5, batch --batch
    nodec_m50    use_decoder=False, mask 0.5, batch --batch        (the decoder-less MaskDiT ablation)
    dit          use_decoder=False, mask 0,   the largest batch whose training workspace fits (--dit-batch overrides)
Each round builds every variant in turn (net + EMA + fused AdamW, seeded inputs), warms it up and times `TrainStep.step`
with CUDA events, then frees it: the variants alternate inside one process on one card.  One JSON line per variant
with the median over rounds: samples/s, ms per step, `mdt_workspace_bytes` of the step, peak allocated memory, and
the card's name, power limit and max SM clock read in the same run.
"""
import argparse
import copy
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from maskdit_b200.maskdit import Precond_models  # noqa: E402
from maskdit_b200.train_step import TrainStep  # noqa: E402

R, C, NCLS, L = 32, 4, 1000, 256


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clk = (s.strip() for s in r.stdout.strip().split(","))
    except Exception:                                   # nvidia-smi missing: the name still comes from the runtime
        name, power, clk = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "sm_clock_max": clk}


def xl2(use_decoder):
    return Precond_models["edm"](R, C, num_classes=NCLS, model_type="DiT-XL/2", use_decoder=use_decoder,
                                 mae_loss_coef=0.1, pad_cls_token=False)


def fixed_bytes(use_decoder):
    """Parameter-sized state of one variant: fp32 weights, bf16 shadow, fp32 gradient, Adam m/v, EMA fp32 + bf16."""
    with torch.device("meta"):
        n = sum(p.numel() for p in xl2(use_decoder).parameters())
    return n * (4 + 2 + 4 + 8 + 4 + 2)


def workspace_bytes(use_decoder, B, mask):
    with torch.device("meta"):
        net = xl2(use_decoder)
    from maskdit_b200.engine import CEngine
    T = int(L * (1 - mask)) if mask > 0 else L
    return CEngine(net._cfg()).workspace_bytes(B, T, True)


def largest_batch(use_decoder, mask, cap):
    """Largest multiple of 32 up to `cap` whose training workspace fits next to the parameter state (10 % headroom)."""
    free, _ = torch.cuda.mem_get_info()
    budget = 0.9 * free - fixed_bytes(use_decoder)
    B = cap
    while B > 32 and workspace_bytes(use_decoder, B, mask) > budget:
        B -= 32
    return B


def run_variant(use_decoder, B, mask, steps, warmup):
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = xl2(use_decoder).train()
    ema = copy.deepcopy(net).eval()
    ts = TrainStep(net, ema, lr=1e-4, global_batch=B)
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    for i in range(warmup):
        ts.step(xs[i % 2], ys[i % 2], mask, 0.1)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        loss = ts.step(xs[i % 2], ys[i % 2], mask, 0.1)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    assert torch.isfinite(loss).all()
    peak = torch.cuda.max_memory_allocated()
    del ts, ema, net, xs, ys, loss
    gc.collect()
    torch.cuda.empty_cache()
    return ms, peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--dit-batch", type=int, default=0, help="batch of the mask-0 DiT (0: largest that fits)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("variant_step_bench.py measures on a CUDA device; none is visible")
    dit_B = args.dit_batch or largest_batch(False, 0.0, args.batch)
    variants = [("maskdit", True, args.batch, 0.5), ("nodec_m50", False, args.batch, 0.5), ("dit", False, dit_B, 0.0)]
    times = {v[0]: [] for v in variants}
    peaks = {}
    for _ in range(args.rounds):
        for name, dec, B, mask in variants:
            ms, peaks[name] = run_variant(dec, B, mask, args.steps, args.warmup)
            times[name].append(ms)
    info = card()
    for name, dec, B, mask in variants:
        ms = statistics.median(times[name])
        print(json.dumps({"variant": name, "use_decoder": dec, "batch": B, "mask_ratio": mask,
                          "samples_per_s": round(B / ms * 1e3, 1), "ms_per_step": round(ms, 2),
                          "ms_per_step_rounds": [round(t, 2) for t in times[name]],
                          "workspace_bytes": workspace_bytes(dec, B, mask), "peak_allocated_bytes": peaks[name],
                          "steps": args.steps, "warmup": args.warmup, **info}))


if __name__ == "__main__":
    main()
