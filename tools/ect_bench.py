#!/usr/bin/env python
"""Cost of consistency tuning (ECT) against EDM training, and of few-step sampling, on one card, in one process:
  * the XL/2 ImageNet-256 MaskDiT training step (32x32x4 latents, batch 256, mask 0.5, MAE 0.1) with the EDM loss and
    with the ECT loss (one extra no-gradient masked forward), alternated round by round; each mode warms up before
    its timed window (CUDA events), medians and the peak memory of each mode's rounds reported;
  * the samplers at batch 64 with CFG 1.5: `consistency_sampler` at 1 and 2 network evaluations against
    `edm_sampler` at 18 steps (35 evaluations); img/s of the median round.

    python tools/ect_bench.py [--steps 10] [--warmup 3] [--rounds 3] [--batch 256] [--sample_batch 64] [--num_steps 18]

Both losses drive the same network and TrainStep (the tuning stage does not change the work of a step).  The card's
name and power limit are read in the same run.  One JSON line per mode.
"""
import argparse
import copy
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from variant_step_bench import C, NCLS, R, card  # noqa: E402

from maskdit_b200.loss import ECTLoss, EDMLoss  # noqa: E402
from maskdit_b200.maskdit import Precond_models  # noqa: E402
from maskdit_b200.sampler import consistency_sampler, edm_sampler  # noqa: E402
from maskdit_b200.train_step import TrainStep  # noqa: E402


def timed(ts, xs, ys, mask, steps, warmup):
    for i in range(warmup):
        ts.step(xs[i % 2], ys[i % 2], mask, 0.1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        loss = ts.step(xs[i % 2], ys[i % 2], mask, 0.1)
    e1.record()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--mask", type=float, default=0.5)
    ap.add_argument("--sample_batch", type=int, default=64)
    ap.add_argument("--num_steps", type=int, default=18)
    ap.add_argument("--iters", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ect_bench.py measures on a CUDA device; none is visible")
    info = card()
    B, mask = args.batch, args.mask
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = Precond_models["edm"](R, C, num_classes=NCLS, model_type="DiT-XL/2", use_decoder=True,
                                    mae_loss_coef=0.1, pad_cls_token=False).train()
    ema = copy.deepcopy(net).eval()
    ect = ECTLoss(stage_steps=1000)
    ts = TrainStep(net, ema, lr=1e-4, global_batch=B, loss_fn=ect)   # owns the stage word the ECT loss reads
    losses = {"edm": EDMLoss(), "ect": ect}
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    times = {"edm": [], "ect": []}
    peak = {"edm": 0, "ect": 0}
    for _ in range(args.rounds):
        for kind in times:
            ts.loss_fn = losses[kind]
            torch.cuda.reset_peak_memory_stats()
            times[kind].append(timed(ts, xs, ys, mask, args.steps, args.warmup))
            peak[kind] = max(peak[kind], torch.cuda.max_memory_allocated())
    base = statistics.median(times["edm"])
    for kind, t in times.items():
        ms = statistics.median(t)
        print(json.dumps({"measure": "train_step", "objective": kind, "model": "DiT-XL/2 (MaskDiT, decoder)",
                          "batch": B, "mask_ratio": mask, "ms_per_step": round(ms, 3),
                          "ms_per_step_rounds": [round(v, 3) for v in t], "relative_to_edm": round(ms / base, 5),
                          "peak_memory_gib": round(peak[kind] / 2 ** 30, 2), "recompute_blocks": ts.recompute_blocks,
                          "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, **info}), flush=True)
    del ts, net, ema, xs
    torch.cuda.empty_cache()

    with torch.device("cuda"):
        net = Precond_models["edm"](R, C, num_classes=NCLS, model_type="DiT-XL/2", use_decoder=True,
                                    mae_loss_coef=0.1, pad_cls_token=False).eval()
    gen = torch.Generator().manual_seed(0)
    lat = torch.randn(args.sample_batch, C, R, R, generator=gen).cuda()
    lab = torch.nn.functional.one_hot(torch.randint(0, NCLS, (args.sample_batch,), generator=gen), NCLS).float().cuda()
    runs = {("edm_sampler", 2 * args.num_steps - 1):
            lambda: edm_sampler(net, lat, lab, cfg_scale=1.5, num_steps=args.num_steps),
            ("consistency_sampler", 1): lambda: consistency_sampler(net, lat, lab, cfg_scale=1.5, sigmas=(80.0,)),
            ("consistency_sampler", 2): lambda: consistency_sampler(net, lat, lab, cfg_scale=1.5,
                                                                    sigmas=(80.0, 0.8))}
    with torch.no_grad():
        for fn in runs.values():      # warm-up: captures the CUDA graphs
            fn()
        torch.cuda.synchronize()
        stimes = {k: [] for k in runs}
        for _ in range(args.rounds):
            for k, fn in runs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.iters):
                    z = fn()
                torch.cuda.synchronize()
                assert torch.isfinite(z).all()
                stimes[k].append((time.perf_counter() - t0) / args.iters)
    for (name, evals), t in stimes.items():
        sec = statistics.median(t)
        print(json.dumps({"measure": "sampler", "sampler": name, "model": "DiT-XL/2 (MaskDiT, decoder)",
                          "batch": args.sample_batch, "cfg_scale": 1.5, "evaluations_per_image": evals,
                          "img_per_s": round(args.sample_batch / sec, 2), "rounds_seconds": [round(v, 4) for v in t],
                          **info}), flush=True)


if __name__ == "__main__":
    main()
