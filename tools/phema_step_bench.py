#!/usr/bin/env python
"""Cost of the power-function EMA profiles (post-hoc EMA): the XL/2 ImageNet-256 training step (32x32x4 latents,
batch 256, mask 0.5) with `TrainStep()` and `TrainStep(phema_sigma_rels=(0.05, 0.10))`, alternated inside one process
on one card.

    python tools/phema_step_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--batch 256]

One network and EMA serve both modes.  Each round builds the mode's TrainStep (Adam moments and, with profiles, their
two 2.92 GB buffers), lets it choose its recompute count from the memory then free (the engine's remembered choice is
cleared first), warms it up, times `TrainStep.step` with CUDA events and frees it again.  With profiles, the
`mdt_power_ema` pass over the flat weights is also timed on its own.  One JSON line per mode (median over rounds,
peak allocated memory, recompute count) and one for the kernel; the card's name and power limit are read in the same
run.
"""
import argparse
import copy
import gc
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from variant_step_bench import C, NCLS, R, card, xl2  # noqa: E402

from maskdit_b200 import ops, phema  # noqa: E402
from maskdit_b200.train_step import TrainStep  # noqa: E402

MODES = {"phema_off": (), "phema_k2": (0.05, 0.10)}


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


def kernel_ms(ts, reps=20):
    """The profile update of one step over the whole trainable region, on its own."""
    w = ts.st.w32[:ts.st.n_train]
    cs = [phema.one_minus_beta(g, 1000) for g in ts.phema_gammas]
    for _ in range(3):
        ops.power_ema(w, ts.phema_emas, cs)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        ops.power_ema(w, ts.phema_emas, cs)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--mask", type=float, default=0.5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("phema_step_bench.py measures on a CUDA device; none is visible")
    B, mask = args.batch, args.mask
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = xl2(True).train()
    ema = copy.deepcopy(net).eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    times, peaks, recompute, kernel = {m: [] for m in MODES}, {m: [] for m in MODES}, {}, []
    for _ in range(args.rounds):
        for name, sigmas in MODES.items():
            ts = TrainStep(net, ema, lr=1e-4, global_batch=B, phema_sigma_rels=sigmas)
            ts._engine._auto_recompute = {}   # each mode picks its own count from the memory it leaves free
            torch.cuda.reset_peak_memory_stats()
            times[name].append(timed(ts, xs, ys, mask, args.steps, args.warmup))
            peaks[name].append(torch.cuda.max_memory_allocated())
            recompute[name] = ts.recompute_blocks
            if sigmas:
                kernel.append(kernel_ms(ts))
            del ts
            gc.collect()
            torch.cuda.empty_cache()
    info = card()
    base = statistics.median(times["phema_off"])
    for name in MODES:
        ms = statistics.median(times[name])
        print(json.dumps({"mode": name, "profiles": len(MODES[name]), "batch": B, "mask_ratio": mask,
                          "ms_per_step": round(ms, 2), "ms_per_step_rounds": [round(t, 2) for t in times[name]],
                          "relative_to_off": round(ms / base, 4), "samples_per_s": round(B / ms * 1e3, 1),
                          "peak_allocated_gib": round(max(peaks[name]) / 2 ** 30, 2),
                          "recompute_blocks": recompute[name], "steps": args.steps, "warmup": args.warmup, **info}))
    n = net.flat_store().n_train
    k = len(MODES["phema_k2"])
    gbytes = n * (4 + 8 * k) / 1e9
    kms = statistics.median(kernel)
    print(json.dumps({"kernel": "mdt_power_ema", "profiles": k, "elements": n, "gbytes_moved": round(gbytes, 3),
                      "ms": round(kms, 3), "gb_per_s": round(gbytes / kms * 1e3, 1),
                      "share_of_off_step": round(kms / base, 4), **info}))


if __name__ == "__main__":
    main()
