#!/usr/bin/env python
"""Cost of activation recomputation in the XL/2 training step at 256 px (32x32x4 latents), one GPU.

    python tools/recompute_step_bench.py [--steps 5] [--warmup 2] [--rounds 2]

Variants (`TrainStep(recompute_blocks=...)`):
    maskdit_r0       MaskDiT (decoder), mask 0.5, batch 256, nothing recomputed
    maskdit_rfull    the same with all 28 + 8 blocks recomputed
    dit_b256_auto    decoder-less DiT, no mask, batch 256, the count TrainStep picks itself (87.9 GB of workspace at
                     r = 0 does not fit one 80 GB card)
    dit_b128x2       the same samples per step as 2 micro-batches of 128 (`grad_accum=2`), nothing recomputed
Each round builds every variant in turn (net + EMA + fused AdamW, seeded inputs), warms it up and times `TrainStep.step`
with CUDA events, then frees it: the variants alternate inside one process on one card.  One JSON line per variant
with the median over rounds: samples/s, ms per step, the recompute count in use, `mdt_workspace_bytes` of a pass at
that count, peak allocated memory, and the card's name, power limit and max SM clock read in the same run.
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

from maskdit_b200.train_step import TrainStep  # noqa: E402

B = 256


def run_variant(use_decoder, mask, recompute, grad_accum, steps, warmup):
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = xl2(use_decoder).train()
    ema = copy.deepcopy(net).eval()
    ts = TrainStep(net, ema, lr=1e-4, global_batch=B, recompute_blocks=recompute)
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    for i in range(warmup):
        ts.step(xs[i % 2], ys[i % 2], mask, 0.1, grad_accum=grad_accum)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        loss = ts.step(xs[i % 2], ys[i % 2], mask, 0.1, grad_accum=grad_accum)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    assert torch.isfinite(loss).all()
    peak = torch.cuda.max_memory_allocated()
    r = ts.recompute_blocks
    mb = B // grad_accum
    T = int(net.model.num_patches * (1 - mask)) if mask > 0 else 0
    ws = net._engine.workspace_bytes(mb, T, True, r)
    del ts, ema, net, xs, ys, loss
    gc.collect()
    torch.cuda.empty_cache()
    return ms, peak, r, ws


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("recompute_step_bench.py measures on a CUDA device; none is visible")
    variants = [("maskdit_r0", True, 0.5, 0, 1), ("maskdit_rfull", True, 0.5, 36, 1),
                ("dit_b256_auto", False, 0.0, None, 1), ("dit_b128x2", False, 0.0, 0, 2)]
    times = {v[0]: [] for v in variants}
    last = {}
    for _ in range(args.rounds):
        for name, dec, mask, rc, acc in variants:
            ms, *last[name] = run_variant(dec, mask, rc, acc, args.steps, args.warmup)
            times[name].append(ms)
    info = card()
    for name, dec, mask, rc, acc in variants:
        ms = statistics.median(times[name])
        peak, r, ws = last[name]
        print(json.dumps({"variant": name, "use_decoder": dec, "batch": B, "grad_accum": acc, "mask_ratio": mask,
                          "recompute_blocks": r, "samples_per_s": round(B / ms * 1e3, 1), "ms_per_step": round(ms, 2),
                          "ms_per_step_rounds": [round(t, 2) for t in times[name]], "workspace_bytes": ws,
                          "peak_allocated_bytes": peak, "steps": args.steps, "warmup": args.warmup, **info}))


if __name__ == "__main__":
    main()
