#!/usr/bin/env python
"""Cost of model guidance (MG) against EDM training on one card, in one process: the XL/2 ImageNet-256 MaskDiT training
step (32x32x4 latents, batch 256, mask 0.5, MAE 0.1) with the EDM loss, the MG loss (one extra no-gradient masked
forward with the null labels) and, for comparison, the ECT loss (one extra no-gradient masked forward of its own),
alternated round by round; each mode warms up before its timed window (CUDA events), medians and the peak memory of
each mode's rounds reported.

    python tools/mg_bench.py [--steps 10] [--warmup 3] [--rounds 3] [--batch 256]

All losses drive the same network and TrainStep.  MG at scale 1.5 over all noise levels: the work of a step does not
depend on the scale or the interval.  The card's name and power limit are read in the same run.  One JSON line per
mode.  An MG network samples on the unguided path, whose rate tools/guided_sampler_bench.py measures.
"""
import argparse
import copy
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ect_bench import timed  # noqa: E402
from variant_step_bench import C, NCLS, R, card  # noqa: E402

from maskdit_b200.loss import ECTLoss, EDMLoss, MGLoss  # noqa: E402
from maskdit_b200.maskdit import Precond_models  # noqa: E402
from maskdit_b200.train_step import TrainStep  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--mask", type=float, default=0.5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mg_bench.py measures on a CUDA device; none is visible")
    info = card()
    B, mask = args.batch, args.mask
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = Precond_models["edm"](R, C, num_classes=NCLS, model_type="DiT-XL/2", use_decoder=True,
                                    mae_loss_coef=0.1, pad_cls_token=False).train()
    ema = copy.deepcopy(net).eval()
    ect = ECTLoss(stage_steps=1000)
    ts = TrainStep(net, ema, lr=1e-4, global_batch=B, loss_fn=ect)   # owns the stage word the ECT loss reads
    losses = {"edm": EDMLoss(), "mg": MGLoss(scale=1.5), "ect": ect}
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    times = {k: [] for k in losses}
    peak = {k: 0 for k in losses}
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


if __name__ == "__main__":
    main()
