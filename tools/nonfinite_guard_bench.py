#!/usr/bin/env python
"""Cost of the non-finite gradient guard: the XL/2 ImageNet-256 training step (32x32x4 latents, batch 256, mask 0.5)
with `TrainStep(skip_nonfinite=False)` and `=True`, alternated inside one process on one card.

    python tools/nonfinite_guard_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--batch 256]

Both modes share one network, so the parameter state is allocated once; each round times `TrainStep.step` with CUDA
events in each mode after its own warm-up.  The world-1 check pass (`mdt_nonfinite_check` over the flat gradient) is
also timed on its own.  The card's name and power limit are read in the same run.  One JSON line per mode and one for
the check kernel.
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
from variant_step_bench import C, NCLS, R, card, xl2  # noqa: E402

from maskdit_b200 import ops  # noqa: E402
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
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--mask", type=float, default=0.5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("nonfinite_guard_bench.py measures on a CUDA device; none is visible")
    B, mask = args.batch, args.mask
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = xl2(True).train()
    ema = copy.deepcopy(net).eval()
    # one TrainStep per mode over the same network: the guarded one adds only its flag and counters
    steps = {"guard_off": TrainStep(net, ema, lr=1e-4, global_batch=B),
             "guard_on": TrainStep(net, ema, lr=1e-4, global_batch=B, skip_nonfinite=True)}
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    times = {m: [] for m in steps}
    for _ in range(args.rounds):
        for name, ts in steps.items():
            times[name].append(timed(ts, xs, ys, mask, args.steps, args.warmup))
    skipped = int(steps["guard_on"].skipped_steps)
    # the check pass alone, over the flat gradient the world-1 step checks
    grad, flag = steps["guard_on"].st.grad[:steps["guard_on"].st.n_train], torch.zeros(1, device="cuda")
    for _ in range(3):
        ops.nonfinite_check(grad, flag)
    reps = 20
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        ops.nonfinite_check(grad, flag)
    e1.record()
    torch.cuda.synchronize()
    check_ms = e0.elapsed_time(e1) / reps
    info = card()
    base = statistics.median(times["guard_off"])
    for name in steps:
        ms = statistics.median(times[name])
        print(json.dumps({"mode": name, "batch": B, "mask_ratio": mask, "ms_per_step": round(ms, 2),
                          "ms_per_step_rounds": [round(t, 2) for t in times[name]],
                          "relative_to_guard_off": round(ms / base, 4), "samples_per_s": round(B / ms * 1e3, 1),
                          "steps": args.steps, "warmup": args.warmup, **info}))
    gbytes = grad.numel() * 4 / 1e9
    print(json.dumps({"kernel": "mdt_nonfinite_check", "elements": grad.numel(), "gbytes_read": round(gbytes, 3),
                      "ms": round(check_ms, 3), "gb_per_s": round(gbytes / check_ms * 1e3, 1),
                      "skipped_steps": skipped, **info}))


if __name__ == "__main__":
    main()
