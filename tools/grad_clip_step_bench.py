#!/usr/bin/env python
"""Cost of gradient-norm clipping: the XL/2 ImageNet-256 training step (32x32x4 latents, batch 256, mask 0.5) at world
1 with `max_grad_norm` None / inf / 1.0, each without and with `skip_nonfinite`, alternated inside one process on one
card.

    python tools/grad_clip_step_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--batch 256]

One TrainStep built with both features serves every mode: its switches (`max_grad_norm`, and the guard's flag and
counters) are set per mode, so the modes share one set of buffers and differ only in what the step launches.  Each
round times `TrainStep.step` with CUDA events in each mode after its own warm-up; the medians over the rounds are
reported.  The norm pass (`mdt_grad_sumsq`) is also timed on its own over the fp32 flat gradient (with and without the
fused check), over a bf16 buffer of the same length, and beside it the check pass it replaces under the guard
(`mdt_nonfinite_check`).  The card's name and power limit are read in the same run.  One JSON line per mode and per
kernel.  The world > 1 cost of a finite bound (every optimizer pass waits for the last chunk's exchange) needs several
GPUs and is not measured here.
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

MODES = {"off": (None, False), "inf": (float("inf"), False), "c1": (1.0, False),
         "off+guard": (None, True), "inf+guard": (float("inf"), True), "c1+guard": (1.0, True)}


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


def kernel_ms(fn, reps=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
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
        sys.exit("grad_clip_step_bench.py measures on a CUDA device; none is visible")
    B, mask = args.batch, args.mask
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = xl2(True).train()
    ema = copy.deepcopy(net).eval()
    ts = TrainStep(net, ema, lr=1e-4, global_batch=B, skip_nonfinite=True, max_grad_norm=1.0)
    flag, counts = ts._flag, ts._counts
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    times = {m: [] for m in MODES}
    norms = {}
    for _ in range(args.rounds):
        for name, (c, guard) in MODES.items():
            ts.max_grad_norm = c
            ts._flag, ts._counts = (flag, counts) if guard else (None, None)
            times[name].append(timed(ts, xs, ys, mask, args.steps, args.warmup))
            if c is not None:
                norms[name] = float(ts.grad_norm)
    skipped = int(counts[1])
    info = card()
    base = statistics.median(times["off"])
    for name, (c, guard) in MODES.items():
        ms = statistics.median(times[name])
        print(json.dumps({"mode": name, "max_grad_norm": c, "skip_nonfinite": guard, "batch": B, "mask_ratio": mask,
                          "ms_per_step": round(ms, 2), "ms_per_step_rounds": [round(t, 2) for t in times[name]],
                          "relative_to_off": round(ms / base, 4), "samples_per_s": round(B / ms * 1e3, 1),
                          "last_grad_norm": norms.get(name), "steps": args.steps, "warmup": args.warmup, **info}))
    # the passes alone, over the flat gradient the world-1 step reads
    n = ts.st.n_train
    grad = ts.st.grad[:n]
    g16 = grad.to(torch.bfloat16)
    slot, f = torch.zeros(1, dtype=torch.float64, device="cuda"), torch.zeros(1, device="cuda")
    kernels = {"mdt_grad_sumsq fp32": (lambda: ops.grad_sumsq(grad, slot, ts._gn_scratch), grad.numel() * 4),
               "mdt_grad_sumsq fp32 + check": (lambda: ops.grad_sumsq(grad, slot, ts._gn_scratch, flag=f),
                                               grad.numel() * 4),
               "mdt_grad_sumsq bf16": (lambda: ops.grad_sumsq(g16, slot, ts._gn_scratch), g16.numel() * 2),
               "mdt_nonfinite_check fp32": (lambda: ops.nonfinite_check(grad, f), grad.numel() * 4)}
    for name, (fn, nbytes) in kernels.items():
        ms = kernel_ms(fn)
        print(json.dumps({"kernel": name, "elements": n, "gbytes_read": round(nbytes / 1e9, 3), "ms": round(ms, 3),
                          "gb_per_s": round(nbytes / 1e9 / ms * 1e3, 1), "skipped_steps": skipped, **info}))


if __name__ == "__main__":
    main()
