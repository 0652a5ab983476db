#!/usr/bin/env python
"""Cost of the learned loss weighting (`EDMPrecond(logvar_channels=128)`): the XL/2 ImageNet-256 MaskDiT training step
(32x32x4 latents, batch 256, mask 0.5, MAE 0.1) with the weighting off and on, alternated inside one process on one
card, and the loss kernels alone.

    python tools/logvar_step_bench.py [--steps 10] [--warmup 3] [--rounds 3] [--batch 256] [--channels 128]

Two XL/2 training states do not fit on one 80 GB card next to a batch-256 workspace, so one network with the weighting
serves both modes: for the "off" mode its `logvar_channels` is set to 0 around the step, which sends the loss down the
unweighted path (the kernels a network without the weighting runs).  Both modes then share every buffer; the off mode's
optimizer passes still cover w's 128 elements (2e-7 of the blob).  Each round times `TrainStep.step` with CUDA events
in each mode after its own warm-up; the medians over the rounds are reported.  The loss kernel is also timed on its own
at the step's shapes: the unweighted forward + gradient seed (two `mdt_edm_loss` launches), the weighted pair
(`mdt_edm_loss_logvar`), and w's gradient (`mdt_logvar_wgrad`).  The card's name and power limit are read in the same
run.  One JSON line per mode and per kernel.
"""
import argparse
import copy
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from variant_step_bench import C, NCLS, R, card  # noqa: E402

from maskdit_b200 import ops  # noqa: E402
from maskdit_b200.maskdit import Precond_models  # noqa: E402
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
    assert torch.isfinite(loss).all() and torch.isfinite(ts.edm_loss).all()
    return e0.elapsed_time(e1) / steps


def kernel_ms(fn, reps=50):
    for _ in range(5):
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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--mask", type=float, default=0.5)
    ap.add_argument("--channels", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("logvar_step_bench.py measures on a CUDA device; none is visible")
    B, mask, Cl = args.batch, args.mask, args.channels
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = Precond_models["edm"](R, C, num_classes=NCLS, model_type="DiT-XL/2", use_decoder=True,
                                    mae_loss_coef=0.1, pad_cls_token=False, logvar_channels=Cl).train()
    ema = copy.deepcopy(net).eval()
    ts = TrainStep(net, ema, lr=1e-4, global_batch=B)
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    times = {"off": [], "on": []}
    for _ in range(args.rounds):
        for name in times:
            net.logvar_channels = Cl if name == "on" else 0
            times[name].append(timed(ts, xs, ys, mask, args.steps, args.warmup))
    net.logvar_channels = Cl
    info = card()
    base = statistics.median(times["off"])
    for name, ts_ in times.items():
        ms = statistics.median(ts_)
        print(json.dumps({"mode": name, "logvar_channels": Cl if name == "on" else 0, "batch": B, "mask_ratio": mask,
                          "ms_per_step": round(ms, 3), "ms_per_step_rounds": [round(t, 3) for t in ts_],
                          "relative_to_off": round(ms / base, 5), "samples_per_s": round(B / ms * 1e3, 1),
                          "recompute_blocks": ts.recompute_blocks, "steps": args.steps, "warmup": args.warmup,
                          "rounds": args.rounds, **info}))
    # the loss kernels alone at the step's shapes (F of the decoder output: B x 256 tokens x 16)
    L, p = (R // 2) ** 2, 2
    F = torch.randn(B * L, p * p * C, device="cuda")
    xin, y = torch.randn(B, C, R, R, device="cuda"), torch.randn(B, C, R, R, device="cuda")
    sigma = torch.exp(torch.randn(B, device="cuda") * 1.2 - 1.2)
    m = ops.mask_indices(torch.rand(B, L, device="cuda"), int(L * (1 - mask)))["mask"]
    gl = torch.full((B,), 1.0 / B, device="cuda")
    freqs, phases = 2 * math.pi * torch.randn(Cl, device="cuda"), 2 * math.pi * torch.rand(Cl, device="cuda")
    w = 0.1 * torch.randn(Cl, device="cuda")
    _, _, _, du, _ = ops.edm_loss_logvar(F, xin, y, sigma, m, gl, 0.5, 0.1, p, freqs, phases, w)
    dw = torch.zeros(Cl, device="cuda")
    kernels = {
        "mdt_edm_loss forward + seed": lambda: (ops.edm_loss(F, xin, y, sigma, m, None, 0.5, 0.1, p, want_dF=False),
                                                ops.edm_loss(F, xin, y, sigma, m, gl, 0.5, 0.1, p)),
        "mdt_edm_loss_logvar forward + seed": lambda: (
            ops.edm_loss_logvar(F, xin, y, sigma, m, None, 0.5, 0.1, p, freqs, phases, w, want_dF=False),
            ops.edm_loss_logvar(F, xin, y, sigma, m, gl, 0.5, 0.1, p, freqs, phases, w)),
        "mdt_logvar_wgrad": lambda: ops.logvar_wgrad(sigma, freqs, phases, du, dw),
    }
    for name, fn in kernels.items():
        print(json.dumps({"kernel": name, "batch": B, "mask_ratio": mask, "logvar_channels": Cl,
                          "us": round(kernel_ms(fn) * 1e3, 2), **info}))


if __name__ == "__main__":
    main()
