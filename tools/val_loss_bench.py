#!/usr/bin/env python
"""Cost of the held-out denoising loss (maskdit_b200/validate.py) on the XL/2 ImageNet-256 network (32x32x4 latents,
1000 classes, decoder), and its effect on the training step's memory plan.

    python tools/val_loss_bench.py [--count 10000] [--levels 8] [--batch 256 64] [--steps 6] [--val_count 256]

1. Throughput: `validate()` of an eval-mode network on `--count` synthetic held-out items x `--levels` levels, timed end
   to end with a host clock (it returns host tensors, so the device work is finished).  Beside it, on the same rows:
   the host side alone (draws, row assembly) through a scorer that launches nothing, and the device side alone (step
   front + eval forward + EDM loss on rows already on the device, CUDA events).  The algorithmic count is the network's
   forward FLOPs per evaluation from its shapes (`forward_flops`), so TFLOP/s = evaluations x that / time.
2. Memory plan: the batch-256, mask-0.5 training step (`TrainStep`, net + EMA + AdamW) without validation and with
   `validate(ema, ...)` at `--val_count` items and the micro-batch as row batch every second step, as
   `train.py --val_every 2` runs it.  Each mode picks its own recompute count (the engine's remembered choice is
   cleared) and reports it with the peak allocated memory and the step time.
One JSON line per measurement; the card's name and power limit are read in the same run.
"""
import argparse
import copy
import gc
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from variant_step_bench import C, NCLS, R, card, xl2  # noqa: E402

from maskdit_b200 import validate as V  # noqa: E402
from maskdit_b200.train_step import TrainStep  # noqa: E402


def forward_flops(net):
    """Multiply-adds x 2 of one unmasked eval forward (one batch row) from the network's shapes: patch embedding,
    timestep / label conditioning, the adaLN projections, every block's linears and attention products, the
    encoder-to-decoder linear and the final layer."""
    m = net.model
    p, D, T = m.patch_size, m.hidden_size, m.num_patches
    d = m.decoder_hidden_size if m.decoder_depth else D
    cin = p * p * m.in_channels

    def block(width, tokens):
        return tokens * (12 * width * width + 2 * tokens * width)  # qkv, proj, fc1, fc2; QK^T and PV

    macs = T * cin * D                                   # patch embedding
    macs += 256 * D + D * D                              # timestep MLP (the label embedding is a table lookup)
    macs += m.depth * (D * 6 * D + block(D, T))          # encoder: adaLN projection + block
    if m.decoder_depth:
        macs += T * D * d                                # decoder_layer
        macs += m.decoder_depth * (D * 6 * d + block(d, T))
    macs += D * 2 * d + T * d * cin                      # final layer: adaLN, linear
    return 2 * macs


class NullScorer:
    def __call__(self, moments, eps, rnd_normal, noise, labels):
        return torch.zeros(moments.shape[0])


def device_ms_per_row(net, held, levels, batch, reps=5):
    """Step front + eval forward + EDM loss on `batch` rows already on the device (CUDA events)."""
    sc = V.CudaScorer(net)
    rows = []
    V.score_items(lambda *a: rows.append(a) or torch.zeros(a[0].shape[0]), held, 0, -(-batch // levels), levels,
                  batch=batch)
    mom, eps, z, noise, lab = (None if t is None else t.cuda() for t in rows[0])
    for _ in range(2):
        sc(mom, eps, z, noise, lab)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        sc(mom, eps, z, noise, lab)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps / mom.shape[0]


def throughput(args, info):
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = xl2(True).eval()
    flops = forward_flops(net)
    held = V.HeldOut.synthetic(args.count, R, C, NCLS, seed=0)
    evals = args.count * args.levels
    for batch in args.batch:
        V.validate(net, V.HeldOut(held.moments[:64], held.labels[:64]), levels=args.levels, batch=batch)   # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = V.validate(net, held, levels=args.levels, batch=batch)
        total = time.perf_counter() - t0
        t0 = time.perf_counter()
        V.validate(NullScorer(), held, levels=args.levels, batch=batch)
        host = time.perf_counter() - t0
        dev_ms = device_ms_per_row(net, held, args.levels, batch)
        print(json.dumps({"measure": "validate", "model": "DiT-XL/2 (MaskDiT, decoder)", "items": args.count,
                          "levels": args.levels, "evaluations": evals, "batch_rows": batch,
                          "gflop_per_evaluation": round(flops / 1e9, 2), "seconds": round(total, 2),
                          "evaluations_per_s": round(evals / total, 1),
                          "tflop_per_s": round(evals * flops / total / 1e12, 1),
                          "host_only_seconds": round(host, 2),
                          "device_ms_per_evaluation": round(dev_ms, 4),
                          "device_only_tflop_per_s": round(flops / dev_ms / 1e9, 1),
                          "device_share_of_total": round(evals * dev_ms / 1e3 / total, 3),
                          "mean_loss": round(res["mean"], 5), **info}), flush=True)
    del net
    gc.collect()
    torch.cuda.empty_cache()


def step_memory(args, info):
    B, mask = 256, 0.5
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = xl2(True).train()
    ema = copy.deepcopy(net).eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    held = V.HeldOut.synthetic(args.val_count, R, C, NCLS, seed=0)
    for mode in ("val_off", "val_on"):
        ts = TrainStep(net, ema, lr=1e-4, global_batch=B)
        ts._engine._auto_recompute = {}
        torch.cuda.reset_peak_memory_stats()
        times, vals = [], []
        for i in range(args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loss = ts.step(xs[i % 2], ys[i % 2], mask, 0.1)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            if mode == "val_on" and (i + 1) % 2 == 0:
                t0 = time.perf_counter()
                vals.append(V.validate(ema, held, levels=8, batch=B)["mean"])
                vals[-1] = (vals[-1], round(time.perf_counter() - t0, 3))
            assert ts.recompute_blocks == ts._engine.recompute_blocks
        assert torch.isfinite(loss).all()
        steady = sorted(times[2:])[len(times[2:]) // 2]
        print(json.dumps({"measure": "train_step_memory", "mode": mode, "batch": B, "mask_ratio": mask,
                          "recompute_blocks": ts.recompute_blocks,
                          "peak_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                          "median_step_ms": round(steady * 1e3, 1), "steps": args.steps,
                          "validations": [{"mean": round(m, 5), "seconds": s} for m, s in vals],
                          "val_items": args.val_count if mode == "val_on" else 0, **info}), flush=True)
        del ts
        gc.collect()
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--count", type=int, default=10000)
    ap.add_argument("--levels", type=int, default=8)
    ap.add_argument("--batch", type=int, nargs="+", default=[256, 64])
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--val_count", type=int, default=256)
    ap.add_argument("--skip", choices=["throughput", "memory"], default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("val_loss_bench.py measures on a CUDA device; none is visible")
    info = card()
    if args.skip != "memory":
        step_memory(args, info)
    if args.skip != "throughput":
        throughput(args, info)


if __name__ == "__main__":
    main()
