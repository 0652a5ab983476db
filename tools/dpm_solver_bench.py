#!/usr/bin/env python
"""Cost and accuracy of multistep DPM-Solver++ (`dpm_solver_sampler`) against the Heun `edm_sampler`, on one card:
  * speed: XL/2 ImageNet-256 (32x32x4 latents) at batch 64 with CFG 1.5, `edm_sampler` at 18 steps (35 evaluations)
    against `dpm_solver_sampler` (order 3) at 10, 15 and 20 evaluations; img/s of the median round;
  * accuracy without FID: a toy DiT-S/2 at R = 8 trained here for 400 EDM steps on four classes of two latents +-P_c,
    and the rms distance of each sampler's output (DPM-Solver++ orders 1-3 at 6, 12 and 24 evaluations, Heun at 3, 6
    and 12 steps) to `edm_sampler` at 256 steps, on 128 seeded latents.  `tests/test_dpm_solver_gpu.py` trains the
    same toy (both in deterministic mode, so the network is the same) and checks that the distance falls with the
    evaluation count for orders 2 and 3.

    python tools/dpm_solver_bench.py [--rounds 3] [--iters 2] [--sample_batch 64]

The card's name and power limit are read in the same run.  One JSON line per measurement.
"""
import argparse
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

from maskdit_b200.maskdit import Precond_models  # noqa: E402
from maskdit_b200.sampler import dpm_solver_sampler, edm_sampler  # noqa: E402


def train_toy(steps=400):
    """DiT-S/2 at R = 8 trained with the EDM loss on four classes of two latents +-P_c (per-element rms 0.5), the
    consistency-tuning toy of tests/test_ect_gpu.py.  Returns (net in eval mode, 128 latents, their one-hot labels)."""
    from maskdit_b200.loss import EDMLoss
    from maskdit_b200.train_step import TrainStep
    ncls, r, B = 4, 8, 64
    gen = torch.Generator().manual_seed(0)
    P = torch.randn(ncls, 4, r, r, generator=gen)
    P = (P * 0.5 / P.pow(2).mean(dim=(1, 2, 3), keepdim=True).sqrt()).cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    torch.manual_seed(0)
    net = Precond_models["edm"](img_resolution=r, img_channels=4, num_classes=ncls, model_type="DiT-S/2",
                                use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False).cuda().train()
    ts = TrainStep(net, None, lr=5e-4, loss_fn=EDMLoss())
    for _ in range(steps):
        c = torch.randint(0, ncls, (B,), device="cuda", generator=g)
        s = torch.randint(0, 2, (B,), device="cuda", generator=g).float() * 2 - 1
        ts.step(P[c] * s.view(-1, 1, 1, 1), torch.eye(ncls, device="cuda")[c], mask_ratio=0.0, mae_loss_coef=0.0)
    c = torch.arange(128, device="cuda") % ncls
    z = torch.randn(128, 4, r, r, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    return net.eval(), z, torch.eye(ncls, device="cuda")[c]


def toy_errors(net, z, lab, evals=(6, 12, 24), orders=(1, 2, 3), heun_steps=256):
    """rms distance of each sampler's output to `edm_sampler` at `heun_steps` steps:
    {(sampler, network evaluations): distance}; Heun runs n / 2 steps (n - 1 evaluations) for each n in `evals`."""
    with torch.no_grad():
        ref = edm_sampler(net, z, lab, num_steps=heun_steps)
        dist = lambda x: (x - ref).pow(2).mean().sqrt().item()  # noqa: E731
        out = {}
        for n in evals:
            for o in orders:
                out[(f"dpm_solver_order{o}", n)] = dist(dpm_solver_sampler(net, z, lab, num_steps=n, order=o))
            out[("edm_heun", n - 1)] = dist(edm_sampler(net, z, lab, num_steps=n // 2))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--sample_batch", type=int, default=64)
    ap.add_argument("--edm_steps", type=int, default=18)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("dpm_solver_bench.py measures on a CUDA device; none is visible")
    info = card()

    torch.use_deterministic_algorithms(True)      # as in the test, so the distances are the test's
    net, z, lab = train_toy()
    errs = toy_errors(net, z, lab)
    torch.use_deterministic_algorithms(False)
    for (name, evals), d in sorted(errs.items(), key=lambda kv: (kv[0][1], kv[0][0])):
        print(json.dumps({"measure": "toy_distance_to_heun256", "sampler": name, "evaluations_per_image": evals,
                          "rms_distance": float(f"{d:.4e}"), "model": "DiT-S/2 toy, R 8, 400 EDM steps", **info}),
              flush=True)
    del net
    torch.cuda.empty_cache()

    with torch.device("cuda"):
        net = Precond_models["edm"](R, C, num_classes=NCLS, model_type="DiT-XL/2", use_decoder=True,
                                    mae_loss_coef=0.1, pad_cls_token=False).eval()
    gen = torch.Generator().manual_seed(0)
    lat = torch.randn(args.sample_batch, C, R, R, generator=gen).cuda()
    lab = torch.nn.functional.one_hot(torch.randint(0, NCLS, (args.sample_batch,), generator=gen), NCLS).float().cuda()
    runs = {("edm_sampler", 2 * args.edm_steps - 1):
            lambda: edm_sampler(net, lat, lab, cfg_scale=1.5, num_steps=args.edm_steps)}
    for n in (10, 15, 20):
        runs[("dpm_solver_sampler", n)] = lambda n=n: dpm_solver_sampler(net, lat, lab, cfg_scale=1.5, num_steps=n)
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
                    out = fn()
                torch.cuda.synchronize()
                assert torch.isfinite(out).all()
                stimes[k].append((time.perf_counter() - t0) / args.iters)
    for (name, evals), t in stimes.items():
        sec = statistics.median(t)
        print(json.dumps({"measure": "sampler", "sampler": name, "model": "DiT-XL/2 (MaskDiT, decoder)",
                          "batch": args.sample_batch, "cfg_scale": 1.5, "evaluations_per_image": evals,
                          "img_per_s": round(args.sample_batch / sec, 2), "rounds_seconds": [round(v, 4) for v in t],
                          **info}), flush=True)


if __name__ == "__main__":
    main()
