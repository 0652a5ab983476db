#!/usr/bin/env python
"""Cost of the sampler's guidance modes on the XL/2 ImageNet-256 network: the configuration of
`bench.py --workload sampler` (random weights, 32x32x4 latents, 1000 classes, decoder, batch 64, 18 Heun steps = 35
network evaluations), run as

    python tools/guided_sampler_bench.py [--batch 64] [--steps 18] [--iters 3] [--rounds 3]

Rows: unguided; classifier-free guidance 1.5 (one pass at batch 2B per evaluation); CFG 1.5 applied only inside the
noise-level interval (0.28, 5.42], an example interval that is not tuned for this model or for sample quality;
autoguidance (weight 2) with a second XL/2 as the guide, and with an S/2 guide (one pass of each network at batch B).
Random weights are enough: the kernels' run time does not depend on the values.  The rows are timed in turn `--rounds`
times in one process (host clock around `--iters` sampler calls ending in a device synchronise, each row warmed up and
its CUDA graphs captured first); the median round is reported.  Per row: img/s, the network passes per image (a CFG
evaluation is two passes of the network, a guided one a pass of each network) and the GFLOP per image from the
networks' shapes (`val_loss_bench.forward_flops`).  One JSON line per row; the card's name and power limit are read
in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from val_loss_bench import forward_flops  # noqa: E402
from variant_step_bench import C, NCLS, R, card, xl2  # noqa: E402

from maskdit_b200.maskdit import Precond_models  # noqa: E402
from maskdit_b200.sampler import edm_sampler  # noqa: E402

INTERVAL = (0.28, 5.42)     # an example: not tuned for this model


def eval_sigmas(num_steps, sigma_min=0.002, sigma_max=80.0, rho=7):
    """The sigma of every network evaluation of edm_sampler without churn (2N - 1 of them)."""
    i = np.arange(num_steps, dtype=np.float64)
    t = (sigma_max ** (1 / rho) + i / (num_steps - 1) * (sigma_min ** (1 / rho) - sigma_max ** (1 / rho))) ** rho
    return [float(t[k]) for k in range(num_steps)] + [float(t[k]) for k in range(1, num_steps)]


def rows(guides):
    return [("unguided", {}, None),
            ("cfg 1.5", dict(cfg_scale=1.5), None),
            ("cfg 1.5, interval (0.28, 5.42] (example, untuned)", dict(cfg_scale=1.5, guidance_interval=INTERVAL), None),
            ("autoguidance 2.0, XL/2 guide", dict(guide_net=guides["XL/2"], guidance=2.0), "XL/2"),
            ("autoguidance 2.0, S/2 guide", dict(guide_net=guides["S/2"], guidance=2.0), "S/2")]


def passes_and_flops(kw, guide, sigmas, f_main, f_guide):
    passes = flops = 0
    for s in sigmas:
        iv = kw.get("guidance_interval")
        inside = iv is None or iv[0] < s <= iv[1]
        if "cfg_scale" in kw and inside:
            passes, flops = passes + 2, flops + 2 * f_main
        elif guide is not None and inside:
            passes, flops = passes + 2, flops + f_main + f_guide[guide]
        else:
            passes, flops = passes + 1, flops + f_main
    return passes, flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=18)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("guided_sampler_bench.py measures on a CUDA device; none is visible")
    info = card()
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = xl2(True).eval()
        guides = {"XL/2": xl2(True).eval(),
                  "S/2": Precond_models["edm"](R, C, num_classes=NCLS, model_type="DiT-S/2", use_decoder=True,
                                               mae_loss_coef=0.1, pad_cls_token=False).eval()}
    f_main = forward_flops(net)
    f_guide = {k: forward_flops(g) for k, g in guides.items()}
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(args.batch, C, R, R, generator=g).cuda()
    lab = torch.nn.functional.one_hot(torch.randint(0, NCLS, (args.batch,), generator=g), NCLS).float().cuda()
    sigmas = eval_sigmas(args.steps)
    table = rows(guides)

    def run(kw):
        with torch.no_grad():
            return edm_sampler(net, lat, lab, num_steps=args.steps, **kw)

    for _, kw, _ in table:      # warm-up: captures every row's CUDA graphs
        run(kw)
    torch.cuda.synchronize()
    times = {name: [] for name, _, _ in table}
    for _ in range(args.rounds):
        for name, kw, _ in table:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.iters):
                run(kw)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) / args.iters)
    for name, kw, guide in table:
        ts = sorted(times[name])
        sec = ts[len(ts) // 2]
        passes, flops = passes_and_flops(kw, guide, sigmas, f_main, f_guide)
        print(json.dumps({"measure": "guided_sampler", "row": name, "model": "DiT-XL/2 (MaskDiT, decoder)",
                          "batch": args.batch, "num_steps": args.steps, "evaluations_per_image": len(sigmas),
                          "network_passes_per_image": passes, "gflop_per_image": round(flops / 1e9, 1),
                          "img_per_s": round(args.batch / sec, 2), "seconds_per_batch": round(sec, 4),
                          "rounds_seconds": [round(t, 4) for t in times[name]],
                          "tflop_per_s": round(args.batch * flops / sec / 1e12, 1), **info}), flush=True)


if __name__ == "__main__":
    main()
