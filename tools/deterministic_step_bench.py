#!/usr/bin/env python
"""Cost of the deterministic mode: the XL/2 ImageNet-256 training step (32x32x4 latents, batch 256, mask 0.5) with
`torch.use_deterministic_algorithms` off and on, alternated inside one process on one card.

    python tools/deterministic_step_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--batch 256]

Each round times `TrainStep.step` with CUDA events in the default mode, then in the deterministic mode (each after its
own warm-up).  Then one step per mode runs with the GEMM probes on (`mdt_gemm_profile_*`): the launch sequence is the
same in both modes, so launch i of one mode is launch i of the other; the launches are grouped by their 2*M*N*K and
the groups whose time changed most are listed (the accumulating GEMMs run one k-slice in the deterministic mode; the
DGELU dgrad's time includes its ordered column sum there).  The card's name and power limit are read in the same run.
One JSON line per mode and one for the GEMM groups.
"""
import argparse
import copy
import ctypes
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from variant_step_bench import C, NCLS, R, card, xl2  # noqa: E402

from maskdit_b200 import _lib  # noqa: E402
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


def gemm_launches(ts, x, y, mask):
    L = _lib.lib()
    L.mdt_gemm_profile_enable(1)
    ts.step(x, y, mask, 0.1)
    torch.cuda.synchronize()
    L.mdt_gemm_profile_enable(0)
    n = L.mdt_gemm_profile_read(None, None, 0)
    ms, fl = (ctypes.c_float * n)(), (ctypes.c_double * n)()
    L.mdt_gemm_profile_read(ms, fl, n)
    return list(ms), list(fl)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--mask", type=float, default=0.5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("deterministic_step_bench.py measures on a CUDA device; none is visible")
    flag = torch.are_deterministic_algorithms_enabled()
    B, mask = args.batch, args.mask
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = xl2(True).train()
    ts = TrainStep(net, copy.deepcopy(net).eval(), lr=1e-4, global_batch=B)
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5 for _ in range(2)]
    ys = [torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), device="cuda", generator=g), NCLS).float()
          for _ in range(2)]
    modes = (("default", False), ("deterministic", True))
    times = {m: [] for m, _ in modes}
    try:
        for _ in range(args.rounds):
            for name, det in modes:
                torch.use_deterministic_algorithms(det)
                times[name].append(timed(ts, xs, ys, mask, args.steps, args.warmup))
        launches = {}
        for name, det in modes:
            torch.use_deterministic_algorithms(det)
            launches[name] = gemm_launches(ts, xs[0], ys[0], mask)
    finally:
        torch.use_deterministic_algorithms(flag)
        _lib.sync_deterministic()
    info = card()
    base = statistics.median(times["default"])
    for name, _ in modes:
        ms = statistics.median(times[name])
        print(json.dumps({"mode": name, "batch": B, "mask_ratio": mask, "ms_per_step": round(ms, 2),
                          "ms_per_step_rounds": [round(t, 2) for t in times[name]],
                          "relative_to_default": round(ms / base, 4), "samples_per_s": round(B / ms * 1e3, 1),
                          "steps": args.steps, "warmup": args.warmup, **info}))
    (ms0, fl0), (ms1, fl1) = launches["default"], launches["deterministic"]
    assert fl0 == fl1, "the GEMM launch sequences of the two modes differ"
    groups = {}
    for a, b, f in zip(ms0, ms1, fl0):
        gr = groups.setdefault(f, [0, 0.0, 0.0])
        gr[0] += 1
        gr[1] += a
        gr[2] += b
    rows = sorted(groups.items(), key=lambda kv: kv[1][1] - kv[1][2])
    print(json.dumps({"gemm_launches": len(fl0), "gemm_ms_default": round(sum(ms0), 2),
                      "gemm_ms_deterministic": round(sum(ms1), 2),
                      "largest_changes": [{"flops": f, "launches": n, "ms_default_per_launch": round(a / n, 4),
                                           "ms_deterministic_per_launch": round(b / n, 4)}
                                          for f, (n, a, b) in rows[:12]], **info}))


if __name__ == "__main__":
    main()
