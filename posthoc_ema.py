#!/usr/bin/env python
"""Post-hoc EMA (Karras et al., "Analyzing and Improving the Training Dynamics of Diffusion Models", CVPR 2024, §3):
reconstruct the EMA of any relative width from the power-function EMA snapshots a run wrote with
`train.py --phema_sigma_rel 0.05,0.10 --phema_every N`.

    python posthoc_ema.py --snapshots <results_dir>/phema --sigma_rel 0.08 [0.12 ...] [--step N] --out ema.pt

Every snapshot up to step N (default: the last one) and every profile in it enters one float64 least-squares fit of
the target profile's weight density (`maskdit_b200/phema.py`); the snapshots are then combined with those coefficients
one file at a time in float64, so at most one snapshot is in memory next to the sum.  The output holds
`{"ema": state_dict, "posthoc": {sigma_rel, step, snapshots, coefficients, fit_residual}}`: `generate.py --ckpt_path`
samples from it unchanged.  With several widths, `--out x.pt` becomes x-<sigma_rel>.pt per width.  Runs on the CPU.
"""
import argparse
import os
import re

import numpy as np
import torch

from maskdit_b200 import phema

_NAME = re.compile(r"phema-(\d+)\.pt$")


def list_snapshots(directory, step=None):
    """[(step, path)] of the snapshot files in `directory` up to `step` (default: all), in step order."""
    found = sorted((int(m.group(1)), os.path.join(directory, f)) for f in os.listdir(directory)
                   if (m := _NAME.fullmatch(f)))
    if step is not None:
        found = [(s, p) for s, p in found if s <= step]
    if not found:
        raise SystemExit(f"no post-hoc EMA snapshots (phema-<step>.pt) in {directory}"
                         + (f" up to step {step}" if step is not None else ""))
    return found


def _load(path):
    return torch.load(path, map_location="cpu", weights_only=True, mmap=True)


def read_index(files):
    """The (t, gamma) of every profile of every file, t counted from the shared origin.  Refuses mixed origins."""
    index, origin = [], None
    for _, path in files:
        snap = _load(path)
        if origin is None:
            origin = int(snap["origin"])
        elif int(snap["origin"]) != origin:
            raise SystemExit(f"{path}: profiles start at step {snap['origin']}, the earlier snapshots at {origin}; "
                             "snapshots of one fit must share their origin")
        t = int(snap["step"]) - origin
        for j, p in enumerate(snap["profiles"]):
            index.append((path, j, t, float(p["gamma"]), float(p["sigma_rel"])))
        del snap
    return index, origin


def reconstruct(files, sigma_rel, step=None):
    """-> (state dict in fp32, info).  `step` (a run step >= the last snapshot's) defaults to the last snapshot."""
    index, origin = read_index(files)
    last = max(origin + t for _, _, t, _, _ in index)
    step = last if step is None else step
    if step > last:
        raise SystemExit(f"the last snapshot is at step {last}: the weights after it are unknown, so no EMA at step {step}")
    gamma = phema.sigma_rel_to_gamma(sigma_rel)
    x, residual = phema.solve([t for *_, t, _, _ in index], [g for *_, g, _ in index], step - origin, gamma)
    acc = None
    for path in dict.fromkeys(p for p, *_ in index):     # one file at a time, in step order
        snap = _load(path)
        for (p, j, *_), xi in zip(index, x):
            if p != path:
                continue
            sd = snap["profiles"][j]["ema"]
            if acc is None:
                acc = {k: torch.zeros(v.shape, dtype=torch.float64) for k, v in sd.items()}
            for k, v in sd.items():
                acc[k].add_(v.double(), alpha=float(xi))
        del snap
    info = {"sigma_rel": float(sigma_rel), "gamma": gamma, "step": int(step), "origin": origin,
            "snapshots": [{"file": os.path.basename(p), "profile": j, "t": t, "gamma": g, "sigma_rel": s}
                          for p, j, t, g, s in index],
            "coefficients": [float(v) for v in x], "fit_residual": residual}
    return {k: v.float() for k, v in acc.items()}, info


def _out_path(out, sigma_rel, several):
    if not several:
        return out
    stem, ext = os.path.splitext(out)
    return f"{stem}-{sigma_rel:g}{ext or '.pt'}"


def main(argv=None):
    ap = argparse.ArgumentParser("Reconstruct an EMA of any width from power-function EMA snapshots")
    ap.add_argument("--snapshots", required=True, help="directory of phema-<step>.pt files (<results_dir>/phema)")
    ap.add_argument("--sigma_rel", type=float, nargs="+", required=True, help="relative EMA width(s) to build")
    ap.add_argument("--step", type=int, default=None, help="run step of the EMA (default: the last snapshot's); "
                                                           "the snapshots up to it enter the fit")
    ap.add_argument("--out", required=True)
    args = ap.parse_args(argv)
    files = list_snapshots(args.snapshots, args.step)
    outs = []
    for s in args.sigma_rel:
        sd, info = reconstruct(files, s, args.step)
        path = _out_path(args.out, s, len(args.sigma_rel) > 1)
        if os.path.dirname(path):
            os.makedirs(os.path.dirname(path), exist_ok=True)
        torch.save({"ema": sd, "posthoc": info}, path)
        big = np.abs(info["coefficients"]).max()
        print(f"sigma_rel {s:g} (gamma {info['gamma']:.3f}) at step {info['step']}: {len(info['snapshots'])} profiles "
              f"from {len(files)} snapshots, largest |coefficient| {big:.3g}, relative L2 residual of the profile fit "
              f"{info['fit_residual']:.3e} -> {path}", flush=True)
        outs.append(path)
    return outs


if __name__ == "__main__":
    main()
