#!/usr/bin/env python
"""Score checkpoints, or EMA widths rebuilt from post-hoc EMA snapshots, by their held-out denoising loss
(`maskdit_b200/validate.py`): the EDM loss of the eval-mode network on the first N items of the latent LMDB split
`<val_root>/val`, at K fixed noise levels with fixed noise, so every row of the table is comparable with every other.
It is a proxy for sample quality, not FID.

    python val_loss.py --config <yaml> --ckpt a.pt b.pt ... [--key ema|model] [--val_root DIR] [--count N] [--levels K]
    python val_loss.py --config <yaml> --snapshots <results_dir>/phema --sigma_rel 0.05 0.075 0.10 0.15 [--step S] ...

The second form rebuilds each width with posthoc_ema.reconstruct and scores it.  One table row per checkpoint or width,
then the best (lowest mean) row; `--json PATH` writes the same numbers.  Under torchrun every rank scores a slice of
the items (as generate.py deals seeds) and rank 0 prints.
"""
import argparse
import json
import os

import torch

from maskdit_b200.config import build_net, load_config
from maskdit_b200.validate import HeldOut, format_levels, validate


def build_parser():
    ap = argparse.ArgumentParser("Held-out denoising loss of checkpoints or post-hoc EMA widths")
    ap.add_argument("--config", required=True)
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--ckpt", nargs="+", help="checkpoints to score (train.py's, posthoc_ema.py's or the reference's)")
    src.add_argument("--snapshots", help="directory of post-hoc EMA snapshots (<results_dir>/phema)")
    ap.add_argument("--sigma_rel", type=float, nargs="+", default=None, help="EMA widths to rebuild and score")
    ap.add_argument("--step", type=int, default=None,
                    help="run step of the rebuilt EMAs (default: the last snapshot's)")
    ap.add_argument("--key", choices=["ema", "model"], default="ema", help="which weights of a checkpoint to score")
    ap.add_argument("--val_root", default=None, help="latent LMDB root holding the val split (default: data.root)")
    ap.add_argument("--synthetic", action="store_true",
                    help="held-out moments drawn from a fixed seed instead of a dataset (as train.py --synthetic)")
    ap.add_argument("--count", type=int, default=10000, help="held-out items: the first N of the split")
    ap.add_argument("--levels", type=int, default=8, help="noise levels per item")
    ap.add_argument("--batch", type=int, default=64, help="network evaluations (item x level rows) per forward")
    ap.add_argument("--seed", type=int, default=0, help="seed of the per-item draws")
    ap.add_argument("--json", default=None, help="also write the numbers to this JSON file")
    return ap


def sources(args):
    """(name, state dict) of every network to score, loaded one at a time."""
    if args.ckpt:
        for path in args.ckpt:
            # trusted checkpoints: train.py's and the reference's hold an argparse.Namespace under 'args'
            ck = torch.load(path, map_location="cpu", weights_only=False)
            if args.key not in ck:
                raise SystemExit(f"{path} has no '{args.key}' weights (keys: {sorted(ck)})")
            yield os.path.basename(path), ck[args.key]
        return
    import posthoc_ema
    if not args.sigma_rel:
        raise SystemExit("--snapshots needs --sigma_rel")
    files = posthoc_ema.list_snapshots(args.snapshots, args.step)
    for s in args.sigma_rel:
        sd, info = posthoc_ema.reconstruct(files, s, args.step)
        yield f"sigma_rel={s:g}@{info['step']}", sd


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.count < 1 or args.levels < 1 or args.batch < 1:
        raise SystemExit("--count, --levels and --batch must be positive")
    cfg = load_config(args.config)
    rank, size = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if size > 1:
        torch.distributed.init_process_group("nccl", device_id=device)
    m = cfg.model
    if args.synthetic:
        held = HeldOut.synthetic(args.count, m.in_size, m.in_channels, m.num_classes)
    else:
        held = HeldOut.from_lmdb(args.val_root or cfg.data.root, args.count, cfg.data.resolution,
                                 cfg.data.num_channels, m.num_classes)
    net = build_net(cfg).to(device).eval()
    rows = []
    for name, sd in sources(args):
        net.load_state_dict({k.replace("_orig_mod.", ""): v for k, v in sd.items()})
        res = validate(net, held, levels=args.levels, seed=args.seed, batch=args.batch)
        rows.append({"name": name, "mean": res["mean"], "per_level": res["per_level"]})
        if rank == 0:
            print(f"{name}: {format_levels(res)}", flush=True)
        sigma = res["sigma"]
    best = min(rows, key=lambda r: r["mean"])
    if rank == 0:
        print(f"best: {best['name']} {best['mean']:.5f} ({len(held)} items x {args.levels} levels, sigma "
              + " ".join(f"{s:.3g}" for s in sigma) + ")", flush=True)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"count": len(held), "levels": args.levels, "seed": args.seed, "sigma": sigma,
                           "rows": rows, "best": best["name"]}, f, indent=1)
    if size > 1:
        torch.distributed.destroy_process_group()
    return rows


if __name__ == "__main__":
    main()
