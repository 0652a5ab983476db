#!/usr/bin/env python
"""Training entry point with the reference's CLI / YAML surface (train.py:294-333, configs/train/*.yaml), driving
the H100 engine.  Launch one process per GPU:

    torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 train.py --config <yaml> [--synthetic]

Differences from the reference driver, all outside the arithmetic: PyYAML instead of OmegaConf; torchrun instead of
`accelerate launch`; bf16 GEMM operands instead of fp16 AMP + GradScaler (`--no_amp` is accepted and ignored: there
is one precision recipe); the DDP wrapper + apex FusedAdam + EMA loop are replaced by `TrainStep` (single flat
all-reduce, fused AdamW+EMA); wandb / FID-during-training are not wired (SURVEY.md §2: out of scope).
Data: the reference's LMDB latent dataset (`data.root`/train: keys z-{i} / y-{i} / length, train_utils/datasets.py:
240-304) through `maskdit_b200.data` (liblmdb when the `lmdb` module exists, otherwise a read-only page walker of
data.mdb); `--wds` reads WebDataset tar shards instead (the reference's train_wds.py twin); `--synthetic` draws VAE
moments of the configured shape (no dataset on the bench boxes).  Either
way the moments -> latent sampling, label dropout and noise injection run as ONE fused kernel (`ops.step_front`),
gradient accumulation (`train.grad_accum`) and the lr ramp follow train.py:211-227.
"""
import argparse
import copy
import os
import time

import torch
import torch.distributed as dist

from maskdit_b200.config import build_net, load_config, mask_ratio_schedule, parse_float_none, parse_int_list
from maskdit_b200.loss import Losses
from maskdit_b200.train_step import TrainStep


def latest_ckpt(d):
    """utils.get_latest_ckpt (utils.py:22-34): highest '<step:07d>.pt'."""
    if not os.path.isdir(d):
        return None
    c = sorted(f for f in os.listdir(d) if f.endswith(".pt") and f[:-3].isdigit())
    return os.path.join(d, c[-1]) if c else None


def synthetic_loader(cfg, batch, device, seed):
    g = torch.Generator(device=device).manual_seed(seed)
    R, C, n = cfg.model.in_size, cfg.model.in_channels, cfg.model.num_classes
    while True:
        moments = torch.randn(batch, 2 * C, R, R, device=device, generator=g)
        labels = torch.nn.functional.one_hot(torch.randint(0, n, (batch,), device=device, generator=g), n).float()
        yield moments, labels


def main():
    ap = argparse.ArgumentParser("training parameters")
    ap.add_argument("--config", required=True)
    ap.add_argument("--results_dir", default="results")
    ap.add_argument("--ckpt_path", default=None)
    ap.add_argument("--global_seed", type=int, default=0)
    ap.add_argument("--num_workers", type=int, default=4)
    ap.add_argument("--no_amp", action="store_true")
    ap.add_argument("--use_wandb", action="store_true")
    ap.add_argument("--use_ckpt_path", default="True")
    ap.add_argument("--use_strict_load", default="True")
    ap.add_argument("--tag", default="")
    ap.add_argument("--enable_eval", action="store_true")
    ap.add_argument("--seeds", type=parse_int_list, default="0-49999")
    ap.add_argument("--cfg_scale", type=parse_float_none, default=None)
    ap.add_argument("--num_steps", type=int, default=40)
    ap.add_argument("--synthetic", action="store_true", help="synthetic latents instead of the LMDB dataset")
    ap.add_argument("--wds", action="store_true",
                    help="data.root holds WebDataset .tar shards (the reference's train_wds.py twin: lmdb2wds.py layout)")
    ap.add_argument("--max_steps", type=int, default=None, help="stop after this many steps (smoke runs)")
    args, _ = ap.parse_known_args()
    cfg = load_config(args.config)

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    torch.manual_seed(args.global_seed)  # same seed on every rank, as the reference (train.py:67-68)

    micro_batch = cfg.train.batchsize                      # train.py:72-75
    rounds = int(cfg.train.get("grad_accum", 1) or 1)
    batch = micro_batch * rounds                           # per-GPU batch of one optimizer step
    global_batch = batch * world
    net = build_net(cfg).to(device).train()
    ema = copy.deepcopy(net).eval()
    for p in ema.parameters():
        p.requires_grad_(False)
    step0 = 0
    ck = args.ckpt_path or latest_ckpt(os.path.join(args.results_dir, "checkpoints"))
    ts = None
    strict = str(args.use_strict_load).lower() in ("true", "1")
    if ck:
        # reference checkpoints store `args` as an argparse.Namespace (train.py:259-265): a full (trusted) unpickle
        sd = torch.load(ck, map_location=device, weights_only=False)
        net.load_state_dict({k.replace("_orig_mod.", ""): v for k, v in sd["model"].items()}, strict=strict)
        ema.load_state_dict({k.replace("_orig_mod.", ""): v for k, v in sd["ema"].items()}, strict=strict)
        step0 = int(os.path.basename(ck)[:-3]) if os.path.basename(ck)[:-3].isdigit() else 0
    ts = TrainStep(net, ema, lr=cfg.train.lr, lr_rampup_kimg=cfg.train.lr_rampup_kimg, global_batch=global_batch,
                   loss_fn=Losses[cfg.model.precond](), reference_lr_schedule=True)
    if ck and strict and "opt" in sd:                      # train.py:150: optimizer state only under strict loading
        ts.load_state_dict(sd["opt"])
    ts.lr_step_offset = step0 - ts.step_count              # lr follows the run's step counter (train.py:223)
    ratio_fn = mask_ratio_schedule(cfg.model.get("mask_ratio_fn", "constant"), cfg.model.mask_ratio,
                                   cfg.model.get("mask_ratio_min", 0) or 0)
    drop = cfg.model.get("class_dropout_prob", 0) or 0
    cfg_max_steps = cfg.train.get("max_num_steps", None) or 10 ** 9
    max_steps = args.max_steps or cfg_max_steps        # --max_steps only shortens the run (smoke runs) ...
    if args.synthetic:
        loader = synthetic_loader(cfg, batch, device, args.global_seed + rank)
    elif args.wds:      # train_wds.py:172-178: shards of config.data.root, split data_list[rank::world]
        from maskdit_b200.data import wds_batches
        shards = sorted(os.path.join(cfg.data.root, f) for f in os.listdir(cfg.data.root) if f.endswith(".tar"))
        if rank == 0:
            print(f"Dataset: {len(shards)} WebDataset shards ({cfg.data.root})", flush=True)
        loader = wds_batches(shards, batch, rank, world, num_classes=cfg.model.num_classes)
    else:
        from maskdit_b200.data import ImageNetLatentDataset, batches
        ds = ImageNetLatentDataset(cfg.data.root, resolution=cfg.data.resolution, num_channels=cfg.data.num_channels,
                                   num_classes=cfg.model.num_classes)
        if rank == 0:
            print(f"Dataset contains {len(ds):,} images ({cfg.data.root})", flush=True)
        loader = batches(ds, batch, rank, world, start=step0)
    log_every = cfg.log.log_every
    running, log_steps, t0, step = 0.0, 0, time.time(), step0
    for moments, labels in loader:
        moments = moments.to(device, non_blocking=True)
        labels = labels.to(device, non_blocking=True)
        ratio = ratio_fn((step - step0) / cfg_max_steps)   # ... the schedule keeps the config's horizon (train.py:208)
        # moments -> latent (train.py:206), label dropout (:209), noise injection (loss.py:35-39): fused step front
        loss = ts.step(moments, labels, ratio, cfg.model.mae_loss_coef, grad_accum=rounds, moments=True,
                       class_dropout_prob=drop)
        running = running + loss.mean()
        log_steps += 1
        step += 1
        if step - step0 > max_steps:
            break
        if step % log_every == 0:
            avg = running / log_steps
            if world > 1:
                dist.all_reduce(avg)
                avg = avg / world
            torch.cuda.synchronize()
            if rank == 0:
                print(f"(step={step:07d}) Train Loss: {float(avg):.4f}, Train Steps/Sec: "
                      f"{log_steps / (time.time() - t0):.2f}", flush=True)
            running, log_steps, t0 = 0.0, 0, time.time()
        if step % cfg.log.ckpt_every == 0 and step > step0:
            if rank == 0:
                d = os.path.join(args.results_dir, "checkpoints")
                os.makedirs(d, exist_ok=True)
                torch.save({"model": net.state_dict(), "ema": ema.state_dict(), "opt": ts.state_dict(), "args": args},
                           os.path.join(d, f"{step:07d}.pt"))
            if world > 1:
                dist.barrier()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
