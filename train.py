#!/usr/bin/env python
"""Training entry point with the reference's CLI / YAML surface (train.py:294-333, configs/train/*.yaml), driving
the H100 engine.  Launch one process per GPU:

    torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 train.py --config <yaml> [--synthetic]

Differences from the reference driver, all outside the arithmetic: PyYAML instead of OmegaConf; torchrun instead of
`accelerate launch`; bf16 GEMM operands instead of fp16 AMP + GradScaler (there is one precision recipe and no loss
scaling, but GradScaler's skip of steps with inf / NaN gradients is kept: `TrainStep(skip_nonfinite=True)` unless
`--no_amp` is given, where the reference has no GradScaler either); the DDP wrapper + apex FusedAdam + EMA loop are replaced by `TrainStep` (single flat
all-reduce, fused AdamW+EMA); wandb / FID-during-training are not wired (SURVEY.md §2: out of scope).
Data: the reference's LMDB latent dataset (`data.root`/train: keys z-{i} / y-{i} / length, train_utils/datasets.py:
240-304) through `maskdit_b200.data` (liblmdb when the `lmdb` module exists, otherwise a read-only page walker of
data.mdb); `--wds` reads WebDataset tar shards instead (the reference's train_wds.py twin); `--synthetic` draws VAE
moments of the configured shape (no dataset on the bench boxes).  Either
way the moments -> latent sampling, label dropout and noise injection run as ONE fused kernel (`ops.step_front`),
gradient accumulation (`train.grad_accum`) and the lr ramp follow train.py:211-227.
Post-hoc EMA (not in the reference): `--phema_sigma_rel 0.05,0.10` keeps power-function EMA profiles next to the
reference-fixed EMA, the checkpoints carry them, and `--phema_every N` writes snapshots that posthoc_ema.py combines
into the EMA of any width after the run.
Held-out validation (not in the reference): `--val_every M` scores the EMA every M steps on the first `--val_count`
items of the latent LMDB split `data.root`/val (`--synthetic`: moments drawn from a fixed seed) at `--val_levels` fixed
noise levels (`maskdit_b200/validate.py`), a loss that compares across steps and runs; val_loss.py scores checkpoints.
Learned loss weighting (not in the reference): `model.logvar_channels: 128` in the YAML trains EDM2's u(sigma) with the
network (`EDMPrecond(logvar_channels=)`); `Train Loss` stays the reference's loss, `Weighted Loss` is the objective, and
the validation line adds the EMA's u at the validation levels.
Gradient-norm clipping (not in the reference): `--max_grad_norm 1.0` clips the global gradient norm as
torch.nn.utils.clip_grad_norm_ does, `--max_grad_norm inf` only measures it; either way the log line reports the
window's mean and maximum norm.
Consistency tuning (not in the reference): `train.objective: ect` with a `train.ect:` block (`stage_steps`, optional `q`,
`k`, `b`, `P_mean`, `P_std`) tunes an EDM network into a one- or two-step generator (`Losses['ect']`); start it from a
trained checkpoint with `--ckpt_path pre.pt --use_strict_load False` (weights and EMA, a fresh optimizer).  `Train Loss`
is then the consistency loss and the log line appends the tuning stage; the `Val Loss` line stays the EDM denoising loss,
which does not measure a tuned network's sample quality.
Model guidance (not in the reference): `train.objective: mg` with a `train.mg:` block (`scale`, the CFG-equivalent
scale s >= 1, and optional `interval: [lo, hi]`) trains a class-conditional EDM or flow network to output the guided
denoiser (`Losses['mg']`, DESIGN §5), so it samples guided at one network pass per step without `--cfg_scale`.  It
needs `model.class_dropout_prob > 0`, and fine-tunes from a trained checkpoint with `--ckpt_path pre.pt
--use_strict_load False` as consistency tuning does.  `Train Loss` stays the plain EDM / flow loss, so it compares with
a run without MG, and the log line appends `MG Loss`, the mean objective.  The `Val Loss` of an MG network is expected
to be higher than without MG, because it learns guided outputs: it is not a quality measure for MG.
"""
import argparse
import copy
import os
import time

import torch
import torch.distributed as dist

from maskdit_b200.config import build_loss, build_net, load_config, mask_ratio_schedule, parse_float_none, \
    parse_int_list
from maskdit_b200.loss import MGLoss
from maskdit_b200.train_step import TrainStep, check_max_grad_norm


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


def skip_nonfinite(args):
    """The reference wraps every optimizer step in GradScaler unless --no_amp is given (train.py:39-42); its skip of
    steps with non-finite gradients follows the same switch."""
    return not args.no_amp


def log_line(step, loss, steps_per_sec, skipped=None, grad_norm=None, weighted=None, ect_stage=None, mg=None):
    """The training log line (the reference's format, train.py:247); `skipped` (a count), `grad_norm` (the
    window's mean and max), `weighted` (the mean objective of a learned loss weighting), `ect_stage` (the
    consistency-tuning stage of the last step) and `mg` (the mean model-guidance objective) are appended only when
    given.  `loss` is the reference's loss, so it compares across runs with and without the weighting or model guidance
    (under consistency tuning, the consistency loss)."""
    line = f"(step={step:07d}) Train Loss: {loss:.4f}, Train Steps/Sec: {steps_per_sec:.2f}"
    if skipped is not None:
        line += f", Skipped Steps: {skipped}"
    if grad_norm is not None:
        line += f", Grad Norm: {grad_norm[0]:.4g} (max {grad_norm[1]:.4g})"
    if weighted is not None:
        line += f", Weighted Loss: {weighted:.4f}"
    if ect_stage is not None:
        line += f", ECT stage: {ect_stage}"
    if mg is not None:
        line += f", MG Loss: {mg:.4f}"
    return line


def parse_sigma_rels(s):
    return tuple(float(v) for v in s.split(",") if v.strip())


def parse_max_grad_norm(s):
    try:
        return check_max_grad_norm(s)
    except ValueError as e:
        raise argparse.ArgumentTypeError(str(e))


def build_parser():
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
    ap.add_argument("--phema_sigma_rel", type=parse_sigma_rels, default=(),
                    help="keep power-function EMA profiles of these relative widths for post-hoc EMA, e.g. 0.05,0.10")
    ap.add_argument("--phema_every", type=int, default=0,
                    help="write a snapshot of the profiles to <results_dir>/phema/phema-<step>.pt every N steps "
                         "(posthoc_ema.py combines them into any EMA width after the run)")
    ap.add_argument("--max_grad_norm", type=parse_max_grad_norm, default=None,
                    help="clip the global gradient norm to this bound (torch's clip_grad_norm_; 'inf' only measures) "
                         "and log its mean and max over each logging window")
    ap.add_argument("--shard_optimizer", action="store_true",
                    help="keep AdamW's moments and the post-hoc EMA profiles sharded across the data-parallel ranks "
                         "(each rank updates 1/world of the weights and the EMA, then the shadow is all-gathered); "
                         "checkpoints and snapshots keep the replicated format")
    ap.add_argument("--val_every", type=int, default=0,
                    help="every N steps, print the held-out denoising loss of the EMA (0: off)")
    ap.add_argument("--val_count", type=int, default=1000,
                    help="held-out items: the first N of data.root/val (with --synthetic: N moments from a fixed seed)")
    ap.add_argument("--val_levels", type=int, default=8, help="noise levels per held-out item")
    return ap


def val_line(step, res, logvar=None):
    """The validation log line (rank 0): the mean over levels, then each level's mean loss; with a learned loss
    weighting, `logvar` = the EMA's u(sigma_k) at the K validation levels."""
    from maskdit_b200.validate import format_levels
    what = "Val Loss (flow)" if res.get("objective") == "flow" else "Val Loss"   # the flow loss is on its own scale
    line = f"(step={step:07d}) {what}: {format_levels(res)} ({res['count']} items, EMA)"
    if logvar is not None:
        line += ", Logvar: [" + " ".join(f"{float(v):.4f}" for v in logvar) + "]"
    return line


def held_out_set(args, cfg):
    """The validation items: the first --val_count of data.root/val, or synthetic moments from a fixed seed."""
    from maskdit_b200.validate import HeldOut
    m = cfg.model
    if args.synthetic:
        return HeldOut.synthetic(args.val_count, m.in_size, m.in_channels, m.num_classes)
    return HeldOut.from_lmdb(cfg.data.root, args.val_count, cfg.data.resolution, cfg.data.num_channels, m.num_classes)


def main():
    args, _ = build_parser().parse_known_args()
    cfg = load_config(args.config)
    try:
        loss_fn = build_loss(cfg)
    except ValueError as e:
        raise SystemExit(f"{args.config}: {e}")

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
                   loss_fn=loss_fn, reference_lr_schedule=True,
                   skip_nonfinite=skip_nonfinite(args), phema_sigma_rels=args.phema_sigma_rel,
                   max_grad_norm=args.max_grad_norm, shard_optimizer=args.shard_optimizer)
    if ck and strict and "opt" in sd:                      # train.py:150: optimizer state only under strict loading
        ts.load_state_dict(sd["opt"])
    ts.lr_step_offset = step0 - ts.step_count              # lr follows the run's step counter (train.py:223)
    if args.phema_every and not ts.phema_emas:
        raise SystemExit("--phema_every needs --phema_sigma_rel")
    if rank == 0 and ts.phema_emas:
        if ts.phema_origin is None:   # a fresh run, or a checkpoint without profiles: they start at this step
            print(f"Post-hoc EMA: new profiles of sigma_rel {list(ts.phema_sigma_rels)} "
                  f"(gamma {[round(g, 3) for g in ts.phema_gammas]}) from step {step0}", flush=True)
        else:
            print(f"Post-hoc EMA: continuing the profiles of sigma_rel {list(ts.phema_sigma_rels)} from step "
                  f"{ts.phema_origin}", flush=True)
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
    held = None
    if args.val_every:
        if args.val_count < 1 or args.val_levels < 1:
            raise SystemExit("--val_count and --val_levels must be positive")
        held = held_out_set(args, cfg)
        if rank == 0:
            print(f"Validation: {len(held)} held-out items x {args.val_levels} noise levels every {args.val_every} "
                  f"steps", flush=True)
    log_every = cfg.log.log_every
    guided = isinstance(loss_fn, MGLoss)
    split = bool(net.logvar_channels) or guided   # the objective differs from the reference's loss
    running, weighted, log_steps, t0, step = 0.0, 0.0, 0, time.time(), step0
    gn_sum = gn_max = None   # the window's gradient norms, accumulated on the device like `running`
    recompute_shown = 0
    for moments, labels in loader:
        moments = moments.to(device, non_blocking=True)
        labels = labels.to(device, non_blocking=True)
        ratio = ratio_fn((step - step0) / cfg_max_steps)   # ... the schedule keeps the config's horizon (train.py:208)
        # moments -> latent (train.py:206), label dropout (:209), noise injection (loss.py:35-39): fused step front
        loss = ts.step(moments, labels, ratio, cfg.model.mae_loss_coef, grad_accum=rounds, moments=True,
                       class_dropout_prob=drop)
        running = running + ts.edm_loss.mean()   # the reference's loss; the objective differs with a weighting or MG
        if split:
            weighted = weighted + loss.mean()
        if ts.grad_norm is not None:
            gn = ts.grad_norm
            gn_sum = gn.clone() if gn_sum is None else gn_sum + gn
            gn_max = gn.clone() if gn_max is None else torch.maximum(gn_max, gn)
        if rank == 0 and ts.recompute_blocks and not recompute_shown:
            recompute_shown = ts.recompute_blocks
            print(f"Activation recomputation: the training workspace of a micro-batch does not fit in device memory, "
                  f"{recompute_shown} of {net.model.depth + net.model.decoder_depth} blocks recompute their forward "
                  f"in the backward", flush=True)
        log_steps += 1
        step += 1
        if step - step0 > max_steps:
            break
        if step % log_every == 0:
            avg = running / log_steps
            wavg = weighted / log_steps if split else None
            if world > 1:
                dist.all_reduce(avg)
                avg = avg / world
                if wavg is not None:
                    dist.all_reduce(wavg)
                    wavg = wavg / world
            torch.cuda.synchronize()
            if rank == 0:
                # every rank takes the same skip decisions, so rank 0's tally is the run's
                skipped = int(ts.skipped_steps) if ts.skipped_steps is not None else None
                # every rank computes the same norm from the same summed gradient
                gnorm = (float(gn_sum) / log_steps, float(gn_max)) if gn_sum is not None else None
                print(log_line(step, float(avg), log_steps / (time.time() - t0), skipped, gnorm,
                               float(wavg) if wavg is not None and not guided else None, ts.ect_stage,
                               float(wavg) if guided else None), flush=True)
            running, weighted, log_steps, t0 = 0.0, 0.0, 0, time.time()
            gn_sum = gn_max = None
        if held is not None and step % args.val_every == 0:
            from maskdit_b200.validate import validate
            ts.materialize(params=False)   # sharded: the EMA's masters from every rank (a no-op otherwise)
            # eager, fixed draws from their own generators: the training step's RNG stream and memory plan are untouched
            res = validate(ema, held, levels=args.val_levels, batch=micro_batch)
            if rank == 0:
                u = ema.logvar(res["sigma"]).tolist() if ema.logvar_channels else None
                print(val_line(step, res, u), flush=True)
        if step % cfg.log.ckpt_every == 0 and step > step0:
            # sharded: every rank gathers the masters, the EMA and the optimizer state (collectives); rank 0 writes
            ts.materialize()
            opt = ts.state_dict() if rank == 0 or ts.sharded else None
            if rank == 0:
                d = os.path.join(args.results_dir, "checkpoints")
                os.makedirs(d, exist_ok=True)
                torch.save({"model": net.state_dict(), "ema": ema.state_dict(), "opt": opt, "args": args},
                           os.path.join(d, f"{step:07d}.pt"))
            if world > 1:
                dist.barrier()
        if args.phema_every and step % args.phema_every == 0 and step > step0:
            # rank 0 writes the profiles; sharded, every rank takes part in gathering them
            snap = ts.phema_snapshot() if rank == 0 or ts.sharded else None
            if rank == 0:
                d = os.path.join(args.results_dir, "phema")
                os.makedirs(d, exist_ok=True)
                path = os.path.join(d, f"phema-{step:07d}.pt")
                torch.save(snap, path)
                print(f"(step={step:07d}) Post-hoc EMA snapshot (origin {ts.phema_origin}): {path}", flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
