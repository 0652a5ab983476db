#!/usr/bin/env python
"""Sampling entry point with the reference's CLI / YAML surface (generate.py:54-87, configs/test/*.yaml).

Builds `Precond_models[config.model.precond]` from the YAML, loads `ckpt['ema']` (reference checkpoints load
unchanged: same state-dict keys), and runs `edm_sampler` on the H100 engine for the requested seeds with
per-sample generators (utils.StackedRandomGenerator, utils.py:119-133).  Under torchrun the seed batches are dealt
to the ranks exactly as generate_with_net does (sample.py:232-235: rank-strided, one barrier per batch); giving any of
--solver / --discretization / --schedule / --scaling selects `ablation_sampler` (sample.py:243-245).  The SD-VAE
decode of the reference (sample.py:275) runs on the same kernels (`maskdit_b200/vae.py`) when `--pretrained_path` names a
FrozenAutoencoderKL checkpoint: images are converted to 8 bit (`ops.to_uint8_nhwc`) and written as `<seed>.png`
(`sampler.write_png`), exactly the tail of generate_with_net (sample.py:275-296).  The latents are always saved as `.npy`
per seed as well; without a VAE checkpoint `--png_preview` writes the raw latent channels as a picture.

Guidance beyond the reference's `--cfg_scale`: `--guide_ckpt` (or `--guide_snapshots` + `--guide_sigma_rel`, a post-hoc
EMA built by `posthoc_ema.reconstruct`) with `--guidance W` guides with a second, weaker network of the same image
geometry and classes (autoguidance; `--guide_config` when its architecture differs), and `--guidance_interval LO HI`
applies CFG or the guide only at evaluations with LO < sigma <= HI.  A rectified-flow config (`model.precond: flow`)
samples with `flow_sampler` (Heun on a uniform t grid, `--num_steps`, `--cfg_scale`, `--guidance_interval` on t) and
refuses the ablation switches, `--S_churn` and autoguidance.  `--consistency_sigmas S0 [S1 ...]` samples a
consistency-tuned EDM network (train.py with `train.objective: ect`) with `consistency_sampler`, one evaluation per
noise level, and refuses the ablation switches, `--S_churn` and flow configs.  `--dpm_order {1,2,3}` samples an EDM or a
flow config with `dpm_solver_sampler` (multistep DPM-Solver++: DDIM, 2M or 3M) in `--num_steps` network evaluations,
with `--cfg_scale`, autoguidance (EDM) and `--guidance_interval` as above, and refuses the ablation switches, `--S_churn`
and `--consistency_sigmas`.  Class-unconditional configs sample with all-zero label rows as the reference does
(sample.py:261-264).  A network trained with model guidance (train.py with `train.objective: mg`) outputs the guided
denoiser itself: every sampler above samples it guided without `--cfg_scale`, at one network pass per evaluation, and
`--cfg_scale` on top compounds the two guidances.
"""
import argparse
import os

import numpy as np
import torch

from maskdit_b200.config import build_net, load_config, parse_float_none, parse_int_list
from maskdit_b200.maskdit import eval_state_dict
from maskdit_b200 import ops
from maskdit_b200.sampler import (ablation_sampler, consistency_sampler, consistency_sigmas, dpm_solver_sampler,
                                  edm_sampler, flow_sampler, rank_seed_batches, write_png)


class StackedRandomGenerator:
    def __init__(self, device, seeds):
        self.generators = [torch.Generator(device).manual_seed(int(s) % (1 << 32)) for s in seeds]

    def randn(self, size, **kw):
        return torch.stack([torch.randn(size[1:], generator=g, **kw) for g in self.generators])

    def randn_like(self, x):
        return self.randn(x.shape, dtype=x.dtype, layout=x.layout, device=x.device)

    def randint(self, *a, size, **kw):
        return torch.stack([torch.randint(*a, size=size[1:], generator=g, **kw) for g in self.generators])


def build_parser():
    ap = argparse.ArgumentParser("Sample from a trained model")
    ap.add_argument("--config", required=True)
    ap.add_argument("--results_dir", default="samples")
    ap.add_argument("--ckpt_path", default=None)
    ap.add_argument("--seeds", type=parse_int_list, default="100-131")
    ap.add_argument("--class_idx", type=int, default=None)
    ap.add_argument("--cfg_scale", type=parse_float_none, default=None)
    ap.add_argument("--num_steps", type=int, default=40)
    ap.add_argument("--S_churn", type=int, default=0)
    ap.add_argument("--max_batch_size", type=int, default=32)
    # ablation_sampler switches (sample.py:358-364): giving any of them selects the generalised sampler
    ap.add_argument("--solver", choices=["euler", "heun"], default=None)
    ap.add_argument("--discretization", choices=["vp", "ve", "iddpm", "edm"], default=None)
    ap.add_argument("--schedule", choices=["vp", "ve", "linear"], default=None)
    ap.add_argument("--scaling", choices=["vp", "none"], default=None)
    ap.add_argument("--pretrained_path", default=None,
                    help="SD-VAE checkpoint (FrozenAutoencoderKL state dict, reference default assets/vae/autoencoder_kl.pth): "
                         "decode the latents and write PNGs as generate_with_net does (sample.py:275-296)")
    ap.add_argument("--subdirs", action="store_true", help="<seed - seed % 1000:06d>/ sub-directories (sample.py:289)")
    ap.add_argument("--png_preview", action="store_true",
                    help="also write channels 0-2 of every latent as an 8-bit PNG (no SD-VAE in this repo)")
    # guidance by a second network (autoguidance) and a noise-level interval for guidance (maskdit_b200/sampler.py)
    ap.add_argument("--guide_ckpt", default=None,
                    help="guide network checkpoint (train.py, posthoc_ema.py or the reference's)")
    ap.add_argument("--guide_key", choices=["ema", "model"], default="ema", help="weights of --guide_ckpt to load")
    ap.add_argument("--guide_config", default=None, help="YAML of the guide's architecture (default: --config)")
    ap.add_argument("--guide_snapshots", default=None,
                    help="build the guide from the post-hoc EMA snapshots in this directory (posthoc_ema.py)")
    ap.add_argument("--guide_sigma_rel", type=float, default=None, help="relative EMA width of the snapshot guide")
    ap.add_argument("--guide_step", type=int, default=None,
                    help="run step of the snapshot guide's EMA (default: the last snapshot's)")
    ap.add_argument("--guidance", type=float, default=None,
                    help="guide weight w: D = D_guide + w (D_net - D_guide); 1 is the unguided network")
    ap.add_argument("--guidance_interval", type=float, nargs=2, default=None, metavar=("LO", "HI"),
                    help="apply the guidance (--cfg_scale or the guide) only at evaluations with LO < sigma <= HI")
    ap.add_argument("--consistency_sigmas", type=float, nargs="+", default=None, metavar="SIGMA",
                    help="sample a consistency-tuned network (train.objective: ect) at these strictly decreasing noise "
                         "levels, one network evaluation each (e.g. 80, or 80 0.8)")
    ap.add_argument("--dpm_order", type=int, choices=[1, 2, 3], default=None,
                    help="sample with multistep DPM-Solver++ of this order (1 DDIM, 2 2M, 3 3M) in --num_steps network "
                         "evaluations, EDM or flow configs")
    return ap


def parse_args(argv=None):
    ap = build_parser()
    args, _ = ap.parse_known_args(argv)
    guide = args.guide_ckpt is not None or args.guide_snapshots is not None
    if args.guide_ckpt is not None and args.guide_snapshots is not None:
        ap.error("--guide_ckpt and --guide_snapshots are mutually exclusive")
    if (args.guide_snapshots is None) != (args.guide_sigma_rel is None):
        ap.error("--guide_snapshots and --guide_sigma_rel go together")
    if args.guide_step is not None and args.guide_snapshots is None:
        ap.error("--guide_step needs --guide_snapshots")
    if args.guide_config is not None and not guide:
        ap.error("--guide_config needs --guide_ckpt or --guide_snapshots")
    if guide and args.cfg_scale is not None:
        ap.error("--cfg_scale and a guide network are mutually exclusive")
    if guide != (args.guidance is not None):
        ap.error("--guidance is the weight of a guide network (--guide_ckpt / --guide_snapshots): give both or neither")
    if args.guidance_interval is not None:
        lo, hi = args.guidance_interval
        if not lo < hi:
            ap.error(f"--guidance_interval needs LO < HI, got {lo:g} {hi:g}")
        if not guide and args.cfg_scale is None:
            ap.error("--guidance_interval needs --cfg_scale or a guide network")
    if args.consistency_sigmas is not None:
        bad = [f"--{k}" for k in ("solver", "discretization", "schedule", "scaling") if getattr(args, k)]
        if args.S_churn:
            bad.append("--S_churn")
        if bad:
            ap.error(f"--consistency_sigmas samples with consistency_sampler: {', '.join(bad)} apply to the EDM "
                     "samplers only")
        try:
            consistency_sigmas(args.consistency_sigmas)
        except ValueError as e:
            ap.error(f"--consistency_sigmas: {e}")
    if args.dpm_order is not None:
        bad = [f"--{k}" for k in ("solver", "discretization", "schedule", "scaling") if getattr(args, k)]
        if args.S_churn:
            bad.append("--S_churn")
        if args.consistency_sigmas is not None:
            bad.append("--consistency_sigmas")
        if bad:
            ap.error(f"--dpm_order samples with dpm_solver_sampler: {', '.join(bad)} do not apply to it")
        if args.num_steps < 1:
            ap.error(f"--dpm_order needs --num_steps >= 1, got {args.num_steps}")
    return args


def check_flow_args(args):
    """A rectified-flow config (`model.precond: flow`) samples with `flow_sampler` (Heun on a uniform t grid,
    `--num_steps`, `--cfg_scale`, `--guidance_interval` on t): refuse the EDM-only switches it has no meaning for."""
    bad = [f"--{k}" for k in ("solver", "discretization", "schedule", "scaling") if getattr(args, k)]
    if args.S_churn:
        bad.append("--S_churn")
    if args.guide_ckpt is not None or args.guide_snapshots is not None or args.guidance is not None:
        bad.append("autoguidance (--guide_ckpt / --guide_snapshots / --guidance)")
    if bad:
        raise SystemExit(f"a flow config (model.precond: flow) samples with flow_sampler: {', '.join(bad)} "
                         "apply to the EDM samplers only")


def guide_state_dict(args):
    """The guide's state dict on the host: `--guide_key` of `--guide_ckpt`, or the post-hoc EMA of width
    `--guide_sigma_rel` at `--guide_step` reconstructed from `--guide_snapshots` (posthoc_ema.reconstruct)."""
    if args.guide_snapshots is not None:
        import posthoc_ema
        files = posthoc_ema.list_snapshots(args.guide_snapshots, args.guide_step)
        sd, _ = posthoc_ema.reconstruct(files, args.guide_sigma_rel, args.guide_step)
        return sd
    ck = torch.load(args.guide_ckpt, map_location="cpu", weights_only=False)   # trusted checkpoint, as --ckpt_path
    if args.guide_key not in ck:
        raise SystemExit(f"{args.guide_ckpt} holds no '{args.guide_key}' weights (keys: {sorted(ck)})")
    return {k.replace("_orig_mod.", ""): v for k, v in ck[args.guide_key].items()}


def main(argv=None):
    args = parse_args(argv)
    cfg = load_config(args.config)
    flow = cfg.model.precond == "flow"
    if flow and args.consistency_sigmas is not None:
        raise SystemExit("--consistency_sigmas samples a consistency-tuned EDM network, not a flow config "
                         "(model.precond: flow)")
    rank, size = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if size > 1:
        torch.distributed.init_process_group("nccl", device_id=device)
    if flow:
        check_flow_args(args)
    net = build_net(cfg).to(device).eval()
    if args.ckpt_path:
        # trusted checkpoint: reference checkpoints hold an argparse.Namespace under 'args' (train.py:259-265)
        ck = torch.load(args.ckpt_path, map_location=device, weights_only=False)
        net.load_state_dict(eval_state_dict(net, ck["ema"]))
    gkw = {}
    if args.guidance is not None:
        guide = build_net(load_config(args.guide_config or args.config)).to(device).eval()
        guide.load_state_dict(eval_state_dict(guide, guide_state_dict(args)))
        net.check_guide(guide)
        gkw = dict(guide_net=guide, guidance=args.guidance)
    if args.guidance_interval is not None:
        gkw["guidance_interval"] = tuple(args.guidance_interval)
    os.makedirs(args.results_dir, exist_ok=True)
    vae = None
    if args.pretrained_path:
        from maskdit_b200.vae import get_model
        vae = get_model(args.pretrained_path, device=device)
    kw = {k: getattr(args, k) for k in ("solver", "discretization", "schedule", "scaling") if getattr(args, k)}
    sampler_fn = ablation_sampler if kw else edm_sampler          # sample.py:243-245
    n_done = 0
    for bs in rank_seed_batches(args.seeds, args.max_batch_size, rank, size):   # sample.py:232-235: rank-strided
        if size > 1:
            torch.distributed.barrier()                          # sample.py:253
        if not bs:
            continue
        rnd = StackedRandomGenerator(device, bs)
        latents = rnd.randn([len(bs), net.img_channels, net.img_resolution, net.img_resolution], device=device)
        labels = torch.zeros([len(bs), net.num_classes], device=device)      # sample.py:261-264
        if net.num_classes:
            labels = torch.eye(net.num_classes, device=device)[rnd.randint(net.num_classes, size=[len(bs)],
                                                                           device=device)]
        if args.class_idx is not None:
            labels[:, :] = 0
            labels[:, args.class_idx] = 1
        with torch.no_grad():
            if args.consistency_sigmas is not None:
                z = consistency_sampler(net, latents.float(), labels.float(), cfg_scale=args.cfg_scale,
                                        randn_like=rnd.randn_like, sigmas=args.consistency_sigmas, **gkw).float()
            elif args.dpm_order is not None:
                z = dpm_solver_sampler(net, latents.float(), labels.float(), cfg_scale=args.cfg_scale,
                                       num_steps=args.num_steps, order=args.dpm_order, **gkw).float()
            elif flow:
                z = flow_sampler(net, latents.float(), labels.float(), cfg_scale=args.cfg_scale,
                                 num_steps=args.num_steps, **gkw).float()
            else:
                z = sampler_fn(net, latents.float(), labels.float(), cfg_scale=args.cfg_scale,
                               randn_like=rnd.randn_like, num_steps=args.num_steps, S_churn=args.S_churn, **kw,
                               **gkw).float()
        if vae is not None:       # images = vae.decode(z); add(1).mul(127.5).clamp(0,255).to(uint8) NHWC; PNG per seed
            px = ops.to_uint8_nhwc(vae.decode(z).contiguous()).cpu().numpy()
            for s, im in zip(bs, px):
                d = os.path.join(args.results_dir, f"{s - s % 1000:06d}") if args.subdirs else args.results_dir
                os.makedirs(d, exist_ok=True)
                write_png(os.path.join(d, f"{s:06d}.png"), im)
        elif args.png_preview:
            px = ops.to_uint8_nhwc((z[:, :3] / z[:, :3].abs().amax().clamp_min(1e-8)).contiguous()).cpu().numpy()
            for s, im in zip(bs, px):
                write_png(os.path.join(args.results_dir, f"{s:06d}.png"), im)
        for s, zi in zip(bs, z.cpu().numpy()):
            np.save(os.path.join(args.results_dir, f"{s:06d}.npy"), zi)
        n_done += len(bs)
    print(f"rank {rank}: wrote {n_done} latents to {args.results_dir}")
    if size > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
