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
"""
import argparse
import os

import numpy as np
import torch

from maskdit_b200.config import build_net, load_config, parse_float_none, parse_int_list
from maskdit_b200 import ops
from maskdit_b200.sampler import ablation_sampler, edm_sampler, rank_seed_batches, write_png


class StackedRandomGenerator:
    def __init__(self, device, seeds):
        self.generators = [torch.Generator(device).manual_seed(int(s) % (1 << 32)) for s in seeds]

    def randn(self, size, **kw):
        return torch.stack([torch.randn(size[1:], generator=g, **kw) for g in self.generators])

    def randn_like(self, x):
        return self.randn(x.shape, dtype=x.dtype, layout=x.layout, device=x.device)

    def randint(self, *a, size, **kw):
        return torch.stack([torch.randint(*a, size=size[1:], generator=g, **kw) for g in self.generators])


def main():
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
    args, _ = ap.parse_known_args()
    cfg = load_config(args.config)
    rank, size = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if size > 1:
        torch.distributed.init_process_group("nccl", device_id=device)
    net = build_net(cfg).to(device).eval()
    if args.ckpt_path:
        # trusted checkpoint: reference checkpoints hold an argparse.Namespace under 'args' (train.py:259-265)
        ck = torch.load(args.ckpt_path, map_location=device, weights_only=False)
        net.load_state_dict({k.replace("_orig_mod.", ""): v for k, v in ck["ema"].items()})
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
        labels = torch.eye(net.num_classes, device=device)[rnd.randint(net.num_classes, size=[len(bs)], device=device)]
        if args.class_idx is not None:
            labels[:, :] = 0
            labels[:, args.class_idx] = 1
        with torch.no_grad():
            z = sampler_fn(net, latents.float(), labels.float(), cfg_scale=args.cfg_scale,
                           randn_like=rnd.randn_like, num_steps=args.num_steps, S_churn=args.S_churn, **kw).float()
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
