#!/usr/bin/env python
"""Throughput of extract_latent.py end to end on 1 GPU and on every GPU of the box (one process per GPU under
torchrun), and of the host's image decoding alone, so the two can be compared.

    python tools/extract_latent_bench.py [--images 3072] [--res 512] [--batch 16] [--num_workers 8] [--out DIR]

Builds a seeded synthetic ImageFolder of JPEGs at ImageNet-like sizes (333-500 px a side) and a stand-in encoder
checkpoint (seeded N(0, 1/fan_in) convolutions; the arithmetic does not depend on the weights), then:
  * host: a DataLoader with the decode + ADM centre crop + normalise of extract_latent.py and no GPU work, with the
    worker count of one rank and of all ranks together -> images/s the host can prepare;
  * extract: `torchrun --nproc-per-node G extract_latent.py` for G = 1 and G = all GPUs; each rank reports the
    images/s of its own share (decode, copy, encode and spill, timed from its first batch request), rank 0 the merge
    time, and the wall time includes start-up.
One JSON line per measurement, with the card names, power limits and CPU count read in the same run.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def cards():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return [dict(zip(("gpu", "power_limit", "sm_clock_max"), (s.strip() for s in line.split(","))))
                for line in r.stdout.strip().splitlines()]
    except Exception:                                   # nvidia-smi missing: the names still come from the runtime
        return [{"gpu": torch.cuda.get_device_name(i), "power_limit": "unknown"} for i in range(torch.cuda.device_count())]


def make_folder(root, n, seed=0):
    """n JPEGs in 10 classes: smooth content (upsampled 24x24 noise) plus fine grain, quality 90, like photographs."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    for i in range(n):
        d = os.path.join(root, "train", f"n{i % 10:08d}")
        os.makedirs(d, exist_ok=True)
        w, h = (500, int(rng.integers(333, 501))) if i % 3 else (int(rng.integers(333, 501)), 500)
        base = Image.fromarray(rng.integers(0, 256, (24, 24, 3), dtype=np.uint8)).resize((w, h), Image.BICUBIC)
        arr = np.clip(np.asarray(base, np.int16) + rng.integers(-12, 13, (h, w, 3)), 0, 255).astype(np.uint8)
        Image.fromarray(arr).save(os.path.join(d, f"img{i:06d}.JPEG"), quality=90)


def host_rate(root, res, batch, workers):
    from extract_latent import ImageFolderImages, make_loader
    ds = ImageFolderImages(os.path.join(root, "train"), res)
    loader = make_loader(ds, batch, workers)
    it = iter(loader)
    next(it)                                            # workers started and warm
    t0, n = time.time(), 0
    for img, _ in it:
        n += img.shape[0]
    return n / (time.time() - t0)


def extract(root, ckpt, outdir, gpus, res, batch, workers):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={gpus}", "--master-addr",
           "127.0.0.1", "--master-port", str(29700 + gpus), os.path.join(ROOT, "extract_latent.py"), "--data_dir", root,
           "--resolution", str(res), "--batch_size", str(batch), "--num_workers", str(workers), "--ckpt", ckpt,
           "--outdir", outdir]
    t0 = time.time()
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), timeout=3600)
    wall = time.time() - t0
    if r.returncode:
        raise SystemExit(r.stdout[-3000:] + r.stderr[-3000:])
    ranks = [(int(a), float(b), float(c)) for a, b, c in
             re.findall(r"rank \d+ of \d+: encoded (\d+) images in ([\d.]+)s \(([\d.]+) img/s\)", r.stdout)]
    merge = re.search(r"merged \d+ shards in ([\d.]+)s", r.stdout)
    assert len(ranks) == gpus, r.stdout
    return {"gpus": gpus, "per_gpu_img_s": [c for _, _, c in ranks],
            "slowest_rank_s": max(b for _, b, _ in ranks),
            "aggregate_img_s": round(sum(a for a, _, _ in ranks) / max(b for _, b, _ in ranks), 1),
            "merge_s": float(merge.group(1)) if merge else None, "wall_s": round(wall, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3072)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--batch", type=int, default=16, help="images per GPU per batch")
    ap.add_argument("--num_workers", type=int, default=8, help="decode workers per GPU")
    ap.add_argument("--out", default=None, help="directory for the JSON records")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("extract_latent_bench needs a CUDA device")
    from vae_encode_bench import stand_in
    from maskdit_b200.vae import AutoencoderKLEncoder
    ngpu = torch.cuda.device_count()
    info = {"cards": cards(), "cpus": os.cpu_count(), "cpus_usable": len(os.sched_getaffinity(0)),
            "images": args.images, "res": args.res, "batch_per_gpu": args.batch, "workers_per_gpu": args.num_workers}
    recs = []
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.time()
        make_folder(tmp, args.images)
        ckpt = os.path.join(tmp, "vae.pth")
        torch.save({k: v.cpu() for k, v in stand_in(AutoencoderKLEncoder()).state_dict().items()}, ckpt)
        torch.cuda.empty_cache()
        print(f"synthetic ImageFolder of {args.images} images in {time.time() - t0:.1f}s", flush=True)
        for g in sorted({1, ngpu}):
            w = g * args.num_workers
            recs.append({"metric": "host_decode", "workers": w,
                         "img_s": round(host_rate(tmp, args.res, args.batch, w), 1), **info})
            print(json.dumps(recs[-1]), flush=True)
        for g in sorted({1, ngpu}):
            recs.append({"metric": "extract_latent", **extract(tmp, ckpt, os.path.join(tmp, f"out{g}"), g, args.res,
                                                               args.batch, args.num_workers), **info})
            print(json.dumps(recs[-1]), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "extract_latent_bench.json"), "w") as f:
            json.dump(recs, f, indent=1)


if __name__ == "__main__":
    main()
