#!/usr/bin/env python
"""Encode an ImageFolder tree into the latent LMDB that `train.py` reads, with the reference's CLI
(extract_latent.py:16-110) and the SD-VAE encoder on the H100 kernels (`maskdit_b200.vae.get_encoder`):

    python extract_latent.py --data_dir <root> --split train --resolution 256 --ckpt assets/vae/autoencoder_kl.pth \\
        --outdir <dir> [--xflip]

Input: `{data_dir}/{split}/<class>/**/<image>` in ImageFolder order (`data.image_folder_samples`).  Host worker
processes decode, centre-crop (ADM rule) and normalise the images into pinned batches; the GPU returns the VAE
moments [8, R/8, R/8] of each.  Output: `{outdir}/{data_name}_{resolution}_latent_lmdb/{split}/data.mdb` with
z-{i} = raw little-endian fp32 moments, y-{i} = decimal class index, and `length`; with --xflip a second pass stores
the moments of the horizontally mirrored images at i = N .. 2N-1.  Values are streamed to disk as they are produced
(`data.MdbWriter`), so the output may be far larger than host memory.
"""
import argparse
import os
import time

import numpy as np
import torch

from maskdit_b200.data import MdbWriter, image_folder_samples, load_image


class ImageFolderImages(torch.utils.data.Dataset):
    def __init__(self, root, resolution):
        self.samples, self.classes = image_folder_samples(root)
        self.resolution = resolution

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        path, label = self.samples[i]
        return torch.from_numpy(load_image(path, self.resolution)), label


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--data_name", default="imagenet", type=str)
    ap.add_argument("--data_dir", default="../datasets", type=str)
    ap.add_argument("--ckpt", default="assets/vae/autoencoder_kl.pth", type=str, help="checkpoint path")
    ap.add_argument("--resolution", default=512, type=int)
    ap.add_argument("--batch_size", default=128, type=int)
    ap.add_argument("--split", default="train", type=str)
    ap.add_argument("--xflip", action="store_true")
    ap.add_argument("--outdir", type=str, default="../data/imagenet512-latent", help="output directory")
    ap.add_argument("--num_workers", default=8, type=int, help="image decoding worker processes")
    args = ap.parse_args(argv)
    if args.split not in ("train", "val"):
        raise SystemExit(f"--split must be train or val, not {args.split!r}")
    if args.resolution % 8:
        raise SystemExit(f"--resolution must be a multiple of 8, not {args.resolution}")

    from maskdit_b200.vae import get_encoder
    dataset = ImageFolderImages(os.path.join(args.data_dir, args.split), args.resolution)
    print(f"data size: {len(dataset)}")
    model = get_encoder(args.ckpt)
    print(f"load vae weights from {args.ckpt}")
    loader = torch.utils.data.DataLoader(dataset, batch_size=args.batch_size, shuffle=False, drop_last=False,
                                         num_workers=args.num_workers, pin_memory=True,
                                         persistent_workers=args.num_workers > 0)
    target = os.path.join(args.outdir, f"{args.data_name}_{args.resolution}_latent_lmdb", args.split)
    idx = 0
    with MdbWriter(target) as db:
        for flip in ((False, True) if args.xflip else (False,)):
            begin = time.time()
            if flip:
                print("starting to store the xflip latents")
            for img, label in loader:
                if img.min() < -1 or img.max() > 1:
                    raise ValueError("preprocessed images left [-1, 1]")
                moments = model.encode_moments(img.cuda(non_blocking=True), flip=flip)
                assert moments.shape[-1] == args.resolution // 8
                for m, lb in zip(moments.cpu().numpy(), label.tolist()):
                    db.put(f"z-{idx}".encode(), np.ascontiguousarray(m, dtype="<f4"))
                    db.put(f"y-{idx}".encode(), str(int(lb)).encode())
                    idx += 1
                    if idx % 5120 == 0:
                        print(f"saved {idx} files with {time.time() - begin:.1f}s elapsed")
                        begin = time.time()
        db.put(b"length", str(idx).encode())
    print(f"[finished] saved {idx} files to {target}")


if __name__ == "__main__":
    main()
