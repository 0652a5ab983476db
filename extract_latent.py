#!/usr/bin/env python
"""Encode an ImageFolder tree into the latent LMDB that `train.py` reads, with the reference's CLI
(extract_latent.py:16-110) and the SD-VAE encoder on the H100 kernels (`maskdit_b200.vae.get_encoder`):

    python extract_latent.py --data_dir <root> --split train --resolution 256 --ckpt assets/vae/autoencoder_kl.pth \\
        --outdir <dir> [--xflip]
    torchrun --nproc-per-node 8 extract_latent.py ...        # one process per GPU, same flags, same data.mdb

Input: `{data_dir}/{split}/<class>/**/<image>` in ImageFolder order (`data.image_folder_samples`).  Host worker
processes decode, centre-crop (ADM rule) and normalise the images into pinned batches; the GPU returns the VAE
moments [8, R/8, R/8] of each.  Output: `{outdir}/{data_name}_{resolution}_latent_lmdb/{split}/data.mdb` with
z-{i} = raw little-endian fp32 moments, y-{i} = decimal class index, and `length`; with --xflip a second pass stores
the moments of the horizontally mirrored images at i = N .. 2N-1.  Values are streamed to disk as they are produced
(`data.MdbWriter`), so the output may be far larger than host memory.

Under `torchrun` with WORLD_SIZE > 1 (where the reference wraps the encoder in `nn.DataParallel`, :40-42), rank r
encodes the contiguous index range `shard_range(N, r, W)` on `cuda:LOCAL_RANK` (and, with --xflip, the mirrored pass of
the same range) and streams its moments and labels to two spill files next to `data.mdb`.  After a barrier, rank 0
merges the spill files in rank order into `data.mdb`, issuing the `put` calls in the one-GPU order, then deletes
them.  The encoder's moments do not depend on how the batch is split, so the file is byte for byte the one a
one-GPU run writes.  The process group (gloo) carries only the rendezvous and barriers; the ranks of a multi-node run
need `--outdir` on a file system they all see.
"""
import argparse
import datetime
import hashlib
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


def make_loader(dataset, batch_size, num_workers):
    return torch.utils.data.DataLoader(dataset, batch_size=batch_size, shuffle=False, drop_last=False,
                                       num_workers=num_workers, pin_memory=True, persistent_workers=num_workers > 0)


def encoded_batches(model, loader, flip, resolution):
    """(moments float32 ndarray [B, 8, R/8, R/8], labels list) per batch of `loader`, mirrored when `flip`."""
    for img, label in loader:
        if img.min() < -1 or img.max() > 1:
            raise ValueError("preprocessed images left [-1, 1]")
        moments = model.encode_moments(img.cuda(non_blocking=True), flip=flip)
        assert moments.shape[-1] == resolution // 8
        yield moments.cpu().numpy(), label.tolist()


def shard_range(n, rank, world):
    """[lo, hi) of the items rank `rank` of `world` encodes: contiguous ranges in rank order, the first n % world ranks
    one item longer.  A rank may get an empty range (n < world)."""
    q, r = divmod(n, world)
    lo = rank * q + min(rank, r)
    return lo, lo + q + (rank < r)


def spill_indices(n, rank, world, xflip):
    """LMDB indices of the records in rank `rank`'s spill files, in file order: its range, then with xflip the same
    range of the mirrored pass, whose item i is stored at n + i."""
    lo, hi = shard_range(n, rank, world)
    return [p * n + i for p in range(1 + xflip) for i in range(lo, hi)]


def spill_paths(target, rank, world):
    """The moments (raw little-endian fp32) and labels (little-endian int64) spill files of one rank."""
    base = os.path.join(target, f"spill-{rank:05d}-of-{world:05d}")
    return base + ".f32", base + ".i64"


def encode_shard(dataset, rank, world, model, target, batch_size, num_workers=0, xflip=False, log=None):
    """Encode rank `rank`'s share of `dataset` (`shard_range`; with xflip also its mirrored pass) into its spill files
    under `target`, in `spill_indices` order.  `log(msg)`, if given, gets the reference's progress messages.
    Returns (records written, seconds)."""
    lo, hi = shard_range(len(dataset), rank, world)
    zpath, ypath = spill_paths(target, rank, world)
    os.makedirs(target, exist_ok=True)
    begin = start = time.time()
    done = 0
    with open(zpath, "wb") as fz, open(ypath, "wb") as fy:
        if hi > lo:
            loader = make_loader(torch.utils.data.Subset(dataset, range(lo, hi)), batch_size, num_workers)
            for flip in ((False, True) if xflip else (False,)):
                if flip and log:
                    log("starting to store the xflip latents")
                for moments, labels in encoded_batches(model, loader, flip, dataset.resolution):
                    fz.write(np.ascontiguousarray(moments, dtype="<f4").tobytes())
                    fy.write(np.asarray(labels, dtype="<i8").tobytes())
                    for _ in labels:
                        done += 1
                        if log and done % 5120 == 0:
                            log(f"saved {done} files with {time.time() - begin:.1f}s elapsed")
                            begin = time.time()
        for f in (fz, fy):                 # rank 0 may read these from another node once the barrier has passed
            f.flush()
            os.fsync(f.fileno())
    return done, time.time() - start


def merge_shards(target, n, world, item_shape, xflip):
    """Write `target/data.mdb` from the spill files of ranks 0 .. world-1: for each pass, z-i then y-i for increasing
    i, then `length` -- the `put` order of the one-GPU loop, which fixes where MdbWriter places every value, so the
    file is byte-identical to a one-GPU run's.  Every spill file is checked for its exact size before `data.mdb` is
    created; the spill files are deleted once `data.mdb` is complete.  Returns the number of records."""
    item_bytes = 4 * int(np.prod(item_shape))
    for r in range(world):
        count = len(spill_indices(n, r, world, xflip))
        for path, size in zip(spill_paths(target, r, world), (count * item_bytes, count * 8)):
            if os.path.getsize(path) != size:
                raise IOError(f"{path}: {os.path.getsize(path)} bytes, expected {size} (rank {r} did not finish)")
    chunk = max(1, (64 << 20) // item_bytes)            # records read at a time, to bound host memory
    idx = 0
    with MdbWriter(target) as db:
        for p in range(1 + xflip):
            for r in range(world):
                lo, hi = shard_range(n, r, world)
                zpath, ypath = spill_paths(target, r, world)
                with open(zpath, "rb") as fz, open(ypath, "rb") as fy:
                    fz.seek(p * (hi - lo) * item_bytes)
                    fy.seek(p * (hi - lo) * 8)
                    for c in range(lo, hi, chunk):
                        k = min(chunk, hi - c)
                        z = fz.read(k * item_bytes)
                        y = np.frombuffer(fy.read(k * 8), dtype="<i8")
                        for j in range(k):
                            db.put(f"z-{idx}".encode(), memoryview(z)[j * item_bytes:(j + 1) * item_bytes])
                            db.put(f"y-{idx}".encode(), str(int(y[j])).encode())
                            idx += 1
        db.put(b"length", str(idx).encode())
    for r in range(world):
        for path in spill_paths(target, r, world):
            os.remove(path)
    return idx


def _dataset_digest(dataset, root):
    h = hashlib.sha256()
    for path, label in dataset.samples:
        h.update(f"{os.path.relpath(path, root)}\0{label}\n".encode())
    return h.hexdigest()


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
    ap.add_argument("--num_workers", default=8, type=int, help="image decoding worker processes (per GPU)")
    args = ap.parse_args(argv)
    if args.split not in ("train", "val"):
        raise SystemExit(f"--split must be train or val, not {args.split!r}")
    if args.resolution % 8:
        raise SystemExit(f"--resolution must be a multiple of 8, not {args.resolution}")

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        # A barrier waits for the slowest rank's share, which can run for hours; torchrun stops the other ranks if
        # one fails, so the long timeout never keeps a failed run alive.
        dist.init_process_group("gloo", timeout=datetime.timedelta(hours=24))
    from maskdit_b200.vae import get_encoder
    root = os.path.join(args.data_dir, args.split)
    dataset = ImageFolderImages(root, args.resolution)
    if rank == 0:
        print(f"data size: {len(dataset)}")
    model = get_encoder(args.ckpt)
    if rank == 0:
        print(f"load vae weights from {args.ckpt}")
    target = os.path.join(args.outdir, f"{args.data_name}_{args.resolution}_latent_lmdb", args.split)
    if world > 1:
        seen = [None] * world
        dist.all_gather_object(seen, _dataset_digest(dataset, root))
        if len(set(seen)) != 1:
            raise RuntimeError(f"the ranks list different images under {root}")
        if rank == 0 and os.path.exists(os.path.join(target, "data.mdb")):
            os.remove(os.path.join(target, "data.mdb"))    # a failed run must not leave an earlier file in place
        done, secs = encode_shard(dataset, rank, world, model, target, args.batch_size, args.num_workers, args.xflip,
                                  log=print if rank == 0 else None)
        print(f"rank {rank} of {world}: encoded {done} images in {secs:.1f}s ({done / max(secs, 1e-9):.1f} img/s)",
              flush=True)
        dist.barrier()
        if rank == 0:
            begin = time.time()
            idx = merge_shards(target, len(dataset), world, (8, args.resolution // 8, args.resolution // 8),
                               args.xflip)
            print(f"merged {world} shards in {time.time() - begin:.1f}s")
            print(f"[finished] saved {idx} files to {target}")
        dist.destroy_process_group()
        return

    loader = make_loader(dataset, args.batch_size, args.num_workers)
    idx = 0
    start = time.time()
    with MdbWriter(target) as db:
        for flip in ((False, True) if args.xflip else (False,)):
            begin = time.time()
            if flip:
                print("starting to store the xflip latents")
            for moments, labels in encoded_batches(model, loader, flip, args.resolution):
                for m, lb in zip(moments, labels):
                    db.put(f"z-{idx}".encode(), np.ascontiguousarray(m, dtype="<f4"))
                    db.put(f"y-{idx}".encode(), str(int(lb)).encode())
                    idx += 1
                    if idx % 5120 == 0:
                        print(f"saved {idx} files with {time.time() - begin:.1f}s elapsed")
                        begin = time.time()
        secs = time.time() - start
        db.put(b"length", str(idx).encode())
    print(f"rank 0 of 1: encoded {idx} images in {secs:.1f}s ({idx / max(secs, 1e-9):.1f} img/s)")
    print(f"[finished] saved {idx} files to {target}")


if __name__ == "__main__":
    main()
