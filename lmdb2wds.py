#!/usr/bin/env python
"""Convert the latent LMDB that `extract_latent.py` writes into the WebDataset tar shards `train.py --wds` reads, with
the reference's CLI (lmdb2wds.py:17-40):

    python lmdb2wds.py --maxcount 10010 --datadir <dir>/imagenet512-latent --outdir <dir>/imagenet512-latent-wds \\
        --resolution 64 --num_channels 8 [--split train] [--maxsize 1e10]

Input: `{datadir}/{split}/data.mdb` (`data.ImageNetLatentDataset`: liblmdb when the `lmdb` module exists, else the
file walker `MdbReader`).  Output: `{outdir}/latent_imagenet_512_{split}-%04d.tar`, sample i under the key `{i:07d}`
(`.latent` = pickle of the float32 [num_channels, R, R] moments, `.cls` = the class index as ASCII), a new shard every
`--maxcount` samples or before a sample that would take the shard's payload past `--maxsize` bytes
(`data.WdsShardWriter`).  Neither webdataset nor tqdm is needed.
"""
import argparse
import os

from maskdit_b200.data import ImageNetLatentDataset, WdsShardWriter


def main(argv=None):
    ap = argparse.ArgumentParser("Convert the latent imagenet dataset to WebDataset")
    ap.add_argument("--maxcount", type=int, default=10010, help="max number of entries per shard")
    ap.add_argument("--maxsize", type=float, default=10 ** 10, help="max size per shard")
    ap.add_argument("--outdir", type=str, default="latent_imagenet_wds", help="path to save the converted dataset")
    ap.add_argument("--datadir", type=str, default="latent_imagenet", help="path to the latent imagenet dataset")
    ap.add_argument("--resolution", type=int, default=64, help="image resolution")
    ap.add_argument("--num_channels", type=int, default=8, help="number of image channels")
    ap.add_argument("--split", type=str, default="train", help="split of the dataset")
    args = ap.parse_args(argv)
    if args.maxcount < 1 or args.maxsize <= 0:
        raise SystemExit(f"--maxcount and --maxsize must be positive, not {args.maxcount} and {args.maxsize}")

    os.makedirs(args.outdir, exist_ok=True)
    pattern = os.path.join(args.outdir, f"latent_imagenet_512_{args.split}-%04d.tar")
    dataset = ImageNetLatentDataset(args.datadir, resolution=args.resolution, num_channels=args.num_channels,
                                    split=args.split)
    shape = (args.num_channels, args.resolution, args.resolution)
    with WdsShardWriter(pattern, maxcount=args.maxcount, maxsize=args.maxsize) as sink:
        for i in range(len(dataset)):
            if i % args.maxcount == 0:
                print(f"writing to the {i // args.maxcount}th shard")
            z, label = dataset.raw(i)
            if z.shape != shape:          # a wrong --resolution reshapes the moments without failing
                raise ValueError(f"z-{i} has shape {z.shape}, not {shape} (--num_channels, --resolution)")
            sink.write(f"{i:07d}", z, label)
    print(f"[finished] wrote {len(dataset)} samples to {len(sink.paths)} shards in {args.outdir}")
    return sink.paths


if __name__ == "__main__":
    main()
