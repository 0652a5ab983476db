"""Step-front data path: the on-disk latent format the reference trains from, and the loader that feeds `TrainStep`.

Reference: `ImageNetLatentDataset` (train_utils/datasets.py:240-304) reads an LMDB environment `<root>/<split>` with
keys `length` (decimal string), `z-{i}` (raw little-endian fp32 bytes of the VAE moments `[2C, R, R]`, written by
extract_latent.py:69-73,106) and `y-{i}` (decimal class index); `train.py:109-115` wraps it in a DataLoader
(`shuffle=False, drop_last=True`, batch = micro-batch x grad_accum) and `helper.get_one_hot` turns the class index
into the float one-hot the label embedder consumes.

The `lmdb` Python module is not part of this image, so `MdbReader` below is a read-only walker of LMDB's on-disk
B+tree (`data.mdb`: two meta pages, branch / leaf / overflow pages) written from the published file format; when
`lmdb` IS importable it is used instead.  PARITY UNPINNED against liblmdb itself (no liblmdb here to produce a
fixture): `tests/test_data.py` round-trips files produced by `MdbWriter` / `write_mdb` (the same format, bulk-loaded).

Nothing here runs on the GPU: batches are assembled in pinned host memory and copied by the caller; the arithmetic
that follows (moments -> latent, label dropout, noise injection) is `ops.step_front` (csrc/loss_optim.cu).
"""
from __future__ import annotations

import mmap
import os
import struct

import numpy as np
import torch

P_BRANCH, P_LEAF, P_OVERFLOW, P_META = 0x01, 0x02, 0x04, 0x08
F_BIGDATA = 0x01
MDB_MAGIC = 0xBEEFC0DE
PAGEHDR = 16
P_INVALID = (1 << 64) - 1


class MdbReader:
    """Read-only point lookups in an LMDB `data.mdb` (main database, default byte-wise key order, 64-bit build)."""

    def __init__(self, path):
        f = os.path.join(path, "data.mdb") if os.path.isdir(path) else path
        self._fh = open(f, "rb")
        self._mm = mmap.mmap(self._fh.fileno(), 0, access=mmap.ACCESS_READ)
        mm = self._mm
        magic, version = struct.unpack_from("<II", mm, PAGEHDR)
        if magic != MDB_MAGIC:
            raise IOError(f"{f}: not an LMDB data file (magic {magic:#x})")
        self.psize = struct.unpack_from("<I", mm, PAGEHDR + 24)[0]   # mm_dbs[FREE_DBI].md_pad holds the page size
        best = None
        for pg in (0, 1):                                            # the meta page with the newer transaction id wins
            base = pg * self.psize + PAGEHDR
            if struct.unpack_from("<I", mm, base)[0] != MDB_MAGIC:
                continue
            txnid = struct.unpack_from("<Q", mm, base + 128)[0]
            if best is None or txnid > best[0]:
                depth = struct.unpack_from("<H", mm, base + 78)[0]
                entries, root = struct.unpack_from("<QQ", mm, base + 104)
                best = (txnid, depth, entries, root)
        self.txnid, self.depth, self.entries, self.root = best

    def close(self):
        self._mm.close()
        self._fh.close()

    def _nodes(self, pgno):
        base = pgno * self.psize
        flags, lower = struct.unpack_from("<HH", self._mm, base + 10)
        n = (lower - PAGEHDR) // 2
        return base, flags, struct.unpack_from(f"<{n}H", self._mm, base + PAGEHDR)

    def _node(self, base, off):
        lo, hi, nflags, ksize = struct.unpack_from("<HHHH", self._mm, base + off)
        key = self._mm[base + off + 8: base + off + 8 + ksize]
        return lo, hi, nflags, key, base + off + 8 + ksize

    def get(self, key: bytes):
        if self.root == P_INVALID:
            return None
        pgno = self.root
        while True:
            base, flags, ptrs = self._nodes(pgno)
            if flags & P_BRANCH:
                lo_i, hi_i = 0, len(ptrs) - 1                       # node 0 of a branch page has an empty key (= -inf)
                while lo_i < hi_i:                                   # last node whose key <= the searched key
                    mid = (lo_i + hi_i + 1) // 2
                    if self._node(base, ptrs[mid])[3] <= key:
                        lo_i = mid
                    else:
                        hi_i = mid - 1
                lo, hi, nflags, _, _ = self._node(base, ptrs[lo_i])
                pgno = lo | (hi << 16) | (nflags << 32)
                continue
            if not flags & P_LEAF:
                raise IOError(f"page {pgno}: unexpected flags {flags:#x}")
            a, b = 0, len(ptrs) - 1
            while a <= b:
                mid = (a + b) // 2
                lo, hi, nflags, k, dpos = self._node(base, ptrs[mid])
                if k == key:
                    size = lo | (hi << 16)
                    if nflags & F_BIGDATA:
                        ov = struct.unpack_from("<Q", self._mm, dpos)[0]
                        start = ov * self.psize + PAGEHDR
                        return self._mm[start:start + size]
                    return self._mm[dpos:dpos + size]
                if k < key:
                    a = mid + 1
                else:
                    b = mid - 1
            return None


class MdbWriter:
    """Stream a fresh single-database LMDB file `<path>/data.mdb` (main database, byte-wise key order, 64-bit layout).

    `put(key, value)` appends a value too large for a leaf node (every latent) to the file at once as overflow pages,
    so memory holds only the keys, their (overflow page, size) pairs and the small inline values; `close()` sorts the
    keys and writes the leaf and branch pages after the overflow pages, then the two meta pages (pages 0 and 1, reserved
    at open).  This is how extract_latent.py writes hundreds of GB of moments; the reference uses liblmdb
    (extract_latent.py:60-106)."""

    def __init__(self, path, psize=4096):
        os.makedirs(path, exist_ok=True)
        self.psize = psize
        self._f = open(os.path.join(path, "data.mdb"), "wb")
        self._f.write(bytes(2 * psize))                      # pages 0 and 1: the meta pages, written by close()
        self._next = 2
        self._small, self._big = {}, {}                      # key -> value bytes | key -> (first overflow page, size)
        self._n_over = 0
        self._nodemax = psize // 2 - PAGEHDR

    def __enter__(self):
        return self

    def __exit__(self, exc_type, *exc):
        if self._f is None:
            return
        if exc_type is None:
            self.close()
        else:                                                # leave an unfinished file rather than a valid-looking one
            self._f.close()
            self._f = None

    def _alloc(self, n=1):
        p = self._next
        self._next += n
        return p

    def put(self, key, value):
        key = bytes(key)
        if key in self._small or key in self._big:
            raise KeyError(f"duplicate key {key!r}")
        mv = memoryview(value).cast("B")
        n = mv.nbytes
        if 8 + len(key) + n <= self._nodemax:
            self._small[key] = mv.tobytes()
            return
        npg = (PAGEHDR + n + self.psize - 1) // self.psize     # value goes to overflow pages
        ov = self._alloc(npg)
        self._f.write(struct.pack("<QHHI", ov, 0, P_OVERFLOW, npg))
        self._f.write(mv)
        self._f.write(bytes(npg * self.psize - PAGEHDR - n))
        self._n_over += npg
        self._big[key] = (ov, n)

    def _page(self, flags, nodes):
        pgno = self._alloc()
        psize = self.psize
        buf = bytearray(psize)
        upper = psize
        ptrs = []
        for nd in nodes:
            upper -= len(nd) + (len(nd) & 1)
            buf[upper:upper + len(nd)] = nd
            ptrs.append(upper)
        lower = PAGEHDR + 2 * len(ptrs)
        assert lower <= upper
        struct.pack_into("<QHHHH", buf, 0, pgno, 0, flags, lower, upper)
        struct.pack_into(f"<{len(ptrs)}H", buf, PAGEHDR, *ptrs)
        self._f.write(buf)
        return pgno

    def _fits(self, used, count, nd):
        return PAGEHDR + 2 * (count + 1) + used + len(nd) + (len(nd) & 1) <= self.psize

    def close(self):
        keys = sorted([*self._small, *self._big])
        n_leaf = n_branch = 0
        level = []          # (first key, pgno)
        cur, used, first = [], 0, None
        for k in keys:
            if k in self._big:
                ov, n = self._big[k]
                nd = struct.pack("<HHHH", n & 0xFFFF, n >> 16, F_BIGDATA, len(k)) + k + struct.pack("<Q", ov)
            else:
                v = self._small[k]
                nd = struct.pack("<HHHH", len(v) & 0xFFFF, len(v) >> 16, 0, len(k)) + k + v
            if cur and not self._fits(used, len(cur), nd):
                level.append((first, self._page(P_LEAF, cur)))
                n_leaf += 1
                cur, used, first = [], 0, None
            if first is None:
                first = k
            cur.append(nd)
            used += len(nd) + (len(nd) & 1)
        if cur:
            level.append((first, self._page(P_LEAF, cur)))
            n_leaf += 1
        depth = 1 if level else 0
        while len(level) > 1:
            nxt, cur, used, first = [], [], 0, None
            for k, pg in level:
                kk = b"" if not cur else k
                nd = struct.pack("<HHHH", pg & 0xFFFF, (pg >> 16) & 0xFFFF, (pg >> 32) & 0xFFFF, len(kk)) + kk
                if cur and not self._fits(used, len(cur), nd):
                    nxt.append((first, self._page(P_BRANCH, cur)))
                    n_branch += 1
                    cur, used, first = [], 0, None
                    nd = struct.pack("<HHHH", pg & 0xFFFF, (pg >> 16) & 0xFFFF, (pg >> 32) & 0xFFFF, 0)
                if first is None:
                    first = k
                cur.append(nd)
                used += len(nd) + (len(nd) & 1)
            nxt.append((first, self._page(P_BRANCH, cur)))
            n_branch += 1
            level = nxt
            depth += 1
        root = level[0][1] if level else P_INVALID
        psize, last_pg = self.psize, self._next - 1
        for m in (0, 1):
            buf = bytearray(psize)
            struct.pack_into("<QHHI", buf, 0, m, 0, P_META, 0)
            b = PAGEHDR
            struct.pack_into("<IIQQ", buf, b, MDB_MAGIC, 1, 0, max(1 << 20, (last_pg + 1) * psize))
            struct.pack_into("<IHHQQQQQ", buf, b + 24, psize, 0, 0, 0, 0, 0, 0, P_INVALID)    # free DB (empty)
            struct.pack_into("<IHHQQQQQ", buf, b + 72, 0, 0, depth, n_branch, n_leaf, self._n_over, len(keys), root)
            struct.pack_into("<QQ", buf, b + 120, last_pg, 1 if m == 1 else 0)
            self._f.seek(m * psize)
            self._f.write(buf)
        self._f.close()
        self._f = None
        self._small, self._big = {}, {}


def write_mdb(path, items, psize=4096):
    """Bulk-load `items` (dict bytes -> bytes) into a fresh single-database LMDB file `<path>/data.mdb` (tests and
    synthetic datasets; the reference writes these with liblmdb, extract_latent.py:60-106)."""
    with MdbWriter(path, psize) as w:
        for k, v in items.items():
            w.put(k, v)


def write_latent_lmdb(root, moments, labels, split="train"):
    """`<root>/<split>` in the layout extract_latent.py produces: z-{i} raw fp32 moments, y-{i} class index, length."""
    items = {b"length": str(len(labels)).encode()}
    for i, (z, y) in enumerate(zip(moments, labels)):
        items[f"z-{i}".encode()] = np.ascontiguousarray(z, dtype="<f4").tobytes()
        items[f"y-{i}".encode()] = str(int(y)).encode()
    write_mdb(os.path.join(root, split), items)


# ---- image side of the latent extraction (extract_latent.py:16-110) --------------------------------------------------
IMG_EXTENSIONS = (".jpg", ".jpeg", ".png", ".ppm", ".bmp", ".pgm", ".tif", ".tiff", ".webp")   # torchvision's list


def image_folder_samples(root):
    """(path, class index) of every image under `root` in ImageFolder order: class directories sorted by name and
    numbered in that order, each walked recursively with sorted directories and sorted file names, files kept by
    (case-insensitive) image extension.  This is the order `ImageFolder.imgs` gives extract_latent.py's dataset
    (train_utils/datasets.py:73-77), so z-{i} / y-{i} are numbered as the reference numbers them."""
    classes = sorted(e.name for e in os.scandir(root) if e.is_dir())
    if not classes:
        raise FileNotFoundError(f"no class directories under {root}")
    out = []
    for idx, c in enumerate(classes):
        for d, _, fnames in sorted(os.walk(os.path.join(root, c), followlinks=True)):
            for f in sorted(fnames):
                if f.lower().endswith(IMG_EXTENSIONS):
                    out.append((os.path.join(d, f), idx))
    return out, classes


def center_crop_arr(pil_image, image_size):
    """ADM centre crop (the rule of train_utils/datasets.py:19-37): halve with a BOX filter while the short side is at
    least twice the target, resize BICUBIC so the short side equals the target, crop the centre.  -> uint8 [R, R, C]."""
    from PIL import Image
    while min(*pil_image.size) >= 2 * image_size:
        pil_image = pil_image.resize(tuple(x // 2 for x in pil_image.size), resample=Image.BOX)
    scale = image_size / min(*pil_image.size)
    pil_image = pil_image.resize(tuple(round(x * scale) for x in pil_image.size), resample=Image.BICUBIC)
    arr = np.asarray(pil_image)
    y0, x0 = (arr.shape[0] - image_size) // 2, (arr.shape[1] - image_size) // 2
    return arr[y0:y0 + image_size, x0:x0 + image_size]


def load_image(path, resolution):
    """One extract_latent.py input: PIL decode, RGB, centre crop, then ToTensor + Normalize(0.5, 0.5) arithmetic
    (x / 255 then (x - 0.5) / 0.5 in fp32) -> float32 [3, R, R] in [-1, 1]."""
    from PIL import Image
    with Image.open(path) as im:
        arr = center_crop_arr(im.convert("RGB"), resolution)
    x = np.ascontiguousarray(arr.transpose(2, 0, 1)).astype(np.float32) / np.float32(255)
    return (x - np.float32(0.5)) / np.float32(0.5)


class ImageNetLatentDataset:
    """train_utils/datasets.py:240-304 (latent + class index; the `feat_path` / `xflip` variants are not used by any
    shipped config and raise).  `__getitem__` -> (moments float32 [2C, R, R], one-hot float32 [num_classes])."""

    def __init__(self, path, resolution=32, num_channels=4, split="train", num_classes=1000, feat_path=None,
                 feat_dim=0, xflip=False):
        if feat_path is not None or feat_dim or xflip:
            raise NotImplementedError("feature-conditioned / x-flipped latent datasets are outside the MaskDiT hot path")
        self._path = os.path.join(path, split)
        if not os.path.exists(os.path.join(self._path, "data.mdb")):
            raise FileNotFoundError(f"no LMDB latent dataset at {self._path} (expected data.mdb; "
                                    "reference layout: extract_latent.py)")
        self.resolution, self.num_channels, self.num_classes = resolution, num_channels, num_classes
        try:
            import lmdb  # noqa: F401 - liblmdb when the module exists
            self._env = lmdb.open(self._path, readonly=True, lock=False, create=False)
            self._txn = self._env.begin(write=False)
            self._get = self._txn.get
        except ImportError:
            self._rd = MdbReader(self._path)
            self._get = self._rd.get
        self.length = int(bytes(self._get(b"length")).decode())

    def __len__(self):
        return self.length

    def raw(self, idx):
        z = np.frombuffer(bytes(self._get(f"z-{idx}".encode())), dtype="<f4").reshape(
            -1, self.resolution, self.resolution).copy()                      # datasets.py:289: .copy()
        return z, int(bytes(self._get(f"y-{idx}".encode())).decode())

    def __getitem__(self, idx):
        z, y = self.raw(idx)
        onehot = np.zeros(self.num_classes, dtype=np.float32)   # helper.get_one_hot (train_utils/helper.py:30-33)
        onehot[y] = 1
        return z, onehot


def batches(dataset, batch, rank=0, world=1, start=0, pin=True):
    """Sequential, rank-strided, drop-last batches forever (train.py:109-115: `shuffle=False, drop_last=True`; the
    reference shards by accelerate's loader wrapper).  Yields pinned host tensors (moments [B,2C,R,R], labels [B,nc])."""
    n = len(dataset)
    per_epoch = n // (batch * world)
    if per_epoch == 0:
        raise ValueError(f"dataset of {n} items is smaller than one global batch ({batch} x {world})")
    z0, y0 = dataset[0]
    zb = torch.empty((batch, *z0.shape), dtype=torch.float32)
    yb = torch.empty((batch, y0.shape[0]), dtype=torch.float32)
    if pin and torch.cuda.is_available():
        zb, yb = zb.pin_memory(), yb.pin_memory()
    it = start
    while True:
        b = it % per_epoch
        base = (b * world + rank) * batch
        for j in range(batch):
            z, y = dataset[base + j]
            zb[j] = torch.from_numpy(np.ascontiguousarray(z))
            yb[j] = torch.from_numpy(y)
        yield zb, yb
        it += 1


# ---- WebDataset shards (lmdb2wds.py:26, train_wds.py:58-64) ------------------------------------------------------------
class WdsShardWriter:
    """Stream samples into the tar shards `pattern % 0`, `pattern % 1`, ... in the layout lmdb2wds.py writes:
    `<key>.latent` = pickle of the [2C,R,R] float32 array, `<key>.cls` = the class index as ASCII (webdataset's default
    encoding of an int).  A shard holds at most `maxcount` samples and at most `maxsize` payload bytes (the member
    contents, as `webdataset.ShardWriter` counts them): a sample that would push the current shard past `maxsize` starts
    the next one, and a sample larger than `maxsize` gets a shard of its own.  The first shard is opened at once, so no
    samples give one empty shard, as with webdataset.  Only the open shard's tar stream is held, so any number of samples
    can be written.  `paths` lists the shards written so far; a run that raises removes the unfinished shard."""

    def __init__(self, pattern, maxcount=100000, maxsize=3e9):
        if maxcount < 1 or maxsize <= 0:
            raise ValueError(f"maxcount ({maxcount}) and maxsize ({maxsize}) must be positive")
        self.pattern, self.maxcount, self.maxsize = pattern, maxcount, maxsize
        self.paths, self._tar = [], None
        self._next_shard()

    def _next_shard(self):
        import tarfile
        self.close()
        self.paths.append(self.pattern % len(self.paths))
        self._tar = tarfile.open(self.paths[-1], "w")
        self._count = self._size = 0

    def __enter__(self):
        return self

    def __exit__(self, exc_type, *exc):
        if self._tar is None:
            return
        if exc_type is None:
            self.close()
        else:
            self._tar.close()
            self._tar = None
            os.remove(self.paths.pop())

    def write(self, key, moments, label):
        import io
        import pickle
        import tarfile
        if self._tar is None:
            raise ValueError("write to a closed WdsShardWriter")
        members = (("latent", pickle.dumps(np.ascontiguousarray(moments, dtype=np.float32))),
                   ("cls", str(int(label)).encode()))
        size = sum(len(p) for _, p in members)
        if self._count >= self.maxcount or (self._count and self._size + size > self.maxsize):
            self._next_shard()
        for ext, payload in members:
            ti = tarfile.TarInfo(f"{key}.{ext}")
            ti.size = len(payload)
            self._tar.addfile(ti, io.BytesIO(payload))
        self._count += 1
        self._size += size

    def close(self):
        if self._tar is not None:
            self._tar.close()
            self._tar = None


def write_wds_shard(path, moments, labels, start=0):
    """One tar shard holding every sample, keys `{start + i:07d}` (`WdsShardWriter`'s layout)."""
    pattern = "%.0s" + path.replace("%", "%%")          # the shard number formats to nothing: the shard is `path`
    with WdsShardWriter(pattern, maxcount=float("inf"), maxsize=float("inf")) as w:
        for i, (z, y) in enumerate(zip(moments, labels)):
            w.write(f"{start + i:07d}", z, y)


def wds_samples(shards, rank=0, world=1, num_classes=1000):
    """Iterate (moments float32 [2C,R,R], one-hot float32 [num_classes]) over this rank's shards, forever
    (train_wds.py:44-48 splits the shard list `data_list[rank::world]`; :58-64 decodes `latent` with pickle and `cls`
    as a decimal string).  Pickle is executed: shards must be trusted, as in the reference."""
    import pickle
    import tarfile
    mine = list(shards)[rank::world]
    if not mine:
        raise ValueError(f"{len(list(shards))} shards cannot be split over {world} ranks")
    while True:
        for path in mine:
            with tarfile.open(path, "r") as tf:
                cur, item = None, {}
                for m in tf:
                    if not m.isfile():
                        continue
                    key, _, ext = m.name.rpartition(".")
                    if key != cur and item:
                        item = {}
                    cur = key
                    item[ext] = tf.extractfile(m).read()
                    if "latent" in item and "cls" in item:
                        z = np.asarray(pickle.loads(item["latent"]), dtype=np.float32)
                        onehot = np.zeros(num_classes, dtype=np.float32)
                        onehot[int(item["cls"].decode("utf-8"))] = 1
                        item = {}
                        yield z, onehot


def wds_batches(shards, batch, rank=0, world=1, num_classes=1000, pin=True):
    """Drop-last batches of pinned host tensors from WebDataset shards (the loader train_wds.py:66-95 builds)."""
    it = wds_samples(shards, rank, world, num_classes)
    z0, y0 = next(it)
    zb = torch.empty((batch, *z0.shape), dtype=torch.float32)
    yb = torch.empty((batch, y0.shape[0]), dtype=torch.float32)
    if pin and torch.cuda.is_available():
        zb, yb = zb.pin_memory(), yb.pin_memory()
    pending = [(z0, y0)]
    while True:
        for j in range(batch):
            z, y = pending.pop() if pending else next(it)
            zb[j] = torch.from_numpy(z)
            yb[j] = torch.from_numpy(y)
        yield zb, yb
