"""GPU: extract_latent.py over W ranks writes the same data.mdb, byte for byte, as a one-GPU run.  Every rank's share
is encoded in this one process on one GPU (`encode_shard`), then merged (`merge_shards`); a real two-process torchrun
run needs two GPUs and is skipped below that."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
RES = 256
SIZES = [(300, 261), (257, 399), (411, 283), (263, 263), (517, 301), (285, 459), (333, 271), (271, 349), (389, 389),
         (301, 513), (260, 290), (455, 277), (281, 281), (267, 405), (359, 263), (299, 311), (275, 500), (421, 333),
         (313, 279), (265, 377)]


def make_folder(root, sizes, classes=3):
    """Synthetic ImageFolder: odd, non-square sizes, JPEG and PNG, `classes` class directories."""
    from PIL import Image
    rng = np.random.default_rng(len(sizes))
    for i, (w, h) in enumerate(sizes):
        d = root / "train" / f"n{i % classes:02d}"
        d.mkdir(parents=True, exist_ok=True)
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(d / f"im{i}.{'png' if i % 2 else 'jpg'}")
    return str(root)


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory):
    from oracle import vae_encode_oracle as VE
    p = tmp_path_factory.mktemp("ckpt") / "vae.pth"
    torch.save(VE.make_vae_encoder_state_dict(4), p)
    return str(p)


def one_gpu(data_dir, ckpt, outdir, xflip, monkeypatch):
    import extract_latent as E
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    E.main(["--data_dir", data_dir, "--resolution", str(RES), "--batch_size", "8", "--ckpt", ckpt, "--outdir", outdir,
            "--num_workers", "0", *(["--xflip"] if xflip else [])])
    return os.path.join(outdir, f"imagenet_{RES}_latent_lmdb", "train", "data.mdb")


def read(path):
    with open(path, "rb") as f:
        return f.read()


@pytest.mark.parametrize("n,xflip", [(20, False), (20, True), (2, True)])
def test_three_ranks_in_one_process_write_the_one_gpu_file(tmp_path, ckpt, monkeypatch, n, xflip):
    """W = 3: 7 / 7 / 6 images, or with n = 2 an empty rank 2; with xflip each rank also runs its mirrored pass."""
    import extract_latent as E
    from maskdit_b200.vae import get_encoder
    data_dir = make_folder(tmp_path / "data", SIZES[:n], classes=min(n, 3))
    want = read(one_gpu(data_dir, ckpt, str(tmp_path / "one"), xflip, monkeypatch))
    dataset = E.ImageFolderImages(os.path.join(data_dir, "train"), RES)
    model = get_encoder(ckpt)
    target = str(tmp_path / "multi")
    for r in range(3):
        done, _ = E.encode_shard(dataset, r, 3, model, target, batch_size=4, num_workers=0, xflip=xflip)
        assert done == len(E.spill_indices(n, r, 3, xflip))
    assert E.merge_shards(target, n, 3, (8, RES // 8, RES // 8), xflip) == n * (1 + xflip)
    got = read(os.path.join(target, "data.mdb"))
    assert len(got) == len(want) and got == want
    assert sorted(os.listdir(target)) == ["data.mdb"]


def test_mirrored_pass_is_encode_moments_with_flip(tmp_path, ckpt, monkeypatch):
    from maskdit_b200 import data as D
    from maskdit_b200.vae import get_encoder
    data_dir = make_folder(tmp_path / "data", SIZES)
    rd = D.MdbReader(one_gpu(data_dir, ckpt, str(tmp_path / "one"), True, monkeypatch))
    samples, _ = D.image_folder_samples(os.path.join(data_dir, "train"))
    n = len(samples)
    assert bytes(rd.get(b"length")) == str(2 * n).encode()
    model = get_encoder(ckpt)
    for i in (0, 7, n - 1):
        x = torch.from_numpy(D.load_image(samples[i][0], RES))[None].cuda()
        for idx, flip in ((i, False), (n + i, True)):
            want = model.encode_moments(x, flip=flip)[0].cpu().numpy()
            got = np.frombuffer(bytes(rd.get(f"z-{idx}".encode())), "<f4").reshape(want.shape)
            assert np.array_equal(got, want), (i, flip)
            assert bytes(rd.get(f"y-{idx}".encode())) == str(samples[i][1]).encode()
    rd.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_torchrun_two_processes_write_the_one_gpu_file(tmp_path, ckpt, monkeypatch):
    data_dir = make_folder(tmp_path / "data", SIZES[:11])
    want = read(one_gpu(data_dir, ckpt, str(tmp_path / "one"), True, monkeypatch))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29643", os.path.join(ROOT, "extract_latent.py"), "--data_dir", data_dir,
           "--resolution", str(RES), "--batch_size", "4", "--ckpt", ckpt, "--outdir", str(tmp_path / "two"),
           "--num_workers", "2", "--xflip"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path),
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "rank 0 of 2" in r.stdout and "rank 1 of 2" in r.stdout and "saved 22 files" in r.stdout, r.stdout
    assert read(str(tmp_path / "two" / f"imagenet_{RES}_latent_lmdb" / "train" / "data.mdb")) == want
