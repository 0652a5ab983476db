"""CPU: lmdb2wds.py turns the latent LMDB into WebDataset tar shards that `data.wds_samples` (train.py --wds) reads
back bit for bit, with the reference's shard names and the webdataset shard-size rules."""
import os
import pickle
import sys
import tarfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lmdb2wds  # noqa: E402
from maskdit_b200 import data as D  # noqa: E402

N, C, R = 23, 8, 8


@pytest.fixture
def latent_db(tmp_path):
    rng = np.random.default_rng(5)
    moments = rng.standard_normal((N, C, R, R)).astype(np.float32)
    labels = rng.integers(0, 1000, N)
    D.write_latent_lmdb(str(tmp_path / "lmdb"), moments, labels)
    return str(tmp_path / "lmdb"), moments, labels


def convert(tmp_path, db, *extra):
    return lmdb2wds.main(["--datadir", db, "--outdir", str(tmp_path / "wds"), "--resolution", str(R),
                          "--num_channels", str(C), *extra])


def read_back(paths):
    it = D.wds_samples(paths, num_classes=1000)
    return [next(it) for _ in range(N)]


def test_round_trip_in_shards_of_maxcount(tmp_path, latent_db):
    db, moments, labels = latent_db
    paths = convert(tmp_path, db, "--maxcount", "10")
    assert [os.path.basename(p) for p in paths] == [f"latent_imagenet_512_train-{s:04d}.tar" for s in range(3)]
    assert sorted(os.listdir(tmp_path / "wds")) == [os.path.basename(p) for p in paths]
    counts = []
    for p in paths:
        with tarfile.open(p) as tf:
            counts.append(len(tf.getnames()) // 2)
    assert counts == [10, 10, 3]
    for i, (z, onehot) in enumerate(read_back(paths)):                  # index order, every moment bit-exact
        assert z.dtype == np.float32 and np.array_equal(z, moments[i]) and onehot.argmax() == labels[i], i


def test_tar_members_parse(tmp_path, latent_db):
    db, moments, labels = latent_db
    paths = convert(tmp_path, db, "--maxcount", "10")
    i = 0
    for p in paths:
        with tarfile.open(p) as tf:
            members = tf.getmembers()
            assert [m.name for m in members] == [f"{j:07d}.{ext}" for j in range(i, i + len(members) // 2)
                                                 for ext in ("latent", "cls")]
            for m in members:
                payload = tf.extractfile(m).read()
                assert m.isfile() and m.size == len(payload) and m.mode == 0o644
                if m.name.endswith(".latent"):
                    z = pickle.loads(payload)
                    assert type(z) is np.ndarray and z.dtype == np.float32 and z.shape == (C, R, R)
                    assert np.array_equal(z, moments[i])
                else:
                    assert payload == str(labels[i]).encode("ascii")
                    i += 1
    assert i == N


def test_maxsize_below_two_samples_gives_one_sample_per_shard(tmp_path, latent_db):
    db, moments, labels = latent_db
    one = len(pickle.dumps(moments[0])) + 1                # the smallest sample: a one-digit class index
    paths = convert(tmp_path, db, "--maxsize", str(2 * one - 1))
    assert len(paths) == N
    for p in paths:
        with tarfile.open(p) as tf:
            assert len(tf.getnames()) == 2
    assert all(np.array_equal(z, moments[i]) for i, (z, _) in enumerate(read_back(paths)))


def test_shard_writer_rules(tmp_path):
    """maxcount and maxsize together; a sample larger than maxsize gets a shard of its own; no samples -> one empty
    shard; a failed run removes its unfinished shard; write_wds_shard is one shard of the same writer."""
    z = np.zeros((2, 2, 2), np.float32)
    one = len(pickle.dumps(z)) + 1
    pattern = str(tmp_path / "s-%02d.tar")
    with D.WdsShardWriter(pattern, maxcount=3, maxsize=2.5 * one) as w:
        for i in range(7):
            w.write(f"{i:07d}", z, i % 10)
    sizes = []
    for p in w.paths:
        with tarfile.open(p) as tf:
            sizes.append(len(tf.getnames()) // 2)
    assert sizes == [2, 2, 2, 1]
    with D.WdsShardWriter(str(tmp_path / "big-%d.tar"), maxsize=one // 2) as w:
        for i in range(3):
            w.write(f"{i:07d}", z, 1)
    assert len(w.paths) == 3
    with D.WdsShardWriter(str(tmp_path / "empty-%d.tar")) as w:
        pass
    with tarfile.open(w.paths[0]) as tf:
        assert w.paths == [str(tmp_path / "empty-0.tar")] and tf.getnames() == []
    with pytest.raises(RuntimeError):
        with D.WdsShardWriter(str(tmp_path / "fail-%d.tar"), maxcount=2) as w:
            for i in range(3):
                w.write(f"{i:07d}", z, 1)
            raise RuntimeError("conversion failed")
    assert sorted(p.name for p in tmp_path.glob("fail-*")) == ["fail-0.tar"]
    D.write_wds_shard(str(tmp_path / "one%.tar"), [z] * 3, [4, 5, 6], start=7)
    with tarfile.open(tmp_path / "one%.tar") as tf:
        assert tf.getnames() == [f"{k:07d}.{e}" for k in (7, 8, 9) for e in ("latent", "cls")]


def test_rejects_a_wrong_resolution(tmp_path, latent_db):
    db, _, _ = latent_db
    with pytest.raises(ValueError):
        convert(tmp_path, db, "--resolution", "4")
