"""CPU: the host side of multi-GPU latent extraction -- how extract_latent.py splits the images over ranks, and the
merge of the ranks' spill files into a data.mdb byte-identical to the one-GPU file."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import extract_latent as E  # noqa: E402
from maskdit_b200 import data as D  # noqa: E402


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("n", [0, 1, 5, 7, 64, 1000])
def test_shard_ranges_are_contiguous_disjoint_and_cover(n, world):
    ranges = [E.shard_range(n, r, world) for r in range(world)]
    assert ranges[0][0] == 0 and ranges[-1][1] == n
    for (lo, hi), (lo2, _) in zip(ranges, ranges[1:]):
        assert hi == lo2                                     # contiguous and disjoint, in rank order
    sizes = [hi - lo for lo, hi in ranges]
    assert sizes == [n // world + (r < n % world) for r in range(world)]   # the first n % world ranks get one more
    if n < world:
        assert sizes.count(0) == world - n
    for xflip in (False, True):
        got = sorted(i for r in range(world) for i in E.spill_indices(n, r, world, xflip))
        assert got == list(range(n * (1 + xflip)))


def test_spill_indices_put_mirrored_item_i_at_n_plus_i():
    assert E.spill_indices(7, 1, 3, False) == [3, 4]
    assert E.spill_indices(7, 1, 3, True) == [3, 4, 10, 11]      # pass 1: item i -> N + i
    assert E.spill_indices(2, 2, 3, True) == []                   # N < W: rank 2 has nothing


def write_spills(target, moments, labels, world, xflip):
    """What encode_shard leaves for each rank: its records in spill_indices order, raw <f4 moments and <i8 labels."""
    n = len(labels)
    for r in range(world):
        idx = E.spill_indices(n, r, world, xflip)
        zpath, ypath = E.spill_paths(target, r, world)
        with open(zpath, "wb") as f:
            f.write(np.ascontiguousarray(moments[idx], dtype="<f4").tobytes())
        with open(ypath, "wb") as f:
            f.write(np.asarray([labels[i % n] for i in idx], dtype="<i8").tobytes())


def one_gpu_file(path, moments, labels, xflip):
    """data.mdb as extract_latent.py's one-GPU loop writes it: per pass z-i, y-i for increasing i, then length."""
    n = len(labels)
    with D.MdbWriter(path) as db:
        for i in range(n * (1 + xflip)):
            db.put(f"z-{i}".encode(), np.ascontiguousarray(moments[i], dtype="<f4"))
            db.put(f"y-{i}".encode(), str(int(labels[i % n])).encode())
        db.put(b"length", str(n * (1 + xflip)).encode())
    with open(os.path.join(path, "data.mdb"), "rb") as f:
        return f.read()


@pytest.mark.parametrize("xflip", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("n,shape", [(2, (8, 8, 8)), (11, (8, 8, 8)), (9, (8, 2, 2))])
def test_merge_is_byte_identical_to_one_gpu_file(tmp_path, n, shape, world, xflip):
    """8x8x8 moments go to overflow pages, 8x2x2 stay inline in the leaves; n = 2 leaves rank 2 of 3 empty."""
    rng = np.random.default_rng(n * 10 + world)
    moments = rng.standard_normal((n * (1 + xflip), *shape)).astype(np.float32)
    labels = rng.integers(0, 1000, n)
    want = one_gpu_file(str(tmp_path / "one"), moments, labels, xflip)
    target = str(tmp_path / "multi")
    os.makedirs(target)
    write_spills(target, moments, labels, world, xflip)
    assert E.merge_shards(target, n, world, shape, xflip) == n * (1 + xflip)
    assert sorted(os.listdir(target)) == ["data.mdb"]                       # spill files removed
    with open(os.path.join(target, "data.mdb"), "rb") as f:
        assert f.read() == want
    readers = [D.MdbReader(target)]
    try:
        import lmdb
        env = lmdb.open(target, readonly=True, lock=False, create=False)
        readers.append(env.begin(write=False))
    except ImportError:
        pass
    for rd in readers:
        assert bytes(rd.get(b"length")) == str(n * (1 + xflip)).encode()
        for i in range(n * (1 + xflip)):
            assert np.array_equal(np.frombuffer(bytes(rd.get(f"z-{i}".encode())), "<f4").reshape(shape), moments[i])
            assert bytes(rd.get(f"y-{i}".encode())) == str(labels[i % n]).encode()


def test_merge_refuses_an_unfinished_rank(tmp_path):
    """A spill file one record short (a rank that did not finish): no data.mdb is written and the spills stay."""
    rng = np.random.default_rng(0)
    moments = rng.standard_normal((5, 8, 2, 2)).astype(np.float32)
    labels = rng.integers(0, 10, 5)
    write_spills(str(tmp_path), moments, labels, 2, False)
    zpath, _ = E.spill_paths(str(tmp_path), 1, 2)
    with open(zpath, "r+b") as f:
        f.truncate(os.path.getsize(zpath) - 4 * 8 * 2 * 2)
    with pytest.raises(IOError, match="did not finish"):
        E.merge_shards(str(tmp_path), 5, 2, (8, 2, 2), False)
    assert not os.path.exists(tmp_path / "data.mdb") and len(os.listdir(tmp_path)) == 4
