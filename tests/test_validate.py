"""CPU: the held-out denoising loss (maskdit_b200/validate.py).

1. The noise levels are the stratified quantiles of the training lognormal; K = 1 gives its median exp(P_mean).
2. The draws of an item depend on (seed, item) alone: any batching and any rank split give every row the same inputs,
   and scoring leaves torch's global RNG untouched.
3. A gloo world-2 run returns every item exactly once, in index order, with the same numbers on both ranks as one
   process.
4. The CPU oracle (oracle/val_oracle.py) matches the unmodified reference's golden (tests/golden/val_s2.npz) at the
   loss tolerance of DESIGN §6, and the batched driver fed the oracle's row scorer matches it too.
5. The new flags of train.py and val_loss.py default to off or to their documented values.
"""
import os
import sys

import numpy as np
import pytest
import torch
from scipy import stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from maskdit_b200 import validate as V  # noqa: E402
from oracle import maskdit_oracle as O  # noqa: E402
from oracle import val_oracle as VO  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "val_s2.npz")
SMALL = O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10)


# ---- 1. levels -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2, 5, 8, 32])
def test_sigma_levels_are_lognormal_quantiles(K):
    s = V.sigma_levels(K)
    assert s.dtype == np.float64 and s.shape == (K,) and np.all(np.diff(s) > 0)
    cdf = stats.lognorm.cdf(s, 1.2, scale=np.exp(-1.2))     # training sigma = exp(N(-1.2, 1.2^2))
    np.testing.assert_allclose(cdf, (np.arange(K) + 0.5) / K, rtol=0, atol=1e-12)
    np.testing.assert_allclose(V.level_normals(K), stats.norm.ppf((np.arange(K) + 0.5) / K), atol=1e-12)
    np.testing.assert_allclose(VO.level_normals(K), V.level_normals(K), rtol=0, atol=0)


def test_one_level_is_the_median():
    assert V.sigma_levels(1)[0] == pytest.approx(np.exp(-1.2), rel=1e-15)
    assert V.level_normals(1)[0] == 0.0
    with pytest.raises(ValueError):
        V.level_normals(0)


# ---- 2. draws --------------------------------------------------------------------------------------------------------
class Recorder:
    """A scorer that records each row's inputs and returns a loss computed from all of them."""

    def __init__(self):
        self.rows = []

    def __call__(self, moments, eps, rnd_normal, noise, labels):
        for j in range(moments.shape[0]):
            self.rows.append((moments[j].clone(), eps[j].clone(), float(rnd_normal[j]), noise[j].clone(),
                              None if labels is None else labels[j].clone()))
        lab = labels.argmax(1).float() if labels is not None else torch.zeros(moments.shape[0])
        return (moments.mean((1, 2, 3)) + eps.pow(2).mean((1, 2, 3)) * rnd_normal.exp()
                + noise.mean((1, 2, 3)) + lab)


def _held(n=7, R=4, C=2, nc=5):
    g = torch.Generator().manual_seed(9)
    return V.HeldOut(torch.randn(n, 2 * C, R, R, generator=g),
                     torch.eye(nc)[torch.randint(0, nc, (n,), generator=g)])


def test_draws_do_not_depend_on_batching_or_rank_split():
    held, K = _held(), 3
    z = V.level_normals(K, np.float32)
    want = None
    for batch in (1, 2, 5, 7, 21, 64):
        for world in (1, 2, 3):
            rec = Recorder()
            parts = [V.score_items(rec, held, *V.rank_slice(len(held), r, world), levels=K, seed=4, batch=batch)
                     for r in range(world)]
            got = torch.cat(parts)
            assert got.shape == (len(held), K)
            assert len(rec.rows) == len(held) * K
            if want is None:
                want = got
            assert torch.equal(got, want), (batch, world)
            for r, (mom, eps, zn, noise, lab) in enumerate(rec.rows):     # rows in (item, level) order
                i, k = divmod(r, K)
                e_i, n_i = V.item_draws(4, i, 2, 4, K)
                assert torch.equal(mom, held.moments[i]) and torch.equal(lab, held.labels[i])
                assert torch.equal(eps, e_i) and torch.equal(noise, n_i[k]) and zn == float(z[k])


def test_draws_are_their_own_stream():
    torch.manual_seed(123)
    before = torch.get_rng_state()
    e1, n1 = V.item_draws(0, 5, 4, 8, 8)
    V.score_items(Recorder(), _held(), 0, 7, levels=2, seed=0, batch=3)
    assert torch.equal(torch.get_rng_state(), before)
    e2, n2 = V.item_draws(0, 5, 4, 8, 8)
    assert torch.equal(e1, e2) and torch.equal(n1, n2)
    e3, _ = V.item_draws(1, 5, 4, 8, 8)
    e4, _ = V.item_draws(0, 6, 4, 8, 8)
    assert not torch.equal(e1, e3) and not torch.equal(e1, e4)
    # more levels extend an item's noise without changing the first ones
    _, n5 = V.item_draws(0, 5, 4, 8, 12)
    assert torch.equal(n5[:8], n1)
    # the oracle's independent statement of the seed rule draws the same numbers
    eo, no = VO.item_draws(0, 5, 4, 8, 8)
    assert torch.equal(eo, e1) and torch.equal(no, n1)


def test_summary_is_float64_in_index_order():
    a = torch.tensor([[1e8, 1.0], [1.0, 2.0], [-1e8, 3.0]], dtype=torch.float32)
    res = V.summarize(a)
    assert res["per_level"] == [(1e8 + 1.0 - 1e8) / 3, 2.0] and res["count"] == 3 and res["levels"] == 2
    assert res["mean"] == pytest.approx((1 / 3 + 2.0) / 2)


# ---- 3. gloo world 2 -------------------------------------------------------------------------------------------------
class IndexScorer:
    """loss = 1000 * item + level, readable from the inputs (the moments of item i are all i)."""

    def __call__(self, moments, eps, rnd_normal, noise, labels):
        return moments[:, 0, 0, 0] * 1000 + torch.round(rnd_normal * 1e4) / 1e4


def _index_held(n):
    return V.HeldOut(torch.arange(n, dtype=torch.float32).reshape(n, 1, 1, 1).expand(n, 2, 4, 4).clone())


def _gloo_worker(rank, world, init, q, done):
    """Puts (rank, {name: numpy array or float}, error) on `q`: plain data, no tensors, so nothing of the result lives
    in this process's shared memory.  It exits only after the parent has taken both results (`done`)."""
    import datetime
    import traceback
    import torch.distributed as dist
    out, err = None, None
    try:
        dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world,
                                timeout=datetime.timedelta(seconds=120))
        out = {}
        for n in (1, 2, 9, 10):
            res = V.validate(IndexScorer(), _index_held(n), levels=3, seed=0, batch=4)
            out[f"index{n}"] = res["per_item"].numpy()
        sd = O.make_state_dict(SMALL, 1)
        g = np.load(GOLD)
        held = V.HeldOut(torch.from_numpy(g["moments"]), torch.from_numpy(g["labels"]))
        res = V.validate(VO.RowScorer(sd, SMALL), held, levels=4, seed=int(g["seed"]), batch=3)
        out["oracle"] = (res["per_item"].numpy(), res["per_level"], res["mean"])
    except Exception:
        err = traceback.format_exc()
    q.put((rank, out, err))
    done.wait(300)
    if dist.is_initialized():
        dist.destroy_process_group()


def test_gloo_world2_every_item_once_in_index_order(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q, done = ctx.Queue(), ctx.Event()
    init = f"file://{tmp_path / 'store'}"
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, init, q, done)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = [q.get(timeout=300) for _ in procs]
    finally:
        done.set()
        for p in procs:
            p.join(120)
    errors = [err for _, _, err in got if err]
    assert not errors, errors[0]
    assert [p.exitcode for p in procs] == [0, 0]
    res = {r: out for r, out, _ in got}
    assert sorted(res) == [0, 1]
    z = torch.from_numpy(V.level_normals(3, np.float32))
    for n in (1, 2, 9, 10):
        want = torch.arange(n, dtype=torch.float32)[:, None] * 1000 + torch.round(z * 1e4) / 1e4
        for r in (0, 1):
            assert np.array_equal(res[r][f"index{n}"], want.numpy()), (n, r)
    # the real estimator (oracle rows) under two ranks: both ranks equal one process, bit for bit
    g = np.load(GOLD)
    held = V.HeldOut(torch.from_numpy(g["moments"]), torch.from_numpy(g["labels"]))
    one = V.validate(VO.RowScorer(O.make_state_dict(SMALL, 1), SMALL), held, levels=4, seed=int(g["seed"]), batch=3)
    for r in (0, 1):
        per_item, per_level, mean = res[r]["oracle"]
        assert np.array_equal(per_item, one["per_item"].numpy())
        assert per_level == one["per_level"] and mean == one["mean"]


# ---- 4. oracle against the reference ---------------------------------------------------------------------------------
def test_golden_draws_are_the_item_draws():
    g = np.load(GOLD)
    N, K = g["per_item"].shape
    C, R = g["eps"].shape[1], g["eps"].shape[2]
    for i in range(N):
        e, n = V.item_draws(int(g["seed"]), i, C, R, K)
        assert np.array_equal(e.numpy(), g["eps"][i]) and np.array_equal(n.numpy(), g["noise"][i])
    assert np.array_equal(V.level_normals(K, np.float32), g["z"])


def test_oracle_matches_reference_golden():
    g = np.load(GOLD)
    N, K = g["per_item"].shape
    sd = O.make_state_dict(SMALL, 1)
    mom, lab = torch.from_numpy(g["moments"]), torch.from_numpy(g["labels"])
    per_item, per_level, mean = VO.estimate(sd, SMALL, mom, lab, levels=K, seed=int(g["seed"]))
    np.testing.assert_allclose(per_item.numpy(), g["per_item"], rtol=2e-5, atol=1e-6)
    want = g["per_item"].astype(np.float64).mean(0)
    np.testing.assert_allclose(per_level, want, rtol=2e-5)
    assert mean == pytest.approx(want.mean(), rel=2e-5)
    # injected draws (the stored ones) give the same numbers bit for bit
    inj = VO.estimate(sd, SMALL, mom, lab, levels=K, draws=lambda i: (torch.from_numpy(g["eps"][i]),
                                                                       torch.from_numpy(g["noise"][i])))
    assert torch.equal(inj[0], per_item)
    # the latent: utils.sample with the clamp (item 0 has logvar -40 < -30)
    eps = torch.from_numpy(g["eps"])
    y, _, _, _ = O.step_front(mom, eps, torch.zeros(N), torch.zeros_like(eps))
    np.testing.assert_allclose(y.numpy(), g["y"], rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("batch", [1, 3, 8, 40])
def test_batched_driver_matches_reference_golden(batch):
    g = np.load(GOLD)
    N, K = g["per_item"].shape
    held = V.HeldOut(torch.from_numpy(g["moments"]), torch.from_numpy(g["labels"]))
    res = V.validate(VO.RowScorer(O.make_state_dict(SMALL, 1), SMALL), held, levels=K, seed=int(g["seed"]),
                     batch=batch)
    np.testing.assert_allclose(res["per_item"].numpy(), g["per_item"], rtol=2e-5, atol=1e-6)
    assert res["count"] == N and res["levels"] == K and len(res["sigma"]) == K


# ---- 5. flags --------------------------------------------------------------------------------------------------------
def test_train_flags_default_off():
    sys.path.insert(0, ROOT)
    import train
    a = train.build_parser().parse_args(["--config", "x.yaml"])
    assert a.val_every == 0 and a.val_count == 1000 and a.val_levels == 8
    res = {"mean": 1.5, "per_level": [1.0, 2.0], "count": 3}
    assert train.val_line(12, res) == "(step=0000012) Val Loss: 1.50000 [1.00000 2.00000] (3 items, EMA)"


def test_val_loss_flags_defaults():
    import val_loss
    a = val_loss.build_parser().parse_args(["--config", "x.yaml", "--ckpt", "a.pt", "b.pt"])
    assert a.ckpt == ["a.pt", "b.pt"] and a.snapshots is None and a.key == "ema" and a.val_root is None
    assert (a.count, a.levels, a.batch, a.seed, a.json, a.synthetic) == (10000, 8, 64, 0, None, False)
    b = val_loss.build_parser().parse_args(["--config", "x.yaml", "--snapshots", "d", "--sigma_rel", "0.05", "0.1"])
    assert b.sigma_rel == [0.05, 0.1] and b.step is None and b.ckpt is None
    with pytest.raises(SystemExit):
        val_loss.build_parser().parse_args(["--config", "x.yaml"])


# ---- 6. the held-out sets -------------------------------------------------------------------------------------------
def test_from_lmdb_reads_the_first_items_of_the_val_split(tmp_path):
    from maskdit_b200.data import write_latent_lmdb
    g = np.random.default_rng(3)
    moments = g.standard_normal((9, 8, 4, 4)).astype(np.float32)
    classes = np.array([3, 0, 6, 6, 1, 2, 5, 4, 6])
    write_latent_lmdb(str(tmp_path), moments, classes, split="val")
    write_latent_lmdb(str(tmp_path), moments[::-1].copy(), classes[::-1].copy(), split="train")   # not read
    held = V.HeldOut.from_lmdb(str(tmp_path), 5, resolution=4, num_channels=4, num_classes=7)
    assert len(held) == 5 and held.moments.dtype == torch.float32
    assert np.array_equal(held.moments.numpy(), moments[:5])
    assert np.array_equal(held.labels.numpy(), np.eye(7, dtype=np.float32)[classes[:5]])
    # a class-unconditional net: the stored class indices are not read, whatever their range
    uncond = V.HeldOut.from_lmdb(str(tmp_path), 9, resolution=4, num_channels=4, num_classes=0)
    assert uncond.labels is None and np.array_equal(uncond.moments.numpy(), moments)
    with pytest.raises(ValueError, match="10 validation items"):
        V.HeldOut.from_lmdb(str(tmp_path), 10, resolution=4, num_channels=4, num_classes=7)
    with pytest.raises(FileNotFoundError):
        V.HeldOut.from_lmdb(str(tmp_path / "missing"), 1, resolution=4, num_channels=4, num_classes=7)


def test_synthetic_set_is_prefix_stable():
    small = V.HeldOut.synthetic(3, 4, 2, 10, seed=7)
    big = V.HeldOut.synthetic(11, 4, 2, 10, seed=7)
    assert small.moments.shape == (3, 4, 4, 4) and small.labels.shape == (3, 10)
    assert torch.equal(big.moments[:3], small.moments) and torch.equal(big.labels[:3], small.labels)
    assert torch.equal(big.labels.sum(1), torch.ones(11))
    other = V.HeldOut.synthetic(3, 4, 2, 10, seed=8)
    assert not torch.equal(other.moments, small.moments)
    assert V.HeldOut.synthetic(3, 4, 2, 0, seed=7).labels is None
    assert torch.equal(V.HeldOut.synthetic(3, 4, 2, 0, seed=7).moments, small.moments)
    # apart from the noise of the same item: the moments are not the item's eps draw
    eps, _ = V.item_draws(7, 0, 4, 4, 1)
    assert not torch.equal(small.moments[0, :4], eps)
