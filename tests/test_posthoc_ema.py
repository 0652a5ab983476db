"""CPU: post-hoc EMA.  The power-function EMA arithmetic (`maskdit_b200/phema.py`), the reconstruction tool
(posthoc_ema.py) on synthetic snapshots, the `mdt_power_ema` argument checks, train.py's flags and TrainStep's host
bookkeeping of the profiles."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from maskdit_b200 import phema  # noqa: E402

MDT_ERR_ARG = -1
A = 1 << 20   # a 256-byte aligned dummy address: the argument checks never dereference it


def test_sigma_rel_gamma_round_trip():
    assert phema.sigma_rel_to_gamma(0.05) == pytest.approx(16.97, abs=1e-2)
    assert phema.sigma_rel_to_gamma(0.10) == pytest.approx(6.94, abs=1e-2)
    for s in (0.005, 0.01, 0.05, 0.08, 0.1, 0.2, 0.29, 0.3):
        g = phema.sigma_rel_to_gamma(s)
        assert phema.gamma_to_sigma_rel(g) == pytest.approx(s, rel=1e-10), s
        assert g > (math.sqrt(5) - 3) / 2        # the EMA branch of the cubic
    for g in (0.0, 1.0, 6.94, 16.97, 100.0):
        assert phema.sigma_rel_to_gamma(phema.gamma_to_sigma_rel(g)) == pytest.approx(g, rel=1e-9)
    for bad in (0.0, -0.1, 0.31, phema.SIGMA_REL_MAX):
        with pytest.raises(ValueError):
            phema.sigma_rel_to_gamma(bad)


def test_one_minus_beta():
    from decimal import Decimal, localcontext
    for g in (0.0, 6.94, 16.97):
        assert phema.one_minus_beta(g, 1) == 1.0                     # the first step copies the weights
        for t in (2, 3, 10, 1000, 2_000_000):
            with localcontext() as ctx:   # 1 - (1 - 1/t)^(g+1) cancels in float64 at large t: 50 digits instead
                ctx.prec = 50
                want = float(1 - (1 - Decimal(1) / t) ** (Decimal(g) + 1))
            assert phema.one_minus_beta(g, t) == pytest.approx(want, rel=1e-14), (g, t)
    with pytest.raises(ValueError):
        phema.one_minus_beta(6.94, 0)


def test_gram_matches_quadrature():
    from scipy.integrate import quad

    def p(tau, t, g):
        return (g + 1) * tau ** g / t ** (g + 1) if tau <= t else 0.0

    cases = [(100, 6.94, 100, 6.94), (100, 16.97, 300, 6.94), (2000, 6.94, 700, 16.97), (5, 0.5, 9, 3.0),
             (1e6, 16.97, 2e6, 6.94)]
    for ta, ga, tb, gb in cases:
        m = min(ta, tb)
        want, err = quad(lambda x: p(x, ta, ga) * p(x, tb, gb), 0, m, limit=200, epsabs=0, epsrel=1e-12)
        got = phema.gram(ta, ga, tb, gb)
        assert got == pytest.approx(want, rel=1e-9), (ta, ga, tb, gb, got, want)
        assert phema.gram(tb, gb, ta, ga) == pytest.approx(got, rel=1e-13)
    # large exponents and steps stay finite (log domain)
    assert np.isfinite(phema.gram(2e6, 200.0, 2e6, 200.0))


# ---- a synthetic run: float64 recurrences over a random walk -------------------------------------------------------------
N, T, EVERY = 1000, 2000, 100
SIGMAS = (0.05, 0.10)


def _walk(seed=0):
    rng = np.random.default_rng(seed)
    return np.cumsum(rng.standard_normal((T, N)), 0) / 30.0 + rng.standard_normal(N)


def _power_ema(w, gammas, every=None):
    """float64 power-function EMA of each gamma over the rows of w; {t: [ema per gamma]} every `every` steps
    (else only the last)."""
    e = [np.zeros(w.shape[1]) for _ in gammas]
    out = {}
    for t in range(1, w.shape[0] + 1):
        for j, g in enumerate(gammas):
            e[j] += phema.one_minus_beta(g, t) * (w[t - 1] - e[j])
        if (every and t % every == 0) or t == w.shape[0]:
            out[t] = [x.copy() for x in e]
    return out


@pytest.fixture(scope="module")
def run():
    w = _walk()
    gammas = [phema.sigma_rel_to_gamma(s) for s in SIGMAS]
    snaps = _power_ema(w, gammas, EVERY)
    ts, gs, vals = [], [], []
    for t, es in snaps.items():
        for g, e in zip(gammas, es):
            ts.append(t), gs.append(g), vals.append(e)
    return w, gammas, snaps, ts, gs, np.array(vals)


def test_reconstructing_a_snapshot_returns_it(run):
    _, _, _, ts, gs, vals = run
    for k in (0, 7, len(ts) // 2 + 1, len(ts) - 1):
        x, res = phema.solve(ts, gs, ts[k], gs[k])
        got = x @ vals
        rel = np.linalg.norm(got - vals[k]) / np.linalg.norm(vals[k])
        assert res < 1e-6 and rel < 1e-6, (k, res, rel)


# Measured on a CPU with numpy's LAPACK: relative L2 of the reconstruction against the directly computed float64
# power EMA, sigma_rel 0.07: 5.6e-5, 0.12: 5.5e-5 (fit residual 2.5e-3 / 2.2e-3).  The discrete beta and the continuous
# density differ most at small t; the random walk makes that early part matter.  Bounds: 3.5x the measurement.
RECON_BOUND = {0.07: 2e-4, 0.12: 2e-4}


@pytest.mark.parametrize("target", [0.07, 0.12])
def test_reconstruction_matches_direct_power_ema(run, target):
    w, _, _, ts, gs, vals = run
    g = phema.sigma_rel_to_gamma(target)
    x, res = phema.solve(ts, gs, T, g)
    got = x @ vals
    want = _power_ema(w, [g])[T][0]
    rel = np.linalg.norm(got - want) / np.linalg.norm(want)
    print(f"sigma_rel {target}: reconstruction rel-L2 {rel:.2e}, fit residual {res:.2e}")
    assert rel < RECON_BOUND[target] and res < 1e-2, (rel, res)
    # a width between the stored ones is not one of them: the stored snapshots alone are far off
    assert min(np.linalg.norm(v - want) for v in vals) / np.linalg.norm(want) > 10 * rel


# ---- posthoc_ema.py on snapshot files -------------------------------------------------------------------------------------
def _write_snapshots(d, run, origin=0, steps=None):
    """The synthetic run's snapshots as train.py writes them: a state dict of two tensors per profile."""
    _, gammas, snaps, _, _, _ = run
    d.mkdir(exist_ok=True)
    for t, es in snaps.items():
        if steps is not None and t not in steps:
            continue
        profiles = [{"sigma_rel": s, "gamma": g, "ema": {"model.a": torch.from_numpy(e[:600]).float().view(20, 30),
                                                          "model.b": torch.from_numpy(e[600:]).float()}}
                    for s, g, e in zip(SIGMAS, gammas, es)]
        torch.save({"step": origin + t, "origin": origin, "profiles": profiles}, d / f"phema-{origin + t:07d}.pt")


def _fp32_vals(run, upto):
    """The snapshot values as stored (fp32), up to step `upto`, in file order."""
    _, _, snaps, _, _, _ = run
    return np.array([np.float32(e).astype(np.float64) for t, es in snaps.items() if t <= upto for e in es])


def test_tool_reconstructs_from_files(tmp_path, run):
    import posthoc_ema
    _write_snapshots(tmp_path / "phema", run, origin=40)
    out = posthoc_ema.main(["--snapshots", str(tmp_path / "phema"), "--sigma_rel", "0.08", "--out",
                            str(tmp_path / "ema.pt")])
    assert out == [str(tmp_path / "ema.pt")]
    ck = torch.load(out[0], weights_only=True)
    info = ck["posthoc"]
    assert info["step"] == 40 + T and info["origin"] == 40 and len(info["snapshots"]) == 2 * (T // EVERY)
    assert set(ck["ema"]) == {"model.a", "model.b"} and ck["ema"]["model.a"].shape == (20, 30)
    assert ck["ema"]["model.a"].dtype == torch.float32
    x = np.array(info["coefficients"])
    want = x @ _fp32_vals(run, T)
    got = torch.cat([ck["ema"]["model.a"].reshape(-1), ck["ema"]["model.b"]]).double().numpy()
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()
    direct = _power_ema(run[0], [phema.sigma_rel_to_gamma(0.08)])[T][0]
    assert np.linalg.norm(got - direct) / np.linalg.norm(direct) < 2e-4
    # several widths: one file each
    outs = posthoc_ema.main(["--snapshots", str(tmp_path / "phema"), "--sigma_rel", "0.07", "0.12", "--out",
                             str(tmp_path / "e.pt")])
    assert outs == [str(tmp_path / "e-0.07.pt"), str(tmp_path / "e-0.12.pt")] and all(map(os.path.exists, outs))


def test_tool_step_picks_the_snapshots_up_to_it(tmp_path, run):
    import posthoc_ema
    _write_snapshots(tmp_path / "phema", run)
    out = posthoc_ema.main(["--snapshots", str(tmp_path / "phema"), "--sigma_rel", "0.08", "--step", "1000",
                            "--out", str(tmp_path / "ema.pt")])
    info = torch.load(out[0], weights_only=True)["posthoc"]
    assert info["step"] == 1000
    assert sorted({s["file"] for s in info["snapshots"]}) == [f"phema-{t:07d}.pt" for t in range(100, 1001, 100)]
    assert max(s["t"] for s in info["snapshots"]) == 1000
    direct = _power_ema(run[0][:1000], [phema.sigma_rel_to_gamma(0.08)])[1000][0]
    ck = torch.load(out[0], weights_only=True)["ema"]
    got = torch.cat([ck["model.a"].reshape(-1), ck["model.b"]]).double().numpy()
    # 10 snapshot files instead of 20: measured 4.6e-4 rel-L2
    assert np.linalg.norm(got - direct) / np.linalg.norm(direct) < 1.5e-3
    # between snapshots: the ones up to the step; past the last: refused (the later weights are unknown)
    files = posthoc_ema.list_snapshots(str(tmp_path / "phema"), 1050)
    assert [s for s, _ in files] == list(range(100, 1001, 100))
    with pytest.raises(SystemExit):
        posthoc_ema.main(["--snapshots", str(tmp_path / "phema"), "--sigma_rel", "0.08", "--step", "50", "--out",
                          str(tmp_path / "x.pt")])
    with pytest.raises(SystemExit):
        posthoc_ema.reconstruct(posthoc_ema.list_snapshots(str(tmp_path / "phema")), 0.08, step=T + 1)


def test_tool_refuses_mixed_origins(tmp_path, run):
    import posthoc_ema
    d = tmp_path / "phema"
    _write_snapshots(d, run, origin=0, steps={100, 200})
    _write_snapshots(d, run, origin=150, steps={100})       # a restarted run: profiles from step 150, file at 250
    with pytest.raises(SystemExit, match="origin"):
        posthoc_ema.main(["--snapshots", str(d), "--sigma_rel", "0.08", "--out", str(tmp_path / "x.pt")])
    # up to step 200 the snapshots agree
    out = posthoc_ema.main(["--snapshots", str(d), "--sigma_rel", "0.08", "--step", "200", "--out",
                            str(tmp_path / "x.pt")])
    assert torch.load(out[0], weights_only=True)["posthoc"]["origin"] == 0


# ---- C ABI, train.py, TrainStep bookkeeping ----------------------------------------------------------------------------------
def test_power_ema_entry_rejects_bad_arguments():
    from maskdit_b200 import _lib
    L = _lib.lib()
    assert "mdt_power_ema" in _lib.exported_symbols() and L.mdt_abi_version() == 2

    def call(w=A, emas=(A, A), cs=(0.5, 0.25), k=None, n=64):
        k = len(emas) if k is None else k
        pe = (ctypes.c_void_p * max(len(emas), 1))(*emas)
        pc = (ctypes.c_float * max(len(cs), 1))(*cs)
        return L.mdt_power_ema(w, pe, pc, k, n, None)

    for bad in (dict(w=None), dict(emas=(A, None)), dict(k=0), dict(emas=(A,) * 5, cs=(0.5,) * 5), dict(n=0),
                dict(n=-4), dict(w=A + 2), dict(emas=(A, A + 1)), dict(cs=(0.5, -0.1)), dict(cs=(1.5, 0.5)),
                dict(cs=(float("nan"), 0.5))):
        assert call(**bad) == MDT_ERR_ARG, bad
    assert L.mdt_power_ema(A, None, (ctypes.c_float * 1)(0.5), 1, 4, None) == MDT_ERR_ARG
    assert L.mdt_power_ema(A, (ctypes.c_void_p * 1)(A), None, 1, 4, None) == MDT_ERR_ARG


def test_train_py_phema_flags():
    import train
    ap = train.build_parser()
    a = ap.parse_known_args(["--config", "c.yaml"])[0]
    assert a.phema_sigma_rel == () and a.phema_every == 0
    a = ap.parse_known_args(["--config", "c.yaml", "--phema_sigma_rel", "0.05,0.10", "--phema_every", "500"])[0]
    assert a.phema_sigma_rel == (0.05, 0.10) and a.phema_every == 500


class _Net:
    """A frozen tensor first (as pos_embed), then one trainable one."""

    def __init__(self):
        self.p = [("pos", torch.nn.Parameter(torch.arange(2.0), requires_grad=False)),
                  ("w", torch.nn.Parameter(torch.zeros(2, 4)))]

    def named_parameters(self):
        return iter(self.p)

    def state_dict(self):
        return {k: p.detach() for k, p in self.p}


def _host_step(sigma_rels):
    """A TrainStep with host tensors in place of its device buffers: the bookkeeping only, no launch."""
    from types import SimpleNamespace

    from maskdit_b200.train_step import TrainStep
    ts = TrainStep.__new__(TrainStep)
    ts.net = _Net()
    ts.st = SimpleNamespace(offsets={"w": (0, 8, (2, 4)), "pos": (64, 2, (2,))}, n_train=8)
    ts.m, ts.v = torch.zeros(8), torch.zeros(8)
    ts.lr, ts.betas, ts.eps, ts.wd = 1e-4, (0.9, 0.999), 1e-8, 0.0
    ts.step_count, ts.lr_step_offset = 0, 0
    ts._flag = ts._counts = None
    if sigma_rels:
        ts.phema_sigma_rels = tuple(sigma_rels)
        ts.phema_gammas = tuple(phema.sigma_rel_to_gamma(s) for s in sigma_rels)
        ts.phema_emas = [torch.zeros(8) for _ in sigma_rels]
        ts.phema_origin, ts.phema_steps = None, 0
    return ts


def test_trainstep_profile_state_round_trip():
    from maskdit_b200.train_step import TrainStep
    assert TrainStep.phema_emas == ()                             # off by default
    assert "phema" not in _host_step(()).state_dict()
    ts = _host_step((0.05, 0.10))
    ts.phema_emas[0].copy_(torch.arange(8.0)), ts.phema_emas[1].copy_(-torch.arange(8.0))
    ts.phema_origin, ts.phema_steps = 10, 5
    sd = ts.state_dict()
    ph = sd["phema"]
    assert ph["origin"] == 10 and ph["steps"] == 5 and ph["sigma_rels"] == [0.05, 0.10]
    assert ph["gammas"] == pytest.approx([16.97, 6.94], abs=1e-2)
    snap = ts.phema_snapshot()
    assert snap["step"] == 15 and snap["origin"] == 10 and [p["sigma_rel"] for p in snap["profiles"]] == [0.05, 0.10]
    ema0 = snap["profiles"][0]["ema"]
    assert list(ema0) == ["pos", "w"] and torch.equal(ema0["w"], torch.arange(8.0).view(2, 4))
    assert torch.equal(ema0["pos"], torch.arange(2.0))            # frozen tensors come from the weights
    ts2 = _host_step((0.05, 0.10))
    ts2.load_state_dict(sd)
    assert ts2.phema_origin == 10 and ts2.phema_steps == 5
    assert all(torch.equal(a, b) for a, b in zip(ts.phema_emas, ts2.phema_emas))
    # a state without profiles (a reference checkpoint): new profiles, origin set by the next step
    del sd["phema"]
    ts2.load_state_dict(sd)
    assert ts2.phema_origin is None and ts2.phema_steps == 0 and all((e == 0).all() for e in ts2.phema_emas)
    with pytest.raises(ValueError, match="not been updated"):
        ts2.phema_snapshot()
    # profiles of other widths are refused rather than silently continued
    ts3 = _host_step((0.05,))
    with pytest.raises(ValueError, match="sigma_rel"):
        ts3.load_state_dict(ts.state_dict())
    # a TrainStep without profiles ignores them
    _host_step(()).load_state_dict(ts.state_dict())
