"""Multistep DPM-Solver++ (DESIGN §5): host logic without a GPU.  The expanded step coefficients against the independent
D1 / D2 form of oracle/dpm_solver_oracle.py, the solver's error and observed order on Gaussian data (where the denoiser
and the probability-flow solution are closed form) for EDM and flow, the noise levels, and the argument refusals of
`dpm_solver_sampler` and generate.py's --dpm_order."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from maskdit_b200.maskdit import EDMPrecond, FlowPrecond  # noqa: E402
from maskdit_b200.sampler import (dpm_solver_coefficients, dpm_solver_levels, dpm_solver_sampler,  # noqa: E402
                                  flow_grid)
from oracle import dpm_solver_oracle as O  # noqa: E402

MU, S = 0.3, 0.5
Z = np.array([1.3, -0.7, 0.2])


def expanded(data_pred, x, alpha, sigma, order, states=None):
    """The product's step, x' = a x + b0 D_i + b1 D_{i-1} + b2 D_{i-2}, in numpy fp64 in the kernel's order."""
    Ds = []
    for i, (k, a, b0, b1, b2) in enumerate(dpm_solver_coefficients(alpha, sigma, order)):
        if states is not None:
            states.append(x)
        Ds.append(np.asarray(data_pred(x, i), dtype=np.float64))
        v = a * x + b0 * Ds[-1]
        if k >= 2:
            v = v + b1 * Ds[-2]
        if k >= 3:
            v = v + b2 * Ds[-3]
        x = v
    return x


def edm_run(levels, order, solver=expanded):
    alpha, sigma = O.edm_alpha_sigma(levels)
    return solver(lambda x, i: O.gauss_edm_D(x, sigma[i], MU, S), sigma[0] * Z, alpha, sigma, order)


def edm_err(levels, order):
    """Max error against the exact D(x(sigma_min); sigma_min) from x(sigma_0) = sigma_0 z."""
    smin = levels[-2]
    exact = O.gauss_edm_D(O.gauss_edm_exact(levels[0] * Z, levels[0], smin, MU, S), smin, MU, S)
    return np.abs(edm_run(levels, order) - exact).max()


def flow_err(levels, order):
    """Max error against the exact D(x(t_last); t_last), starting on the exact path at levels[0] (x(1) = z)."""
    alpha, sigma = O.flow_alpha_sigma(levels)
    x0 = O.gauss_flow_exact(Z, 1.0, sigma[0], MU, S)
    got = expanded(lambda x, i: O.gauss_flow_D(x, sigma[i], MU, S), x0, alpha, sigma, order)
    t = sigma[-2]
    return np.abs(got - O.gauss_flow_D(O.gauss_flow_exact(Z, 1.0, t, MU, S), t, MU, S)).max()


def edm_heun(num_steps):
    """edm_sampler's Heun steps (Euler last step) in fp64."""
    t = O.karras_levels(num_steps)
    x = t[0] * Z
    for k in range(num_steps):
        d = (x - O.gauss_edm_D(x, t[k], MU, S)) / t[k]
        xn = x + (t[k + 1] - t[k]) * d
        if k < num_steps - 1:
            dp = (xn - O.gauss_edm_D(xn, t[k + 1], MU, S)) / t[k + 1]
            xn = x + (t[k + 1] - t[k]) * (0.5 * d + 0.5 * dp)
        x = xn
    return x


def uniform_lambda_edm(n, smax=80.0, smin=0.002):
    return np.append(np.exp(np.linspace(math.log(smax), math.log(smin), n)), 0.0)


def uniform_lambda_flow(n, t_hi=0.98, t_lo=0.002):
    lam = np.linspace(math.log((1 - t_hi) / t_hi), math.log((1 - t_lo) / t_lo), n)
    return np.append(1.0 / (1.0 + np.exp(lam)), 0.0)


# ---- the expanded coefficients against the D1 / D2 form ---------------------------------------------------------------
@pytest.mark.parametrize("kind", ["edm", "flow", "edm_uniform"])
@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 7])
def test_expanded_coefficients_match_oracle(kind, order, n):
    """Arbitrary data predictions D_i: every state the solver passes through (warm-up, full-order and final steps, the
    flow's t = 1 limits) and the result agree to 1e-13 of the state's size."""
    levels = {"edm": O.karras_levels(n), "flow": flow_grid(n), "edm_uniform": uniform_lambda_edm(n)}[kind]
    if kind == "edm_uniform" and n == 1:
        levels = np.array([80.0, 0.0])
    alpha, sigma = (O.flow_alpha_sigma if kind == "flow" else O.edm_alpha_sigma)(levels)
    rng = np.random.default_rng(100 * order + n)
    Ds = [rng.standard_normal(16) for _ in range(n)]
    x = sigma[0] * rng.standard_normal(16)
    want, got = [], []
    ref = O.dpm_solver(lambda xx, i: (want.append(xx), Ds[i])[1], x, alpha, sigma, order)
    out = expanded(lambda xx, i: Ds[i], x, alpha, sigma, order, states=got)
    for i, (a, b) in enumerate(zip(got + [out], want + [ref])):
        assert np.abs(a - b).max() <= 1e-13 * np.abs(b).max(), (kind, order, n, i)
    assert np.array_equal(out, alpha[-1] * Ds[-1])                     # the step into sigma = 0: x' = alpha D


def test_step_orders_and_limits():
    st = dpm_solver_coefficients(*O.edm_alpha_sigma(O.karras_levels(6)), 3)
    assert [s[0] for s in st] == [1, 2, 3, 3, 2, 1]                   # warm-up, full order, then N - i
    assert st[-1] == (1, 0.0, 1.0, 0.0, 0.0)
    assert [s[0] for s in dpm_solver_coefficients(*O.edm_alpha_sigma(O.karras_levels(4)), 2)] == [1, 2, 2, 1]
    # flow: the first evaluation at t = 1 (lambda = -inf) is a DDIM step into t_1 = 0.8, x' = t_1 x + (1 - t_1) D_0,
    # and no later step reads D_0
    st = dpm_solver_coefficients(*O.flow_alpha_sigma(flow_grid(5)), 3)
    assert st[0][1:] == pytest.approx((0.8, 0.2, 0.0, 0.0), rel=1e-15)
    assert st[1][3] == 0.0 and st[2][4] == 0.0 and st[2][3] != 0.0
    assert all(np.isfinite(v) for s in st for v in s)
    # order 1 is DDIM: x' = (sigma'/sigma) x + alpha' (1 - sigma' alpha / (sigma alpha')) D
    lv = O.karras_levels(5)
    for i, (k, a, b0, b1, b2) in enumerate(dpm_solver_coefficients(*O.edm_alpha_sigma(lv), 1)[:-1]):
        assert (k, b1, b2) == (1, 0.0, 0.0)
        assert a == lv[i + 1] / lv[i] and b0 == pytest.approx(1 - lv[i + 1] / lv[i], rel=1e-14)
    with pytest.raises(ValueError):
        dpm_solver_coefficients([1.0, 1.0], [1.0, 0.0], 4)


# ---- Gaussian data -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("evals, heun, m2, m3", [(15, 2.6e-1, 5.9e-2, 9.9e-3), (35, 3.6e-2, 9.0e-3, 8.4e-4)])
def test_error_table(evals, heun, m2, m3):
    """The Karras grid sigma 80 -> 0.002, rho 7, from 80 z: Heun (edm_sampler) with (evals + 1) / 2 steps against 2M
    and 3M with `evals` evaluations, to the two digits quoted in DESIGN §5; the oracle gives the same errors."""
    exact = O.gauss_edm_D(O.gauss_edm_exact(80 * Z, 80.0, 0.002, MU, S), 0.002, MU, S)
    assert float(f"{np.abs(edm_heun((evals + 1) // 2) - exact).max():.1e}") == heun
    lv = O.karras_levels(evals)
    for order, want in ((2, m2), (3, m3)):
        assert float(f"{edm_err(lv, order):.1e}") == want
        assert np.abs(edm_run(lv, order, O.dpm_solver) - edm_run(lv, order)).max() < 1e-13


@pytest.mark.parametrize("kind", ["edm", "flow"])
def test_observed_order_uniform_lambda(kind):
    """log2 of the error ratio between 32 -> 64 and 64 -> 128 evaluations on a uniform-lambda grid: >= 1.9 for 2M and
    3M (the first-order warm-up step limits 3M to order 2), >= 0.95 for DDIM."""
    for order, lo in ((1, 0.95), (2, 1.9), (3, 1.9)):
        if kind == "edm":
            e = [edm_err(uniform_lambda_edm(n), order) for n in (32, 64, 128)]
        else:
            e = [flow_err(uniform_lambda_flow(n), order) for n in (32, 64, 128)]
        rates = np.log2(np.array(e[:-1]) / np.array(e[1:]))
        assert (rates >= lo).all(), (kind, order, rates, e)


def test_third_order_beats_second_on_the_default_grids():
    for n in range(16, 65):
        assert edm_err(O.karras_levels(n), 3) < edm_err(O.karras_levels(n), 2), n
        assert flow_err(flow_grid(n), 3) < flow_err(flow_grid(n), 2), n


# ---- the levels and the refusals ---------------------------------------------------------------------------------------
def _small(cls, **kw):
    return cls(8, 4, num_classes=10, model_type="DiT-S/2", use_decoder=True, mae_loss_coef=0.1, **kw)


def test_levels():
    edm, flow = _small(EDMPrecond), _small(FlowPrecond)
    f, lv = dpm_solver_levels(edm, 18)
    assert not f and np.array_equal(lv, O.karras_levels(18))
    f, lv = dpm_solver_levels(flow, 7)
    assert f and np.array_equal(lv, flow_grid(7))
    assert dpm_solver_levels(edm, 1)[1].tolist() == [80.0, 0.0]
    clamped = _small(EDMPrecond, sigma_min=0.01, sigma_max=40.0)
    assert np.array_equal(dpm_solver_levels(clamped, 9)[1], O.karras_levels(9, 0.01, 40.0))


def test_sampler_refusals():
    edm, flow = _small(EDMPrecond), _small(FlowPrecond)
    z = torch.zeros(1, 4, 8, 8)
    for kw in (dict(order=0), dict(order=4), dict(num_steps=0)):
        for net in (edm, flow):
            with pytest.raises(ValueError):
                dpm_solver_sampler(net, z, **kw)
    with pytest.raises(ValueError, match="flow networks"):
        dpm_solver_sampler(flow, z, guide_net=_small(FlowPrecond), guidance=2.0)
    with pytest.raises(ValueError):
        dpm_solver_sampler(edm, z, guidance=2.0)                          # a guidance weight without a guide


@pytest.mark.parametrize("argv, what", [
    (["--dpm_order", "3", "--S_churn", "10"], "--S_churn"),
    (["--dpm_order", "3", "--solver", "euler"], "--solver"),
    (["--dpm_order", "2", "--schedule", "vp"], "--schedule"),
    (["--dpm_order", "3", "--consistency_sigmas", "80"], "--consistency_sigmas"),
    (["--dpm_order", "4"], "invalid choice"),
    (["--dpm_order", "3", "--num_steps", "0"], "--num_steps"),
])
def test_generate_dpm_order_validation(argv, what, capsys):
    import generate
    with pytest.raises(SystemExit):
        generate.parse_args(["--config", "x.yaml", *argv])
    assert what in capsys.readouterr().err
    a = generate.parse_args(["--config", "x.yaml", "--dpm_order", "3", "--num_steps", "15", "--cfg_scale", "1.5"])
    assert (a.dpm_order, a.num_steps) == (3, 15)
    assert generate.parse_args(["--config", "x.yaml"]).dpm_order is None
