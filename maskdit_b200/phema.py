"""Power-function EMA profiles and their post-hoc combination (Karras et al., "Analyzing and Improving the Training
Dynamics of Diffusion Models", CVPR 2024, §3 and the appendix on power-function EMA).

A profile of exponent gamma averages the weights of optimizer steps 1..t (counted from the profile's origin) with
    beta(t) = (1 - 1/t)^(gamma + 1),    ema <- beta * ema + (1 - beta) * w,
so step 1 copies the weights.  Its continuous model is the weight density p(tau) = (gamma + 1) tau^gamma / t^(gamma + 1)
on (0, t], whose relative width (standard deviation over t) is
    sigma_rel = sqrt((gamma + 1) / ((gamma + 2)^2 (gamma + 3))).
Snapshots of a few profiles taken during training span a space of such densities: the combination of snapshots that is
closest in L2 to the density of any other (gamma, t) is the EMA of that width, reconstructed after the run.  Everything
here is host arithmetic in float64.
"""
from __future__ import annotations

import math

import numpy as np

# sigma_rel as a function of gamma > -1 peaks at gamma = (sqrt(5) - 3) / 2 (the root of gamma^2 + 3 gamma + 1); the
# larger-gamma branch beyond that point is the one an EMA uses.
_GAMMA_PEAK = (math.sqrt(5.0) - 3.0) / 2.0


def gamma_to_sigma_rel(gamma):
    g = np.asarray(gamma, dtype=np.float64)
    out = np.sqrt((g + 1) / ((g + 2) ** 2 * (g + 3)))
    return float(out) if out.ndim == 0 else out


SIGMA_REL_MAX = gamma_to_sigma_rel(_GAMMA_PEAK)   # 0.3003


def sigma_rel_to_gamma(sigma_rel: float) -> float:
    """The exponent of the profile of relative width `sigma_rel`: the largest real root of
    gamma^3 + 7 gamma^2 + (16 - s^-2) gamma + (12 - s^-2) = 0, s = sigma_rel."""
    s = float(sigma_rel)
    if not 0.0 < s < SIGMA_REL_MAX:
        raise ValueError(f"sigma_rel {s} outside (0, {SIGMA_REL_MAX:.4f})")
    t = s ** -2
    roots = np.roots([1.0, 7.0, 16.0 - t, 12.0 - t])
    return float(max(r.real for r in roots if abs(r.imag) <= 1e-9 * max(1.0, abs(r.real))))


def one_minus_beta(gamma: float, t: int) -> float:
    """1 - beta(t) = 1 - (1 - 1/t)^(gamma + 1) in float64 (1 at t = 1)."""
    if t < 1:
        raise ValueError(f"profile step {t} < 1")
    if t == 1:
        return 1.0
    return -math.expm1((gamma + 1.0) * math.log1p(-1.0 / t))


def gram(t_a, g_a, t_b, g_b):
    """Inner products of the densities of profiles (t_a, g_a) and (t_b, g_b) over tau (numpy broadcasting):
    (g_a+1)(g_b+1) min(t_a,t_b)^(g_a+g_b+1) / ((g_a+g_b+1) t_a^(g_a+1) t_b^(g_b+1)), evaluated in the log domain so that
    large exponents and step counts do not overflow."""
    t_a, g_a, t_b, g_b = (np.asarray(v, dtype=np.float64) for v in (t_a, g_a, t_b, g_b))
    m = np.minimum(t_a, t_b)
    s = g_a + g_b + 1
    return (g_a + 1) * (g_b + 1) / s * np.exp(s * np.log(m) - (g_a + 1) * np.log(t_a) - (g_b + 1) * np.log(t_b))


def solve(ts, gammas, t_target, gamma_target):
    """Coefficients x minimising || sum_i x_i p_i - p_target ||^2 over tau for snapshot densities (ts[i], gammas[i]),
    and the fit's relative L2 residual || sum_i x_i p_i - p_target || / || p_target ||.  Float64 least squares on the
    Gram matrix scaled to a unit diagonal (the densities' norms scale as 1/t)."""
    ts, gammas = np.asarray(ts, dtype=np.float64), np.asarray(gammas, dtype=np.float64)
    if ts.ndim != 1 or ts.shape != gammas.shape or ts.size == 0:
        raise ValueError("need one (t, gamma) per snapshot and at least one snapshot")
    if (ts < 1).any() or t_target < 1:
        raise ValueError("profile steps start at 1")
    A = gram(ts[:, None], gammas[:, None], ts[None, :], gammas[None, :])
    b = gram(ts, gammas, t_target, gamma_target)
    c = float(gram(t_target, gamma_target, t_target, gamma_target))
    d = 1.0 / np.sqrt(np.diag(A))
    y = np.linalg.lstsq(A * d[:, None] * d[None, :], b * d, rcond=None)[0]
    x = y * d
    r2 = float(x @ A @ x - 2.0 * x @ b + c)
    return x, math.sqrt(max(r2, 0.0) / c)
