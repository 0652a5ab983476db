"""CPU float64 restatement of multistep DPM-Solver++ (Lu et al., 2022; DESIGN §5) in its D1 / D2 form.

Independent of `maskdit_b200.sampler`, which expands every step into x' = a x + b0 D_i + b1 D_{i-1} + b2 D_{i-2} with
host-computed coefficients; the tests hold the two against each other.  The state follows x = alpha x0 + sigma eps with
lambda = log(alpha / sigma).  `alpha` and `sigma` hold the N + 1 levels (the last sigma is 0); the network is evaluated
at the first N.  Infinite lambdas (alpha = 0 at flow time t = 1, sigma = 0 at the end) are left to IEEE arithmetic: a
difference divided by an infinite ratio r is 0, and the step into sigma = 0 returns alpha D.
"""
import numpy as np


def karras_levels(num_steps, sigma_min=0.002, sigma_max=80.0, rho=7.0):
    """The EDM sampler's noise levels (sample.py:40-43) with num_steps positive levels, then 0."""
    if num_steps == 1:
        return np.array([sigma_max, 0.0])
    i = np.arange(num_steps, dtype=np.float64)
    s = (sigma_max ** (1 / rho) + i / (num_steps - 1) * (sigma_min ** (1 / rho) - sigma_max ** (1 / rho))) ** rho
    return np.append(s, 0.0)


def edm_alpha_sigma(levels):
    levels = np.asarray(levels, dtype=np.float64)
    return np.ones_like(levels), levels


def flow_alpha_sigma(levels):
    t = np.asarray(levels, dtype=np.float64)
    return 1.0 - t, t


def dpm_solver(data_pred, x, alpha, sigma, order):
    """Multistep DPM-Solver++ of order 1-3 from the fp64 state `x` at level 0.  data_pred(x, i) is D at level i.
    Step i uses order k = min(order, i + 1, N - i).  Returns the state after the last step (alpha_N D_{N-1})."""
    alpha, sigma = np.asarray(alpha, np.float64), np.asarray(sigma, np.float64)
    N = len(sigma) - 1
    with np.errstate(divide="ignore"):
        lam = np.log(alpha) - np.log(sigma)
    x = np.asarray(x, dtype=np.float64)
    Ds = []
    for i in range(N):
        D = np.asarray(data_pred(x, i), dtype=np.float64)
        Ds.append(D)
        if sigma[i + 1] == 0:
            x = alpha[i + 1] * D
            continue
        h = lam[i + 1] - lam[i]
        E = np.expm1(-h)
        a1 = alpha[i + 1]
        base = sigma[i + 1] / sigma[i] * x - a1 * E * D
        k = min(order, i + 1, N - i)
        if k == 1:
            x = base
        elif k == 2:
            r0 = (lam[i] - lam[i - 1]) / h
            D1 = (D - Ds[-2]) / r0
            x = base - 0.5 * a1 * E * D1
        else:
            r0 = (lam[i] - lam[i - 1]) / h
            r1 = (lam[i - 1] - lam[i - 2]) / h
            D1_0 = (D - Ds[-2]) / r0
            D1_1 = (Ds[-2] - Ds[-3]) / r1
            D1 = D1_0 + r0 / (r0 + r1) * (D1_0 - D1_1)
            D2 = (D1_0 - D1_1) / (r0 + r1)
            x = base + a1 * (E / h + 1) * D1 - a1 * ((E + h) / h ** 2 - 0.5) * D2
    return x


# ---- Gaussian data: the denoiser and the probability-flow solution in closed form ---------------------------------------
def gauss_edm_D(x, sigma, mu, s):
    """E[x0 | x0 + sigma eps = x] for x0 ~ N(mu, s^2)."""
    return mu + s * s / (s * s + sigma * sigma) * (x - mu)


def gauss_edm_exact(x_start, sigma_start, sigma, mu, s):
    """The probability-flow ODE dx/dsigma = (x - D) / sigma from (sigma_start, x_start) to sigma."""
    return mu + (x_start - mu) * np.sqrt((s * s + sigma * sigma) / (s * s + sigma_start * sigma_start))


def gauss_flow_D(x, t, mu, s):
    """E[x0 | (1 - t) x0 + t eps = x] for x0 ~ N(mu, s^2)."""
    a = 1.0 - t
    return mu + a * s * s / (a * a * s * s + t * t) * (x - a * mu)


def gauss_flow_exact(x_start, t_start, t, mu, s):
    """The flow ODE dx/dt = (x - D) / t solved in closed form: x(t) = (1 - t) mu + sqrt((1 - t)^2 s^2 + t^2) xi
    with xi constant along the path."""
    sd = lambda tt: np.sqrt((1.0 - tt) ** 2 * s * s + tt * tt)  # noqa: E731
    xi = (x_start - (1.0 - t_start) * mu) / sd(t_start)
    return (1.0 - t) * mu + sd(t) * xi
