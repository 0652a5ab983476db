"""EDM Heun sampler (reference: sample.py:30-66) driving the H100 engine.

Same signature and semantics as the reference `edm_sampler` (fp64 state, 2N-1 network evaluations, `randn_like`
consumed once per step even when S_churn = 0).  With a `maskdit_b200.EDMPrecond` network each evaluation is one
eval-mode engine pass at batch 2B with the classifier-free-guidance combine fused into the output kernel, and the
fp64 Euler/Heun state updates are single fused kernels.  Both samplers can instead guide with a second network
(`guide_net`, `guidance`: autoguidance) and apply either guidance only inside a noise-level interval
(`guidance_interval`); see `_denoiser`.  `flow_sampler` integrates a rectified-flow network's velocity instead,
`consistency_sampler` samples a consistency-tuned network in one evaluation per noise level, and `dpm_solver_sampler`
(multistep DPM-Solver++) samples an EDM or a flow network in one evaluation per noise level.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops


def _denoiser(net, class_labels, cfg_scale, feat, guide_net, guidance, guidance_interval):
    """The sampler's network evaluation D(x; sigma) as a function of (x, sigma as a Python float).

    Without guide_net / guidance_interval it is the reference's call `net(x, sigma, labels, cfg_scale)`.  With a guide
    network, D = D_guide + guidance (D_net - D_guide) (autoguidance, Karras et al., NeurIPS 2024); guidance == 1 is the
    unguided network and evaluates no guide.  guidance_interval = (lo, hi) applies the active guidance (CFG or the
    guide) only where lo < sigma <= hi (Kynkaanniemi et al., NeurIPS 2024), decided per evaluation; elsewhere the
    evaluation is the unguided `net(x, sigma, labels, None)`."""
    if guide_net is not None:
        if cfg_scale is not None:
            raise ValueError("cfg_scale and guide_net are mutually exclusive")
        if guidance is None:
            raise ValueError("guide_net needs a guidance weight")
        net.check_guide(guide_net)
        guidance = float(guidance)
        if not np.isfinite(guidance):
            raise ValueError(f"guidance must be finite, got {guidance}")
    elif guidance is not None:
        raise ValueError("guidance is the weight of guide_net; classifier-free guidance takes cfg_scale")
    if guidance_interval is not None:
        lo, hi = (float(v) for v in guidance_interval)
        if not lo < hi:
            raise ValueError(f"guidance_interval needs sigma_lo < sigma_hi, got ({lo}, {hi})")
        if guide_net is None and cfg_scale is None:
            raise ValueError("guidance_interval needs cfg_scale or guide_net")

    def denoise(x, sigma):
        s = torch.tensor(sigma, dtype=torch.float64, device=x.device)
        if (guidance_interval is not None and not lo < sigma <= hi) or (guide_net is not None and guidance == 1):
            return net(x, s, class_labels, None, feat=feat)["x"]
        if guide_net is None:
            return net(x, s, class_labels, cfg_scale, feat=feat)["x"]
        return net.forward_guided(x, s, class_labels, guide_net, guidance)

    return denoise


def edm_sampler(net, latents, class_labels=None, cfg_scale=None, feat=None, randn_like=torch.randn_like,
                num_steps=18, sigma_min=0.002, sigma_max=80, rho=7, S_churn=0, S_min=0, S_max=float("inf"),
                S_noise=1, guide_net=None, guidance=None, guidance_interval=None):
    """`guide_net`, `guidance` and `guidance_interval` (all opt-in) select guidance by a second network and limit the
    guidance to a noise-level interval: see `_denoiser`.  Without them every evaluation is the reference's call."""
    denoise = _denoiser(net, class_labels, cfg_scale, feat, guide_net, guidance, guidance_interval)
    sigma_min = max(sigma_min, net.sigma_min)
    sigma_max = min(sigma_max, net.sigma_max)
    dev = latents.device
    # Karras schedule in fp64 on the host (sample.py:40-43); t_N = 0
    i = np.arange(num_steps, dtype=np.float64)
    t = (sigma_max ** (1 / rho) + i / (num_steps - 1) * (sigma_min ** (1 / rho) - sigma_max ** (1 / rho))) ** rho
    t = np.concatenate([t, [0.0]])

    x_next = (latents.to(torch.float64) * t[0]).contiguous()
    d_cur = torch.empty_like(x_next)
    x32 = torch.empty(x_next.shape, dtype=torch.float32, device=dev)
    for k in range(num_steps):
        t_cur, t_next = float(t[k]), float(t[k + 1])
        gamma = min(S_churn / num_steps, np.sqrt(2) - 1) if S_min <= t_cur <= S_max else 0
        t_hat = t_cur + gamma * t_cur
        noise = randn_like(x_next)  # drawn every step, as in the reference (sample.py:53)
        if gamma > 0:
            x_hat = (x_next + float(np.sqrt(t_hat ** 2 - t_cur ** 2)) * S_noise * noise).contiguous()
        else:
            x_hat = x_next.clone()
        den = denoise(x_hat.float(), t_hat).float().contiguous()
        ops.heun_update(0, x_hat, den, d_cur, x_next, x32, t_hat, t_next)          # Euler step (sample.py:56-58)
        if k < num_steps - 1:
            den = denoise(x32, t_next).float().contiguous()
            ops.heun_update(1, x_hat, den, d_cur, x_next, x32, t_hat, t_next)      # 2nd-order correction (:61-64)
    return x_next


def consistency_sigmas(sigmas, sigma_max=float("inf")):
    """The noise levels of `consistency_sampler`: each clamped to `sigma_max` as `edm_sampler` clamps its largest, then
    required positive, finite and strictly decreasing.  Returns a list of floats."""
    out = [min(float(s), float(sigma_max)) for s in sigmas]
    if not out:
        raise ValueError("consistency sampling needs at least one noise level")
    if not all(np.isfinite(s) and s > 0 for s in out):
        raise ValueError(f"consistency sampling needs positive, finite noise levels, got {out}")
    if any(a <= b for a, b in zip(out, out[1:])):
        raise ValueError(f"consistency sampling needs strictly decreasing noise levels, got {out}")
    return out


@torch.no_grad()
def consistency_sampler(net, latents, class_labels=None, cfg_scale=None, randn_like=torch.randn_like, sigmas=(80.0,),
                        guide_net=None, guidance=None, guidance_interval=None):
    """Few-step sampler of a consistency-tuned network (`Losses['ect']`, DESIGN §5), one network evaluation per noise
    level: x = sigma_0 z, D = f(x, sigma_0); then for each following sigma_i, x = D + sigma_i eps_i (one `randn_like`
    per re-noising) and D = f(x, sigma_i).  Returns the last D (fp64).  Every evaluation is `edm_sampler`'s, so
    `cfg_scale`, `guide_net` / `guidance` and `guidance_interval` apply as there; the state is fp64 and every update is
    one `mdt_lincomb_f64` launch that also writes the next fp32 network input."""
    denoise = _denoiser(net, class_labels, cfg_scale, None, guide_net, guidance, guidance_interval)
    sig = consistency_sigmas(sigmas, net.sigma_max)
    x = latents.to(torch.float64).contiguous().clone()
    xin = torch.empty(latents.shape, dtype=torch.float32, device=latents.device)
    ops.lincomb_f64(sig[0], x, out=x, out_f32=xin)                                                # sigma_0 z
    D = denoise(xin, sig[0]).float().contiguous()
    for s in sig[1:]:
        noise = randn_like(x).contiguous()
        ops.lincomb_f64(s, noise, 0.0, None, 1.0, D, out=x, out_f32=xin)                         # D + sigma_i eps_i
        D = denoise(xin, s).float().contiguous()
    return D.double()


def flow_grid(num_steps):
    """The flow sampler's time grid: num_steps + 1 uniform points from t = 1 (noise) to t = 0 (data), fp64."""
    if num_steps < 1:
        raise ValueError(f"num_steps must be at least 1, got {num_steps}")
    return 1.0 - np.arange(num_steps + 1, dtype=np.float64) / num_steps


@torch.no_grad()
def flow_sampler(net, latents, class_labels=None, cfg_scale=None, num_steps=50, solver="heun",
                 guidance_interval=None):
    """ODE sampler of a rectified-flow network (`FlowPrecond`): integrates dx/dt = v^(x, t) from x(1) = `latents` to
    t = 0 on `flow_grid(num_steps)`.  The state is fp64 and every update is one `mdt_lincomb_f64` launch that also
    writes the next fp32 network input.  solver 'euler': num_steps evaluations; 'heun': Heun's second-order step with
    an Euler last step (the corrector would evaluate at t = 0), 2 num_steps - 1 evaluations.  `cfg_scale` and
    `guidance_interval` = (lo, hi), which applies CFG only where lo < t <= hi, are those of `edm_sampler` with t in
    place of sigma."""
    if solver not in ("euler", "heun"):
        raise ValueError(f"solver must be 'euler' or 'heun', got {solver!r}")
    denoise = _denoiser(net, class_labels, cfg_scale, None, None, None, guidance_interval)
    t = flow_grid(num_steps)
    x = latents.to(torch.float64).contiguous().clone()
    xin = x.float().contiguous()
    for k in range(num_steps):
        t_cur, t_next = float(t[k]), float(t[k + 1])
        h = t_next - t_cur
        v = denoise(xin, t_cur).float().contiguous()
        if solver == "euler" or k == num_steps - 1:
            ops.lincomb_f64(1.0, x, 0.0, None, h, v, out=x, out_f32=xin)                 # x + h v
            continue
        ops.lincomb_f64(1.0, x, 0.0, None, h, v, out_f32=xin)                           # predictor input x + h v
        ops.lincomb_f64(1.0, x, 0.0, None, 0.5 * h, v, out=x)                           # x + h/2 v
        v2 = denoise(xin, t_next).float().contiguous()
        ops.lincomb_f64(1.0, x, 0.0, None, 0.5 * h, v2, out=x, out_f32=xin)             # ... + h/2 v'
    return x


def _lambda(alpha, sigma):
    """log(alpha / sigma), with the limits -inf at alpha = 0 (flow time t = 1) and +inf at sigma = 0."""
    if alpha == 0:
        return -math.inf
    if sigma == 0:
        return math.inf
    return math.log(alpha / sigma)


def dpm_solver_coefficients(alpha, sigma, order):
    """The steps of multistep DPM-Solver++ (DESIGN §5) on the levels x = alpha_i x0 + sigma_i eps, i = 0..N (sigma_N = 0),
    expanded to x' = a x + b0 D_i + b1 D_{i-1} + b2 D_{i-2}: one (k, a, b0, b1, b2) per step i = 0..N-1, in fp64.
    k = min(order, i + 1, N - i) is the step's order (the terms k does not use have coefficient 0).  The step into
    sigma = 0 is x' = alpha_N D; a history term whose lambda gap is infinite (flow time t = 1) drops out (its ratio r
    is infinite)."""
    if order not in (1, 2, 3):
        raise ValueError(f"order must be 1, 2 or 3, got {order}")
    alpha, sigma = [float(v) for v in alpha], [float(v) for v in sigma]
    N = len(sigma) - 1
    lam = [_lambda(a, s) for a, s in zip(alpha, sigma)]
    out = []
    for i in range(N):
        a1 = alpha[i + 1]
        if sigma[i + 1] == 0:
            out.append((1, 0.0, a1, 0.0, 0.0))
            continue
        h = lam[i + 1] - lam[i]
        E = math.expm1(-h)
        a, b0, b1, b2 = sigma[i + 1] / sigma[i], -a1 * E, 0.0, 0.0
        k = min(order, i + 1, N - i)
        if k == 2:
            r0 = (lam[i] - lam[i - 1]) / h
            # - a1 E / 2 * (D_i - D_{i-1}) / r0
            c = -0.5 * a1 * E / r0
            b0, b1 = b0 + c, -c
        elif k == 3:
            r0 = (lam[i] - lam[i - 1]) / h
            r1 = (lam[i - 1] - lam[i - 2]) / h
            c1 = a1 * (E / h + 1)                       # weight of D1
            c2 = -a1 * ((E + h) / (h * h) - 0.5)        # weight of D2
            # D1 = (1 + r0/(r0+r1)) D1_0 - r0/(r0+r1) D1_1,  D2 = (D1_0 - D1_1)/(r0+r1),  D1_j = difference / r_j
            w0 = c1 * (1 + r0 / (r0 + r1)) + c2 / (r0 + r1)
            w1 = -c1 * r0 / (r0 + r1) - c2 / (r0 + r1)
            b0, b1, b2 = b0 + w0 / r0, -w0 / r0 + w1 / r1, -w1 / r1
        out.append((k, a, b0, b1, b2))
    return out


def dpm_solver_levels(net, num_steps, sigma_min=0.002, sigma_max=80, rho=7):
    """(flow, levels): the N = num_steps noise levels of `dpm_solver_sampler` followed by 0.  EDM: `edm_sampler`'s
    Karras grid, clamped to the network's sigma range (a single level is sigma_max); flow (`FlowPrecond`):
    `flow_grid(N)`."""
    if num_steps < 1:
        raise ValueError(f"num_steps must be at least 1, got {num_steps}")
    from .maskdit import FlowPrecond
    if isinstance(net, FlowPrecond):
        return True, flow_grid(num_steps)
    sigma_min = max(sigma_min, net.sigma_min)
    sigma_max = min(sigma_max, net.sigma_max)
    if num_steps == 1:
        return False, np.array([float(sigma_max), 0.0])
    i = np.arange(num_steps, dtype=np.float64)
    t = (sigma_max ** (1 / rho) + i / (num_steps - 1) * (sigma_min ** (1 / rho) - sigma_max ** (1 / rho))) ** rho
    return False, np.concatenate([t, [0.0]])


def _dpm_solve(denoise, x, levels, flow, order):
    """Multistep DPM-Solver++ from the fp64 state `x` at levels[0] through `levels` (the last one 0).  denoise(x32,
    level) is the network output at the fp32 input x32: D (EDM) or the velocity v^ (flow, D = x - t v^ from the fp64
    state).  One network evaluation and one `mdt_dpm_update` launch per positive level; x is updated in place."""
    levels = np.asarray(levels, dtype=np.float64)
    alpha, sigma = (1.0 - levels, levels) if flow else (np.ones_like(levels), levels)
    steps = dpm_solver_coefficients(alpha, sigma, order)
    hist = [torch.empty_like(x) for _ in range(min(order, len(steps)))]
    xin = x.float().contiguous()
    for i, (k, a, b0, b1, b2) in enumerate(steps):
        lv = float(levels[i])
        F = denoise(xin, lv).float().contiguous()
        slot = lambda j: hist[(i - j) % len(hist)]  # noqa: E731  D_{i-j}
        last = i == len(steps) - 1
        ops.dpm_update(F, x, slot(0), a, b0, slot(1) if k >= 2 else None, b1, slot(2) if k >= 3 else None, b2,
                       velocity=flow, t=lv, out_f32=None if last else xin)
    return x


@torch.no_grad()
def dpm_solver_sampler(net, latents, class_labels=None, cfg_scale=None, num_steps=10, order=3, sigma_min=0.002,
                       sigma_max=80, rho=7, guide_net=None, guidance=None, guidance_interval=None):
    """Multistep DPM-Solver++ (Lu et al., 2022; DESIGN §5), a training-free ODE sampler of an EDM (`EDMPrecond`) or a
    rectified-flow (`FlowPrecond`) network in `num_steps` network evaluations, one per level of
    `dpm_solver_levels`: order 1 is DDIM, 2 and 3 are 2M and 3M.  The state is fp64, every step is one `mdt_dpm_update`
    launch, and the returned fp64 value is D at the last positive level.  Each evaluation is `edm_sampler`'s, so
    `cfg_scale`, `guide_net` / `guidance` (EDM only: a flow network refuses a guide) and `guidance_interval` apply as
    there; for a flow network the interval is decided on t."""
    if order not in (1, 2, 3):
        raise ValueError(f"order must be 1, 2 or 3, got {order}")
    flow, levels = dpm_solver_levels(net, num_steps, sigma_min, sigma_max, rho)
    denoise = _denoiser(net, class_labels, cfg_scale, None, guide_net, guidance, guidance_interval)
    x = latents.to(torch.float64).contiguous().clone()
    ops.lincomb_f64(float(levels[0]), x, out=x)                                                  # sigma_0 z
    return _dpm_solve(denoise, x, levels, flow, order)


class _Schedules:
    """Noise-level schedule sigma(t), scaling s(t), their derivatives and sigma^-1 as plain fp64 host functions
    (sample.py:86-92,131-152).  The reference evaluates them on 0-d fp64 tensors; the values are identical."""

    def __init__(self, schedule, scaling, beta_d, beta_min):
        e = np.e
        if schedule == "vp":
            self.sigma = lambda t: float((e ** (0.5 * beta_d * (t ** 2) + beta_min * t) - 1) ** 0.5)
            self.sigma_deriv = lambda t: 0.5 * (beta_min + beta_d * t) * (self.sigma(t) + 1 / self.sigma(t))
            self.sigma_inv = lambda s: float((np.sqrt(beta_min ** 2 + 2 * beta_d * np.log(s ** 2 + 1)) - beta_min) / beta_d)
        elif schedule == "ve":
            self.sigma = lambda t: float(np.sqrt(t))
            self.sigma_deriv = lambda t: float(0.5 / np.sqrt(t))
            self.sigma_inv = lambda s: float(s ** 2)
        elif schedule == "linear":
            self.sigma, self.sigma_deriv, self.sigma_inv = (lambda t: float(t)), (lambda t: 1.0), (lambda s: float(s))
        else:
            raise AssertionError(schedule)
        if scaling == "vp":
            self.s = lambda t: float(1 / np.sqrt(1 + self.sigma(t) ** 2))
            self.s_deriv = lambda t: -self.sigma(t) * self.sigma_deriv(t) * (self.s(t) ** 3)
        elif scaling == "none":
            self.s, self.s_deriv = (lambda t: 1.0), (lambda t: 0.0)
        else:
            raise AssertionError(scaling)

    def ode_coeffs(self, t):
        """dx/dt = A(t) x - B(t) D(x / s(t); sigma(t))   (sample.py:171-172)."""
        sg, sd, sc = self.sigma(t), self.sigma_deriv(t), self.s(t)
        return sd / sg + self.s_deriv(t) / sc, sd * sc / sg


def _iddpm_sigmas(M, C_1, C_2, sigma_min, sigma_max, num_steps):
    # sample.py:117-123.  `j` is an int64 tensor there, so alpha_bar is evaluated in torch's default float32 while u is
    # fp64: that promotion is part of the reference's step sequence, hence torch (host tensors) here as well.
    u = torch.zeros(M + 1, dtype=torch.float64)
    abar = lambda j: (0.5 * np.pi * j / M / (C_2 + 1)).sin() ** 2  # noqa: E731
    for j in torch.arange(M, 0, -1):
        u[j - 1] = ((u[j] ** 2 + 1) / (abar(j - 1) / abar(j)).clip(min=C_1) - 1).sqrt()
    uf = u[torch.logical_and(u >= sigma_min, u <= sigma_max)].numpy()
    return uf[np.round((len(uf) - 1) / (num_steps - 1) * np.arange(num_steps, dtype=np.float64)).astype(np.int64)]


def ablation_sampler(net, latents, class_labels=None, cfg_scale=None, feat=None, randn_like=torch.randn_like,
                     num_steps=18, sigma_min=None, sigma_max=None, rho=7, solver="heun", discretization="edm",
                     schedule="linear", scaling="none", epsilon_s=1e-3, C_1=0.001, C_2=0.008, M=1000, alpha=1,
                     S_churn=0, S_min=0, S_max=float("inf"), S_noise=1, guide_net=None, guidance=None,
                     guidance_interval=None):
    """Generalised sampler (reference: sample.py:73-188), same signature.  All schedule quantities are fp64 host
    scalars; the state lives on the device in fp64 and every update (churn, Euler, the alpha-weighted 2nd-order
    correction) is one `mdt_lincomb_f64` launch that also emits the next fp32 network input x / s(t).  The opt-in
    `guide_net`, `guidance` and `guidance_interval` are those of `edm_sampler`; the interval is decided on sigma(t)."""
    denoise = _denoiser(net, class_labels, cfg_scale, feat, guide_net, guidance, guidance_interval)
    assert solver in ("euler", "heun") and discretization in ("vp", "ve", "iddpm", "edm")
    assert schedule in ("vp", "ve", "linear") and scaling in ("vp", "none")
    vp_sig = lambda bd, bm, t: float((np.e ** (0.5 * bd * (t ** 2) + bm * t) - 1) ** 0.5)  # noqa: E731
    if sigma_min is None:
        sigma_min = {"vp": vp_sig(19.1, 0.1, epsilon_s), "ve": 0.02, "iddpm": 0.002, "edm": 0.002}[discretization]
    if sigma_max is None:
        sigma_max = {"vp": vp_sig(19.1, 0.1, 1), "ve": 100, "iddpm": 81, "edm": 80}[discretization]
    sigma_min, sigma_max = max(sigma_min, net.sigma_min), min(sigma_max, net.sigma_max)
    beta_d = 2 * (np.log(sigma_min ** 2 + 1) / epsilon_s - np.log(sigma_max ** 2 + 1)) / (epsilon_s - 1)
    beta_min = np.log(sigma_max ** 2 + 1) - 0.5 * beta_d
    idx = np.arange(num_steps, dtype=np.float64)
    if discretization == "vp":
        sig_steps = [vp_sig(beta_d, beta_min, t) for t in 1 + idx / (num_steps - 1) * (epsilon_s - 1)]
    elif discretization == "ve":
        sig_steps = np.sqrt((sigma_max ** 2) * ((sigma_min ** 2 / sigma_max ** 2) ** (idx / (num_steps - 1))))
    elif discretization == "iddpm":
        sig_steps = _iddpm_sigmas(M, C_1, C_2, sigma_min, sigma_max, num_steps)
    else:
        sig_steps = (sigma_max ** (1 / rho) + idx / (num_steps - 1) * (sigma_min ** (1 / rho) - sigma_max ** (1 / rho))) ** rho
    sch = _Schedules(schedule, scaling, beta_d, beta_min)
    t_steps = [sch.sigma_inv(float(net.round_sigma(torch.as_tensor(v, dtype=torch.float64)))) for v in sig_steps] + [0.0]
    dev = latents.device
    f64 = lambda v: torch.tensor(v, dtype=torch.float64, device=dev)  # noqa: E731

    x_next = (latents.to(torch.float64) * (sch.sigma(t_steps[0]) * sch.s(t_steps[0]))).contiguous()
    x_hat, d_cur, x_prime = torch.empty_like(x_next), torch.empty_like(x_next), torch.empty_like(x_next)
    xin = torch.empty(x_next.shape, dtype=torch.float32, device=dev)
    for i in range(num_steps):
        t_cur, t_next = t_steps[i], t_steps[i + 1]
        sg_cur = sch.sigma(t_cur)
        gamma = min(S_churn / num_steps, np.sqrt(2) - 1) if S_min <= sg_cur <= S_max else 0
        t_hat = sch.sigma_inv(float(net.round_sigma(f64(sg_cur + gamma * sg_cur))))
        churn = float(np.sqrt(max(sch.sigma(t_hat) ** 2 - sg_cur ** 2, 0.0))) * sch.s(t_hat) * S_noise
        noise = randn_like(x_next).contiguous()        # consumed every step (sample.py:166), also when churn == 0
        ops.lincomb_f64(sch.s(t_hat) / sch.s(t_cur), x_next, churn, noise, out=x_hat, out_f32=xin,
                        f32_scale=1.0 / sch.s(t_hat))
        h = t_next - t_hat
        den = denoise(xin, sch.sigma(t_hat)).float().contiguous()
        A, Bc = sch.ode_coeffs(t_hat)
        ops.lincomb_f64(A, x_hat, 0.0, None, -Bc, den, out=d_cur)                       # d_cur = A x_hat - B D
        if solver == "euler" or i == num_steps - 1:
            ops.lincomb_f64(1.0, x_hat, h, d_cur, out=x_next)                           # x_hat + h d_cur
            continue
        t_prime = t_hat + alpha * h
        ops.lincomb_f64(1.0, x_hat, alpha * h, d_cur, out=x_prime, out_f32=xin, f32_scale=1.0 / sch.s(t_prime))
        den = denoise(xin, sch.sigma(t_prime)).float().contiguous()
        A2, B2 = sch.ode_coeffs(t_prime)
        w1, w2 = h * (1 - 1 / (2 * alpha)), h / (2 * alpha)
        ops.lincomb_f64(w2 * A2, x_prime, w1, d_cur, -w2 * B2, den, out=x_prime)       # w1 d_cur + w2 d_prime
        ops.lincomb_f64(1.0, x_hat, 1.0, x_prime, out=x_next)
    return x_next


def rank_seed_batches(seeds, max_batch_size, rank=0, size=1):
    """This rank's seed batches (generate_with_net, sample.py:232-235): the seed list is cut into a multiple-of-`size`
    number of near-equal batches no larger than `max_batch_size`, dealt to the ranks round robin."""
    seeds = list(seeds)
    if not seeds:
        return []
    num_batches = ((len(seeds) - 1) // (max_batch_size * size) + 1) * size
    q, r = divmod(len(seeds), num_batches)          # tensor_split: the first r parts hold q + 1 elements
    out, pos = [], 0
    for b in range(num_batches):
        n = q + (1 if b < r else 0)
        if b % size == rank:
            out.append(seeds[pos:pos + n])
        pos += n
    return out


def write_png(path, image_hwc_uint8):
    """8-bit RGB / grey PNG (what PIL.Image.save writes at sample.py:291-296), stdlib only."""
    import struct
    import zlib
    a = np.ascontiguousarray(image_hwc_uint8, dtype=np.uint8)
    if a.ndim == 2:
        a = a[:, :, None]
    H, W, C = a.shape
    if C not in (1, 3):
        raise ValueError("PNG writer handles 1 or 3 channels")
    raw = np.concatenate([np.zeros((H, 1), np.uint8), a.reshape(H, W * C)], axis=1).tobytes()  # filter type 0 rows

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 0 if C == 1 else 2, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))
