"""EDM Heun sampler (reference: sample.py:30-66) driving the H100 engine.

Same signature and semantics as the reference `edm_sampler` (fp64 state, 2N-1 network evaluations, `randn_like`
consumed once per step even when S_churn = 0).  With a `maskdit_b200.EDMPrecond` network each evaluation is one
eval-mode engine pass at batch 2B with the classifier-free-guidance combine fused into the output kernel, and the
fp64 Euler/Heun state updates are single fused kernels.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def edm_sampler(net, latents, class_labels=None, cfg_scale=None, feat=None, randn_like=torch.randn_like,
                num_steps=18, sigma_min=0.002, sigma_max=80, rho=7, S_churn=0, S_min=0, S_max=float("inf"),
                S_noise=1):
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
        den = net(x_hat.float(), torch.tensor(t_hat, dtype=torch.float64, device=dev), class_labels, cfg_scale,
                  feat=feat)["x"].float().contiguous()
        ops.heun_update(0, x_hat, den, d_cur, x_next, x32, t_hat, t_next)          # Euler step (sample.py:56-58)
        if k < num_steps - 1:
            den = net(x32, torch.tensor(t_next, dtype=torch.float64, device=dev), class_labels, cfg_scale,
                      feat=feat)["x"].float().contiguous()
            ops.heun_update(1, x_hat, den, d_cur, x_next, x32, t_hat, t_next)      # 2nd-order correction (:61-64)
    return x_next


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
                     S_churn=0, S_min=0, S_max=float("inf"), S_noise=1):
    """Generalised sampler (reference: sample.py:73-188), same signature.  All schedule quantities are fp64 host
    scalars; the state lives on the device in fp64 and every update (churn, Euler, the alpha-weighted 2nd-order
    correction) is one `mdt_lincomb_f64` launch that also emits the next fp32 network input x / s(t)."""
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
        den = net(xin, f64(sch.sigma(t_hat)), class_labels, cfg_scale, feat=feat)["x"].float().contiguous()
        A, Bc = sch.ode_coeffs(t_hat)
        ops.lincomb_f64(A, x_hat, 0.0, None, -Bc, den, out=d_cur)                       # d_cur = A x_hat - B D
        if solver == "euler" or i == num_steps - 1:
            ops.lincomb_f64(1.0, x_hat, h, d_cur, out=x_next)                           # x_hat + h d_cur
            continue
        t_prime = t_hat + alpha * h
        ops.lincomb_f64(1.0, x_hat, alpha * h, d_cur, out=x_prime, out_f32=xin, f32_scale=1.0 / sch.s(t_prime))
        den = net(xin, f64(sch.sigma(t_prime)), class_labels, cfg_scale, feat=feat)["x"].float().contiguous()
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
