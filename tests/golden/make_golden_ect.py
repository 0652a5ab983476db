"""Golden vectors of Easy Consistency Tuning (ECT, DESIGN §5) around the UNMODIFIED reference network.

Run in the dev container only (the GPU box has no /root/reference):  python tests/golden/make_golden_ect.py
The reference's own EDMPrecond (make_golden.py's `build_ref`, weights from oracle.maskdit_oracle.make_state_dict),
`patchify` and `mae_loss` run in CPU fp32 with the ECT objective applied around `net(x, sigma, y, mask_ratio=...)`:
  t = exp(P_mean + P_std n) (P_mean -1.1, P_std 2), r = t max(0, 1 - q^-(s+1) (1 + k sigmoid(-b t))) (q 2, k 8, b 1),
  x_t = x + t eps, x_r = x + r eps; student D_t = net(x_t, t) with gradient; target net(x_r, r) without gradient, with
  the same mask (same ids_keep) and labels, fed sigma = t where r = 0 and replaced there by x;
  S = (L / T) sum over kept patches of (D_t - D_r)^2, c = 0.00054 sqrt(C R R),
  loss = (sqrt(S + c^2) - c) / (t - r) + mae_coef * mae_loss(net, x_t, D_t, mask)   (unmasked: T = L, no MAE term).
The draws (n, eps, the mask noise) and the stage are stored, with every gradient norm, make_golden.py's full gradients
and 4x8 slices of the other matrices.  The sampler case runs the two-step consistency sampler with CFG through the
reference's `net(x, sigma, labels, cfg_scale)`.  Writes tests/golden/ect_*.npz.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (installs the timm stand-in and imports the reference)
from make_golden import O, rl  # noqa: E402

P_MEAN, P_STD, Q, K, BB = -1.1, 2.0, 2.0, 8.0, 1.0


def ect_r(t, stage):
    qs = Q ** -(stage + 1)
    return t * (1.0 - qs * (1.0 + K / (1.0 + torch.exp(BB * t)))).clamp_min(0.0)


def train_case(name, cfg, B, mask_ratio, mae_coef, stage, rnd=None, grads="full"):
    net = MG.build_ref(cfg).train()
    x, labels = MG.inputs(cfg, B, seed=7)
    g = torch.Generator().manual_seed(321)
    if rnd is None:
        rnd = torch.randn(B, generator=g)
    eps = torch.randn(x.shape, generator=g)
    t = (rnd * P_STD + P_MEAN).exp()
    r = ect_r(t, stage)
    t4, r4 = t.reshape(B, 1, 1, 1), r.reshape(B, 1, 1, 1)
    xt, xr = x + t4 * eps, x + r4 * eps
    sr = torch.where(r > 0, r, t)
    out = dict(images=x.numpy(), rnd_normal=rnd.numpy(), noise_unit=eps.numpy(), t=t.numpy(), r=r.numpy(),
               stage=np.int64(stage), mask_ratio=np.float32(mask_ratio), mae_coef=np.float32(mae_coef))
    if labels is not None:
        out["labels"] = labels.numpy()
    kw = {}
    if mask_ratio > 0:
        mn = torch.rand(B, cfg.num_patches, generator=g)
        md = O.mask_from_noise(mn, mask_ratio)
        out.update(mask_noise=mn.numpy(), mask=md["mask"].numpy())
        kw = dict(mask_ratio=mask_ratio, mask_dict=md)
    D_t = net(xt, t, labels, **kw)["x"]
    with torch.no_grad():
        D_r = torch.where(r4 > 0, net(xr, sr, labels, **kw)["x"], x)
    p = net.model.patch_size
    se = rl.patchify((D_t - D_r) ** 2, p, cfg.img_channels).sum(-1)            # [B, L]
    L = se.shape[1]
    if mask_ratio > 0:
        keep = 1 - md["mask"]
        S = (se * keep).sum(1) * (L / keep.sum(1))
    else:
        S = se.sum(1)
    c = 0.00054 * (cfg.img_channels * cfg.img_resolution ** 2) ** 0.5
    loss = ((S + c * c).sqrt() - c) / (t - r)
    if mask_ratio > 0 and mae_coef > 0:
        loss = loss + mae_coef * rl.mae_loss(net, xt, D_t, md["mask"])
    out.update(D_t=D_t.detach().numpy(), loss=loss.detach().numpy())
    net.zero_grad()
    loss.mean().backward()
    for k, prm in net.named_parameters():
        if prm.grad is None:
            continue
        out[f"gnorm/{k}"] = np.float64(prm.grad.double().norm().item())
        if grads == "full" and k in MG.GRAD_KEYS_FULL:
            out[f"grad/{k}"] = prm.grad.numpy()
        elif prm.grad.ndim >= 2:
            out[f"gslice/{k}"] = prm.grad.reshape(prm.grad.shape[0], -1)[:4, :8].numpy().copy()
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **out)
    print(name, "t", t.numpy(), "r", r.numpy(), "loss", loss.detach().numpy())


def sampler_case(name, cfg, B, sigmas=(80.0, 0.8), cfg_scale=1.5):
    """x = sigma_0 z, D = f(x, sigma_0); x = D + sigma_1 eps_1, D = f(x, sigma_1); fp64 state, CFG."""
    net = MG.build_ref(cfg).eval()
    _, labels = MG.inputs(cfg, B, seed=11)
    g = torch.Generator().manual_seed(99)
    latents = torch.randn(B, cfg.img_channels, cfg.img_resolution, cfg.img_resolution, generator=g)
    noises = [torch.randn(latents.shape, dtype=torch.float64, generator=g) for _ in sigmas[1:]]

    def f(x, s):
        return net(x.float(), torch.tensor(s, dtype=torch.float64), labels, cfg_scale)["x"].double()

    with torch.no_grad():
        D = f(latents.double() * sigmas[0], sigmas[0])
        for s, n in zip(sigmas[1:], noises):
            D = f(D + s * n, s)
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), labels=labels.numpy(), latents=latents.numpy(),
                        noises=np.stack([n.numpy() for n in noises]), z=D.numpy(), sigmas=np.array(sigmas),
                        cfg_scale=np.float64(cfg_scale))
    print(name, "sampler |z|", D.abs().mean().item())


# The stages are those of early tuning: the gradient seed is proportional to delta = D_t - D_r, so the bf16 noise of the
# two network outputs weighs 1 / gap more in it than in the loss (DESIGN §5); the kernel tests cover the small gaps.
if __name__ == "__main__":
    # stage 0: the two small-t rows have r = 0 (the denoising limit), the two large-t rows r > 0
    train_case("ect_s2_train_mask", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10), B=4,
               mask_ratio=0.5, mae_coef=0.1, stage=0, rnd=torch.tensor([-1.0, 0.3, 1.5, 0.9]))
    train_case("ect_nd_s2_uncond", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=0, use_decoder=False),
               B=2, mask_ratio=0.0, mae_coef=0.0, stage=0, rnd=torch.tensor([0.8, 1.6]))
    train_case("ect_xl2_mask", O.Cfg(model_type="DiT-XL/2", img_resolution=32, num_classes=1000), B=2,
               mask_ratio=0.5, mae_coef=0.1, stage=0, rnd=torch.tensor([1.2, -0.4]), grads="slices")
    sampler_case("ect_s2_sampler", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10), B=2)
