"""Golden vectors of model guidance (MG, DESIGN §5) around the UNMODIFIED reference network.

Run in the dev container only (the GPU box has no /root/reference):  python tests/golden/make_golden_mg.py
The reference's own EDMPrecond (make_golden.py's `build_ref`, weights from oracle.maskdit_oracle.make_state_dict),
`patchify` and `mae_loss` run in CPU fp32 with the MG objective applied around `net(x, sigma, y, mask_ratio=...)`:
  EDM: sigma = exp(P_mean + P_std n) (P_mean -1.2, P_std 1.2), x_n = x + sigma eps; the student D_c = net(x_n, sigma, y)
  with gradient; D_u = net(x_n, sigma, 0) without gradient, with the same mask (same ids_keep) and the all-zero label
  row; w_b = 1 - 1/scale where the label row is non-zero and lo < sigma <= hi, else 0;
  target = x + w_b (D_c - D_u) (a constant); loss = the reference EDMLoss with y replaced by the target in the denoising
  term, plus mae_coef * mae_loss(net, x_n, D_c, mask) unchanged.
  Flow (around `net.model`, as make_golden_flow.py): t = sigmoid(n), x_t = (1 - t) x + t eps, v' = (eps - x) +
  w_b (v_c - v_u), the interval on t; the MAE term on x^ = x_t - t v_c unchanged.
The draws (n, eps, the mask noise), the scale and the interval are stored, with D_u (flow: v_u), the plain loss against
the unguided target, every gradient norm, make_golden.py's full gradients and 4x8 slices of the other matrices.
Writes tests/golden/mg_*.npz.
"""
import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as Fn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (installs the timm stand-in and imports the reference)
from make_golden import O, rl  # noqa: E402


def edm_term(net, D, target, weight, mask):
    l = weight * (D - target) ** 2
    if mask is None:
        return l.mean(dim=(1, 2, 3))
    l = Fn.avg_pool2d(l.mean(dim=1), net.model.patch_size).flatten(1)
    keep = 1 - mask
    return (l * keep).sum(dim=1) / keep.sum(dim=1)


def flow_term(net, v, target, mask):
    l = (v - target) ** 2
    if mask is None:
        return l.mean(dim=(1, 2, 3))
    l = Fn.avg_pool2d(l.mean(dim=1), net.model.patch_size).flatten(1)
    keep = 1 - mask
    return (l * keep).sum(dim=1) / keep.sum(dim=1)


def train_case(name, cfg, B, mask_ratio, mae_coef, scale, interval, rnd, flow=False, grads="full"):
    net = MG.build_ref(cfg).train()
    x, labels = MG.inputs(cfg, B, seed=7)       # the last label row is dropped (all zero)
    g = torch.Generator().manual_seed(321)
    eps = torch.randn(x.shape, generator=g)
    lo, hi = interval
    w = 1.0 - 1.0 / scale
    if flow:
        level = 1.0 / (1.0 + torch.exp(-rnd))
        l4 = level.reshape(B, 1, 1, 1)
        xin = (1 - l4) * x + l4 * eps
    else:
        level = (rnd * 1.2 - 1.2).exp()
        l4 = level.reshape(B, 1, 1, 1)
        xin = x + l4 * eps
    wb = torch.where((labels.abs().sum(1) > 0) & (level > lo) & (level <= hi), torch.tensor(w), torch.tensor(0.0))
    w4 = wb.reshape(B, 1, 1, 1)
    out = dict(images=x.numpy(), labels=labels.numpy(), rnd_normal=rnd.numpy(), noise_unit=eps.numpy(),
               level=level.numpy(), w_b=wb.numpy(), scale=np.float64(scale), lo=np.float64(lo), hi=np.float64(hi),
               mask_ratio=np.float32(mask_ratio), mae_coef=np.float32(mae_coef))
    kw, md = {}, None
    if mask_ratio > 0:
        mn = torch.rand(B, cfg.num_patches, generator=g)
        md = O.mask_from_noise(mn, mask_ratio)
        out.update(mask_noise=mn.numpy(), mask=md["mask"].numpy())
        kw = dict(mask_ratio=mask_ratio, mask_dict=md)
    mask = md["mask"] if md else None
    null = torch.zeros_like(labels)
    if flow:
        v = net.model(xin, level, labels, **kw)["x"]
        with torch.no_grad():
            vu = net.model(xin, level, null, **kw)["x"]
        target = (eps - x) + w4 * (v.detach() - vu)
        plain = flow_term(net, v, eps - x, mask)
        loss = flow_term(net, v, target, mask)
        if mask is not None and mae_coef > 0:
            mae = mae_coef * rl.mae_loss(net, xin, xin - l4 * v, mask)
            plain, loss = plain + mae, loss + mae
        out["F_u"] = vu.numpy()
    else:
        D = net(xin, level, labels, **kw)["x"]
        with torch.no_grad():
            Du = net(xin, level, null, **kw)["x"]
        weight = (l4 ** 2 + 0.25) / (l4 * 0.5) ** 2
        target = x + w4 * (D.detach() - Du)
        plain = edm_term(net, D, x, weight, mask)
        loss = edm_term(net, D, target, weight, mask)
        if mask is not None and mae_coef > 0:
            mae = mae_coef * rl.mae_loss(net, xin, D, mask)
            plain, loss = plain + mae, loss + mae
        out["D_u"] = Du.numpy()
    out.update(loss=loss.detach().numpy(), edm_loss=plain.detach().numpy())
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
    print(name, "level", level.numpy(), "w_b", wb.numpy(), "loss", loss.detach().numpy(), "plain",
          plain.detach().numpy())


if __name__ == "__main__":
    # sigma = 0.091 (below the interval), 0.43 and 1.82 (guided), 0.89 (inside, but its label was dropped)
    train_case("mg_s2_train_mask", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10), B=4,
               mask_ratio=0.5, mae_coef=0.1, scale=2.0, interval=(0.3, 2.0), rnd=torch.tensor([-1.0, 0.3, 1.5, 0.9]))
    train_case("mg_nd_s2_cond", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10, use_decoder=False),
               B=2, mask_ratio=0.0, mae_coef=0.0, scale=3.0, interval=(0.0, math.inf), rnd=torch.tensor([0.8, -0.3]))
    train_case("mg_xl2_mask", O.Cfg(model_type="DiT-XL/2", img_resolution=32, num_classes=1000), B=3,
               mask_ratio=0.5, mae_coef=0.1, scale=2.0, interval=(0.0, math.inf), rnd=torch.tensor([1.2, -0.4, 0.5]),
               grads="slices")
    train_case("mg_flow_s2_mask", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10), B=3,
               mask_ratio=0.5, mae_coef=0.1, scale=1.5, interval=(0.0, math.inf), rnd=torch.tensor([0.4, -0.7, 1.1]),
               flow=True)
