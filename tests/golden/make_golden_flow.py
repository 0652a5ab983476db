"""Golden vectors of the rectified-flow objective (DESIGN §5) around the UNMODIFIED reference network.

Run in the dev container only (the GPU box has no /root/reference):  python tests/golden/make_golden_flow.py
The reference's own DiT (`DiT_models` through the EDMPrecond built by make_golden.py's `build_ref`, weights from
oracle.maskdit_oracle.make_state_dict), `patchify` and `mae_loss` run in CPU fp32 with the flow definition applied
around `model(x_t, t, y, mask_ratio=...)`:
  t = sigmoid(P_mean + P_std n) (P_mean 0, P_std 1), x_t = (1 - t) x + t eps, v^ = model output, v = eps - x,
  x^ = x_t - t v^; masked: mean over kept patches of the per-patch mean of (v^ - v)^2 + mae_coef * mae_loss(x_t, x^);
  unmasked: mean((v^ - v)^2).
The draws (n, eps, the mask noise) are stored, with every gradient norm, make_golden.py's full gradients and 4x8 slices
of the other matrices.  Writes tests/golden/flow_*.npz.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as Fn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (installs the timm stand-in and imports the reference)
from make_golden import O, rl  # noqa: E402


def flow_loss(net, x, xt, eps, t4, v_hat, mask, mae_coef):
    l = (v_hat - (eps - x)) ** 2
    if mask is None:
        return l.mean(dim=(1, 2, 3))
    loss = Fn.avg_pool2d(l.mean(dim=1), net.model.patch_size).flatten(1)
    keep = 1 - mask
    loss = (loss * keep).sum(dim=1) / keep.sum(dim=1)
    if mae_coef > 0:
        loss = loss + mae_coef * rl.mae_loss(net, xt, xt - t4 * v_hat, mask)
    return loss


def train_case(name, cfg, B, mask_ratio, mae_coef, grads="full"):
    net = MG.build_ref(cfg).train()
    x, labels = MG.inputs(cfg, B, seed=7)
    g = torch.Generator().manual_seed(321)
    rnd = torch.randn(B, generator=g)
    eps = torch.randn(x.shape, generator=g)
    t = 1.0 / (1.0 + torch.exp(-(rnd * 1.0 + 0.0)))
    t4 = t.reshape(B, 1, 1, 1)
    xt = (1 - t4) * x + t4 * eps
    md = None
    out = dict(images=x.numpy(), rnd_normal=rnd.numpy(), noise_unit=eps.numpy(), t=t.numpy(),
               mask_ratio=np.float32(mask_ratio), mae_coef=np.float32(mae_coef))
    if labels is not None:
        out["labels"] = labels.numpy()
    if mask_ratio > 0:
        mn = torch.rand(B, cfg.num_patches, generator=g)
        md = O.mask_from_noise(mn, mask_ratio)
        out.update(mask_noise=mn.numpy(), mask=md["mask"].numpy())
        res = net.model(xt, t, labels, mask_ratio=mask_ratio, mask_dict=md)
    else:
        res = net.model(xt, t, labels)
    v_hat = res["x"]
    loss = flow_loss(net, x, xt, eps, t4, v_hat, md["mask"] if md else None, mae_coef)
    out.update(F=v_hat.detach().numpy(), loss=loss.detach().numpy(), x_hat=(xt - t4 * v_hat).detach().numpy())
    net.zero_grad()
    loss.mean().backward()
    for k, p in net.named_parameters():
        if p.grad is None:
            continue
        out[f"gnorm/{k}"] = np.float64(p.grad.double().norm().item())
        if grads == "full" and k in MG.GRAD_KEYS_FULL:
            out[f"grad/{k}"] = p.grad.numpy()
        elif p.grad.ndim >= 2:
            out[f"gslice/{k}"] = p.grad.reshape(p.grad.shape[0], -1)[:4, :8].numpy().copy()
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **out)
    print(name, "loss", loss.detach().numpy())


def sampler_case(name, cfg, B, num_steps=3, cfg_scale=1.5):
    """Heun on the uniform grid t_i = 1 - i / N with an Euler last step, CFG through forward_with_cfg, fp64 state."""
    net = MG.build_ref(cfg).eval()
    _, labels = MG.inputs(cfg, B, seed=11)
    g = torch.Generator().manual_seed(99)
    latents = torch.randn(B, cfg.img_channels, cfg.img_resolution, cfg.img_resolution, generator=g)
    grid = 1.0 - np.arange(num_steps + 1, dtype=np.float64) / num_steps
    seen = []

    def v(xx, tc):
        seen.append(tc)
        tt = torch.full((2 * B,), tc, dtype=torch.float32)
        return net.model.forward_with_cfg(xx.float(), tt, labels, cfg_scale)["x"].double()

    with torch.no_grad():
        x = latents.double()
        for k in range(num_steps):
            tc, tn = float(grid[k]), float(grid[k + 1])
            h = tn - tc
            d = v(x, tc)
            if k == num_steps - 1:
                x = x + h * d
            else:
                d2 = v(x + h * d, tn)
                x = x + 0.5 * h * d + 0.5 * h * d2
    assert len(seen) == 2 * num_steps - 1
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), labels=labels.numpy(), latents=latents.numpy(),
                        z=x.numpy(), sampler_t=np.array(seen), num_steps=np.int64(num_steps),
                        cfg_scale=np.float64(cfg_scale))
    print(name, "sampler |z|", x.abs().mean().item())


if __name__ == "__main__":
    train_case("flow_s2_train_mask", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10), B=2,
               mask_ratio=0.5, mae_coef=0.1)
    train_case("flow_nd_s2_uncond", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=0, use_decoder=False),
               B=2, mask_ratio=0.0, mae_coef=0.0)
    train_case("flow_xl2_mask", O.Cfg(model_type="DiT-XL/2", img_resolution=32, num_classes=1000), B=2,
               mask_ratio=0.5, mae_coef=0.1, grads="slices")
    sampler_case("flow_s2_sampler", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10), B=2)
