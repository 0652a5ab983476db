"""Golden vectors of multistep DPM-Solver++ (DESIGN §5) around the UNMODIFIED reference network.

Run in the dev container only (the GPU box has no /root/reference):  python tests/golden/make_golden_dpm.py
The reference's own DiT (the EDMPrecond built by make_golden.py's `build_ref`, weights from
oracle.maskdit_oracle.make_state_dict) runs in CPU fp32 inside the float64 solver of oracle/dpm_solver_oracle.py, in
its D1 / D2 form:
  * EDM, DiT-S/2 with decoder, class-conditional, CFG 1.5 through the reference's `forward(x, sigma, labels, cfg_scale)`,
    order 3 on the 6-level Karras grid (sigma 80 -> 0.002, rho 7);
  * rectified flow, the decoder-less class-unconditional DiT-S/2, D = x - t v^ with v^ = `model(x, t, None)`, order 2
    on flow_grid(5) (t = 1, 0.8, ..., 0.2).
The network reads the state rounded to fp32, as the H100 sampler's network does.  Writes tests/golden/dpm_*.npz.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (installs the timm stand-in and imports the reference)
from make_golden import O  # noqa: E402
from oracle import dpm_solver_oracle as DPM  # noqa: E402


def edm_case(name, cfg, B, num_steps=6, order=3, cfg_scale=1.5):
    net = MG.build_ref(cfg).eval()
    _, labels = MG.inputs(cfg, B, seed=11)
    g = torch.Generator().manual_seed(99)
    latents = torch.randn(B, cfg.img_channels, cfg.img_resolution, cfg.img_resolution, generator=g)
    levels = DPM.karras_levels(num_steps)
    alpha, sigma = DPM.edm_alpha_sigma(levels)

    def D(x, i):
        s = torch.tensor(sigma[i], dtype=torch.float64)
        return net(torch.from_numpy(x).float(), s, labels, cfg_scale)["x"].double().numpy()

    with torch.no_grad():
        z = DPM.dpm_solver(D, sigma[0] * latents.double().numpy(), alpha, sigma, order)
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), labels=labels.numpy(), latents=latents.numpy(), z=z,
                        levels=levels, num_steps=np.int64(num_steps), order=np.int64(order),
                        cfg_scale=np.float64(cfg_scale))
    print(name, "|z|", np.abs(z).mean())


def flow_case(name, cfg, B, num_steps=5, order=2):
    net = MG.build_ref(cfg).eval()
    g = torch.Generator().manual_seed(98)
    latents = torch.randn(B, cfg.img_channels, cfg.img_resolution, cfg.img_resolution, generator=g)
    levels = 1.0 - np.arange(num_steps + 1, dtype=np.float64) / num_steps
    alpha, sigma = DPM.flow_alpha_sigma(levels)

    def D(x, i):
        t = torch.full((B,), sigma[i], dtype=torch.float32)
        v = net.model(torch.from_numpy(x).float(), t, None)["x"].double().numpy()
        return x - sigma[i] * v

    with torch.no_grad():
        z = DPM.dpm_solver(D, latents.double().numpy(), alpha, sigma, order)
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), latents=latents.numpy(), z=z, levels=levels,
                        num_steps=np.int64(num_steps), order=np.int64(order))
    print(name, "|z|", np.abs(z).mean())


if __name__ == "__main__":
    edm_case("dpm_s2_sampler", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10), B=2)
    flow_case("dpm_nd_s2_flow", O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=0, use_decoder=False), B=2)
