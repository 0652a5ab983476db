"""Golden vectors of the decoder-less DiT (use_decoder=False, models/maskdit.py:254) from the UNMODIFIED reference.

Run in the dev container only (the GPU box has no /root/reference):  python tests/golden/make_golden_nodecoder.py
Reuses make_golden.py's `train_case` / `eval_case` (same weights from oracle.maskdit_oracle.make_state_dict, same
recorded random draws) with `use_decoder=False`; writes tests/golden/nd_*.npz.  `nd_xl2_bf16.npz` holds the
reference's XL/2 outputs under CPU bf16 autocast: the bf16-operand yardstick the GPU bounds are derived from.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (installs the timm stand-in and imports the reference)
from make_golden import O  # noqa: E402


def nd(model_type, R, ncls):
    return O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls, use_decoder=False)


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def bf16_case(name, cfg, train_gold, eval_gold):
    """The XL/2 forwards of `train_gold` (masked training) and `eval_gold` (plain eval, CFG) again under CPU bf16
    autocast, with their rel-L2 distance from the fp32 outputs."""
    g, e = np.load(os.path.join(HERE, train_gold + ".npz")), np.load(os.path.join(HERE, eval_gold + ".npz"))
    t = lambda k, src: torch.from_numpy(np.asarray(src[k]))   # noqa: E731
    net = MG.build_ref(cfg).train()
    sigma = (t("rnd_normal", g) * 1.2 - 1.2).exp()
    md = O.mask_from_noise(t("mask_noise", g), float(g["mask_ratio"]))
    out = {}
    with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16):
        D = net(t("images", g) + t("noise_unit", g) * sigma, sigma, t("labels", g), mask_ratio=float(g["mask_ratio"]),
                mask_dict=md)["x"].float()
        net.eval()
        plain = net(t("images", e), t("sigma", e), t("labels", e))["x"].float()
        cfgout = net(t("images", e), torch.tensor(1.7, dtype=torch.float64), t("labels", e), 1.5)["x"].float()
    for k, v, ref in (("D_train", D, t("D", g)), ("D_plain", plain, t("D_plain", e)), ("D_cfg", cfgout, t("D_cfg", e))):
        out[k] = v.numpy()
        out[f"bf16_rel_{k}"] = np.float64(rel(v, ref))
        print(name, k, "bf16-autocast rel-L2", out[f"bf16_rel_{k}"])
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **out)


if __name__ == "__main__":
    small = nd("DiT-S/2", 8, 10)
    MG.train_case("nd_s2_train_mask", small, B=2, mask_ratio=0.5, with_grads=True)
    MG.train_case("nd_s2_train_nomask", small, B=2, mask_ratio=0.0, with_grads=True)
    # class-unconditional, 30 % masking: T = int(256 * 0.7) = 179 kept tokens (ragged scatter / gather, mma.sync)
    MG.train_case("nd_s2_uncond_mask30", nd("DiT-S/2", 32, 0), B=3, mask_ratio=0.3, with_grads=True)
    xl = nd("DiT-XL/2", 32, 1000)
    MG.train_case("nd_xl2_grads", xl, B=2, mask_ratio=0.5, with_grads=True)    # T = 128
    MG.eval_case("nd_xl2_eval", xl, B=2, num_steps=3)                           # T = 256, 3-step CFG sampler
    bf16_case("nd_xl2_bf16", xl, "nd_xl2_grads", "nd_xl2_eval")
