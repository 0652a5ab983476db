"""Golden vectors of the DiT_models geometries the other goldens do not reach, from the UNMODIFIED reference.

Run in the dev container only (the GPU box has no /root/reference):  python tests/golden/make_golden_geometry.py
Reuses make_golden.py's `train_case` / `eval_case` (weights from oracle.maskdit_oracle.make_state_dict, recorded
random draws); writes tests/golden/geo_*.npz and touches no other golden.

  geo_s8_mask50            DiT-S/8 MaskDiT, mask 0.5   pd 256 masked loss + MAE, patch-embed backward at cpp 256,
                                                       T = 8 encoder / 16 decoder tokens
  geo_s8_eval              DiT-S/8 MaskDiT             eval, CFG and a 3-step CFG sampler at patch 8
  geo_b8_nd_nomask         DiT-B/8 decoder-less        unmasked loss at pd 256, final layer N = 256 on D = 768
  geo_l4_nd_uncond_mask30  DiT-L/4 decoder-less, no classes, mask 0.3
                                                       D = 1024, T = 44 (ragged), kept-row scatter / gather at pd 64
  geo_h2_mask50            DiT-H/2 MaskDiT, mask 0.5   head_dim 80 encoder attention at T = 128, D = 1280, decoder
                                                       at T = 256
  geo_h2_bf16              the geo_h2_mask50 forward under CPU bf16 autocast: the precision yardstick of the 32-block
                           DiT-H encoder
"""
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (installs the timm stand-in and imports the reference)
from make_golden import O  # noqa: E402


def savez_fixed(path, **arrays):
    """np.savez_compressed with a fixed member timestamp, so a rerun writes the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k, v in arrays.items():
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            with zf.open(info, "w", force_zip64=True) as f:
                np.lib.format.write_array(f, np.asanyarray(v), allow_pickle=False)


np.savez_compressed = savez_fixed   # make_golden's cases write through this name


def cfg(model_type, R, ncls, use_decoder=True):
    return O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls, use_decoder=use_decoder)


def bf16_train_case(name, c, train_gold):
    """The masked training forward of `train_gold` again under CPU bf16 autocast, with its rel-L2 distance from the
    fp32 output."""
    g = np.load(os.path.join(HERE, train_gold + ".npz"))
    t = lambda k: torch.from_numpy(np.asarray(g[k]))   # noqa: E731
    net = MG.build_ref(c).train()
    sigma = (t("rnd_normal") * 1.2 - 1.2).exp()
    mr = float(g["mask_ratio"])
    md = O.mask_from_noise(t("mask_noise"), mr)
    with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16):
        D = net(t("images") + t("noise_unit") * sigma, sigma, t("labels"), mask_ratio=mr, mask_dict=md)["x"].float()
    ref = t("D")
    r = ((D.double() - ref.double()).norm() / ref.double().norm()).item()
    print(name, "D_train bf16-autocast rel-L2", r)
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), D_train=D.numpy(), bf16_rel_D_train=np.float64(r))


if __name__ == "__main__":
    s8 = cfg("DiT-S/8", 32, 10)
    MG.train_case("geo_s8_mask50", s8, B=3, mask_ratio=0.5, with_grads=True)
    MG.eval_case("geo_s8_eval", s8, B=2, num_steps=3)
    MG.train_case("geo_b8_nd_nomask", cfg("DiT-B/8", 32, 10, use_decoder=False), B=2, mask_ratio=0.0,
                  with_grads=True)
    MG.train_case("geo_l4_nd_uncond_mask30", cfg("DiT-L/4", 32, 0, use_decoder=False), B=2, mask_ratio=0.3,
                  with_grads=True)
    h2 = cfg("DiT-H/2", 32, 1000)
    MG.train_case("geo_h2_mask50", h2, B=2, mask_ratio=0.5, with_grads=True)
    bf16_train_case("geo_h2_bf16", h2, "geo_h2_mask50")
