"""Golden vectors of the held-out denoising loss (maskdit_b200/validate.py) from the UNMODIFIED reference on CPU fp32.

Run in the dev container only (the GPU box has no /root/reference):  python tests/golden/make_golden_val.py
Writes tests/golden/val_s2.npz.  The reference's own `utils.sample`, `EDMPrecond` (eval mode) and `EDMLoss` run on a
batch of (item, level) rows; their random draws (randn_like in utils.sample, randn [B,1,1,1] and randn_like in
EDMLoss.__call__, train_utils/loss.py:35,39) are injected with the held-out set's fixed draws: each item's generator
seeded by (seed, item) (validate.item_draws: numpy PCG64), the levels' rnd_normal = Phi^-1((k + 1/2) / K).
Weights are not stored: oracle.maskdit_oracle.make_state_dict(cfg, 1) is deterministic on CPU.
"""
import contextlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from maskdit_b200 import validate as V  # noqa: E402
from oracle import maskdit_oracle as O  # noqa: E402
from oracle import timm_standin  # noqa: E402

timm_standin.install()
sys.path.insert(0, "/root/reference")
import train_utils.loss as rl  # noqa: E402
import utils as ru  # noqa: E402

from make_golden import Wrap, build_ref  # noqa: E402

N, K, SEED = 5, 8, 3


@contextlib.contextmanager
def injected(randn=None, randn_like=None):
    """torch.randn / torch.randn_like return the given tensors (checked against the requested shapes)."""
    orig_randn, orig_like = torch.randn, torch.randn_like

    def fake_randn(*shape, **kw):
        shape = tuple(shape[0]) if len(shape) == 1 and isinstance(shape[0], (list, tuple)) else tuple(shape)
        assert randn is not None and tuple(randn.shape) == shape, shape
        return randn.clone()

    def fake_like(x, **kw):
        assert randn_like is not None and randn_like.shape == x.shape, x.shape
        return randn_like.clone()

    torch.randn, torch.randn_like = fake_randn, fake_like
    try:
        yield
    finally:
        torch.randn, torch.randn_like = orig_randn, orig_like


def main():
    cfg = O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=10)
    C, R = cfg.img_channels, cfg.img_resolution
    g = torch.Generator().manual_seed(41)
    moments = torch.cat([torch.randn(N, C, R, R, generator=g), torch.randn(N, C, R, R, generator=g) * 2 - 3], 1)
    moments[0, C:] = -40.0         # a logvar below utils.sample's clamp (-30)
    labels = torch.eye(cfg.num_classes)[torch.randint(0, cfg.num_classes, (N,), generator=g)]
    draws = [V.item_draws(SEED, i, C, R, K) for i in range(N)]
    eps = torch.stack([d[0] for d in draws])
    noise = torch.stack([d[1] for d in draws])                          # [N, K, C, R, R]
    z = torch.tensor(V.level_normals(K), dtype=torch.float32)
    # rows in (item, level) order, item-major
    mom_rows = moments.repeat_interleave(K, 0)
    lab_rows = labels.repeat_interleave(K, 0)
    eps_rows = eps.repeat_interleave(K, 0)
    with torch.no_grad():
        with injected(randn_like=eps_rows):
            y = ru.sample(mom_rows)                                     # utils.py:59-65
        net = build_ref(cfg).eval()
        with injected(randn=z.repeat(N).reshape(N * K, 1, 1, 1), randn_like=noise.reshape(N * K, C, R, R)):
            loss = rl.Losses["edm"]()(net=Wrap(net), images=y, labels=lab_rows)   # mask_ratio 0: mean_flat
    per_item = loss.reshape(N, K)
    np.savez_compressed(os.path.join(HERE, "val_s2.npz"), moments=moments.numpy(), labels=labels.numpy(),
                        eps=eps.numpy(), noise=noise.numpy(), z=z.numpy(), seed=np.int64(SEED),
                        per_item=per_item.numpy(), y=y.reshape(N, K, C, R, R)[:, 0].numpy())
    print("val_s2 per-level", per_item.double().mean(0).numpy(), "mean", per_item.double().mean().item())


if __name__ == "__main__":
    main()
