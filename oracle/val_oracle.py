"""CPU fp32 restatement of the held-out denoising loss (maskdit_b200/validate.py), written independently of it: one
item at a time, its draws from the item's own generator, the reference's step front and EDM loss (maskdit_oracle), and
the per-level sums in float64 in index order.  tests/golden/make_golden_val.py pins it to the unmodified reference."""
import math
from statistics import NormalDist

import numpy as np
import torch

from oracle import maskdit_oracle as O


def level_normals(levels):
    """Phi^-1((k + 1/2) / K) in float64."""
    return [NormalDist().inv_cdf((k + 0.5) / levels) for k in range(levels)]


def item_draws(seed, index, channels, resolution, levels):
    """eps [C, R, R] then noise [K, C, R, R]: float32 standard normals of numpy's default generator (PCG64) seeded
    with the entropy [seed, index]."""
    g = np.random.Generator(np.random.PCG64(np.random.SeedSequence([seed, index])))
    eps = torch.tensor(g.standard_normal((channels, resolution, resolution), dtype=np.float32))
    return eps, torch.tensor(g.standard_normal((levels, channels, resolution, resolution), dtype=np.float32))


def item_losses(sd, cfg: O.Cfg, moments, labels, eps, noise, z, P_mean=-1.2, P_std=1.2, scale_factor=0.18215):
    """Losses [K] of one item: moments [2C, R, R], labels [nc] or None, z [K] float32 (rnd_normal of each level)."""
    K = z.shape[0]
    y, _, _, _ = O.step_front(moments[None], eps[None], z[:1], noise[:1], scale_factor=scale_factor)
    lab = None if labels is None else labels[None].expand(K, -1)
    loss, _ = O.edm_loss(sd, cfg, y.expand(K, -1, -1, -1), lab, z.reshape(K, 1, 1, 1), noise, None, 0.0,
                         P_mean=P_mean, P_std=P_std)
    return loss


class RowScorer:
    """The per-row loss on CPU for maskdit_b200.validate's batched driver: (moments, eps, rnd_normal, noise, labels)
    of B rows -> losses [B]."""

    def __init__(self, sd, cfg: O.Cfg):
        self.sd, self.cfg = sd, cfg

    def __call__(self, moments, eps, rnd_normal, noise, labels):
        with torch.no_grad():
            y, _, _, _ = O.step_front(moments, eps, rnd_normal, noise)
            loss, _ = O.edm_loss(self.sd, self.cfg, y, labels, rnd_normal.reshape(-1, 1, 1, 1), noise, None, 0.0)
        return loss


def estimate(sd, cfg: O.Cfg, moments, labels, levels=8, seed=0, draws=None):
    """-> (per_item float32 [N, K], per_level float64 [K], mean).  `draws(i)` -> (eps, noise) replaces the generator
    (golden tests inject the reference's)."""
    N, C2, R, _ = moments.shape
    z = torch.tensor(level_normals(levels), dtype=torch.float32)
    rows = []
    with torch.no_grad():
        for i in range(N):
            eps, noise = draws(i) if draws is not None else item_draws(seed, i, C2 // 2, R, levels)
            rows.append(item_losses(sd, cfg, moments[i], None if labels is None else labels[i], eps, noise, z))
    per_item = torch.stack(rows)
    acc = [0.0] * levels
    for row in per_item.double().tolist():            # float64, item by item in index order
        acc = [a + v for a, v in zip(acc, row)]
    per_level = np.array(acc) / N
    return per_item, per_level, float(math.fsum(per_level) / levels)
