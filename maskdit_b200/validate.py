"""Held-out denoising loss: a fixed estimate of the EDM training objective of the network the sampler runs.

The training loss cannot be compared across a run: it is a one-batch estimate over random sigma draws, and it depends
on the mask ratio, which a schedule such as the fine-tune's `cos4` changes every step.  This module scores a network on
a fixed held-out set instead, with every draw fixed, so two checkpoints, two EMA widths or two runs scored with the same
settings can be compared directly.  It is a proxy for sample quality, not FID.

For item i of the held-out set (the first N items of a latent split, in index order) and level k of K:
  * the latent is `y_i = 0.18215 * (mean + exp(0.5 * clamp(logvar, -30, 20)) * eps_i)` (utils.sample);
  * `sigma_k = exp(P_mean + P_std * z_k)` with `z_k = Phi^-1((k + 1/2) / K)`: stratified quantiles of the training
    sigma distribution (P_mean -1.2, P_std 1.2), so the mean over levels estimates the objective's mean over sigma;
  * the loss is `mean(lambda(sigma_k) * (D(y_i + sigma_k * n_ik) - y_i)^2)`, `lambda = (s^2 + sd^2) / (s * sd)^2`: the
    unmasked EDM loss of the eval-mode network (every token kept) with the item's class label.
`eps_i` and `n_ik` come from a CPU generator (numpy's PCG64) seeded by (seed, i) alone, never from torch's global
RNG.  So the numbers do not depend on the batch size, the rank count or how often validation ran, and validating
leaves a training run's random stream untouched.

One network evaluation is one batch row (item, level).  On the GPU a row runs through the training path's own kernels:
`mdt_step_front` (sigma_k enters as `rnd_normal = z_k`), the eval forward `mdt_forward` and `mdt_edm_loss` without a
mask.  Under torch.distributed each rank scores a contiguous slice of the items and one all_gather puts the per-item
losses back in index order, so every rank returns the same numbers.  The per-level means are float64 sums over the
items in index order.
"""
from __future__ import annotations

import os
from statistics import NormalDist

import numpy as np
import torch

P_MEAN, P_STD = -1.2, 1.2
SCALE_FACTOR = 0.18215


# ---- the fixed draws -------------------------------------------------------------------------------------------------
def level_normals(levels, dtype=np.float64):
    """z_k = Phi^-1((k + 1/2) / K), k = 0 .. K-1: the standard-normal quantiles at the centres of K equal strata."""
    if levels < 1:
        raise ValueError(f"levels must be at least 1, got {levels}")
    return np.array([NormalDist().inv_cdf((k + 0.5) / levels) for k in range(levels)], dtype=dtype)


def sigma_levels(levels, P_mean=P_MEAN, P_std=P_STD):
    """sigma_k = exp(P_mean + P_std * z_k) in float64: quantiles of the training lognormal (K = 1: its median)."""
    return np.exp(P_mean + P_std * level_normals(levels))


def item_draws(seed, index, channels, resolution, levels):
    """(eps [C, R, R], noise [K, C, R, R]) float32 on the CPU for item `index`: eps first, then the K noise fields,
    from numpy's PCG64 seeded with the entropy (seed, index).  (torch's CPU generator keeps only 32 bits of its seed, so
    it cannot give every (seed, index) pair a stream of its own.)"""
    if int(seed) < 0 or int(index) < 0:
        raise ValueError(f"seed {seed} and item {index} must be non-negative")
    g = np.random.default_rng([int(seed), int(index)])
    eps = g.standard_normal((channels, resolution, resolution), dtype=np.float32)
    noise = g.standard_normal((levels, channels, resolution, resolution), dtype=np.float32)
    return torch.from_numpy(eps), torch.from_numpy(noise)


# ---- the held-out set ------------------------------------------------------------------------------------------------
class HeldOut:
    """N VAE moments [N, 2C, R, R] and one-hot labels [N, num_classes] (None for a class-unconditional net), float32 on
    the CPU, in index order."""

    def __init__(self, moments, labels=None):
        self.moments = moments.float().contiguous()
        self.labels = None if labels is None else labels.float().contiguous()
        if self.labels is not None and self.labels.shape[0] != self.moments.shape[0]:
            raise ValueError(f"{self.moments.shape[0]} moments but {self.labels.shape[0]} labels")

    def __len__(self):
        return self.moments.shape[0]

    @classmethod
    def from_lmdb(cls, root, count, resolution=32, num_channels=4, num_classes=1000, split="val"):
        """The first `count` items of the latent LMDB `<root>/<split>` (the layout extract_latent.py writes).  With
        num_classes = 0 (a class-unconditional net) the stored class indices are not read and labels is None."""
        from .data import ImageNetLatentDataset
        ds = ImageNetLatentDataset(root, resolution=resolution, num_channels=num_channels, split=split,
                                   num_classes=max(num_classes, 1))
        if count > len(ds):
            raise ValueError(f"{count} validation items requested, {os.path.join(root, split)} holds {len(ds)}")
        if not num_classes:
            return cls(torch.from_numpy(np.stack([ds.raw(i)[0] for i in range(count)])))
        zs, ys = zip(*(ds[i] for i in range(count)))
        return cls(torch.from_numpy(np.stack(zs)), torch.from_numpy(np.stack(ys)))

    @classmethod
    def synthetic(cls, count, resolution=32, num_channels=4, num_classes=1000, seed=0):
        """`count` moments and labels drawn from a fixed seed (for runs without a dataset).  Item i's moments and label
        come from a generator of its own (numpy's PCG64 with the entropy (seed, i, 1), apart from the noise draws of
        `item_draws`), so the set of N items is the first N items of any larger one."""
        zs, ys = [], []
        for i in range(count):
            g = np.random.default_rng([int(seed), i, 1])
            zs.append(g.standard_normal((2 * num_channels, resolution, resolution), dtype=np.float32))
            ys.append(int(g.integers(num_classes)) if num_classes else 0)
        moments = torch.from_numpy(np.stack(zs)) if zs else torch.zeros(0, 2 * num_channels, resolution, resolution)
        labels = None
        if num_classes:
            labels = torch.nn.functional.one_hot(torch.tensor(ys, dtype=torch.int64), num_classes).float()
        return cls(moments, labels)


# ---- scoring ---------------------------------------------------------------------------------------------------------
class CudaScorer:
    """Per-row losses of a `maskdit_b200.EDMPrecond` in eval mode on its device: step front, eval forward, EDM loss."""

    def __init__(self, net, P_mean=P_MEAN, P_std=P_STD, scale_factor=SCALE_FACTOR):
        from .loss import _unwrap
        from .maskdit import EDMPrecond
        raw = _unwrap(net)
        if not isinstance(raw, EDMPrecond):
            raise TypeError("CudaScorer scores a maskdit_b200.EDMPrecond network")
        if raw.training:
            raise ValueError("the held-out loss is that of the eval-mode network: call net.eval() first")
        self.net = raw
        self.device = next(raw.parameters()).device
        if self.device.type != "cuda":
            raise ValueError("CudaScorer needs the network on a CUDA device")
        self.P_mean, self.P_std, self.scale_factor = P_mean, P_std, scale_factor

    def __call__(self, moments, eps, rnd_normal, noise, labels):
        from . import ops
        net, dev = self.net, self.device
        net._ready(dev)                                   # the bf16 weight shadow follows the fp32 weights
        to = lambda t: None if t is None else t.to(dev, non_blocking=True).contiguous()  # noqa: E731
        with torch.no_grad():
            y, yn, sigma = ops.step_front(to(moments), to(eps), to(rnd_normal), to(noise), None, None, 0.0,
                                          self.scale_factor, self.P_mean, self.P_std)
            _, _, lab = net._norm_inputs(y, sigma, to(labels))
            Fo, _ = net._engine.forward(yn, sigma, lab, None, save=False)
            loss, _, _ = ops.edm_loss(Fo, yn, y, sigma, None, None, net.sigma_data, 0.0, net.model.patch_size,
                                      want_dF=False)
        return loss


def rank_slice(count, rank, world):
    """[lo, hi): the contiguous slice of the items that `rank` of `world` scores (ceil(N / world) per rank)."""
    per = -(-count // world)
    lo = min(rank * per, count)
    return lo, min(lo + per, count)


def score_items(scorer, held, lo, hi, levels=8, seed=0, batch=64):
    """Per-item losses [hi - lo, K] (float32, CPU) of items lo .. hi-1.  The (item, level) rows are taken in index
    order, item-major, `batch` rows per scorer call; the last call takes the remainder."""
    if batch < 1:
        raise ValueError(f"batch must be at least 1, got {batch}")
    n = hi - lo
    if n <= 0:
        return torch.zeros(0, levels)
    _, C2, R, _ = held.moments.shape
    z = torch.from_numpy(level_normals(levels, np.float32))
    out = []
    draws = {}
    for r0 in range(0, n * levels, batch):
        rows = range(r0, min(r0 + batch, n * levels))
        items = [lo + r // levels for r in rows]
        ks = torch.tensor([r % levels for r in rows])
        for i in dict.fromkeys(items):
            if i not in draws:
                draws[i] = item_draws(seed, i, C2 // 2, R, levels)
        idx = torch.tensor(items)
        eps = torch.stack([draws[i][0] for i in items])
        noise = torch.stack([draws[i][1][k] for i, k in zip(items, ks.tolist())])
        labels = held.labels[idx] if held.labels is not None else None
        out.append(scorer(held.moments[idx], eps, z[ks], noise, labels).float().cpu())
        for i in [i for i in draws if i < items[-1]]:     # an item whose rows are all scored
            del draws[i]
    return torch.cat(out).reshape(n, levels)


def gather_items(local, count, group=None):
    """Concatenate every rank's `rank_slice` of the per-item losses in rank order -> [count, K] on every rank (one
    all_gather of equal-sized, padded slices on the device of the process group's backend)."""
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    per, K = -(-count // world), local.shape[1]
    nccl = dist.get_backend(group) == "nccl"
    dev = torch.device("cuda", torch.cuda.current_device()) if nccl else torch.device("cpu")
    buf = torch.zeros(per, K, dtype=torch.float32, device=dev)
    lo, hi = rank_slice(count, rank, world)
    if local.shape[0] != hi - lo:
        raise ValueError(f"rank {rank} holds {local.shape[0]} items, its slice is {hi - lo}")
    buf[:hi - lo] = local.to(dev)
    parts = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(parts, buf, group=group)
    return torch.cat([p[:rank_slice(count, r, world)[1] - rank_slice(count, r, world)[0]].cpu()
                      for r, p in enumerate(parts)])


def summarize(per_item, P_mean=P_MEAN, P_std=P_STD):
    """{sigma, per_level, mean, count, levels} of per-item losses [N, K]: per-level means of float64 sums taken
    item by item in index order, and their mean over the levels."""
    a = per_item.double().numpy()
    N, K = a.shape
    if N == 0:
        raise ValueError("no items to summarize")
    per_level = np.cumsum(a, axis=0)[-1] / N             # sequential, in index order
    return {"sigma": sigma_levels(K, P_mean, P_std).tolist(), "per_level": per_level.tolist(),
            "mean": float(per_level.mean()), "count": N, "levels": K}


def validate(net_or_scorer, held, levels=8, seed=0, batch=64, group=None):
    """Score the first len(held) items at K = `levels` noise levels.  `net_or_scorer`: an eval-mode EDMPrecond on a
    CUDA device, or any callable (moments, eps, rnd_normal, noise, labels) -> per-row losses.  Under an initialised
    torch.distributed process group (or `group`) each rank scores its slice and every rank returns the whole result.
    Returns `summarize(...)` plus `per_item` [N, K] (float32)."""
    import torch.distributed as dist
    scorer = net_or_scorer if not hasattr(net_or_scorer, "parameters") else CudaScorer(net_or_scorer)
    count = len(held)
    if count < 1:
        raise ValueError("the held-out set is empty")
    distributed = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
    if distributed:
        lo, hi = rank_slice(count, dist.get_rank(group), dist.get_world_size(group))
        per_item = gather_items(score_items(scorer, held, lo, hi, levels, seed, batch), count, group)
    else:
        per_item = score_items(scorer, held, 0, count, levels, seed, batch)
    res = summarize(per_item)
    res["per_item"] = per_item
    return res


def format_levels(res):
    """'<mean> [<L_0> ... <L_{K-1}>]'."""
    return f"{res['mean']:.5f} [" + " ".join(f"{v:.5f}" for v in res["per_level"]) + "]"
