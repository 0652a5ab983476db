"""EDM training loss (reference: train_utils/loss.py) on the H100 engine.

`Losses['edm']` has the reference's constructor and call signature.  When `net` is a `maskdit_b200.EDMPrecond`
(bare, or wrapped in anything exposing `.module` like DDP / `DataParallelB200`), the loss runs fused:
noise injection -> engine forward -> ONE kernel for unpatchify + EDM output scaling + weighted-SE / per-patch
means / masked means / MAE term, whose backward seeds the hand-written network backward.  The random draws are
made with torch's generator in the reference's order (loss.py:35 randn[B,1,1,1]; loss.py:39 randn_like; then
maskdit.py:102 rand[B,L]) so a seeded run consumes the same RNG stream positions as the reference.
"""
from __future__ import annotations

import torch

from . import ops
from .maskdit import EDMPrecond


def _unwrap(net):
    """unwrap_model (train_utils/helper.py:61-68) generalised to any wrapper exposing .module / ._orig_mod."""
    seen = 0
    while not isinstance(net, EDMPrecond) and seen < 4:
        if hasattr(net, "_orig_mod"):
            net = net._orig_mod
        elif hasattr(net, "module"):
            net = net.module
        else:
            break
        seen += 1
    return net


class _FusedLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, net, yn, y, sigma, labels, mask_dict, mae_coef):
        Fo, saved = net._engine.forward(yn, sigma, labels, mask_dict, save=True)
        mask = mask_dict["mask"] if mask_dict is not None else None
        p = net.model.patch_size
        loss, _, _ = ops.edm_loss(Fo, yn, y, sigma, mask, None, net.sigma_data, mae_coef, p, want_D=False,
                                  want_dF=False)
        ctx.net, ctx.saved = net, saved
        ctx.args = (Fo, yn, y, sigma, mask, mae_coef, p)
        return loss

    @staticmethod
    def backward(ctx, gl):
        net = ctx.net
        Fo, yn, y, sigma, mask, mae_coef, p = ctx.args
        _, _, dF = ops.edm_loss(Fo, yn, y, sigma, mask, gl.contiguous().float(), net.sigma_data, mae_coef, p,
                                want_D=False, want_dF=True)
        net._run_backward(ctx.saved, dF.view(-1, dF.shape[-1]))
        ctx.saved = ctx.args = None
        return (torch.zeros(1, device=gl.device),) + (None,) * 7


class EDMLoss:
    """train_utils/loss.py:22-60."""

    def __init__(self, P_mean=-1.2, P_std=1.2, sigma_data=0.5):
        self.P_mean, self.P_std, self.sigma_data = P_mean, P_std, sigma_data

    # RNG hooks (tests replace them to inject the golden draws)
    def _randn(self, shape, device):
        return torch.randn(shape, device=device)

    def _rand(self, shape, device):
        return torch.rand(shape, device=device)

    def __call__(self, net, images, labels=None, mask_ratio=0, mae_loss_coef=0, feat=None, augment_pipe=None):
        if feat is not None or augment_pipe is not None:
            raise NotImplementedError("feat / augment_pipe are not part of the MaskDiT latent training path")
        raw = self._net(net, images.device)
        B = images.shape[0]
        y = images.contiguous().float()
        rnd_normal = self._randn([B, 1, 1, 1], images.device)            # loss.py:35
        sigma4 = (rnd_normal * self.P_std + self.P_mean).exp()            # loss.py:36
        yn = (y + self._randn(tuple(y.shape), images.device) * sigma4).contiguous()  # loss.py:39,41
        return self._finish(raw, y, yn, sigma4.reshape(B).contiguous(), labels, mask_ratio, mae_loss_coef)

    def from_moments(self, net, moments, labels=None, mask_ratio=0, mae_loss_coef=0, class_dropout_prob=0.0,
                     scale_factor=0.18215, eps=None, drop_u=None):
        """The whole step front of the reference's training loop in one kernel (`ops.step_front`): `x = sample(x)`
        (train.py:206, utils.py:59-65) -> label dropout (train.py:209) -> sigma draw + noise injection (loss.py:35-39),
        then the same fused loss as `__call__`.  Random draws are made here in the reference's order: randn_like(mean),
        rand[B,1] (only when class_dropout_prob > 0), randn[B,1,1,1], randn_like(images), then rand[B,L] for the mask.
        `labels` is modified in place (dropped rows zeroed), as `y = y * (...)` rebinds it in the reference.
        `eps` / `drop_u`: pre-drawn slices (gradient accumulation draws them once for the whole per-GPU batch before
        the micro-batch rounds, train.py:206-209, so `TrainStep.step` passes them in)."""
        dev = moments.device
        raw = self._net(net, dev)
        B, C2, R, _ = moments.shape
        moments = moments.contiguous().float()
        if eps is None:
            eps = self._randn((B, C2 // 2, R, R), dev)
        if class_dropout_prob > 0 and labels is not None:
            if drop_u is None:
                drop_u = self._rand((B, 1), dev).reshape(B)
            drop_u = drop_u.contiguous()
            if labels.dtype != torch.float32 or not labels.is_contiguous():
                labels = labels.contiguous().float()
        else:
            drop_u = None
        rnd_normal = self._randn([B, 1, 1, 1], dev).reshape(B).contiguous()
        noise = self._randn((B, C2 // 2, R, R), dev)
        y, yn, sigma = ops.step_front(moments, eps, rnd_normal, noise, labels, drop_u, float(class_dropout_prob),
                                      scale_factor, self.P_mean, self.P_std)
        return self._finish(raw, y, yn, sigma, labels, mask_ratio, mae_loss_coef)

    def _net(self, net, dev):
        raw = _unwrap(net)
        if not isinstance(raw, EDMPrecond):
            raise TypeError("maskdit_b200.Losses['edm'] drives a maskdit_b200.EDMPrecond network")
        raw._ready(dev)
        return raw

    def _finish(self, raw, y, yn, sigma, labels, mask_ratio, mae_loss_coef):
        dev, B = y.device, y.shape[0]
        _, _, lab = raw._norm_inputs(y, sigma, labels)
        md = None
        if mask_ratio > 0:
            assert raw.training, "masked loss needs net.train() (loss.py:46)"
            L = raw.model.num_patches
            md = ops.mask_indices(self._rand((B, L), dev), int(L * (1 - mask_ratio)))  # maskdit.py:101-104
        coef = float(mae_loss_coef) if (mask_ratio > 0 and mae_loss_coef > 0) else 0.0
        if torch.is_grad_enabled():
            loss = _FusedLossFn.apply(raw._anchor, raw, yn, y, sigma, lab, md, coef)
        else:
            Fo, _ = raw._engine.forward(yn, sigma, lab, md, save=False)
            loss, _, _ = ops.edm_loss(Fo, yn, y, sigma, md["mask"] if md else None, None, raw.sigma_data, coef,
                                      raw.model.patch_size, want_dF=False)
        self.last_mask_dict = md
        return loss


Losses = {"edm": EDMLoss}
