"""EDM training loss (reference: train_utils/loss.py) on the H100 engine, the rectified-flow loss (`FlowLoss`) and
Easy Consistency Tuning of an EDM network (`ECTLoss`).

`Losses['edm']` has the reference's constructor and call signature.  When `net` is a `maskdit_b200.EDMPrecond`
(bare, or wrapped in anything exposing `.module` like DDP / `DataParallelB200`), the loss runs fused:
noise injection -> engine forward -> ONE kernel for unpatchify + EDM output scaling + weighted-SE / per-patch
means / masked means / MAE term, whose backward seeds the hand-written network backward.  A network with a learned loss
weighting (`EDMPrecond(logvar_channels=C)`) returns the per-sample objective exp(-u) E + u + mae_coef M when gradients
are enabled; `last_edm_loss` always holds the reference's per-sample loss E + mae_coef M of the last call (without a
gradient, and without a weighting, the returned loss itself).  The random draws are
made with torch's generator in the reference's order (loss.py:35 randn[B,1,1,1]; loss.py:39 randn_like; then
maskdit.py:102 rand[B,L]) so a seeded run consumes the same RNG stream positions as the reference.
"""
from __future__ import annotations

import math

import torch

from . import ops
from .maskdit import EDMPrecond, FlowPrecond


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


class _FusedLogvarLossFn(torch.autograd.Function):
    """`_FusedLossFn` with the learned loss weighting: returns (objective, reference loss); the reference loss carries
    no gradient.  The backward seeds the network with exp(-u)-scaled EDM gradients and adds w's gradient to the flat
    buffer after the network backward."""

    @staticmethod
    def forward(ctx, anchor, net, yn, y, sigma, labels, mask_dict, mae_coef):
        Fo, saved = net._engine.forward(yn, sigma, labels, mask_dict, save=True)
        mask = mask_dict["mask"] if mask_dict is not None else None
        p = net.model.patch_size
        obj, loss, _, _, _ = ops.edm_loss_logvar(Fo, yn, y, sigma, mask, None, net.sigma_data, mae_coef, p,
                                                 *net._logvar_tensors(), want_dF=False)
        ctx.net, ctx.saved = net, saved
        ctx.args = (Fo, yn, y, sigma, mask, mae_coef, p)
        ctx.mark_non_differentiable(loss)
        return obj, loss

    @staticmethod
    def backward(ctx, gl, _):
        net = ctx.net
        Fo, yn, y, sigma, mask, mae_coef, p = ctx.args
        freqs, phases, w = net._logvar_tensors()
        _, _, _, du, dF = ops.edm_loss_logvar(Fo, yn, y, sigma, mask, gl.contiguous().float(), net.sigma_data,
                                              mae_coef, p, freqs, phases, w, want_dF=True)
        net._run_backward(ctx.saved, dF.view(-1, dF.shape[-1]))   # also (re)attaches a zeroed gradient buffer
        ops.logvar_wgrad(sigma, freqs, phases, du, net._store.gview("logvar_linear.weight").view(-1))
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
        if not isinstance(raw, EDMPrecond) or isinstance(raw, FlowPrecond):
            raise TypeError("maskdit_b200.Losses['edm'] drives a maskdit_b200.EDMPrecond network"
                            + (" (this one is a FlowPrecond: use Losses['flow'])" if isinstance(raw, FlowPrecond)
                               else ""))
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
        if torch.is_grad_enabled() and raw.logvar_channels:
            # learned weighting: the objective is what the gradient follows, the reference loss is kept for logging
            loss, self.last_edm_loss = _FusedLogvarLossFn.apply(raw._anchor, raw, yn, y, sigma, lab, md, coef)
            self.last_mask_dict = md
            return loss
        if torch.is_grad_enabled():
            loss = _FusedLossFn.apply(raw._anchor, raw, yn, y, sigma, lab, md, coef)
        else:
            Fo, _ = raw._engine.forward(yn, sigma, lab, md, save=False)
            loss, _, _ = ops.edm_loss(Fo, yn, y, sigma, md["mask"] if md else None, None, raw.sigma_data, coef,
                                      raw.model.patch_size, want_dF=False)
        self.last_mask_dict = md
        self.last_edm_loss = loss
        return loss


class _FusedFlowLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, net, xt, y, eps, t, labels, mask_dict, mae_coef):
        Fo, saved = net._engine.forward(xt, t, labels, mask_dict, save=True)
        mask = mask_dict["mask"] if mask_dict is not None else None
        p = net.model.patch_size
        loss, _, _ = ops.flow_loss(Fo, xt, y, eps, t, mask, None, mae_coef, p, want_dF=False)
        ctx.net, ctx.saved = net, saved
        ctx.args = (Fo, xt, y, eps, t, mask, mae_coef, p)
        return loss

    @staticmethod
    def backward(ctx, gl):
        net = ctx.net
        Fo, xt, y, eps, t, mask, mae_coef, p = ctx.args
        _, _, dF = ops.flow_loss(Fo, xt, y, eps, t, mask, gl.contiguous().float(), mae_coef, p, want_dF=True)
        net._run_backward(ctx.saved, dF.view(-1, dF.shape[-1]))
        ctx.saved = ctx.args = None
        return (torch.zeros(1, device=gl.device),) + (None,) * 8


class FlowLoss:
    """Rectified-flow training loss of a `FlowPrecond` (DESIGN §5), with `EDMLoss`'s constructor style and call
    signature.  t = sigmoid(P_mean + P_std n) (logit-normal) with n drawn where EDMLoss draws its `rnd_normal`,
    x_t = (1 - t) x + t eps, and per sample: the mean over kept patches of the per-patch mean of (v^ - v)^2, v = eps - x,
    plus mae_coef times MaskDiT's MAE term on the removed patches with D replaced by x^ = x_t - t v^; without a mask
    mean((v^ - v)^2).  Forward, loss and gradient seed run fused as in `EDMLoss`; the draws are made in EDMLoss's order.
    `last_edm_loss` holds the per-sample loss of the last call (for the training log)."""

    def __init__(self, P_mean=0.0, P_std=1.0):
        self.P_mean, self.P_std = P_mean, P_std

    def _randn(self, shape, device):
        return torch.randn(shape, device=device)

    def _rand(self, shape, device):
        return torch.rand(shape, device=device)

    def __call__(self, net, images, labels=None, mask_ratio=0, mae_loss_coef=0, feat=None, augment_pipe=None):
        if feat is not None or augment_pipe is not None:
            raise NotImplementedError("feat / augment_pipe are not part of the MaskDiT latent training path")
        raw = self._net(net, images.device)
        B = images.shape[0]
        x = images.contiguous().float()
        rnd = self._randn([B, 1, 1, 1], images.device)
        t4 = 1.0 / (1.0 + torch.exp(-(rnd * self.P_std + self.P_mean)))
        eps = self._randn(tuple(x.shape), images.device).contiguous()
        xt = ((1.0 - t4) * x + t4 * eps).contiguous()
        return self._finish(raw, x, xt, eps, t4.reshape(B).contiguous(), labels, mask_ratio, mae_loss_coef)

    def from_moments(self, net, moments, labels=None, mask_ratio=0, mae_loss_coef=0, class_dropout_prob=0.0,
                     scale_factor=0.18215, eps=None, drop_u=None):
        """`EDMLoss.from_moments` with the flow step front (`ops.flow_step_front`): latent, label dropout, t draw and
        x_t in one launch, the same draws in the same order, `eps` / `drop_u` as there."""
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
        noise = self._randn((B, C2 // 2, R, R), dev).contiguous()
        x, xt, t = ops.flow_step_front(moments, eps, rnd_normal, noise, labels, drop_u, float(class_dropout_prob),
                                       scale_factor, self.P_mean, self.P_std)
        return self._finish(raw, x, xt, noise, t, labels, mask_ratio, mae_loss_coef)

    def _net(self, net, dev):
        raw = _unwrap(net)
        if not isinstance(raw, FlowPrecond):
            raise TypeError("maskdit_b200.Losses['flow'] drives a maskdit_b200.FlowPrecond network"
                            + (" (this one is an EDMPrecond: use Losses['edm'])" if isinstance(raw, EDMPrecond)
                               else ""))
        raw._ready(dev)
        return raw

    def _finish(self, raw, x, xt, eps, t, labels, mask_ratio, mae_loss_coef):
        dev, B = x.device, x.shape[0]
        _, _, lab = raw._norm_inputs(x, t, labels)
        md = None
        if mask_ratio > 0:
            assert raw.training, "masked loss needs net.train()"
            L = raw.model.num_patches
            md = ops.mask_indices(self._rand((B, L), dev), int(L * (1 - mask_ratio)))
        coef = float(mae_loss_coef) if (mask_ratio > 0 and mae_loss_coef > 0) else 0.0
        if torch.is_grad_enabled():
            loss = _FusedFlowLossFn.apply(raw._anchor, raw, xt, x, eps, t, lab, md, coef)
        else:
            Fo, _ = raw._engine.forward(xt, t, lab, md, save=False)
            loss, _, _ = ops.flow_loss(Fo, xt, x, eps, t, md["mask"] if md else None, None, coef,
                                       raw.model.patch_size, want_dF=False)
        self.last_mask_dict = md
        self.last_edm_loss = loss
        return loss


def ect_r(t, qs, k=8.0, b=1.0):
    """ECT's target noise level r = t max(0, 1 - qs (1 + k sigmoid(-b t))), qs = q^-(s+1) of the tuning stage s (a
    float or a device tensor), evaluated op by op as `mdt_ect_step_front` does."""
    sig = 1.0 / (1.0 + torch.exp(b * t))
    return t * (1.0 - qs * (1.0 + k * sig)).clamp_min(0.0)


class _FusedECTLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, net, xt, xr, sr, y, t, r, labels, mask_dict, mae_coef, c):
        # the target first: the student's saving forward must be the handle's last, its backward reads that workspace
        Fr, _ = net._engine.forward(xr, sr, labels, mask_dict, save=False)
        Ft, saved = net._engine.forward(xt, t, labels, mask_dict, save=True)
        mask = mask_dict["mask"] if mask_dict is not None else None
        p = net.model.patch_size
        loss, _, _ = ops.ect_loss(Ft, Fr, xt, xr, y, t, r, mask, None, net.sigma_data, c, mae_coef, p,
                                  want_dF=False)
        ctx.net, ctx.saved = net, saved
        ctx.args = (Ft, Fr, xt, xr, y, t, r, mask, mae_coef, c, p)
        return loss

    @staticmethod
    def backward(ctx, gl):
        net = ctx.net
        Ft, Fr, xt, xr, y, t, r, mask, mae_coef, c, p = ctx.args
        _, _, dF = ops.ect_loss(Ft, Fr, xt, xr, y, t, r, mask, gl.contiguous().float(), net.sigma_data, c, mae_coef, p,
                                want_dF=True)
        net._run_backward(ctx.saved, dF.view(-1, dF.shape[-1]))
        ctx.saved = ctx.args = None
        return (torch.zeros(1, device=gl.device),) + (None,) * 11


class ECTLoss:
    """Easy Consistency Tuning (ECT; Geng et al., ICLR 2025) of a trained `EDMPrecond`, whose output D(x; sigma) is
    the consistency function f (DESIGN §5), with `EDMLoss`'s call signature.  Per sample: t = exp(P_mean + P_std n)
    with n drawn where EDMLoss draws `rnd_normal`, r = `ect_r(t, q^-(s+1), k, b)` at the tuning stage s, one eps for
    x_t = x + t eps and x_r = x + r eps.  The student D_t = D(x_t; t) carries the gradient; the target D_r = D(x_r; r)
    is a no-gradient forward of the same weights with the same kept tokens and labels (x itself where r = 0).  The
    loss is (sqrt(S + c^2) - c) / (t - r) + mae_coef M, S = (L / T) sum over kept patches of (D_t - D_r)^2,
    c = 0.00054 sqrt(C R R), M MaskDiT's MAE term on the removed patches with D = D_t.  `last_edm_loss` holds the
    per-sample loss of the last call (for the training log).

    The stage enters as one fp32 device word, q^-(s+1): `stage_scale` when set (`TrainStep` owns it and moves it
    with the run's step), otherwise built from `stage`."""

    def __init__(self, stage_steps, q=2.0, k=8.0, b=1.0, P_mean=-1.1, P_std=2.0, sigma_data=0.5):
        if int(stage_steps) != stage_steps or stage_steps < 1:
            raise ValueError(f"ECT needs stage_steps >= 1 (steps per tuning stage), got {stage_steps}")
        if not q > 1:
            raise ValueError(f"ECT needs q > 1 (the gap t - r shrinks by q per stage), got {q}")
        self.stage_steps = int(stage_steps)
        self.q, self.k, self.b = float(q), float(k), float(b)
        self.P_mean, self.P_std, self.sigma_data = P_mean, P_std, sigma_data
        self.stage = 0
        self.stage_scale = None

    def stage_at(self, step, origin):
        """The tuning stage s = floor((step - origin) / stage_steps) of run step `step` (origin: the first tuned)."""
        return (int(step) - int(origin)) // self.stage_steps

    def scale_of(self, stage):
        """q^-(s+1) of stage s, the word the step front reads."""
        return self.q ** -(int(stage) + 1)

    def _qs(self, dev):
        if self.stage_scale is not None:
            return self.stage_scale
        return torch.full((1,), self.scale_of(self.stage), dtype=torch.float32, device=dev)

    def _randn(self, shape, device):
        return torch.randn(shape, device=device)

    def _rand(self, shape, device):
        return torch.rand(shape, device=device)

    def __call__(self, net, images, labels=None, mask_ratio=0, mae_loss_coef=0, feat=None, augment_pipe=None):
        if feat is not None or augment_pipe is not None:
            raise NotImplementedError("feat / augment_pipe are not part of the MaskDiT latent training path")
        dev = images.device
        raw = self._net(net, dev)
        B = images.shape[0]
        y = images.contiguous().float()
        t4 = (self._randn([B, 1, 1, 1], dev) * self.P_std + self.P_mean).exp()
        eps = self._randn(tuple(y.shape), dev)
        r4 = ect_r(t4, self._qs(dev), self.k, self.b)
        xt, xr = (y + t4 * eps).contiguous(), (y + r4 * eps).contiguous()
        sr = torch.where(r4 > 0, r4, t4)
        return self._finish(raw, y, xt, xr, sr.reshape(B).contiguous(), t4.reshape(B).contiguous(),
                            r4.reshape(B).contiguous(), labels, mask_ratio, mae_loss_coef)

    def from_moments(self, net, moments, labels=None, mask_ratio=0, mae_loss_coef=0, class_dropout_prob=0.0,
                     scale_factor=0.18215, eps=None, drop_u=None):
        """`EDMLoss.from_moments` with the ECT step front (`ops.ect_step_front`): latent, label dropout, t, r, x_t and
        x_r in one launch, the same draws in the same order, `eps` / `drop_u` as there."""
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
        noise = self._randn((B, C2 // 2, R, R), dev).contiguous()
        y, xt, xr, sr, t, r = ops.ect_step_front(moments, eps, rnd_normal, noise, self._qs(dev), labels, drop_u,
                                                 float(class_dropout_prob), scale_factor, self.P_mean, self.P_std,
                                                 self.k, self.b)
        return self._finish(raw, y, xt, xr, sr, t, r, labels, mask_ratio, mae_loss_coef)

    def _net(self, net, dev):
        raw = _unwrap(net)
        if not isinstance(raw, EDMPrecond) or isinstance(raw, FlowPrecond):
            raise TypeError("maskdit_b200.Losses['ect'] tunes a maskdit_b200.EDMPrecond network"
                            + (" (consistency tuning of a FlowPrecond is not supported)"
                               if isinstance(raw, FlowPrecond) else ""))
        if raw.logvar_channels:
            raise ValueError("Losses['ect'] does not train a learned loss weighting: build the network with "
                             "logvar_channels=0")
        raw._ready(dev)
        return raw

    def _finish(self, raw, y, xt, xr, sr, t, r, labels, mask_ratio, mae_loss_coef):
        dev, B = y.device, y.shape[0]
        _, _, lab = raw._norm_inputs(y, t, labels)
        md = None
        if mask_ratio > 0:
            assert raw.training, "masked loss needs net.train()"
            L = raw.model.num_patches
            md = ops.mask_indices(self._rand((B, L), dev), int(L * (1 - mask_ratio)))
        coef = float(mae_loss_coef) if (mask_ratio > 0 and mae_loss_coef > 0) else 0.0
        c = 0.00054 * math.sqrt(y[0].numel())
        if torch.is_grad_enabled():
            loss = _FusedECTLossFn.apply(raw._anchor, raw, xt, xr, sr, y, t, r, lab, md, coef, c)
        else:
            Fr, _ = raw._engine.forward(xr, sr, lab, md, save=False)
            Ft, _ = raw._engine.forward(xt, t, lab, md, save=False)
            loss, _, _ = ops.ect_loss(Ft, Fr, xt, xr, y, t, r, md["mask"] if md else None, None, raw.sigma_data, c,
                                      coef, raw.model.patch_size, want_dF=False)
        self.last_mask_dict = md
        self.last_edm_loss = loss
        return loss


def mg_weight(scale):
    """Model guidance's w = 1 - 1/s of the CFG-equivalent scale s >= 1 (DESIGN §5)."""
    s = float(scale)
    if not s >= 1 or math.isinf(s):
        raise ValueError(f"model guidance needs a finite scale s >= 1 (the CFG-equivalent scale), got {scale}")
    return 1.0 - 1.0 / s


class _FusedMGLossFn(torch.autograd.Function):
    """Returns (objective, plain loss); the plain loss carries no gradient.  `eps` is None for EDM, the noise for
    flow."""

    @staticmethod
    def forward(ctx, anchor, net, mg, xin, y, eps, sigma, labels, mask_dict, mae_coef):
        # the null-label forward first: the student's saving forward must be the handle's last, its backward reads
        # that workspace
        Fu, _ = net._engine.forward(xin, sigma, torch.zeros_like(labels), mask_dict, save=False)
        Fc, saved = net._engine.forward(xin, sigma, labels, mask_dict, save=True)
        mask = mask_dict["mask"] if mask_dict is not None else None
        loss, plain, _ = mg._kernel(net, Fc, Fu, xin, y, eps, sigma, labels, mask, None, mae_coef)
        ctx.net, ctx.mg, ctx.saved = net, mg, saved
        ctx.args = (Fc, Fu, xin, y, eps, sigma, labels, mask, mae_coef)
        ctx.mark_non_differentiable(plain)
        return loss, plain

    @staticmethod
    def backward(ctx, gl, _):
        _, _, dF = ctx.mg._kernel(ctx.net, *ctx.args[:8], gl.contiguous().float(), ctx.args[8])
        ctx.net._run_backward(ctx.saved, dF.view(-1, dF.shape[-1]))
        ctx.saved = ctx.args = None
        return (torch.zeros(1, device=gl.device),) + (None,) * 9


class MGLoss:
    """Model guidance (MG; Tang et al. 2025, in this repository's own definition, DESIGN §5) of a class-conditional
    `EDMPrecond` or `FlowPrecond`: the network learns to output the guided denoiser, so it samples guided without
    CFG's second pass.  The draws and the step front are those of `EDMLoss` / `FlowLoss` for the network given (MG
    draws nothing more).  The student D_c carries the gradient; D_u is a no-gradient forward of the same weights on the
    same input, noise level and kept tokens with the null (all-zero) label row.  Row b's target is
    y + w_b sg(D_c - D_u), w_b = w = 1 - 1/scale where its label was kept and lo < sigma_b <= hi (flow: t), else 0;
    the objective is MaskDiT's loss with that target in the denoising term (flow: v' = (eps - y) + w_b (F_c - F_u)).
    The call returns the per-sample objective; `last_edm_loss` holds the plain loss against y (for the training log)
    and `last_objective` the objective."""

    def __init__(self, scale, interval=None, P_mean=None, P_std=None, sigma_data=0.5):
        self.scale = float(scale)
        self.w = mg_weight(scale)
        lo, hi = (0.0, math.inf) if interval is None else (float(interval[0]), float(interval[1]))
        if not lo < hi:
            raise ValueError(f"model guidance needs an interval lo < hi, got [{lo}, {hi}]")
        self.lo, self.hi = lo, hi
        self.P_mean, self.P_std, self.sigma_data = P_mean, P_std, sigma_data

    def _randn(self, shape, device):
        return torch.randn(shape, device=device)

    def _rand(self, shape, device):
        return torch.rand(shape, device=device)

    def _front(self, net):
        """An `EDMLoss` or `FlowLoss` for `net` that draws through this object's hooks and finishes with MG."""
        flow = isinstance(_unwrap(net), FlowPrecond)
        kw = {k: v for k, v in (("P_mean", self.P_mean), ("P_std", self.P_std)) if v is not None}
        front = FlowLoss(**kw) if flow else EDMLoss(sigma_data=self.sigma_data, **kw)
        front._randn, front._rand = self._randn, self._rand
        front._finish = self._finish_flow if flow else self._finish_edm
        return front

    def __call__(self, net, images, labels=None, mask_ratio=0, mae_loss_coef=0, feat=None, augment_pipe=None):
        return self._front(net)(net, images, labels, mask_ratio, mae_loss_coef, feat, augment_pipe)

    def from_moments(self, net, moments, labels=None, mask_ratio=0, mae_loss_coef=0, class_dropout_prob=0.0,
                     scale_factor=0.18215, eps=None, drop_u=None):
        """`EDMLoss.from_moments` / `FlowLoss.from_moments` of the network given, finished with MG."""
        return self._front(net).from_moments(net, moments, labels, mask_ratio, mae_loss_coef, class_dropout_prob,
                                             scale_factor, eps, drop_u)

    def _kernel(self, raw, F, Fu, xin, y, eps, sigma, lab, mask, gl, coef):
        p, want = raw.model.patch_size, gl is not None
        if eps is None:
            loss, plain, _, dF = ops.mg_loss(F, Fu, xin, y, sigma, lab, mask, gl, raw.sigma_data, coef, self.w,
                                             self.lo, self.hi, p, want_dF=want)
        else:
            loss, plain, _, dF = ops.flow_mg_loss(F, Fu, xin, y, eps, sigma, lab, mask, gl, coef, self.w, self.lo,
                                                  self.hi, p, want_dF=want)
        return loss, plain, dF

    def _finish_edm(self, raw, y, yn, sigma, labels, mask_ratio, mae_loss_coef):
        return self._finish(raw, yn, y, None, sigma, labels, mask_ratio, mae_loss_coef)

    def _finish_flow(self, raw, x, xt, eps, t, labels, mask_ratio, mae_loss_coef):
        return self._finish(raw, xt, x, eps, t, labels, mask_ratio, mae_loss_coef)

    def _finish(self, raw, xin, y, eps, sigma, labels, mask_ratio, mae_loss_coef):
        if not raw.num_classes:
            raise ValueError("Losses['mg'] guides a class-conditional network: this one has num_classes=0")
        if raw.logvar_channels:
            raise ValueError("Losses['mg'] does not train a learned loss weighting: build the network with "
                             "logvar_channels=0")
        dev, B = y.device, y.shape[0]
        _, _, lab = raw._norm_inputs(y, sigma, labels)
        md = None
        if mask_ratio > 0:
            assert raw.training, "masked loss needs net.train()"
            L = raw.model.num_patches
            md = ops.mask_indices(self._rand((B, L), dev), int(L * (1 - mask_ratio)))
        coef = float(mae_loss_coef) if (mask_ratio > 0 and mae_loss_coef > 0) else 0.0
        if torch.is_grad_enabled():
            loss, plain = _FusedMGLossFn.apply(raw._anchor, raw, self, xin, y, eps, sigma, lab, md, coef)
        else:
            Fu, _ = raw._engine.forward(xin, sigma, torch.zeros_like(lab), md, save=False)
            Fc, _ = raw._engine.forward(xin, sigma, lab, md, save=False)
            loss, plain, _ = self._kernel(raw, Fc, Fu, xin, y, eps, sigma, lab, md["mask"] if md else None, None,
                                          coef)
        self.last_mask_dict = md
        self.last_edm_loss = plain
        self.last_objective = loss
        return loss


Losses = {"edm": EDMLoss, "flow": FlowLoss, "ect": ECTLoss, "mg": MGLoss}
