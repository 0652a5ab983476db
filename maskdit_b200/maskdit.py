"""Host-side mirror of the reference model interface (models/maskdit.py) over the H100 engine.

Exports the same registries the reference's entry points consume (SURVEY.md §8b):
    DiT_models      name -> constructor            (models/maskdit.py:709-715)
    Precond_models  {'edm': EDMPrecond}            (models/maskdit.py:779-781), plus 'flow': FlowPrecond
`EDMPrecond` is an `nn.Module` with the reference's constructor signature, attributes and state-dict key set
(378 entries for XL/2), so `train.py`/`generate.py`-style drivers, `deepcopy` (EMA), `load_state_dict` of reference
checkpoints and the reference's own `EDMLoss`/`edm_sampler` work against it unchanged.  Its arithmetic is the
CUDA engine (`engine.py`); there is no PyTorch fallback: calling it with CPU tensors raises.

Scope: the asymmetric encoder-decoder MaskDiT (use_decoder=True, every config the reference ships) and the plain
decoder-less DiT (use_decoder=False, the reference's default: the final layer runs on the encoder width, and training
with a mask fills the removed patches of the output with zeros, models/maskdit.py:550-553), each at any mask ratio,
with or without classes.  pad_cls_token, direct_cls_token, ext_feature_dim, use_encoder_feat and learn_sigma must be
off; other flag combinations raise NotImplementedError.
"""
from __future__ import annotations

import copy
import os
import math
from functools import partial

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .engine import CEngine
from .flat import FlatStore

# (depth, hidden, heads) — models/maskdit.py:649-706
_ARCH = {"H": (32, 1280, 16), "XL": (28, 1152, 16), "L": (24, 1024, 16), "B": (12, 768, 12), "S": (12, 384, 6)}


def sincos_2d(dim, grid):
    """Fixed 2-D sin-cos table (get_2d_sincos_pos_embed, models/maskdit.py:595-642): [grid*grid, dim] float32;
    first half from the column (w) index, second half from the row (h) index, each [sin | cos]."""
    k = np.arange(dim // 4, dtype=np.float64)
    omega = np.power(10000.0, -k / (dim // 4))
    rows, cols = np.divmod(np.arange(grid * grid), grid)

    def half(pos):
        ang = pos.astype(np.float32).astype(np.float64)[:, None] * omega[None]
        return np.concatenate([np.sin(ang), np.cos(ang)], 1)

    return torch.from_numpy(np.concatenate([half(cols), half(rows)], 1)).float()


class _Node(nn.Module):
    """Parameter container; children are named after the reference's module tree so state-dict keys match."""


class _Cfg:
    pass


class DiT(nn.Module):
    """Parameter/attribute holder matching the reference `DiT` (models/maskdit.py:237-332).  The forward pass is
    executed by `EDMPrecond` through the engine (the EDM scalings are fused into the first/last kernels)."""

    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4.0, class_dropout_prob=0.1, num_classes=1000, learn_sigma=False, use_decoder=False,
                 mae_loss_coef=0, pad_cls_token=False, direct_cls_token=False, ext_feature_dim=0,
                 use_encoder_feat=False, norm_layer=None):
        super().__init__()
        if learn_sigma or pad_cls_token or direct_cls_token or ext_feature_dim or use_encoder_feat:
            raise NotImplementedError("maskdit_b200 covers the shipped configs: learn_sigma/pad_cls_token/"
                                      "ext_feature_dim/use_encoder_feat must be off")
        self.learn_sigma, self.in_channels, self.out_channels = learn_sigma, in_channels, in_channels
        self.patch_size, self.num_heads, self.class_dropout_prob = patch_size, num_heads, class_dropout_prob
        self.num_classes, self.use_decoder, self.mae_loss_coef = num_classes, use_decoder, mae_loss_coef
        self.pad_cls_token = self.direct_cls_token = False
        self.ext_feature_dim, self.use_encoder_feat = 0, False
        self.cls_token, self.extras, self.decoder_extras = None, 0, 0
        self.input_size, self.hidden_size, self.depth, self.mlp_ratio = input_size, hidden_size, depth, mlp_ratio
        # decoder: maskdit.py:310-312; none without use_decoder (final layer on the encoder width, :308,329-331)
        self.decoder_hidden_size, self.decoder_depth, self.decoder_num_heads = (512, 8, 16) if use_decoder else (0, 0, 0)
        grid = input_size // patch_size
        self.num_patches = grid * grid
        D, Dd, L = hidden_size, self.decoder_hidden_size, self.num_patches

        def P(*shape, grad=True):
            return nn.Parameter(torch.zeros(*shape), requires_grad=grad)

        def linear(out_f, in_f, bias=True):
            n = _Node()
            n.weight = P(out_f, in_f)
            if bias:
                n.bias = P(out_f)
            return n

        def seq(**children):
            n = _Node()
            for name, child in children.items():
                n.add_module(name.lstrip("_"), child)
            return n

        def block(d, cond):
            n = _Node()
            n.attn = seq(qkv=linear(3 * d, d), proj=linear(d, d))
            n.mlp = seq(fc1=linear(int(d * mlp_ratio), d), fc2=linear(d, int(d * mlp_ratio)))
            n.adaLN_modulation = seq(_1=linear(6 * d, cond))
            return n

        self.pos_embed = P(1, L, D, grad=False)
        pe = _Node()
        pe.weight, pe.bias = P(D, in_channels, patch_size, patch_size), P(D)
        self.x_embedder = seq(proj=pe)
        self.x_embedder.patch_size = (patch_size, patch_size)  # read at loss.py via net.model.patch_size only
        self.x_embedder.num_patches = L
        self.t_embedder = seq(mlp=seq(_0=linear(D, 256), _2=linear(D, D)))
        self.y_embedder = seq(embedding_table=linear(D, num_classes, bias=False)) if num_classes else None
        self.blocks = nn.ModuleList([block(D, D) for _ in range(depth)])
        self.decoder_pos_embed = self.decoder_layer = self.decoder_blocks = self.mask_token = None
        if use_decoder:
            self.decoder_pos_embed = P(1, L, Dd, grad=False)
            self.decoder_layer = seq(linear=linear(Dd, D), adaLN_modulation=seq(_1=linear(2 * D, D)))
            self.decoder_blocks = nn.ModuleList([block(Dd, D) for _ in range(self.decoder_depth)])
            self.mask_token = P(1, 1, Dd) if mae_loss_coef > 0 else None
        Df = Dd if use_decoder else D
        self.final_layer = seq(linear=linear(patch_size * patch_size * self.out_channels, Df),
                               adaLN_modulation=seq(_1=linear(2 * Df, D)))
        self.reset_parameters()

    @torch.no_grad()
    def reset_parameters(self):
        """Same initial distribution as DiT.initialize_weights (models/maskdit.py:334-409): Xavier-uniform matrices
        with zero biases; N(0, 0.02) label table / timestep MLP / mask token; zeros for every adaLN projection and
        for the final and decoder-entry linears (adaLN-Zero); fixed sin-cos position tables."""
        grid = int(round(self.num_patches ** 0.5))
        for name, prm in self.named_parameters():
            if name.endswith("pos_embed"):
                prm.copy_(sincos_2d(prm.shape[-1], grid).unsqueeze(0))
            elif name.endswith(".bias"):
                prm.zero_()
            elif "adaLN_modulation" in name or name.startswith(("final_layer.linear", "decoder_layer.linear")):
                prm.zero_()
            elif name.startswith(("y_embedder", "t_embedder")) or name == "mask_token":
                prm.normal_(std=0.02)
            else:
                nn.init.xavier_uniform_(prm.view(prm.shape[0], -1))

    def forward(self, *a, **k):
        raise RuntimeError("call the EDMPrecond wrapper: the H100 engine fuses the EDM scalings into the network "
                           "kernels, the bare DiT is a parameter holder")


def _dit(arch, patch):
    depth, hidden, heads = _ARCH[arch]
    return lambda **kw: DiT(depth=depth, hidden_size=hidden, patch_size=patch, num_heads=heads, **kw)


DiT_models = {f"DiT-{a}/{p}": _dit(a, p) for a in ("H", "XL", "L", "B", "S") for p in (2, 4, 8)}


class _NetFn(torch.autograd.Function):
    """D_x = EDMPrecond(x) with a hand-written backward: gradients go straight into the flat gradient buffer."""

    @staticmethod
    def forward(ctx, anchor, net, x, sigma, labels, mask_dict):
        Fo, saved = net._engine.forward(x, sigma, labels, mask_dict, save=True)
        ctx.net, ctx.saved, ctx.sigma = net, saved, sigma
        return ops.edm_precond_out(Fo, x, sigma, net.sigma_data, net.model.patch_size)

    @staticmethod
    def backward(ctx, gD):
        net = ctx.net
        dF = ops.edm_precond_out_bwd(gD.contiguous().float(), ctx.sigma, net.sigma_data, net.model.patch_size)
        net._run_backward(ctx.saved, dF)
        ctx.saved = None
        return (torch.zeros(1, device=gD.device),) + (None,) * 5


LOGVAR_MAX_CHANNELS = 256


class EDMPrecond(nn.Module):
    """EDM preconditioning wrapper (reference: models/maskdit.py:722-776) running on the sm_90a engine.

    `logvar_channels` C > 0 adds EDM2's learned loss weighting (Karras et al., CVPR 2024; Kendall et al.'s uncertainty
    weighting), which the reference does not have: a tiny network u(sigma) = sum_j w_j phi_j(c), c = ln(sigma) / 4,
    phi_j(c) = sqrt(2) cos(freqs_j c + phases_j), j < C <= 256.  `freqs = 2 pi randn(C)` and `phases = 2 pi rand(C)` are
    drawn in that order at construction from `torch.Generator().manual_seed(0)` on the CPU, so two nets of one config
    agree; they are frozen (`logvar_fourier.freqs`, `logvar_fourier.phases`).  `w` (`logvar_linear.weight` [1, C], no
    bias) is trained and starts at zero.  Unlike EDM2 the linear has no forced weight normalisation: no other layer here
    is magnitude-preserving, and AdamW treats w like every other weight.  The training loss (`Losses['edm']` with
    gradients) then returns the per-sample objective exp(-u) E + u + mae_coef M, E and M being the EDM and MAE terms;
    at the optimum exp(u(sigma)) is the expected E at sigma.  The three tensors are registered after `model.*`, so the
    reference's parameters keep their positions.  0 (the default): none of this exists."""

    PRECOND = 0   # the C handle's precondition kind (mdt_model_set_precond): MDT_PRECOND_EDM

    def __init__(self, img_resolution, img_channels, num_classes=0, sigma_min=0, sigma_max=float("inf"),
                 sigma_data=0.5, model_type="DiT-B/2", logvar_channels=0, **model_kwargs):
        super().__init__()
        self.img_resolution, self.img_channels, self.num_classes = img_resolution, img_channels, num_classes
        self.sigma_min, self.sigma_max, self.sigma_data = sigma_min, sigma_max, sigma_data
        self.model_type = model_type
        self.logvar_channels = int(logvar_channels)
        if not 0 <= self.logvar_channels <= LOGVAR_MAX_CHANNELS:
            raise ValueError(f"logvar_channels must be in [0, {LOGVAR_MAX_CHANNELS}], got {logvar_channels}")
        self._ctor = dict(img_resolution=img_resolution, img_channels=img_channels, num_classes=num_classes,
                          sigma_min=sigma_min, sigma_max=sigma_max, sigma_data=sigma_data, model_type=model_type,
                          logvar_channels=self.logvar_channels, **model_kwargs)
        self.model = DiT_models[model_type](input_size=img_resolution, in_channels=img_channels,
                                            num_classes=num_classes, **model_kwargs)
        if self.logvar_channels:
            C, g = self.logvar_channels, torch.Generator().manual_seed(0)
            self.logvar_fourier = _Node()
            # on the CPU (the generator's device) also under a `with torch.device(...)` context
            self.logvar_fourier.freqs = nn.Parameter(2 * np.pi * torch.randn(C, generator=g, device="cpu"),
                                                     requires_grad=False)
            self.logvar_fourier.phases = nn.Parameter(2 * np.pi * torch.rand(C, generator=g, device="cpu"),
                                                      requires_grad=False)
            self.logvar_linear = _Node()
            self.logvar_linear.weight = nn.Parameter(torch.zeros(1, C))
        self._store, self._engine, self._anchor = None, None, None
        self._graphs = {}  # CUDA graphs of the eval-mode forward, keyed by input shapes (see _eval_graphed)

    # -- engine plumbing ---------------------------------------------------------------------------------------
    def _cfg(self):
        c, m = _Cfg(), self.model
        c.hidden, c.depth, c.heads, c.patch = m.hidden_size, m.depth, m.num_heads, m.patch_size
        c.dec_hidden, c.dec_depth, c.dec_heads = m.decoder_hidden_size, m.decoder_depth, m.decoder_num_heads
        # MLP widths as DiT.__init__ sizes fc1 (0 without a decoder)
        c.mlp_hidden, c.dec_mlp_hidden = int(m.hidden_size * m.mlp_ratio), int(m.decoder_hidden_size * m.mlp_ratio)
        c.has_mask_token = m.mask_token is not None
        c.num_patches, c.num_classes, c.sigma_data = m.num_patches, self.num_classes, self.sigma_data
        c.img_resolution, c.img_channels = self.img_resolution, self.img_channels
        c.patch_dim = m.patch_size * m.patch_size * m.out_channels
        c.logvar_channels = self.logvar_channels
        c.precond = self.PRECOND
        return c

    def _params(self):
        return dict(self.named_parameters())

    def _layout(self):
        """The step driver (its C model handle) and the flat store it lays out.  Both depend only on the config, so
        they are built once, without a device."""
        if self._engine is None:
            self._engine = CEngine(self._cfg())
            self._store = self._engine.store = FlatStore(self._engine,
                                                         {k: tuple(p.shape) for k, p in self.named_parameters()})
        return self._engine, self._store

    def _ready(self, device):
        """Flatten parameters on `device` (once / after .to()) and refresh the bf16 weight shadow when any
        parameter was modified through PyTorch (optimizer step, load_state_dict, EMA copy...)."""
        if device.type != "cuda":
            raise ops.L.MdtError("maskdit_b200 runs on CUDA (sm_90a) only — there is no CPU fallback")
        params = self._params()
        _, st = self._layout()
        if not st.is_attached(params) or st.device != device:
            st.attach(params, device)
            self._anchor = torch.zeros(1, device=device, requires_grad=True)
            self._graphs = {}
        if st.shadow_stale(params):
            ops.cast_bf16(st.w32, out=st.w16)
            st.mark_shadow_fresh(params)
        return st

    def flat_store(self):
        """The flat parameter store (after the first CUDA call / `prepare()`): used by the fused training step."""
        return self._store

    def prepare(self, device=None):
        device = torch.device(device) if device is not None else next(self.parameters()).device
        return self._ready(device)

    def _run_backward(self, saved, dF16):
        st = self._store
        params = self._params()
        first = next(q for q in params.values() if q.requires_grad)
        if first.grad is None:  # fresh / zero_grad(set_to_none=True): start from zero and (re)attach .grad views
            st.ensure_grad().zero_()
            for k, p in params.items():
                if p.requires_grad:
                    p.grad = st.gview(k)
        self._engine.backward(saved, dF16)

    def __deepcopy__(self, memo):
        new = type(self)(**copy.deepcopy(self._ctor))
        dev = next(self.parameters()).device
        new.to(dev)
        with torch.no_grad():   # every parameter, the frozen logvar features included
            for (k, p), (_, q) in zip(self.named_parameters(), new.named_parameters()):
                q.copy_(p)
                q.requires_grad_(p.requires_grad)
        new.train(self.training)
        return new

    # -- reference interface -------------------------------------------------------------------------------------
    def round_sigma(self, sigma):
        return torch.as_tensor(sigma)

    def _norm_inputs(self, x, sigma, class_labels):
        B = x.shape[0]
        xf = x.contiguous().float()
        sig = torch.as_tensor(sigma, device=x.device).to(torch.float32).reshape(-1)
        if sig.numel() == 1:
            sig = sig.expand(B)
        sig = sig.contiguous()
        if self.num_classes:
            if class_labels is None:
                lab = torch.zeros(B, self.num_classes, device=x.device, dtype=torch.float32)
            else:
                lab = class_labels.to(torch.float32).reshape(-1, self.num_classes).contiguous()
                if lab.data_ptr() % 16:   # a row slice of a narrow label matrix: the vectorised kernels need 16 B
                    lab = lab.clone()
        else:
            lab = None
        return xf, sig, lab

    # -- eval-mode forward (no autograd): eager, or replayed from a CUDA graph ---------------------------------------
    def _eval_eager(self, xf, sig, lab, cfg_scale, guide=None):
        p = self.model.patch_size
        if guide is not None:
            # guidance by a second network: one eval pass of each at batch B, `cfg_scale` is the guide weight w
            Fm, _ = self._engine.forward(xf, sig, lab, None, save=False)
            Fg, _ = guide._engine.forward(xf, sig, lab, None, save=False)
            return ops.guided_precond_out(Fm, p, Fg, guide.model.patch_size, xf, sig, self.sigma_data, cfg_scale)
        if cfg_scale is not None:
            # forward_with_cfg (models/maskdit.py:559-587): one eval pass at batch 2B, guidance fused in the output
            x2 = torch.cat([xf, xf], 0)
            s2 = torch.cat([sig, sig], 0)
            y2 = torch.cat([lab, torch.zeros_like(lab)], 0)
            Fo, _ = self._engine.forward(x2, s2, y2, None, save=False)
            return ops.cfg_precond_out(Fo, xf, sig, self.sigma_data, float(cfg_scale), p)
        Fo, _ = self._engine.forward(xf, sig, lab, None, save=False)
        return ops.edm_precond_out(Fo, xf, sig, self.sigma_data, p)

    def _eval_graphed(self, xf, sig, lab, cfg_scale, guide=None):
        """The eval forward is ~280 launches with static shapes: the sampler calls it 35 times per batch and the host
        enqueue time (35 ms per evaluation at B=64) is as long as the device time (38 ms).  It is therefore captured
        once per (shapes, cfg_scale, guide) into a CUDA graph with static input buffers and replayed.  Weights are read
        from the flat bf16 shadows, whose storage is stable: the cache is dropped when this store is re-attached, and a
        guide's entry is keyed by its shadow's address too.  The entry holds the guide, so its id is not reused while
        the entry exists.  MDT_CUDA_GRAPH=0 disables the graphs."""
        key = (tuple(xf.shape), None if lab is None else tuple(lab.shape), cfg_scale)
        if guide is not None:
            key += (id(guide), guide._store.w16.data_ptr())
        ent = self._graphs.get(key)
        if ent is None:
            sx, ss = torch.empty_like(xf), torch.empty_like(sig)
            sl = None if lab is None else torch.empty_like(lab)
            sx.copy_(xf), ss.copy_(sig)
            if sl is not None:
                sl.copy_(lab)
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):  # warm-up outside the capture (lazy kernel attributes, allocator pools)
                self._eval_eager(sx, ss, sl, cfg_scale, guide)
            cur.wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            n0 = ops.L.LAUNCHES
            with torch.cuda.graph(graph):
                out = self._eval_eager(sx, ss, sl, cfg_scale, guide)
            ent = (graph, sx, ss, sl, out, ops.L.LAUNCHES - n0, guide)
            self._graphs[key] = ent
        graph, sx, ss, sl, out, n_launch, _ = ent
        sx.copy_(xf), ss.copy_(sig)
        if sl is not None:
            sl.copy_(lab)
        graph.replay()
        ops.L.LAUNCHES += n_launch
        return out.clone()

    def forward(self, x, sigma, class_labels=None, cfg_scale=None, **model_kwargs):
        """Same call contract as the reference (models/maskdit.py:756-773): returns {'x': D_x [, 'mask': mask]}."""
        mask_ratio = model_kwargs.pop("mask_ratio", 0)
        mask_dict = model_kwargs.pop("mask_dict", None)
        feat = model_kwargs.pop("feat", None)
        if feat is not None or model_kwargs:
            raise NotImplementedError(f"unsupported arguments: feat / {list(model_kwargs)}")
        self._ready(x.device)
        xf, sig, lab = self._norm_inputs(x, sigma, class_labels)
        B = xf.shape[0]
        out = {}
        p = self.model.patch_size
        use_graph = not self.training and os.environ.get("MDT_CUDA_GRAPH", "1") != "0" \
            and not torch.cuda.is_current_stream_capturing()
        if cfg_scale is not None:
            assert self.num_classes and lab is not None
            with torch.no_grad():
                fn = self._eval_graphed if use_graph else self._eval_eager
                out["x"] = fn(xf, sig, lab, cfg_scale).to(x.dtype)
            return out
        md = None
        if mask_ratio > 0:
            L = self.model.num_patches
            if mask_dict is None:
                noise = torch.rand(B, L, device=x.device)  # get_mask, models/maskdit.py:102
                mask_dict = ops.mask_indices(noise, int(L * (1 - mask_ratio)))
            out["mask"] = mask_dict["mask"]
            if self.training:
                md = mask_dict  # eval with mask_ratio > 0 keeps all tokens (train=self.training, maskdit.py:482)
        if torch.is_grad_enabled() and any(q.requires_grad for q in self.parameters()):
            out["x"] = _NetFn.apply(self._anchor, self, xf, sig, lab, md).to(x.dtype)
        elif md is None and use_graph:
            out["x"] = self._eval_graphed(xf, sig, lab, None).to(x.dtype)
        else:
            Fo, _ = self._engine.forward(xf, sig, lab, md, save=False)
            out["x"] = ops.edm_precond_out(Fo, xf, sig, self.sigma_data, p).to(x.dtype)
        return out

    # -- learned loss weighting ------------------------------------------------------------------------------------
    def _logvar_tensors(self):
        """(freqs, phases, w) as flat fp32 views of the store (w: [C])."""
        st = self._store
        return (st.view32("logvar_fourier.freqs"), st.view32("logvar_fourier.phases"),
                st.view32("logvar_linear.weight").view(-1))

    @torch.no_grad()
    def logvar(self, sigma):
        """u(sigma) [N] fp32 of the learned loss weighting (see the class docstring), one value per element of `sigma`
        (a tensor or a sequence), on the network's CUDA device (`mdt_logvar`).  Inspection only: no gradient."""
        if not self.logvar_channels:
            raise ValueError("this network has no learned loss weighting (logvar_channels = 0)")
        dev = next(self.parameters()).device
        self._ready(dev)
        sig = torch.as_tensor(sigma, dtype=torch.float32).to(dev).reshape(-1).contiguous()
        return ops.logvar(sig, *self._logvar_tensors())

    def check_guide(self, guide):
        """Raise ValueError unless `guide` can guide this network: an EDMPrecond with the same image geometry, classes
        and sigma_data.  Depth, width, patch size and use_decoder may differ."""
        if not isinstance(guide, EDMPrecond):
            raise ValueError(f"the guide must be an EDMPrecond, not {type(guide).__name__}")
        for k in ("img_resolution", "img_channels", "num_classes", "sigma_data"):
            if getattr(guide, k) != getattr(self, k):
                raise ValueError(f"the guide's {k} is {getattr(guide, k)}, the network's {getattr(self, k)}")

    def forward_guided(self, x, sigma, class_labels, guide, guidance):
        """D_x guided by a second network (autoguidance, Karras et al., NeurIPS 2024):
        D = D_guide + guidance * (D_self - D_guide), from one eval pass of each network at batch B with the same
        labels (None for unconditional networks), combined in fp32 with the EDM output scaling.  Returns D_x like
        `forward(...)['x']`."""
        self.check_guide(guide)
        w = float(guidance)
        if not math.isfinite(w):
            raise ValueError(f"guidance must be finite, got {guidance}")
        self._ready(x.device)
        guide._ready(x.device)
        xf, sig, lab = self._norm_inputs(x, sigma, class_labels)
        use_graph = not self.training and os.environ.get("MDT_CUDA_GRAPH", "1") != "0" \
            and not torch.cuda.is_current_stream_capturing()
        with torch.no_grad():
            fn = self._eval_graphed if use_graph else self._eval_eager
            return fn(xf, sig, lab, w, guide).to(x.dtype)


class FlowPrecond(EDMPrecond):
    """The DiT trained with the rectified-flow objective (linear interpolant, velocity prediction; SiT, Ma et al. 2024)
    on the same engine, flat store, state-dict keys and CUDA-graph eval path as `EDMPrecond`.

    t in [0, 1], t = 0 is data and t = 1 is noise: x_t = (1 - t) x + t eps.  The network reads x_t unscaled (c_in = 1)
    with c_noise = t in the unchanged timestep embedder, and `forward(x_t, t, class_labels, cfg_scale)` returns
    {'x': v^ [, 'mask': mask]}: the unpatchified network output is the velocity, whose target is v = eps - x; the
    denoised estimate is x_t - t v^.  `Losses['flow']` trains it and `flow_sampler` integrates dx/dt = v^ from t = 1 to 0.
    There is no autograd path through `forward` (train through `Losses['flow']`), no autoguidance and no learned loss
    weighting (defined over sigma).  `sigma_data`, `sigma_min` and `sigma_max` are kept for the shared constructor and
    are not read."""

    PRECOND = 1   # MDT_PRECOND_FLOW

    def __init__(self, img_resolution, img_channels, num_classes=0, sigma_min=0, sigma_max=float("inf"),
                 sigma_data=0.5, model_type="DiT-B/2", logvar_channels=0, **model_kwargs):
        if logvar_channels:
            raise ValueError("the learned loss weighting (logvar_channels) is defined over the EDM noise level sigma: "
                             "flow networks do not have it")
        super().__init__(img_resolution, img_channels, num_classes, sigma_min, sigma_max, sigma_data, model_type, 0,
                         **model_kwargs)

    def _eval_eager(self, xf, t, lab, cfg_scale, guide=None):
        if guide is not None:
            raise ValueError("autoguidance is not available for flow networks")
        B, p = xf.shape[0], self.model.patch_size
        C, R = self.img_channels, self.img_resolution
        if cfg_scale is not None:
            # forward_with_cfg (models/maskdit.py:559-587): one eval pass at batch 2B, guidance fused in the output
            Fo, _ = self._engine.forward(torch.cat([xf, xf], 0), torch.cat([t, t], 0),
                                         torch.cat([lab, torch.zeros_like(lab)], 0), None, save=False)
            return ops.flow_cfg_out(Fo, B, C, R, p, float(cfg_scale))
        Fo, _ = self._engine.forward(xf, t, lab, None, save=False)
        return ops.flow_cfg_out(Fo, B, C, R, p)

    def forward(self, x, t, class_labels=None, cfg_scale=None, **model_kwargs):
        """{'x': v^ [, 'mask': mask]} of x = x_t at flow time t (a scalar or [B]); the call contract of
        `EDMPrecond.forward` with t in place of sigma."""
        mask_ratio = model_kwargs.pop("mask_ratio", 0)
        mask_dict = model_kwargs.pop("mask_dict", None)
        feat = model_kwargs.pop("feat", None)
        if feat is not None or model_kwargs:
            raise NotImplementedError(f"unsupported arguments: feat / {list(model_kwargs)}")
        self._ready(x.device)
        xf, tt, lab = self._norm_inputs(x, t, class_labels)
        B, p = xf.shape[0], self.model.patch_size
        out = {}
        use_graph = not self.training and os.environ.get("MDT_CUDA_GRAPH", "1") != "0" \
            and not torch.cuda.is_current_stream_capturing()
        if cfg_scale is not None:
            assert self.num_classes and lab is not None
            with torch.no_grad():
                fn = self._eval_graphed if use_graph else self._eval_eager
                out["x"] = fn(xf, tt, lab, cfg_scale).to(x.dtype)
            return out
        if torch.is_grad_enabled() and any(q.requires_grad for q in self.parameters()):
            raise RuntimeError("FlowPrecond.forward has no autograd path: train through Losses['flow'] and evaluate "
                               "under torch.no_grad()")
        md = None
        if mask_ratio > 0:
            L = self.model.num_patches
            if mask_dict is None:
                noise = torch.rand(B, L, device=x.device)  # get_mask, models/maskdit.py:102
                mask_dict = ops.mask_indices(noise, int(L * (1 - mask_ratio)))
            out["mask"] = mask_dict["mask"]
            if self.training:
                md = mask_dict
        if md is None and use_graph:
            out["x"] = self._eval_graphed(xf, tt, lab, None).to(x.dtype)
        else:
            Fo, _ = self._engine.forward(xf, tt, lab, md, save=False)
            out["x"] = ops.flow_cfg_out(Fo, B, self.img_channels, self.img_resolution, p).to(x.dtype)
        return out

    def check_guide(self, guide):
        raise ValueError("autoguidance is not available for flow networks")

    def forward_guided(self, x, sigma, class_labels, guide, guidance):
        raise ValueError("autoguidance is not available for flow networks")


Precond_models = {"edm": EDMPrecond, "flow": FlowPrecond}


def eval_state_dict(net, sd):
    """`sd` ready for `net.load_state_dict` where a network is only evaluated (sampling, guides, the held-out loss):
    `_orig_mod.` prefixes (torch.compile'd checkpoints) removed and, when `net` has no learned loss weighting, the
    `logvar_*` tensors of a run trained with one dropped.  Sampling never reads u(sigma), so such a checkpoint samples
    the same with or without them."""
    sd = {k.replace("_orig_mod.", ""): v for k, v in sd.items()}
    if not getattr(net, "logvar_channels", 0):
        sd = {k: v for k, v in sd.items() if not k.startswith(("logvar_fourier.", "logvar_linear."))}
    return sd
