"""Host-side mirror of the reference model interface (models/maskdit.py) over the H100 engine.

Exports the same registries the reference's entry points consume (SURVEY.md §8b):
    DiT_models      name -> constructor            (models/maskdit.py:709-715)
    Precond_models  {'edm': EDMPrecond}            (models/maskdit.py:779-781)
`EDMPrecond` is an `nn.Module` with the reference's constructor signature, attributes and state-dict key set
(378 entries for XL/2), so `train.py`/`generate.py`-style drivers, `deepcopy` (EMA), `load_state_dict` of reference
checkpoints and the reference's own `EDMLoss`/`edm_sampler` work against it unchanged.  Its arithmetic is the
CUDA engine (`engine.py`); there is no PyTorch fallback: calling it with CPU tensors raises.

Scope (matches every config the reference ships): use_decoder=True, pad_cls_token=False, ext_feature_dim=0,
use_encoder_feat=False, learn_sigma=False.  Other flag combinations raise NotImplementedError.
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
from .engine import Engine, make_engine  # noqa: F401
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
        if not use_decoder:
            raise NotImplementedError("maskdit_b200 implements the asymmetric encoder-decoder MaskDiT "
                                      "(use_decoder=True), as in every reference config")
        self.learn_sigma, self.in_channels, self.out_channels = learn_sigma, in_channels, in_channels
        self.patch_size, self.num_heads, self.class_dropout_prob = patch_size, num_heads, class_dropout_prob
        self.num_classes, self.use_decoder, self.mae_loss_coef = num_classes, use_decoder, mae_loss_coef
        self.pad_cls_token = self.direct_cls_token = False
        self.ext_feature_dim, self.use_encoder_feat = 0, False
        self.cls_token, self.extras, self.decoder_extras = None, 0, 0
        self.input_size, self.hidden_size, self.depth, self.mlp_ratio = input_size, hidden_size, depth, mlp_ratio
        self.decoder_hidden_size, self.decoder_depth, self.decoder_num_heads = 512, 8, 16  # maskdit.py:310-312
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
        self.decoder_pos_embed = P(1, L, Dd, grad=False)
        self.decoder_layer = seq(linear=linear(Dd, D), adaLN_modulation=seq(_1=linear(2 * D, D)))
        self.decoder_blocks = nn.ModuleList([block(Dd, D) for _ in range(self.decoder_depth)])
        self.mask_token = P(1, 1, Dd) if mae_loss_coef > 0 else None
        self.final_layer = seq(linear=linear(patch_size * patch_size * self.out_channels, Dd),
                               adaLN_modulation=seq(_1=linear(2 * Dd, D)))
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


class EDMPrecond(nn.Module):
    """EDM preconditioning wrapper (reference: models/maskdit.py:722-776) running on the sm_90a engine."""

    def __init__(self, img_resolution, img_channels, num_classes=0, sigma_min=0, sigma_max=float("inf"),
                 sigma_data=0.5, model_type="DiT-B/2", **model_kwargs):
        super().__init__()
        self.img_resolution, self.img_channels, self.num_classes = img_resolution, img_channels, num_classes
        self.sigma_min, self.sigma_max, self.sigma_data = sigma_min, sigma_max, sigma_data
        self.model_type = model_type
        self._ctor = dict(img_resolution=img_resolution, img_channels=img_channels, num_classes=num_classes,
                          sigma_min=sigma_min, sigma_max=sigma_max, sigma_data=sigma_data, model_type=model_type,
                          **model_kwargs)
        self.model = DiT_models[model_type](input_size=img_resolution, in_channels=img_channels,
                                            num_classes=num_classes, **model_kwargs)
        self._store, self._engine, self._anchor = None, None, None
        self._graphs = {}  # CUDA graphs of the eval-mode forward, keyed by input shapes (see _eval_graphed)
        self._grad_ready_hook = None  # set by TrainStep: called with (lo, hi) when a gradient range is final

    # -- engine plumbing ---------------------------------------------------------------------------------------
    def _cfg(self):
        c, m = _Cfg(), self.model
        c.hidden, c.depth, c.heads, c.patch = m.hidden_size, m.depth, m.num_heads, m.patch_size
        c.dec_hidden, c.dec_depth, c.dec_heads = m.decoder_hidden_size, m.decoder_depth, m.decoder_num_heads
        c.num_patches, c.num_classes, c.sigma_data = m.num_patches, self.num_classes, self.sigma_data
        c.img_channels, c.patch_dim = self.img_channels, m.patch_size * m.patch_size * m.out_channels
        return c

    def _params(self):
        return dict(self.named_parameters())

    def _ready(self, device):
        """Flatten parameters on `device` (once / after .to()) and refresh the bf16 weight shadow when any
        parameter was modified through PyTorch (optimizer step, load_state_dict, EMA copy...)."""
        if device.type != "cuda":
            raise ops.L.MdtError("maskdit_b200 runs on CUDA (sm_90a) only — there is no CPU fallback")
        params = self._params()
        if self._store is None:
            self._store = FlatStore()
            self._store.plan({k: tuple(p.shape) for k, p in params.items()})
        st = self._store
        if not st.is_attached(params) or st.device != device:
            st.attach(params, device)
            self._engine = make_engine(self._cfg(), st)
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
        self._engine.backward(saved, dF16, on_ready=self._grad_ready_hook)

    def __deepcopy__(self, memo):
        new = EDMPrecond(**copy.deepcopy(self._ctor))
        dev = next(self.parameters()).device
        new.to(dev)
        with torch.no_grad():
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
    def _eval_eager(self, xf, sig, lab, cfg_scale):
        p = self.model.patch_size
        if cfg_scale is not None:
            # forward_with_cfg (models/maskdit.py:559-587): one eval pass at batch 2B, guidance fused in the output
            x2 = torch.cat([xf, xf], 0)
            s2 = torch.cat([sig, sig], 0)
            y2 = torch.cat([lab, torch.zeros_like(lab)], 0)
            Fo, _ = self._engine.forward(x2, s2, y2, None, save=False)
            return ops.cfg_precond_out(Fo, xf, sig, self.sigma_data, float(cfg_scale), p)
        Fo, _ = self._engine.forward(xf, sig, lab, None, save=False)
        return ops.edm_precond_out(Fo, xf, sig, self.sigma_data, p)

    def _eval_graphed(self, xf, sig, lab, cfg_scale):
        """The eval forward is ~280 launches with static shapes: the sampler calls it 35 times per batch and the host
        enqueue time (35 ms per evaluation at B=64) is as long as the device time (38 ms).  It is therefore captured
        once per (shapes, cfg_scale) into a CUDA graph with static input buffers and replayed.  Weights are read from
        the flat bf16 shadow, whose storage is stable (the cache is dropped when the store is re-attached).
        MDT_CUDA_GRAPH=0 disables the graphs."""
        key = (tuple(xf.shape), None if lab is None else tuple(lab.shape), cfg_scale)
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
                self._eval_eager(sx, ss, sl, cfg_scale)
            cur.wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            n0 = ops.L.LAUNCHES
            with torch.cuda.graph(graph):
                out = self._eval_eager(sx, ss, sl, cfg_scale)
            ent = (graph, sx, ss, sl, out, ops.L.LAUNCHES - n0)
            self._graphs[key] = ent
        graph, sx, ss, sl, out, n_launch = ent
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


Precond_models = {"edm": EDMPrecond}
