"""TEST INFRASTRUCTURE ONLY — CPU fp32 restatement (plain PyTorch, functional style) of the reference hot path.

Used by tests/, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline leg as the CHECKER; the product path
(`maskdit_b200/`) never imports it.  It is pinned against the real reference (`/root/reference`, executed
unmodified through oracle/timm_standin.py) by tests/golden/make_golden.py + tests/test_oracle_golden.py.

Every function cites the reference code it restates (file:line under /root/reference).  Parameters are taken from
a flat dict keyed exactly like `EDMPrecond.state_dict()` (SURVEY.md §8 a21).
"""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn.functional as F

# models/maskdit.py:645-715 — (depth, hidden, patch, heads) per registry name
_DIT_TABLE = {
    "DiT-H": (32, 1280, 16), "DiT-XL": (28, 1152, 16), "DiT-L": (24, 1024, 16), "DiT-B": (12, 768, 12),
    "DiT-S": (12, 384, 6),
}


@dataclass
class Cfg:
    """Shape configuration of EDMPrecond(model_type=...) (models/maskdit.py:242-332, 722-741)."""
    model_type: str = "DiT-XL/2"
    img_resolution: int = 32
    img_channels: int = 4
    num_classes: int = 1000
    use_decoder: bool = True
    mae_loss_coef: float = 0.1
    sigma_data: float = 0.5
    # decoder is hard-coded in the reference (models/maskdit.py:310-312)
    dec_hidden: int = 512
    dec_depth: int = 8
    dec_heads: int = 16
    mlp_ratio: float = 4.0

    @property
    def depth(self):
        return _DIT_TABLE[self.model_type.split("/")[0]][0]

    @property
    def hidden(self):
        return _DIT_TABLE[self.model_type.split("/")[0]][1]

    @property
    def heads(self):
        return _DIT_TABLE[self.model_type.split("/")[0]][2]

    @property
    def patch(self):
        return int(self.model_type.split("/")[1])

    @property
    def grid(self):
        return self.img_resolution // self.patch

    @property
    def num_patches(self):
        return self.grid * self.grid

    @property
    def patch_dim(self):
        return self.patch * self.patch * self.img_channels


# ------------------------------------------------------------------------------------------------------------
# fixed tables
# ------------------------------------------------------------------------------------------------------------
def sincos_pos_embed(dim: int, grid: int) -> torch.Tensor:
    """get_2d_sincos_pos_embed (models/maskdit.py:595-642): [grid*grid, dim] fp32.
    First half encodes the w coordinate ("w goes first", :603), second half h; each half = [sin | cos] with
    omega_k = 10000^(-k/(dim/4)), computed in float64 then cast."""
    quarter = dim // 4
    omega = 1.0 / 10000 ** (np.arange(quarter, dtype=np.float64) / quarter)
    hh, ww = np.meshgrid(np.arange(grid, dtype=np.float32), np.arange(grid, dtype=np.float32), indexing="ij")

    def enc(pos):
        out = pos.reshape(-1).astype(np.float64)[:, None] * omega[None, :]
        return np.concatenate([np.sin(out), np.cos(out)], axis=1)

    emb = np.concatenate([enc(ww), enc(hh)], axis=1)
    return torch.from_numpy(emb).float()


def timestep_embedding(t: torch.Tensor, dim: int = 256, max_period: float = 10000.0) -> torch.Tensor:
    """TimestepEmbedder.timestep_embedding (models/maskdit.py:41-58): [cos | sin], freqs exp(-ln(P) k/half)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


# ------------------------------------------------------------------------------------------------------------
# parameters
# ------------------------------------------------------------------------------------------------------------
def param_shapes(cfg: Cfg) -> dict:
    """Key -> shape of `EDMPrecond.state_dict()` for the configs in scope (pad_cls_token=False, no ext features):
    DiT.__init__ models/maskdit.py:242-332."""
    D, Dd, P = cfg.hidden, cfg.dec_hidden, cfg.patch
    H4, Hd4 = int(D * cfg.mlp_ratio), int(Dd * cfg.mlp_ratio)
    s = {}
    s["model.pos_embed"] = (1, cfg.num_patches, D)
    s["model.x_embedder.proj.weight"] = (D, cfg.img_channels, P, P)
    s["model.x_embedder.proj.bias"] = (D,)
    s["model.t_embedder.mlp.0.weight"] = (D, 256)
    s["model.t_embedder.mlp.0.bias"] = (D,)
    s["model.t_embedder.mlp.2.weight"] = (D, D)
    s["model.t_embedder.mlp.2.bias"] = (D,)
    if cfg.num_classes:
        s["model.y_embedder.embedding_table.weight"] = (D, cfg.num_classes)

    def block(prefix, d, h4, cond):
        s[f"{prefix}.attn.qkv.weight"] = (3 * d, d)
        s[f"{prefix}.attn.qkv.bias"] = (3 * d,)
        s[f"{prefix}.attn.proj.weight"] = (d, d)
        s[f"{prefix}.attn.proj.bias"] = (d,)
        s[f"{prefix}.mlp.fc1.weight"] = (h4, d)
        s[f"{prefix}.mlp.fc1.bias"] = (h4,)
        s[f"{prefix}.mlp.fc2.weight"] = (d, h4)
        s[f"{prefix}.mlp.fc2.bias"] = (d,)
        s[f"{prefix}.adaLN_modulation.1.weight"] = (6 * d, cond)
        s[f"{prefix}.adaLN_modulation.1.bias"] = (6 * d,)

    for i in range(cfg.depth):
        block(f"model.blocks.{i}", D, H4, D)
    fin = D
    if cfg.use_decoder:
        s["model.decoder_pos_embed"] = (1, cfg.num_patches, Dd)
        s["model.decoder_layer.linear.weight"] = (Dd, D)
        s["model.decoder_layer.linear.bias"] = (Dd,)
        s["model.decoder_layer.adaLN_modulation.1.weight"] = (2 * D, D)
        s["model.decoder_layer.adaLN_modulation.1.bias"] = (2 * D,)
        for i in range(cfg.dec_depth):
            block(f"model.decoder_blocks.{i}", Dd, Hd4, D)
        if cfg.mae_loss_coef > 0:
            s["model.mask_token"] = (1, 1, Dd)
        fin = Dd
    s["model.final_layer.linear.weight"] = (cfg.patch_dim, fin)
    s["model.final_layer.linear.bias"] = (cfg.patch_dim,)
    s["model.final_layer.adaLN_modulation.1.weight"] = (2 * fin, D)
    s["model.final_layer.adaLN_modulation.1.bias"] = (2 * fin,)
    return s


def make_state_dict(cfg: Cfg, seed: int = 1, dtype=torch.float32) -> dict:
    """Deterministic, structure-independent weights for parity work: every trainable tensor ~ N(0, std) drawn from
    a CPU generator seeded by (seed, crc32(key)).  This ALSO randomises the 227 tensors the reference zero-inits
    (models/maskdit.py:375-408) — with those at zero the net is the identity and any comparison is vacuous
    (SURVEY.md §3.3).  pos-embeds are the fixed sin-cos tables."""
    sd = {}
    for key, shape in param_shapes(cfg).items():
        if key.endswith("pos_embed"):
            sd[key] = sincos_pos_embed(shape[-1], cfg.grid).unsqueeze(0).to(dtype)
            continue
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(key.encode())) % (1 << 31))
        fan_in = int(np.prod(shape[1:])) if len(shape) > 1 else shape[0]
        if key.endswith(".bias") or "mask_token" in key:
            std = 0.02
        elif "adaLN_modulation" in key:
            std = 0.5 / math.sqrt(fan_in)      # keeps shift/scale/gate O(0.5) so every branch matters
        else:
            std = 1.0 / math.sqrt(fan_in)
        sd[key] = (torch.randn(shape, generator=g, dtype=torch.float32) * std).to(dtype)
    return sd


# ------------------------------------------------------------------------------------------------------------
# mask path (integer; bit-exact contract)
# ------------------------------------------------------------------------------------------------------------
def mask_from_noise(noise: torch.Tensor, mask_ratio: float) -> dict:
    """get_mask (models/maskdit.py:88-113) for a GIVEN noise tensor [B, L]; ties broken by ascending index."""
    B, L = noise.shape
    len_keep = int(L * (1 - mask_ratio))
    ids_shuffle = torch.argsort(noise, dim=1, stable=True)
    ids_restore = torch.argsort(ids_shuffle, dim=1, stable=True)
    ids_keep = ids_shuffle[:, :len_keep]
    mask = (ids_restore >= len_keep).to(torch.float32)
    return {"mask": mask, "ids_keep": ids_keep, "ids_restore": ids_restore}


# ------------------------------------------------------------------------------------------------------------
# network
# ------------------------------------------------------------------------------------------------------------
def _ln(x, eps=1e-6):
    return F.layer_norm(x, (x.shape[-1],), eps=eps)


def _modulate(x, shift, scale):
    """modulate (models/maskdit.py:19-20)."""
    return x * (1 + scale.unsqueeze(1)) + shift.unsqueeze(1)


def _attention(sd, p, x, heads):
    """timm Attention as constructed at models/maskdit.py:178 (qkv_bias=True)."""
    B, N, C = x.shape
    qkv = F.linear(x, sd[f"{p}.qkv.weight"], sd[f"{p}.qkv.bias"]).reshape(B, N, 3, heads, C // heads)
    q, k, v = qkv.permute(2, 0, 3, 1, 4).unbind(0)
    att = torch.softmax((q @ k.transpose(-2, -1)) * (C // heads) ** -0.5, dim=-1)
    o = (att @ v).transpose(1, 2).reshape(B, N, C)
    return F.linear(o, sd[f"{p}.proj.weight"], sd[f"{p}.proj.bias"])


def _block(sd, p, x, c, heads):
    """DiTBlock.forward (models/maskdit.py:188-192)."""
    mod = F.linear(F.silu(c), sd[f"{p}.adaLN_modulation.1.weight"], sd[f"{p}.adaLN_modulation.1.bias"])
    sh1, sc1, g1, sh2, sc2, g2 = mod.chunk(6, dim=1)
    x = x + g1.unsqueeze(1) * _attention(sd, f"{p}.attn", _modulate(_ln(x), sh1, sc1), heads)
    h = F.linear(_modulate(_ln(x), sh2, sc2), sd[f"{p}.mlp.fc1.weight"], sd[f"{p}.mlp.fc1.bias"])
    h = F.linear(F.gelu(h, approximate="tanh"), sd[f"{p}.mlp.fc2.weight"], sd[f"{p}.mlp.fc2.bias"])
    return x + g2.unsqueeze(1) * h


def patchify(imgs, p, c):
    """train_utils/loss.py:73-85: [N,C,H,W] -> [N, L, p*p*C], patch vector ordered (ph, pw, c)."""
    n, _, hh, ww = imgs.shape
    h, w = hh // p, ww // p
    return imgs.reshape(n, c, h, p, w, p).permute(0, 2, 4, 3, 5, 1).reshape(n, h * w, p * p * c)


def unpatchify(x, p, c):
    """DiT.unpatchify (models/maskdit.py:411-424): inverse of patchify."""
    n, L, _ = x.shape
    h = w = int(round(L ** 0.5))
    return x.reshape(n, h, w, p, p, c).permute(0, 5, 1, 3, 2, 4).reshape(n, c, h * p, w * p)


def dit_forward(sd, cfg: Cfg, x, t, y, mask_dict=None, training=True):
    """DiT.forward + forward_encoder (models/maskdit.py:467-557) for pad_cls_token=False, no external features.
    `mask_dict` None => no masking.  Returns F_x [B,C,R,R]."""
    D, P = cfg.hidden, cfg.patch
    B = x.shape[0]
    # PatchEmbed == Linear over (c, ph, pw)-ordered patches (timm PatchEmbed, ctor :278) + pos_embed (:475)
    w = sd["model.x_embedder.proj.weight"].reshape(D, -1)
    patches = x.reshape(B, cfg.img_channels, cfg.grid, P, cfg.grid, P).permute(0, 2, 4, 1, 3, 5).reshape(
        B, cfg.num_patches, -1)
    h = F.linear(patches, w, sd["model.x_embedder.proj.bias"]) + sd["model.pos_embed"]
    masked = mask_dict is not None
    if masked and training:  # mask_out_token (:116-127, :482-483)
        idx = mask_dict["ids_keep"].unsqueeze(-1).expand(-1, -1, D)
        h = torch.gather(h, 1, idx)
    # conditioning (:491-495): t-MLP (:34-38) + label table (:75,80)
    # the frequency embedding is computed in float32 as the reference does; a float64 run casts it up
    te = F.linear(timestep_embedding(t, 256).to(x.dtype), sd["model.t_embedder.mlp.0.weight"],
                  sd["model.t_embedder.mlp.0.bias"])
    c = F.linear(F.silu(te), sd["model.t_embedder.mlp.2.weight"], sd["model.t_embedder.mlp.2.bias"])
    if cfg.num_classes:
        c = c + F.linear(y, sd["model.y_embedder.embedding_table.weight"])
    for i in range(cfg.depth):
        h = _block(sd, f"model.blocks.{i}", h, c, cfg.heads)
    if cfg.use_decoder:
        # DecoderLayer (:209-213)
        sh, sc = F.linear(F.silu(c), sd["model.decoder_layer.adaLN_modulation.1.weight"],
                          sd["model.decoder_layer.adaLN_modulation.1.bias"]).chunk(2, dim=1)
        h = F.linear(_modulate(_ln(h), sh, sc), sd["model.decoder_layer.linear.weight"],
                     sd["model.decoder_layer.linear.bias"])
        if masked and training:  # unmask_tokens (:157-163, :539-543) == scatter + mask_token fill
            L, Dd = cfg.num_patches, cfg.dec_hidden
            tok = sd.get("model.mask_token", torch.zeros(1, 1, Dd, dtype=h.dtype))
            full = tok.expand(B, L, Dd).clone()
            full = full.scatter(1, mask_dict["ids_keep"].unsqueeze(-1).expand(-1, -1, Dd), h)
            h = full
        h = h + sd["model.decoder_pos_embed"]
        for i in range(cfg.dec_depth):
            h = _block(sd, f"model.decoder_blocks.{i}", h, c, cfg.dec_heads)
    # FinalLayer (:230-234)
    sh, sc = F.linear(F.silu(c), sd["model.final_layer.adaLN_modulation.1.weight"],
                      sd["model.final_layer.adaLN_modulation.1.bias"]).chunk(2, dim=1)
    out = F.linear(_modulate(_ln(h), sh, sc), sd["model.final_layer.linear.weight"],
                   sd["model.final_layer.linear.bias"])
    return unpatchify(out, P, cfg.img_channels)


def edm_precond(sd, cfg: Cfg, x, sigma, labels=None, cfg_scale=None, mask_dict=None, training=True):
    """EDMPrecond.forward (models/maskdit.py:756-773) incl. forward_with_cfg (:559-587).  Returns D_x."""
    sd_ = cfg.sigma_data
    sigma = sigma.to(x.dtype).reshape(-1, 1, 1, 1)
    B = x.shape[0]
    if labels is None:
        labels = torch.zeros(B, cfg.num_classes, dtype=x.dtype)
    c_skip = sd_ ** 2 / (sigma ** 2 + sd_ ** 2)
    c_out = sigma * sd_ / (sigma ** 2 + sd_ ** 2).sqrt()
    c_in = 1 / (sd_ ** 2 + sigma ** 2).sqrt()
    c_noise = (sigma.log() / 4).flatten()
    xin = c_in * x
    if cfg_scale is None:
        t = c_noise.expand(B) if c_noise.numel() == 1 else c_noise
        Fx = dit_forward(sd, cfg, xin, t, labels, mask_dict=mask_dict, training=training)
    else:
        x2 = torch.cat([xin, xin], 0)
        y2 = torch.cat([labels, torch.zeros_like(labels)], 0)
        t = c_noise.expand(2 * B) if c_noise.numel() == 1 else torch.cat([c_noise, c_noise], 0)
        out = dit_forward(sd, cfg, x2, t, y2, mask_dict=None, training=False)
        cond, unc = out[:B], out[B:]
        Fx = unc + cfg_scale * (cond - unc)
    return c_skip * x + c_out * Fx


def edm_loss(sd, cfg: Cfg, images, labels, rnd_normal, noise_unit, mask_dict, mae_loss_coef,
             P_mean=-1.2, P_std=1.2):
    """EDMLoss.__call__ (train_utils/loss.py:28-60) with the random draws passed in:
    rnd_normal [B,1,1,1] (loss.py:35), noise_unit = randn_like(images) (loss.py:39)."""
    sd_ = cfg.sigma_data
    sigma = (rnd_normal * P_std + P_mean).exp()
    weight = (sigma ** 2 + sd_ ** 2) / (sigma * sd_) ** 2
    yn = images + noise_unit * sigma
    D = edm_precond(sd, cfg, yn, sigma, labels, mask_dict=mask_dict, training=True)
    loss = weight * (D - images) ** 2
    if mask_dict is None:
        return loss.mean(dim=(1, 2, 3)), D
    p = cfg.patch
    per_patch = F.avg_pool2d(loss.mean(dim=1), p).flatten(1)       # loss.py:47
    unmask = 1 - mask_dict["mask"]
    out = (per_patch * unmask).sum(1) / unmask.sum(1)               # loss.py:48-49
    if mae_loss_coef > 0:                                           # mae_loss, loss.py:87-101
        tgt = patchify(yn, p, cfg.img_channels)
        prd = patchify(D, p, cfg.img_channels)
        tgt = (tgt - tgt.mean(-1, keepdim=True)) / (tgt.var(-1, keepdim=True) + 1e-6) ** 0.5
        mae = ((prd - tgt) ** 2).mean(-1)
        m = mask_dict["mask"]
        out = out + mae_loss_coef * (mae * m).sum(1) / m.sum(1)
    return out, D


def edm_sampler(denoise, latents, num_steps=18, sigma_min=0.002, sigma_max=80.0, rho=7.0, net_sigma_min=0.0,
                net_sigma_max=float("inf"), S_churn=0.0, S_min=0.0, S_max=float("inf"), S_noise=1.0,
                randn_like=torch.randn_like):
    """edm_sampler (sample.py:30-66), including the stochastic churn (sample.py:50-53: gamma, t_hat, noise
    injection; `randn_like` is consumed once per step even when gamma = 0, as in the reference).
    `denoise(x_f32, sigma_f64)` returns the network output; state is float64.
    Returns (x_final, list of sigmas evaluated)."""
    sigma_min, sigma_max = max(sigma_min, net_sigma_min), min(sigma_max, net_sigma_max)
    idx = torch.arange(num_steps, dtype=torch.float64)
    t_steps = (sigma_max ** (1 / rho) + idx / (num_steps - 1) * (sigma_min ** (1 / rho) - sigma_max ** (1 / rho))) ** rho
    t_steps = torch.cat([t_steps, torch.zeros_like(t_steps[:1])])
    x_next = latents.to(torch.float64) * t_steps[0]
    evals = []
    for i, (t_cur, t_next) in enumerate(zip(t_steps[:-1], t_steps[1:])):
        x_cur = x_next
        gamma = min(S_churn / num_steps, math.sqrt(2.0) - 1) if S_min <= t_cur <= S_max else 0
        t_hat = t_cur + gamma * t_cur
        x_hat = x_cur + (t_hat ** 2 - t_cur ** 2).sqrt() * S_noise * randn_like(x_cur)
        evals.append(float(t_hat))
        den = denoise(x_hat.float(), t_hat).to(torch.float64)
        d_cur = (x_hat - den) / t_hat
        x_next = x_hat + (t_next - t_hat) * d_cur
        if i < num_steps - 1:
            evals.append(float(t_next))
            den = denoise(x_next.float(), t_next).to(torch.float64)
            d_prime = (x_next - den) / t_next
            x_next = x_hat + (t_next - t_hat) * (0.5 * d_cur + 0.5 * d_prime)
    return x_next, evals


def adamw_ema_step(w, g, m, v, ema, step, lr=1e-4, b1=0.9, b2=0.999, eps=1e-8, wd=0.0, ema_decay=0.9999):
    """apex FusedAdam(adam_w_mode=True) as configured at train.py:141 (== torch.optim.AdamW) followed by
    update_ema (train_utils/helper.py:47-58).  In-place on fp32 tensors."""
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    w.mul_(1 - lr * wd)
    w.addcdiv_(m / bc1, (v / bc2).sqrt() + eps, value=-lr)
    if ema is not None:
        ema.mul_(ema_decay).add_(w, alpha=1 - ema_decay)


def step_front(moments, eps, rnd_normal, noise_unit, labels=None, drop_u=None, drop_prob=0.0, scale_factor=0.18215,
               P_mean=-1.2, P_std=1.2):
    """The step front of the reference's training loop given the pre-drawn randoms: utils.sample (utils.py:59-65),
    label dropout (train.py:209), sigma draw + noise injection (train_utils/loss.py:35-39).
    Returns (y, yn, sigma [B], labels)."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    std = torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0))
    y = scale_factor * (mean + std * eps)
    if labels is not None and drop_u is not None and drop_prob > 0:
        labels = labels * (drop_u.reshape(-1, 1) >= drop_prob)
    sigma = (rnd_normal.reshape(-1, 1, 1, 1) * P_std + P_mean).exp()
    return y, y + noise_unit * sigma, sigma.reshape(-1), labels


def lr_schedule(train_steps, base_lr, global_batch, rampup_kimg):
    """train.py:223, with `train_steps` the 0-based counter incremented after the update (train.py:232)."""
    return base_lr * min(train_steps * global_batch / max(rampup_kimg * 1000, 1e-8), 1)


def rank_batches(seeds, max_batch_size, rank, size):
    """sample.py:232-235: seeds -> this rank's batches (tensor_split into a multiple of `size` parts, rank-strided)."""
    num_batches = ((len(seeds) - 1) // (max_batch_size * size) + 1) * size
    return [b.tolist() for b in torch.as_tensor(seeds).tensor_split(num_batches)[rank::size]]


def ablation_sampler(denoise, latents, randn_like=torch.randn_like, num_steps=18, sigma_min=None, sigma_max=None,
                     rho=7, solver="heun", discretization="edm", schedule="linear", scaling="none", epsilon_s=1e-3,
                     C_1=0.001, C_2=0.008, M=1000, alpha=1, S_churn=0, S_min=0, S_max=float("inf"), S_noise=1,
                     net_sigma_min=0.0, net_sigma_max=float("inf")):
    """sample.py:73-188 restated with every schedule quantity a host-side fp64 scalar (the reference keeps them as
    0-d fp64 tensors; `round_sigma` is the identity for EDMPrecond, models/maskdit.py:775).
    `denoise(x_f32, sigma_float)` -> D.  Returns (x fp64, list of evaluated sigmas)."""
    t64 = lambda v: torch.as_tensor(v, dtype=torch.float64)  # noqa: E731
    vp_sigma = lambda bd, bm: (lambda t: float((np.e ** (0.5 * bd * (t ** 2) + bm * t) - 1) ** 0.5))  # noqa: E731
    if sigma_min is None:
        sigma_min = {"vp": vp_sigma(19.1, 0.1)(epsilon_s), "ve": 0.02, "iddpm": 0.002, "edm": 0.002}[discretization]
    if sigma_max is None:
        sigma_max = {"vp": vp_sigma(19.1, 0.1)(1), "ve": 100, "iddpm": 81, "edm": 80}[discretization]
    sigma_min, sigma_max = max(sigma_min, net_sigma_min), min(sigma_max, net_sigma_max)
    bd = 2 * (np.log(sigma_min ** 2 + 1) / epsilon_s - np.log(sigma_max ** 2 + 1)) / (epsilon_s - 1)   # sample.py:109
    bm = np.log(sigma_max ** 2 + 1) - 0.5 * bd
    idx = np.arange(num_steps, dtype=np.float64)
    if discretization == "vp":
        sig_steps = np.array([vp_sigma(bd, bm)(t) for t in 1 + idx / (num_steps - 1) * (epsilon_s - 1)])
    elif discretization == "ve":
        sig_steps = np.sqrt((sigma_max ** 2) * ((sigma_min ** 2 / sigma_max ** 2) ** (idx / (num_steps - 1))))
    elif discretization == "iddpm":
        # sample.py:118-121: `j` is an int64 tensor, so alpha_bar is evaluated in torch's default FLOAT32 (int tensor x
        # python float) while u accumulates in fp64 - the type promotion is part of the reference's numbers.
        ut = torch.zeros(M + 1, dtype=torch.float64)
        abar = lambda j: (0.5 * np.pi * j / M / (C_2 + 1)).sin() ** 2  # noqa: E731
        for j in torch.arange(M, 0, -1):
            ut[j - 1] = ((ut[j] ** 2 + 1) / (abar(j - 1) / abar(j)).clip(min=C_1) - 1).sqrt()
        u = ut.numpy()
        uf = u[np.logical_and(u >= sigma_min, u <= sigma_max)]
        sig_steps = uf[np.round((len(uf) - 1) / (num_steps - 1) * idx).astype(np.int64)]
    else:
        sig_steps = (sigma_max ** (1 / rho) + idx / (num_steps - 1) * (sigma_min ** (1 / rho) - sigma_max ** (1 / rho))) ** rho
    if schedule == "vp":
        sigma = vp_sigma(bd, bm)
        sigma_deriv = lambda t: 0.5 * (bm + bd * t) * (sigma(t) + 1 / sigma(t))  # noqa: E731
        sigma_inv = lambda s_: (np.sqrt(bm ** 2 + 2 * bd * np.log(s_ ** 2 + 1)) - bm) / bd  # noqa: E731
    elif schedule == "ve":
        sigma, sigma_deriv, sigma_inv = (lambda t: np.sqrt(t)), (lambda t: 0.5 / np.sqrt(t)), (lambda s_: s_ ** 2)
    else:
        sigma, sigma_deriv, sigma_inv = (lambda t: t), (lambda t: 1.0), (lambda s_: s_)
    if scaling == "vp":
        s = lambda t: 1 / np.sqrt(1 + sigma(t) ** 2)  # noqa: E731
        s_deriv = lambda t: -sigma(t) * sigma_deriv(t) * (s(t) ** 3)  # noqa: E731
    else:
        s, s_deriv = (lambda t: 1.0), (lambda t: 0.0)
    t_steps = [float(sigma_inv(v)) for v in sig_steps] + [0.0]
    evals = []
    x_next = latents.to(torch.float64) * (sigma(t_steps[0]) * s(t_steps[0]))
    for i in range(num_steps):
        t_cur, t_next = t_steps[i], t_steps[i + 1]
        x_cur = x_next
        gamma = min(S_churn / num_steps, np.sqrt(2) - 1) if S_min <= sigma(t_cur) <= S_max else 0
        t_hat = float(sigma_inv(sigma(t_cur) + gamma * sigma(t_cur)))
        x_hat = s(t_hat) / s(t_cur) * x_cur + float(np.sqrt(max(sigma(t_hat) ** 2 - sigma(t_cur) ** 2, 0))) * s(
            t_hat) * S_noise * randn_like(x_cur)
        h = t_next - t_hat
        evals.append(float(sigma(t_hat)))
        den = denoise((x_hat / s(t_hat)).float(), t64(sigma(t_hat))).to(torch.float64)
        d_cur = (sigma_deriv(t_hat) / sigma(t_hat) + s_deriv(t_hat) / s(t_hat)) * x_hat - sigma_deriv(t_hat) * s(
            t_hat) / sigma(t_hat) * den
        x_prime, t_prime = x_hat + alpha * h * d_cur, t_hat + alpha * h
        if solver == "euler" or i == num_steps - 1:
            x_next = x_hat + h * d_cur
        else:
            evals.append(float(sigma(t_prime)))
            den = denoise((x_prime / s(t_prime)).float(), t64(sigma(t_prime))).to(torch.float64)
            d_prime = (sigma_deriv(t_prime) / sigma(t_prime) + s_deriv(t_prime) / s(t_prime)) * x_prime - \
                sigma_deriv(t_prime) * s(t_prime) / sigma(t_prime) * den
            x_next = x_hat + h * ((1 - 1 / (2 * alpha)) * d_cur + 1 / (2 * alpha) * d_prime)
    return x_next, evals
