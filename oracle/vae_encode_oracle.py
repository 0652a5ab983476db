"""TEST INFRASTRUCTURE ONLY — CPU fp32 restatement of the reference's SD-VAE ENCODE path (Encoder.forward + quant_conv
+ sample, autoencoder.py:212-303,431-446), the data preparation that extract_latent.py:66 runs on every image.
The product path (`maskdit_b200/vae.py`) never imports it; it is pinned against the unmodified reference module
(`autoencoder.FrozenAutoencoderKL`) by tests/golden/make_golden_encode.py + tests/test_vae_encode.py.

Parameters are a flat dict keyed like `FrozenAutoencoderKL.state_dict()` (`encoder.*`, `quant_conv.*`).  The building
blocks (GroupNorm, swish, ResnetBlock, AttnBlock) are the decode oracle's.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.vae_oracle import CH, CH_MULT, NUM_RES_BLOCKS, Z_CH, _attn, _conv, _gn, _resblock, _swish

IN_CH = 3


def encoder_param_shapes():
    """Key -> shape of `encoder` + `quant_conv` (autoencoder.py:212-279, :422), in registration order."""
    out = {"encoder.conv_in.weight": (CH, IN_CH, 3, 3), "encoder.conv_in.bias": (CH,)}

    def res(p, cin, cout):
        out[f"{p}.norm1.weight"], out[f"{p}.norm1.bias"] = (cin,), (cin,)
        out[f"{p}.conv1.weight"], out[f"{p}.conv1.bias"] = (cout, cin, 3, 3), (cout,)
        out[f"{p}.norm2.weight"], out[f"{p}.norm2.bias"] = (cout,), (cout,)
        out[f"{p}.conv2.weight"], out[f"{p}.conv2.bias"] = (cout, cout, 3, 3), (cout,)
        if cin != cout:
            out[f"{p}.nin_shortcut.weight"], out[f"{p}.nin_shortcut.bias"] = (cout, cin, 1, 1), (cout,)

    block_in = CH
    for lvl, mult in enumerate(CH_MULT):
        for i in range(NUM_RES_BLOCKS):
            res(f"encoder.down.{lvl}.block.{i}", block_in, CH * mult)
            block_in = CH * mult
        if lvl != len(CH_MULT) - 1:
            out[f"encoder.down.{lvl}.downsample.conv.weight"] = (block_in, block_in, 3, 3)
            out[f"encoder.down.{lvl}.downsample.conv.bias"] = (block_in,)
    res("encoder.mid.block_1", block_in, block_in)
    p = "encoder.mid.attn_1"
    out[f"{p}.norm.weight"], out[f"{p}.norm.bias"] = (block_in,), (block_in,)
    for n in ("q", "k", "v", "proj_out"):
        out[f"{p}.{n}.weight"], out[f"{p}.{n}.bias"] = (block_in, block_in, 1, 1), (block_in,)
    res("encoder.mid.block_2", block_in, block_in)
    out["encoder.norm_out.weight"], out["encoder.norm_out.bias"] = (block_in,), (block_in,)
    out["encoder.conv_out.weight"], out["encoder.conv_out.bias"] = (2 * Z_CH, block_in, 3, 3), (2 * Z_CH,)
    out["quant_conv.weight"], out["quant_conv.bias"] = (2 * Z_CH, 2 * Z_CH, 1, 1), (2 * Z_CH,)
    return out


def make_vae_encoder_state_dict(seed=4):
    """Deterministic stand-in weights for the encode half, drawn from their own generator with the decode stand-in's
    rule (conv weights N(0, 1/fan_in), GroupNorm scales 1 + 0.1 N(0,1), biases 0.05 N(0,1))."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in encoder_param_shapes().items():
        if k.endswith("weight") and len(shp) == 4:
            fan_in = shp[1] * shp[2] * shp[3]
            sd[k] = torch.randn(shp, generator=g) * fan_in ** -0.5
        elif k.endswith("weight"):
            sd[k] = 1 + 0.1 * torch.randn(shp, generator=g)
        else:
            sd[k] = 0.05 * torch.randn(shp, generator=g)
    return sd


def encode_moments(sd, x):
    """FrozenAutoencoderKL.encode_moments (autoencoder.py:431-434): images [B,3,H,W] -> moments [B,8,H/8,W/8]."""
    h = _conv(sd, "encoder.conv_in", x, 1)
    for lvl in range(len(CH_MULT)):
        for i in range(NUM_RES_BLOCKS):
            h = _resblock(sd, f"encoder.down.{lvl}.block.{i}", h)
        if lvl != len(CH_MULT) - 1:                                                      # Downsample.forward, :68-72
            p = f"encoder.down.{lvl}.downsample.conv"
            h = F.conv2d(F.pad(h, (0, 1, 0, 1)), sd[f"{p}.weight"], sd[f"{p}.bias"], stride=2)
    h = _resblock(sd, "encoder.mid.block_1", h)
    h = _attn(sd, "encoder.mid.attn_1", h)
    h = _resblock(sd, "encoder.mid.block_2", h)
    h = _conv(sd, "encoder.conv_out", _swish(_gn(sd, "encoder.norm_out", h)), 1)
    return _conv(sd, "quant_conv", h, 0)


def sample(moments, eps, scale_factor=0.18215):
    """FrozenAutoencoderKL.sample (autoencoder.py:436-442) with the normal draw given."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    return scale_factor * (mean + torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0)) * eps)
