"""SD-VAE on the H100 kernels: both halves of the reference's `FrozenAutoencoderKL` (autoencoder.py:415-463).

Decode is the sampler tail (sample.py:275 `images = vae.decode(z)`, autoencoder.py:306-453), so that `generate.py` ends
in images as `generate_with_net` does.  `AutoencoderKLDecoder` holds `post_quant_conv.*` and `decoder.*` under the
reference's state-dict keys (an `autoencoder_kl.pth` written for `FrozenAutoencoderKL` loads with `strict=False`: the
encoder half is ignored) and `decode(z)` returns the `[B, 3, 8h, 8w]` image the reference's `decode` returns.

Encode is the data preparation in front of training (extract_latent.py:66 `model(img, fn='encode_moments')`,
autoencoder.py:212-303,431-446): `AutoencoderKLEncoder` holds `encoder.*` and `quant_conv.*` and returns the
`[B, 8, H/8, W/8]` moments that `train.py` reads from the latent LMDB.

Every convolution is the wgmma GEMM on an im2col operand with GroupNorm + swish + nearest upsample (decode) or the
stride-2 Downsample window (encode) fused into its construction (csrc/vae.cu); activations are pixel-major fp32 row
matrices.  No PyTorch arithmetic on the path (torch only lays out the weights once).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops
from .ops import bf16, f32

CH, CH_MULT, NUM_RES_BLOCKS, Z_CH, OUT_CH = 128, (1, 2, 4, 4), 2, 4, 3   # autoencoder.py:466-479 (get_model)


class _Node(nn.Module):
    """Container whose children are created on demand, so parameters can live under the reference's dotted names."""

    def child(self, name):
        if name not in self._modules:
            self.add_module(name, _Node())
        return self._modules[name]


def _res_shapes(out, p, cin, cout):
    """ResnetBlock parameters (autoencoder.py:79-115, temb_channels = 0) appended to `out` in registration order."""
    out.extend([(f"{p}.norm1.weight", (cin,)), (f"{p}.norm1.bias", (cin,)), (f"{p}.conv1.weight", (cout, cin, 3, 3)),
                (f"{p}.conv1.bias", (cout,)), (f"{p}.norm2.weight", (cout,)), (f"{p}.norm2.bias", (cout,)),
                (f"{p}.conv2.weight", (cout, cout, 3, 3)), (f"{p}.conv2.bias", (cout,))])
    if cin != cout:
        out.extend([(f"{p}.nin_shortcut.weight", (cout, cin, 1, 1)), (f"{p}.nin_shortcut.bias", (cout,))])


def _attn_shapes(out, p, c):
    """AttnBlock parameters (autoencoder.py:141-172)."""
    out.extend([(f"{p}.norm.weight", (c,)), (f"{p}.norm.bias", (c,))])
    for n in ("q", "k", "v", "proj_out"):
        out.extend([(f"{p}.{n}.weight", (c, c, 1, 1)), (f"{p}.{n}.bias", (c,))])


def _shapes():
    """(key, shape) of post_quant_conv + decoder in the reference's registration order (autoencoder.py:307-377, :424)."""
    out = []
    out.extend([("post_quant_conv.weight", (Z_CH, 4, 1, 1)), ("post_quant_conv.bias", (Z_CH,))])
    c = CH * CH_MULT[-1]
    out.extend([("decoder.conv_in.weight", (c, Z_CH, 3, 3)), ("decoder.conv_in.bias", (c,))])
    _res_shapes(out, "decoder.mid.block_1", c, c)
    _attn_shapes(out, "decoder.mid.attn_1", c)
    _res_shapes(out, "decoder.mid.block_2", c, c)
    plan, cur = {}, c
    for lvl in reversed(range(len(CH_MULT))):
        for i in range(NUM_RES_BLOCKS + 1):
            plan[(lvl, i)] = (cur, CH * CH_MULT[lvl])
            cur = CH * CH_MULT[lvl]
        plan[(lvl, "up")] = cur
    for lvl in range(len(CH_MULT)):
        for i in range(NUM_RES_BLOCKS + 1):
            _res_shapes(out, f"decoder.up.{lvl}.block.{i}", *plan[(lvl, i)])
        if lvl != 0:
            cu = plan[(lvl, "up")]
            out.extend([(f"decoder.up.{lvl}.upsample.conv.weight", (cu, cu, 3, 3)),
                        (f"decoder.up.{lvl}.upsample.conv.bias", (cu,))])
    out.extend([("decoder.norm_out.weight", (CH,)), ("decoder.norm_out.bias", (CH,)),
                ("decoder.conv_out.weight", (OUT_CH, CH, 3, 3)), ("decoder.conv_out.bias", (OUT_CH,))])
    return out, plan


def _encoder_shapes():
    """(key, shape) of encoder + quant_conv in the reference's registration order (autoencoder.py:212-279, :422):
    conv_in, down.{0..3} (two ResnetBlocks each, a Downsample conv below the last level), mid, norm_out, conv_out."""
    out = []
    out.extend([("encoder.conv_in.weight", (CH, OUT_CH, 3, 3)), ("encoder.conv_in.bias", (CH,))])
    block_in = CH
    for lvl, mult in enumerate(CH_MULT):
        for i in range(NUM_RES_BLOCKS):
            _res_shapes(out, f"encoder.down.{lvl}.block.{i}", block_in, CH * mult)
            block_in = CH * mult
        if lvl != len(CH_MULT) - 1:
            out.extend([(f"encoder.down.{lvl}.downsample.conv.weight", (block_in, block_in, 3, 3)),
                        (f"encoder.down.{lvl}.downsample.conv.bias", (block_in,))])
    _res_shapes(out, "encoder.mid.block_1", block_in, block_in)
    _attn_shapes(out, "encoder.mid.attn_1", block_in)
    _res_shapes(out, "encoder.mid.block_2", block_in, block_in)
    out.extend([("encoder.norm_out.weight", (block_in,)), ("encoder.norm_out.bias", (block_in,)),
                ("encoder.conv_out.weight", (2 * Z_CH, block_in, 3, 3)), ("encoder.conv_out.bias", (2 * Z_CH,)),
                ("quant_conv.weight", (2 * Z_CH, 2 * Z_CH, 1, 1)), ("quant_conv.bias", (2 * Z_CH,))])
    return out


class _AutoencoderKLHalf(nn.Module):
    """What both halves share: parameters under the reference's dotted keys, their GEMM-layout bf16 packing, and the
    convolution / ResnetBlock / AttnBlock building blocks over pixel-major fp32 rows."""

    _UNPACKED = ()      # 1x1 convolutions run by a dedicated kernel on fp32 weights (post_quant_conv / quant_conv)
    _CIN_PAD = {}       # conv weight key -> input channels it is zero-padded to before packing

    def __init__(self, shapes, scale_factor, max_rows):
        super().__init__()
        self.scale_factor = scale_factor
        self.max_rows = max_rows          # im2col operands are built for at most this many output pixels at a time
        self._keys = [k for k, _ in shapes]
        for k, shp in shapes:
            node, parts = self, k.split(".")
            for part in parts[:-1]:
                node = node.child(part) if isinstance(node, _Node) else self._root_child(part)
            node.register_parameter(parts[-1], nn.Parameter(torch.zeros(shp), requires_grad=False))
        self._packed, self._versions = {}, None

    def _root_child(self, name):
        if name not in self._modules:
            self.add_module(name, _Node())
        return self._modules[name]

    # -- weights ---------------------------------------------------------------------------------------------------
    def _p(self, key):
        node = self
        for part in key.split("."):
            node = node._modules[part] if part in node._modules else node._parameters[part]
        return node

    def _ready(self):
        """(Re)build the GEMM-layout bf16 weights when a parameter changed: conv weight [Co,Ci,kh,kw] -> [Co, (kh,kw,Ci)]
        padded to a multiple of 8 columns."""
        ver = (sum(self._p(k)._version for k in self._keys), self._p(self._keys[0]).data_ptr())
        if self._versions == ver:
            return
        self._packed = {}
        for k in self._keys:
            w = self._p(k)
            if not w.is_cuda:
                raise ops.L.MdtError("maskdit_b200 runs on CUDA (sm_90a) only — there is no CPU fallback")
            if k.endswith(".weight") and w.ndim == 4 and not k.startswith(self._UNPACKED):
                w = w.detach()
                co, ci, kh, kw = w.shape
                if k in self._CIN_PAD:
                    ci = self._CIN_PAD[k]
                    w = torch.cat([w, w.new_zeros(co, ci - w.shape[1], kh, kw)], dim=1)
                K = kh * kw * ci
                Kp = (K + 7) // 8 * 8
                flat = torch.zeros(co, Kp, dtype=f32, device=w.device)
                flat[:, :K] = w.permute(0, 2, 3, 1).reshape(co, K)
                self._packed[k] = (ops.cast_bf16(flat.contiguous()), K, Kp)
            else:
                self._packed[k] = w.detach().float().contiguous()
        self._versions = ver

    # -- building blocks -------------------------------------------------------------------------------------------
    def _conv(self, x, B, H, W, cin, name, norm=None, silu=False, up=1, resid=None, ks=3, stride=1):
        """x [B*(H/up)*(W/up), cin] f32 -> [B*H*W, cout] f32 = conv_ks(f(upsample(x))) + bias (+ resid).
        stride = 2: x [B*2H*2W, cin] -> the Downsample convolution (pad (0,1,0,1), 3x3 stride 2, autoencoder.py:68-72)."""
        wq, K, Kp = self._packed[f"{name}.weight"]
        bias = self._packed[f"{name}.bias"]
        cout = wq.shape[0]
        ldo = (cout + 7) // 8 * 8
        M = B * H * W
        out = torch.empty(M, ldo, dtype=f32, device=x.device)
        sums = gamma = beta = None
        src_rows = (stride * H // up) * (stride * W // up)
        if norm is not None:
            sums = self._gn_stats(x, B, src_rows, cin)
            gamma, beta = self._packed[f"{norm}.weight"], self._packed[f"{norm}.bias"]
        per = max(1, min(B, self.max_rows // (H * W)))        # images per im2col operand
        A = torch.empty(per * H * W, Kp, dtype=bf16, device=x.device)
        for b0 in range(0, B, per):
            nb = min(per, B - b0)
            src = ops.ptr(x) + 4 * b0 * src_rows * cin
            sp = (ops.ptr(sums) + 8 * b0 * 64) if sums is not None else 0
            if stride == 1:
                ops.check(ops.lib().mdt_vae_im2col(src, sp, ops.ptr(gamma), ops.ptr(beta), int(silu), ks, up,
                                                   ops.ptr(A), nb, H, W, cin, Kp, ops.stream_ptr()), "mdt_vae_im2col")
            else:
                ops.check(ops.lib().mdt_vae_im2col_strided(src, sp, ops.ptr(gamma), ops.ptr(beta), int(silu), ks, up,
                                                           stride, 0, ops.ptr(A), nb, H, W, cin, Kp, ops.stream_ptr()),
                          "mdt_vae_im2col_strided")
            m = nb * H * W
            ops.gemm(A, wq, m, cout, Kp, out=out[b0 * H * W:], ldo=ldo, bias=bias,
                     resid=resid[b0 * H * W:] if resid is not None else None, ld_resid=cout)
        return out   # (ldo > cout only for conv_out: the caller reads the first cout columns)

    def _gn_stats(self, x, B, P, C):
        """GroupNorm(32) sums [B,32,2] f64 of x [B*P, C] (deterministic two-pass reduction: decode is run-to-run stable)."""
        sums = torch.empty(B, 32, 2, dtype=torch.float64, device=x.device)
        scratch = torch.empty(B * ((P + 255) // 256) * 64, dtype=f32, device=x.device)
        ops.check(ops.lib().mdt_vae_gn_stats(ops.ptr(x), ops.ptr(sums), ops.ptr(scratch), B, P, C, ops.stream_ptr()),
                  "mdt_vae_gn_stats", 2)
        return sums

    def _resblock(self, x, B, H, W, name, cin, cout):
        """ResnetBlock.forward with temb = None (autoencoder.py:117-137)."""
        h = self._conv(x, B, H, W, cin, f"{name}.conv1", norm=f"{name}.norm1", silu=True)
        sc = x
        if cin != cout:   # nin_shortcut: 1x1 convolution of the block input
            sc = self._conv(x, B, H, W, cin, f"{name}.nin_shortcut", ks=1)
        return self._conv(h, B, H, W, cout, f"{name}.conv2", norm=f"{name}.norm2", silu=True, resid=sc)

    def _attn(self, x, B, H, W, name, c):
        """AttnBlock.forward (autoencoder.py:174-198): one head over the H*W positions, head_dim = c."""
        T, M = H * W, B * H * W
        dev = x.device
        q, k, v = (torch.empty(M, c, dtype=bf16, device=dev) for _ in range(3))
        sums = self._gn_stats(x, B, T, c)
        xn = torch.empty(M, c, dtype=bf16, device=dev)
        ops.check(ops.lib().mdt_vae_im2col(ops.ptr(x), ops.ptr(sums), ops.ptr(self._packed[f"{name}.norm.weight"]),
                                           ops.ptr(self._packed[f"{name}.norm.bias"]), 0, 1, 1, ops.ptr(xn), B, H, W, c,
                                           c, ops.stream_ptr()), "mdt_vae_im2col")
        for t, n in ((q, "q"), (k, "k"), (v, "v")):
            ops.gemm(xn, self._packed[f"{name}.{n}.weight"][0], M, c, c, out=t, bias=self._packed[f"{name}.{n}.bias"])
        S = torch.empty(T, T, dtype=f32, device=dev)
        P = torch.empty(T, T, dtype=bf16, device=dev)
        o = torch.empty(M, c, dtype=bf16, device=dev)
        for b in range(B):
            qb, kb, vb = q[b * T:(b + 1) * T], k[b * T:(b + 1) * T], v[b * T:(b + 1) * T]
            ops.gemm(qb, kb, T, T, c, out=S)                                          # w_ = q k^T
            ops.check(ops.lib().mdt_vae_softmax_rows(ops.ptr(S), float(c) ** -0.5, ops.ptr(P), T, T, ops.stream_ptr()),
                      "mdt_vae_softmax_rows")
            ops.gemm(P, vb, T, c, T, b_mn=True, out=o[b * T:(b + 1) * T])             # h_ = softmax(w_) v
        out = torch.empty(M, c, dtype=f32, device=dev)
        ops.gemm(o, self._packed[f"{name}.proj_out.weight"][0], M, c, c, out=out,
                 bias=self._packed[f"{name}.proj_out.bias"], resid=x, ld_resid=c)
        return out


class AutoencoderKLDecoder(_AutoencoderKLHalf):
    _UNPACKED = ("post_quant_conv",)

    def __init__(self, scale_factor=0.18215, max_rows=1 << 21):
        shapes, plan = _shapes()
        super().__init__(shapes, scale_factor, max_rows)
        self._plan = plan

    # -- reference interface ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def decode(self, z):
        """FrozenAutoencoderKL.decode (autoencoder.py:449-453): z [B,4,h,w] -> images [B,3,8h,8w] f32."""
        self._ready()
        z = z.contiguous().float()
        ops._c(z, f32)
        B, C, H, W = z.shape
        x = torch.empty(B * H * W, C, dtype=f32, device=z.device)
        ops.check(ops.lib().mdt_vae_post_quant(ops.ptr(z), ops.ptr(self._packed["post_quant_conv.weight"]),
                                               ops.ptr(self._packed["post_quant_conv.bias"]), self.scale_factor,
                                               ops.ptr(x), B, C, H * W, ops.stream_ptr()), "mdt_vae_post_quant")
        c = CH * CH_MULT[-1]
        h = self._conv(x, B, H, W, C, "decoder.conv_in")
        h = self._resblock(h, B, H, W, "decoder.mid.block_1", c, c)
        h = self._attn(h, B, H, W, "decoder.mid.attn_1", c)
        h = self._resblock(h, B, H, W, "decoder.mid.block_2", c, c)
        for lvl in reversed(range(len(CH_MULT))):
            for i in range(NUM_RES_BLOCKS + 1):
                cin, cout = self._plan[(lvl, i)]
                h = self._resblock(h, B, H, W, f"decoder.up.{lvl}.block.{i}", cin, cout)
            if lvl != 0:
                H, W = 2 * H, 2 * W
                cu = self._plan[(lvl, "up")]
                h = self._conv(h, B, H, W, cu, f"decoder.up.{lvl}.upsample.conv", up=2)
        y = self._conv(h, B, H, W, CH, "decoder.conv_out", norm="decoder.norm_out", silu=True)   # [M, 8], 3 valid
        img = torch.empty(B, OUT_CH, H, W, dtype=f32, device=z.device)
        ops.check(ops.lib().mdt_vae_rows_to_nchw(ops.ptr(y), ops.ptr(img), B, H * W, OUT_CH, y.shape[1],
                                                 ops.stream_ptr()), "mdt_vae_rows_to_nchw")
        return img

    def forward(self, inputs, fn="decode"):
        if fn != "decode":
            raise NotImplementedError("only the decode half of the autoencoder is on the sampling path")
        return self.decode(inputs)


class AutoencoderKLEncoder(_AutoencoderKLHalf):
    """The encode half of FrozenAutoencoderKL (Encoder.forward + quant_conv, autoencoder.py:212-303,431-446).

    Images are processed in chunks of at most `max_pixels` input pixels (at least one image per chunk), so the
    activations stay within a fixed budget whatever the batch: one fp32 [512*512, 128] activation is 134 MB per image.
    Every kernel on the path is per image and the GEMMs do not split K, so the moments are bit-identical for any chunk
    size and any `max_rows`."""

    _UNPACKED = ("quant_conv",)
    _CIN_PAD = {"encoder.conv_in.weight": 4}     # the image rows carry a zero fourth channel (C % 4 im2col rule)

    def __init__(self, scale_factor=0.18215, max_rows=1 << 21, max_pixels=1 << 22):
        super().__init__(_encoder_shapes(), scale_factor, max_rows)
        self.max_pixels = max_pixels

    def _check(self, x):
        if x.ndim != 4 or x.shape[1] != OUT_CH:
            raise ValueError(f"expected images [B, {OUT_CH}, H, W], got {tuple(x.shape)}")
        if x.shape[2] % 8 or x.shape[3] % 8:
            raise ValueError(f"image height and width must be multiples of 8, got {x.shape[2]}x{x.shape[3]}")
        self._ready()
        x = x.contiguous().float()
        ops._c(x, f32)
        return x

    def _chunk(self, x, flip, moments, eps, z):
        """Encoder.forward + quant_conv (+ sample) of the images x [b,3,H,W] into moments [b,8,H/8,W/8] (z [b,4,..])."""
        B, _, H, W = x.shape
        rows = torch.empty(B * H * W, 4, dtype=f32, device=x.device)
        ops.check(ops.lib().mdt_vae_image_to_rows(ops.ptr(x), ops.ptr(rows), B, H, W, int(flip), ops.stream_ptr()),
                  "mdt_vae_image_to_rows")
        h = self._conv(rows, B, H, W, 4, "encoder.conv_in")
        block_in = CH
        for lvl, mult in enumerate(CH_MULT):
            for i in range(NUM_RES_BLOCKS):
                h = self._resblock(h, B, H, W, f"encoder.down.{lvl}.block.{i}", block_in, CH * mult)
                block_in = CH * mult
            if lvl != len(CH_MULT) - 1:
                H, W = H // 2, W // 2
                h = self._conv(h, B, H, W, block_in, f"encoder.down.{lvl}.downsample.conv", stride=2)
        h = self._resblock(h, B, H, W, "encoder.mid.block_1", block_in, block_in)
        h = self._attn(h, B, H, W, "encoder.mid.attn_1", block_in)
        h = self._resblock(h, B, H, W, "encoder.mid.block_2", block_in, block_in)
        y = self._conv(h, B, H, W, block_in, "encoder.conv_out", norm="encoder.norm_out", silu=True)   # [M, 8]
        ops.check(ops.lib().mdt_vae_quant_moments(ops.ptr(y), y.shape[1], ops.ptr(self._packed["quant_conv.weight"]),
                                                  ops.ptr(self._packed["quant_conv.bias"]), ops.ptr(eps),
                                                  self.scale_factor, ops.ptr(moments), ops.ptr(z), B, 2 * Z_CH, H * W,
                                                  ops.stream_ptr()), "mdt_vae_quant_moments")

    def _run(self, x, flip=False, eps=None):
        B, _, H, W = x.shape
        moments = torch.empty(B, 2 * Z_CH, H // 8, W // 8, dtype=f32, device=x.device)
        z = None
        if eps is not None:
            if tuple(eps.shape) != (B, Z_CH, H // 8, W // 8):
                raise ValueError(f"eps must be [{B}, {Z_CH}, {H // 8}, {W // 8}], got {tuple(eps.shape)}")
            eps = eps.contiguous().float()
            ops._c(eps, f32)
            z = torch.empty_like(eps)
        per = max(1, min(B, self.max_pixels // (H * W)))     # images per chunk
        for b0 in range(0, B, per):
            b1 = min(B, b0 + per)
            self._chunk(x[b0:b1], flip, moments[b0:b1], eps[b0:b1] if eps is not None else None,
                        z[b0:b1] if z is not None else None)
        return moments, z

    # -- reference interface ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def encode_moments(self, x, flip=False):
        """FrozenAutoencoderKL.encode_moments (autoencoder.py:431-434): images [B,3,H,W] f32 in [-1,1] ->
        moments [B,8,H/8,W/8] f32 (mean | logvar).  flip=True encodes `x.flip(-1)` without materialising it."""
        return self._run(self._check(x), flip)[0]

    @torch.no_grad()
    def encode(self, x, eps=None):
        """FrozenAutoencoderKL.encode (autoencoder.py:436-446): z = scale_factor * (mean + std * eps) [B,4,H/8,W/8];
        eps is drawn on the device (standard normal) when not given."""
        x = self._check(x)
        B, _, H, W = x.shape
        if eps is None:
            eps = torch.randn(B, Z_CH, H // 8, W // 8, dtype=f32, device=x.device)
        return self._run(x, False, eps)[1]

    def forward(self, inputs, fn="encode_moments"):
        if fn == "encode_moments":
            return self.encode_moments(inputs)
        if fn == "encode":
            return self.encode(inputs)
        raise NotImplementedError(f"the encoder half serves fn='encode_moments' / 'encode', not {fn!r}")


def _load_half(m, pretrained_path, what):
    sd = torch.load(pretrained_path, map_location="cpu", weights_only=True)
    own = set(m.state_dict().keys())
    missing = own - set(sd.keys())
    if missing:
        raise KeyError(f"checkpoint lacks {what} tensors: {sorted(missing)[:4]} ...")
    m.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=True)


def get_encoder(pretrained_path=None, scale_factor=0.18215, device="cuda"):
    """autoencoder.get_model (autoencoder.py:466-479) for the encode half, as extract_latent.py:40 uses it: loads
    `encoder.*` / `quant_conv.*` from a FrozenAutoencoderKL checkpoint (decoder / post_quant_conv entries are ignored)."""
    m = AutoencoderKLEncoder(scale_factor)
    if pretrained_path is not None:
        _load_half(m, pretrained_path, "encoder")
    return m.to(device).eval()


def get_model(pretrained_path=None, scale_factor=0.18215, device="cuda"):
    """autoencoder.get_model (autoencoder.py:466-479) for the decode half: loads `decoder.*` / `post_quant_conv.*` from a
    FrozenAutoencoderKL checkpoint (encoder / quant_conv entries are ignored)."""
    m = AutoencoderKLDecoder(scale_factor)
    if pretrained_path is not None:
        _load_half(m, pretrained_path, "decoder")
    return m.to(device).eval()
