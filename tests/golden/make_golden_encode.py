"""Generate the SD-VAE encode goldens by executing the UNMODIFIED reference (/root/reference) on CPU fp32.

Run in the dev container only (the GPU box has no /root/reference):  python tests/golden/make_golden_encode.py
Writes tests/golden/vae_encode.npz and tests/golden/center_crop.npz; no other golden is touched.  Weights are not
stored: the encoder stand-in is oracle.vae_encode_oracle.make_vae_encoder_state_dict(4), the decoder half (loaded only
because FrozenAutoencoderKL insists on a complete checkpoint) is oracle.vae_oracle.make_vae_state_dict(3).
"""
import contextlib
import io
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import vae_encode_oracle as VE  # noqa: E402
from oracle import vae_oracle as VO  # noqa: E402

sys.path.insert(0, "/root/reference")
import autoencoder as ra  # noqa: E402

ENC_SEED = 4


def encode_case(name="vae_encode"):
    """FrozenAutoencoderKL.encode_moments / encode (autoencoder.py:431-446) on B = 2 images at 64x64: the vae_decode
    golden's first image clamped to [-1, 1] (structured) and uniform noise in [-1, 1]."""
    sd = {**VE.make_vae_encoder_state_dict(ENC_SEED), **VO.make_vae_state_dict(3)}
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "autoencoder_kl.pth")
        torch.save(sd, ck)
        with contextlib.redirect_stdout(io.StringIO()):
            model = ra.get_model(ck)                      # asserts len(missing) == 0 and len(unexpected) == 0 itself
    keys = [k for k in model.state_dict().keys() if k.startswith(("encoder.", "quant_conv."))]
    assert keys == list(VE.encoder_param_shapes().keys())
    dec = np.load(os.path.join(HERE, "vae_decode.npz"))
    g = torch.Generator().manual_seed(41)
    x = torch.stack([torch.from_numpy(dec["images"][0]).clamp(-1, 1),
                     torch.rand(3, 64, 64, generator=g) * 2 - 1]).contiguous()
    eps = torch.randn(2, 4, 8, 8, generator=g)
    with torch.no_grad():
        m = model(x, fn="encode_moments")
        mf = model(x.flip(dims=[-1]), fn="encode_moments")
        torch.manual_seed(0)
        z_ref = model(x, fn="encode")                     # the reference's own draw: check `sample` against it
        torch.manual_seed(0)
        assert torch.allclose(z_ref, VE.sample(m, torch.randn_like(m[:, :4])), rtol=0, atol=0)
        mean, logvar = torch.chunk(m, 2, dim=1)
        z = model.scale_factor * (mean + torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0)) * eps)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            m16 = model(x, fn="encode_moments").float()
    rel = lambda a, b: ((a - b).norm() / b.norm()).item()   # noqa: E731
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), x=x.numpy(), moments=m.numpy(), moments_flip=mf.numpy(),
                        eps=eps.numpy(), z=z.numpy(), keys=np.array(keys),
                        shapes=np.array([str(tuple(model.state_dict()[k].shape)) for k in keys]),
                        moments_bf16=m16.numpy(),
                        bf16_rel_mean=np.float64(rel(m16[:, :4], m[:, :4])),
                        bf16_rel_logvar=np.float64(rel(m16[:, 4:], m[:, 4:])))
    print(name, "moments range", m.min().item(), m.max().item(), "bf16-autocast rel-L2 mean / logvar",
          rel(m16[:, :4], m[:, :4]), rel(m16[:, 4:], m[:, 4:]))


def center_crop_case(name="center_crop"):
    """center_crop_arr (train_utils/datasets.py:19-37) at res 64 on three synthetic RGB images: 160x136 (one BOX halving
    first), 90x70 (bicubic down-scale) and 48x56 (bicubic up-scale)."""
    sys.modules.setdefault("lmdb", types.ModuleType("lmdb"))    # datasets.py imports lmdb at the top; unused here
    from PIL import Image
    from train_utils.datasets import center_crop_arr
    rng = np.random.default_rng(5)
    out = {}
    for i, (w, h) in enumerate(((160, 136), (90, 70), (48, 56))):
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // max(1, w - 1), yy * 255 // max(1, h - 1), (xx + yy) * 127 // (w + h)], -1)
        arr = np.clip(base + rng.integers(-20, 21, size=base.shape), 0, 255).astype(np.uint8)
        out[f"in{i}"] = arr
        out[f"out{i}"] = np.asarray(center_crop_arr(Image.fromarray(arr), 64))
        assert out[f"out{i}"].shape == (64, 64, 3)
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **out)
    print(name, "ok")


if __name__ == "__main__":
    encode_case()
    center_crop_case()
