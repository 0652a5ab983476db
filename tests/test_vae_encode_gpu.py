"""GPU: SD-VAE encode on the wgmma GEMM + fused im2col — against the unmodified reference's moments
(tests/golden/vae_encode.npz), its new kernels against torch, its determinism, and extract_latent.py end to end into
train.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def load(name):
    return {k: torch.from_numpy(v) if v.dtype.kind == "f" else v
            for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm()).item()


def encoder():
    from maskdit_b200.vae import AutoencoderKLEncoder
    from oracle import vae_encode_oracle as VE
    e = AutoencoderKLEncoder()
    e.load_state_dict(VE.make_vae_encoder_state_dict(4), strict=True)
    return e.cuda().eval()


def test_encode_moments_vs_reference_golden():
    """Moments of the stand-in encoder on the golden 64x64 images vs the reference's fp32 output, bounded relative to
    the reference under CPU bf16 autocast (the same bf16-operand precision class); mirrored images and z too."""
    from maskdit_b200 import _lib
    g = load("vae_encode")
    e = encoder()
    bound = {"mean": min(2e-2, 1.5 * float(g["bf16_rel_mean"])), "logvar": min(2e-2, 1.5 * float(g["bf16_rel_logvar"]))}
    x = g["x"].cuda()
    e.encode_moments(x)                                   # packs the weights (no GEMM) before the recording starts
    _lib.lib().mdt_gemm_configs_seen(1)
    _lib.GEMM_PROFILE = []                                # ops.gemm records every launch while this is a list
    try:
        m = e.encode_moments(x)
        torch.cuda.synchronize()
        n_gemm = len(_lib.GEMM_PROFILE)
    finally:
        _lib.GEMM_PROFILE = None
    seen = _lib.lib().mdt_gemm_configs_seen(1)
    convs = sum(1 for k, v in e.state_dict().items() if v.ndim == 4 and not k.startswith("quant_conv"))
    assert n_gemm == convs + 2 * x.shape[0] and seen != 0, (n_gemm, convs, seen)   # + q k^T and P v per image
    assert m.shape == (2, 8, 8, 8) and torch.isfinite(m).all()
    for what, got, want in (("", m, g["moments"]), (" (flip)", e.encode_moments(x, flip=True), g["moments_flip"])):
        rm, rl = rel(got[:, :4], want[:, :4]), rel(got[:, 4:], want[:, 4:])
        print(f"encode_moments{what} rel-L2 mean {rm:.3e} logvar {rl:.3e}; bounds {bound}")
        assert rm <= bound["mean"] and rl <= bound["logvar"], (what, rm, rl, bound)
    z = e.encode(x, eps=g["eps"].cuda())
    rz = rel(z, g["z"])
    print(f"encode z rel-L2 {rz:.3e}")
    assert z.shape == (2, 4, 8, 8) and rz <= max(bound.values())
    assert e(x, "encode").shape == (2, 4, 8, 8) and torch.equal(e(x, "encode_moments"), m)


def test_encode_is_bit_deterministic_and_chunking_invariant():
    g = load("vae_encode")
    e = encoder()
    x = torch.cat([g["x"], g["x"].flip(-1), -g["x"]]).cuda()          # 6 images
    m = e.encode_moments(x)
    assert torch.equal(e.encode_moments(x), m)
    e.max_rows = 2048                                   # several im2col operands / GEMM launches per convolution
    assert torch.equal(e.encode_moments(x), m)
    e.max_rows, e.max_pixels = 1 << 21, 1               # one image per chunk
    assert torch.equal(e.encode_moments(x), m)
    e.max_pixels = 2 * 64 * 64                          # chunks of 2
    assert torch.equal(e.encode_moments(x), m)
    assert torch.equal(e.encode_moments(x[:2], flip=True), m[2:4])


def bf16_round(t):
    return t.to(torch.bfloat16).float()


@pytest.mark.parametrize("C,H,W", [(128, 8, 8), (256, 5, 7), (4, 4, 6)])
def test_stride2_im2col_matches_pad_unfold(C, H, W):
    """Downsample's operand: F.pad(x, (0,1,0,1)) then a 3x3 stride-2 window, bit for bit; columns past 9C are zero."""
    from maskdit_b200 import ops
    B = 2
    g = torch.Generator().manual_seed(C + H)
    x = bf16_round(torch.randn(B, C, 2 * H, 2 * W, generator=g))
    src = x.permute(0, 2, 3, 1).contiguous().cuda()                       # rows [B, 2H, 2W, C]
    Kp = (9 * C + 7) // 8 * 8 + 8
    A = torch.full((B * H * W, Kp), 7.0, dtype=torch.bfloat16, device="cuda")
    ops.check(ops.lib().mdt_vae_im2col_strided(ops.ptr(src), 0, 0, 0, 0, 3, 1, 2, 0, ops.ptr(A), B, H, W, C, Kp,
                                               ops.stream_ptr()), "mdt_vae_im2col_strided")
    u = F.unfold(F.pad(x, (0, 1, 0, 1)), kernel_size=3, stride=2)          # [B, C*9, H*W], (c, ky, kx)
    want = u.view(B, C, 3, 3, H * W).permute(0, 4, 2, 3, 1).reshape(B * H * W, 9 * C)
    got = A.float().cpu()
    assert torch.equal(got[:, :9 * C], want)
    assert not got[:, 9 * C:].any()
    # stride 1 with the "same" padding is the original entry point, bit for bit
    A1, A2 = (torch.empty(B * 4 * H * W, Kp, dtype=torch.bfloat16, device="cuda") for _ in range(2))
    ops.check(ops.lib().mdt_vae_im2col(ops.ptr(src), 0, 0, 0, 0, 3, 1, ops.ptr(A1), B, 2 * H, 2 * W, C, Kp,
                                       ops.stream_ptr()), "mdt_vae_im2col")
    ops.check(ops.lib().mdt_vae_im2col_strided(ops.ptr(src), 0, 0, 0, 0, 3, 1, 1, 1, ops.ptr(A2), B, 2 * H, 2 * W, C,
                                               Kp, ops.stream_ptr()), "mdt_vae_im2col_strided")
    assert torch.equal(A1, A2)


@pytest.mark.parametrize("flip", [0, 1])
def test_image_to_rows_exact(flip):
    from maskdit_b200 import ops
    B, H, W = 3, 16, 24
    img = (torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(2)) * 2 - 1).cuda()
    rows = torch.full((B * H * W, 4), 5.0, device="cuda")
    ops.check(ops.lib().mdt_vae_image_to_rows(ops.ptr(img), ops.ptr(rows), B, H, W, flip, ops.stream_ptr()),
              "mdt_vae_image_to_rows")
    src = img.flip(-1) if flip else img
    want = torch.cat([src.permute(0, 2, 3, 1).reshape(-1, 3), torch.zeros(B * H * W, 1, device="cuda")], 1)
    assert torch.equal(rows, want)


def test_quant_moments_and_sample_vs_torch():
    from maskdit_b200 import ops
    B, C, P, ld = 3, 8, 40, 8
    g = torch.Generator().manual_seed(9)
    x = torch.randn(B * P, ld, generator=g)
    W = torch.randn(C, C, generator=g) * C ** -0.5
    bias = 0.05 * torch.randn(C, generator=g)
    x[:P, 4:] += 30.0                                        # logvar above the clamp for the first image
    x[P:2 * P, 4:] -= 45.0                                   # below it for the second
    eps = torch.randn(B, C // 2, P, generator=g)
    mom, z = torch.empty(B, C, P, device="cuda"), torch.empty(B, C // 2, P, device="cuda")
    dev = [t.cuda().contiguous() for t in (x, W, bias, eps)]
    ops.check(ops.lib().mdt_vae_quant_moments(ops.ptr(dev[0]), ld, ops.ptr(dev[1]), ops.ptr(dev[2]), ops.ptr(dev[3]),
                                              0.18215, ops.ptr(mom), ops.ptr(z), B, C, P, ops.stream_ptr()),
              "mdt_vae_quant_moments")
    want = (x.double().view(B, P, ld) @ W.double().t() + bias.double()).permute(0, 2, 1)
    assert rel(mom, want) <= 1e-6
    mean, logvar = want[:, :4], want[:, 4:].clamp(-30, 20)
    zw = 0.18215 * (mean + torch.exp(0.5 * logvar) * eps.double())
    assert rel(z, zw) <= 1e-6
    mom2 = torch.empty_like(mom)                             # eps = NULL: moments only, z untouched
    ops.check(ops.lib().mdt_vae_quant_moments(ops.ptr(dev[0]), ld, ops.ptr(dev[1]), ops.ptr(dev[2]), 0, 0.18215,
                                              ops.ptr(mom2), 0, B, C, P, ops.stream_ptr()), "mdt_vae_quant_moments")
    assert torch.equal(mom2, mom)


YAML = """
data: {dataset: imagenet256-latent, category: lmdb, resolution: 16, num_channels: 4, root: none, feat_path: None}
model:
  precond: edm
  model_type: DiT-S/2
  in_size: 16
  in_channels: 4
  num_classes: 1000
  use_decoder: True
  ext_feature_dim: 0
  pad_cls_token: False
  mask_ratio: 0.5
  mask_ratio_fn: constant
  mask_ratio_min: 0
  mae_loss_coef: 0.1
  class_dropout_prob: 0.1
train: {tf32: False, amp: True, batchsize: 8, grad_accum: 1, epochs: 1, lr: 0.0001, lr_rampup_kimg: 0, xflip: False,
        max_num_steps: 4}
log: {log_every: 2, ckpt_every: 4, tag: t}
"""


def run(cmd, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, *cmd], cwd=cwd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def test_extract_latent_end_to_end_then_train(tmp_path):
    """extract_latent.py --xflip on a small ImageFolder of mixed sizes and formats: the LMDB holds 2N entries, labels in
    folder order, moments bit-equal to in-process encode_moments (mirrored for the second half); train.py trains on it."""
    from PIL import Image
    from maskdit_b200 import data as D
    from oracle import vae_encode_oracle as VE
    from oracle import vae_oracle as VO
    rng = np.random.default_rng(0)
    sizes = [(160, 128), (128, 200), (300, 260), (140, 140), (97, 131), (256, 128), (129, 170), (400, 300), (128, 128),
             (150, 220)]
    for i, (w, h) in enumerate(sizes):
        d = tmp_path / "data" / "train" / f"n0{i % 3}"
        d.mkdir(parents=True, exist_ok=True)
        arr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        Image.fromarray(arr).save(d / f"img{i}.{'png' if i % 2 else 'jpg'}")
    ck = tmp_path / "vae.pth"
    torch.save({**VE.make_vae_encoder_state_dict(4), **VO.make_vae_state_dict(3)}, ck)
    out = run([os.path.join(ROOT, "extract_latent.py"), "--data_dir", str(tmp_path / "data"), "--resolution", "128",
               "--batch_size", "4", "--xflip", "--ckpt", str(ck), "--outdir", str(tmp_path / "out"), "--num_workers",
               "2"], str(tmp_path))
    assert "saved 20 files" in out, out
    db = tmp_path / "out" / "imagenet_128_latent_lmdb"
    samples, _ = D.image_folder_samples(str(tmp_path / "data" / "train"))
    N = len(samples)
    rd = D.MdbReader(str(db / "train"))
    assert bytes(rd.get(b"length")) == str(2 * N).encode() and rd.entries == 4 * N + 1
    x = torch.stack([torch.from_numpy(D.load_image(p, 128)) for p, _ in samples]).cuda()
    e = encoder()
    want = torch.cat([e.encode_moments(x), e.encode_moments(x, flip=True)]).cpu().numpy()
    for i in range(2 * N):
        assert bytes(rd.get(f"y-{i}".encode())) == str(samples[i % N][1]).encode(), i
        got = np.frombuffer(bytes(rd.get(f"z-{i}".encode())), dtype="<f4").reshape(8, 16, 16)
        assert np.array_equal(got, want[i]), i
    rd.close()
    cfg = tmp_path / "cfg.yaml"
    cfg.write_text(YAML.replace("root: none", f"root: {db}"))
    out = run([os.path.join(ROOT, "train.py"), "--config", str(cfg), "--max_steps", "2", "--results_dir",
               str(tmp_path / "res")], str(tmp_path))
    assert f"Dataset contains {2 * N} images" in out and "(step=0000002)" in out, out[-2000:]
