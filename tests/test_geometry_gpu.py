"""GPU: the DiT_models geometries beyond the shipped XL/2 on the CUDA path against the unmodified reference's goldens
(tests/golden/make_golden_geometry.py): patch 8 (pd = cpp = 256) with and without the decoder, DiT-L/4 decoder-less
at T = 44, and DiT-H/2, whose head_dim 80 runs on the mma.sync attention kernels.  Also the C driver against the
Python engine, the S/8 eval / CFG / sampler, and two training steps of DiT-S/8 on the C driver.

Bounds: the constants of support.py; for DiT-H/2's 32-block forward, where the reference's own CPU bf16-autocast
output (geo_h2_bf16.npz) is further from its fp32 output, 1.5x that measured distance."""
import copy
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
from support import (CFG_TOL, EVAL_TOL, FWD_TOL, LOSS_TOL, GoldenLoss, ImplRecorder,  # noqa: E402
                     check_c_driver_matches_engine, check_grads, load, rel_l2)

pytestmark = pytest.mark.gpu


def build_geo(model_type, R, ncls, use_decoder, seed=1):
    from maskdit_b200.maskdit import Precond_models
    from oracle import maskdit_oracle as O
    cfg = O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls, use_decoder=use_decoder)
    net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=ncls, model_type=model_type,
                                use_decoder=use_decoder, mae_loss_coef=0.1, pad_cls_token=False)
    net.load_state_dict(O.make_state_dict(cfg, seed), strict=True)
    return net.cuda(), cfg


# name -> (model_type, R, ncls, use_decoder), attention (T, head_dim, family) forward and backward (1 = wgmma,
# 0 = mma.sync), forward bound
CASES = {
    # encoder T = 8 (16 patches, half kept), decoder T = 16 at head_dim 32
    "geo_s8_mask50": (("DiT-S/8", 32, 10, True), {(8, 64, 0), (16, 32, 0)}, FWD_TOL),
    "geo_b8_nd_nomask": (("DiT-B/8", 32, 10, False), {(16, 64, 0)}, FWD_TOL),
    "geo_l4_nd_uncond_mask30": (("DiT-L/4", 32, 0, False), {(44, 64, 0)}, FWD_TOL),
    # head_dim 80 has no wgmma instance: the encoder runs mma.sync even at T = 128; the decoder (T = 256, 32) wgmma
    "geo_h2_mask50": (("DiT-H/2", 32, 1000, True), {(128, 80, 0), (256, 32, 1)},
                      max(FWD_TOL, 1.5 * float(load("geo_h2_bf16")["bf16_rel_D_train"]))),
}


def inputs(g):
    sigma = (g["rnd_normal"].cuda() * 1.2 - 1.2).exp()
    yn = g["images"].cuda() + g["noise_unit"].cuda() * sigma
    lab = g["labels"].cuda() if "labels" in g else None
    md = {k: g[k].cuda() for k in ("mask", "ids_keep", "ids_restore")} if "ids_keep" in g else None
    return sigma, yn, lab, md


@pytest.mark.parametrize("name", list(CASES))
def test_loss_D_and_grads_vs_reference_golden(name):
    (mt, R, ncls, dec), attn, fwd_tol = CASES[name]
    g = load(name)
    net, cfg = build_geo(mt, R, ncls, dec)
    net.train()
    lf = GoldenLoss(g)
    mr = float(g["mask_ratio"])
    lab = g["labels"].cuda() if "labels" in g else None
    with ImplRecorder() as rec:
        loss = lf(net, g["images"].cuda(), lab, mask_ratio=mr, mae_loss_coef=0.1)
        loss.mean().backward()
    if mr > 0:
        for k in ("mask", "ids_keep", "ids_restore"):
            assert torch.equal(lf.last_mask_dict[k].cpu(), g[k]), k
    print(name, "loss", loss.tolist(), "ref", g["loss"].tolist(), "attn", sorted(rec.attn_fwd), sorted(rec.attn_bwd))
    assert torch.allclose(loss.cpu(), g["loss"], rtol=LOSS_TOL), (loss, g["loss"])
    assert rec.attn_fwd == attn and rec.attn_bwd == attn, (rec.attn_fwd, rec.attn_bwd)
    check_grads(net, g, what=name)
    sigma, yn, lab, md = inputs(g)
    with torch.no_grad():
        D = net(yn, sigma, lab, mask_ratio=mr, mask_dict=md)["x"] if md else net(yn, sigma, lab)["x"]
    r = rel_l2(D, g["D"])
    print(name, "D rel-L2", r, "bound", fwd_tol)
    assert r <= fwd_tol


@pytest.mark.parametrize("name", ["geo_s8_mask50", "geo_l4_nd_uncond_mask30"])
def test_c_driver_matches_python_engine(name):
    """`mdt_forward` == `Engine.forward` bit for bit; backward within the fp32-atomics order noise
    (test_model_gpu.py::check_c_driver_matches_engine).  Decoder-less with a mask: the removed tokens' rows of F are
    exactly zero."""
    (mt, R, ncls, dec), _, _ = CASES[name]
    g = load(name)
    net, cfg = build_geo(mt, R, ncls, dec)
    net.train()
    sigma, x, lab, md = inputs(g)
    sigma, x = sigma.reshape(-1).contiguous(), x.contiguous()
    _, _, Fc = check_c_driver_matches_engine(net, x, sigma, lab, md, name)
    assert Fc.shape[-1] == cfg.patch_dim
    if not dec:
        removed = md["mask"].bool().reshape(-1)
        assert (Fc[removed] == 0).all() and (Fc[~removed] != 0).any(dim=1).all()


def test_s8_eval_cfg_and_short_sampler_vs_reference_golden():
    """DiT-S/8 unmasked eval (T = 16 encoder and decoder tokens), CFG at 2B, and a 3-step CFG sampler."""
    from maskdit_b200.sampler import edm_sampler
    g = load("geo_s8_eval")
    net, cfg = build_geo("DiT-S/8", 32, 10, True)
    net.eval()
    with torch.no_grad(), ImplRecorder() as rec:
        plain = net(g["images"].cuda(), g["sigma"].cuda(), g["labels"].cuda())["x"]
        c = net(g["images"].cuda(), torch.tensor(1.7, dtype=torch.float64).cuda(), g["labels"].cuda(), 1.5)["x"]
    r1, r2 = rel_l2(plain, g["D_plain"]), rel_l2(c, g["D_cfg"])
    print("S/8 eval rel-L2 plain", r1, "cfg", r2, sorted(rec.attn_fwd))
    assert rec.attn_fwd == {(16, 64, 0), (16, 32, 0)}, rec.attn_fwd
    assert r1 <= EVAL_TOL and r2 <= CFG_TOL
    calls = []
    orig = net.forward

    def spy(x, s, *a, **k):
        calls.append(float(s))
        return orig(x, s, *a, **k)

    net.forward = spy
    with torch.no_grad():
        z = edm_sampler(net, g["latents"].cuda(), g["labels"].cuda(), cfg_scale=1.5, num_steps=int(g["num_steps"]))
    net.forward = orig
    assert calls == pytest.approx(g["sampler_sigmas"].tolist(), rel=1e-12)
    rz = rel_l2(z, g["z"])
    print("S/8 3-step sampler rel-L2", rz)
    assert z.dtype == torch.float64 and rz <= max(1e-2, CFG_TOL)


def test_s8_train_steps_on_c_driver():
    """Two TrainStep steps of DiT-S/8 (the EDM + MAE loss at pd 256, the patch-embed backward at cpp 256) on the C
    driver: finite losses, and the patch embedding and final layer move."""
    from maskdit_b200.engine import CEngine
    from maskdit_b200.train_step import TrainStep
    g = load("geo_s8_mask50")
    net, cfg = build_geo("DiT-S/8", 32, 10, True)
    net.train()
    ema = copy.deepcopy(net).eval()
    before = {k: v.detach().clone() for k, v in net.state_dict().items()}
    ts = TrainStep(net, ema, lr=1e-3, loss_fn=GoldenLoss(g))
    x, y = g["images"].cuda(), g["labels"].cuda()
    losses = [ts.step(x, y, 0.5, 0.1) for _ in range(2)]
    assert isinstance(net._engine, CEngine)
    for l in losses:
        assert torch.isfinite(l).all(), losses
    assert torch.allclose(losses[0].cpu(), g["loss"], rtol=LOSS_TOL), (losses[0], g["loss"])
    after = net.state_dict()
    for k in ("model.x_embedder.proj.weight", "model.x_embedder.proj.bias", "model.final_layer.linear.weight",
              "model.blocks.0.attn.qkv.weight", "model.decoder_blocks.7.mlp.fc2.weight"):
        assert torch.isfinite(after[k]).all() and not torch.equal(after[k], before[k]), k
