"""GPU: the decoder-less DiT (use_decoder=False) on the CUDA path against the unmodified reference's goldens
(tests/golden/make_golden_nodecoder.py), the C driver against the Python engine, the zero-filled output scatter, the
eval CUDA graph, the optimizer-state layout and the train.py / generate.py entry points.

Bounds: the existing constants of support.py; where the reference's own CPU bf16-autocast output of the same
XL/2 forward (nd_xl2_bf16.npz) is further from its fp32 output, 1.5x that measured distance."""
import copy
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
from support import (CFG_TOL, EVAL_TOL, FWD_TOL, LOSS_TOL, GoldenLoss, ImplRecorder,  # noqa: E402
                     check_c_driver_matches_engine, check_grads, load, rel_l2)

pytestmark = pytest.mark.gpu


def build_nd(model_type="DiT-S/2", R=8, ncls=10, seed=1):
    from maskdit_b200.maskdit import Precond_models
    from oracle import maskdit_oracle as O
    cfg = O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls, use_decoder=False)
    net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=ncls, model_type=model_type,
                                use_decoder=False, mae_loss_coef=0.1, pad_cls_token=False)
    sd = O.make_state_dict(cfg, seed)
    net.load_state_dict(sd, strict=True)
    return net.cuda(), cfg, sd


def yardstick(key, const):
    return max(const, 1.5 * float(load("nd_xl2_bf16")[f"bf16_rel_{key}"]))


# name, (model_type, R, ncls), attention (T, head_dim, family) forward and backward; family 1 = wgmma, 0 = mma.sync
CASES = {
    "nd_s2_train_mask": (("DiT-S/2", 8, 10), {(8, 64, 0)}),
    "nd_s2_train_nomask": (("DiT-S/2", 8, 10), {(16, 64, 0)}),
    "nd_s2_uncond_mask30": (("DiT-S/2", 32, 0), {(179, 64, 0)}),
    "nd_xl2_grads": (("DiT-XL/2", 32, 1000), {(128, 72, 1)}),
}


def inputs(g):
    sigma = (g["rnd_normal"].cuda() * 1.2 - 1.2).exp()
    yn = g["images"].cuda() + g["noise_unit"].cuda() * sigma
    lab = g["labels"].cuda() if "labels" in g else None
    md = {k: g[k].cuda() for k in ("mask", "ids_keep", "ids_restore")} if "ids_keep" in g else None
    return sigma, yn, lab, md


@pytest.mark.parametrize("name", list(CASES))
def test_loss_D_and_grads_vs_reference_golden(name):
    (mt, R, ncls), attn = CASES[name]
    g = load(name)
    net, cfg, _ = build_nd(mt, R, ncls)
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
    tol = yardstick("D_train", FWD_TOL) if name.startswith("nd_xl2") else FWD_TOL
    print(name, "D rel-L2", r, "bound", tol)
    assert r <= tol


@pytest.mark.parametrize("name", list(CASES))
def test_c_driver_matches_python_engine_and_masked_rows(name):
    """`mdt_forward` == `Engine.forward` bit for bit; backward within the fp32-atomics order noise
    (test_model_gpu.py::check_c_driver_matches_engine).  Masked training: the removed tokens' rows of F are exactly
    zero, and their dF reaches no parameter (a large dF there leaves every gradient unchanged)."""
    (mt, R, ncls), _ = CASES[name]
    g = load(name)
    net, cfg, _ = build_nd(mt, R, ncls)
    net.train()
    sigma, x, lab, md = inputs(g)
    sigma, x = sigma.reshape(-1).contiguous(), x.contiguous()
    B, L = x.shape[0], cfg.num_patches
    removed = md["mask"].bool().reshape(-1) if md else torch.zeros(B * L, dtype=torch.bool, device="cuda")
    ce, ctx_c, Fc = check_c_driver_matches_engine(net, x, sigma, lab, md, name,
                                                  dF_same_grads=lambda dF: dF.masked_fill(removed[:, None], 1e3))
    if md:
        assert int(removed.sum()) == B * (L - md["ids_keep"].shape[1])
        assert (Fc[removed] == 0).all() and (Fc[~removed] != 0).any(dim=1).all()
    T = md["ids_keep"].shape[1] if md else L
    assert ctx_c["nbytes"] == ce.workspace_bytes(B, T, True) > ce.workspace_bytes(B, T, False)
    assert ce._count(md is not None) == (9 + 2 * bool(ncls) + 7 * cfg.depth + bool(md),
                                         16 + 13 * cfg.depth + bool(ncls) + bool(md))


def test_xl2_eval_cfg_and_short_sampler_vs_reference_golden():
    """XL/2 unmasked eval (T = 256, 16 heads of 72, 28 wide blocks over every token), CFG at 2B, 3-step sampler."""
    from maskdit_b200.sampler import edm_sampler
    g = load("nd_xl2_eval")
    net, cfg, _ = build_nd("DiT-XL/2", 32, 1000)
    net.eval()
    with torch.no_grad(), ImplRecorder() as rec:
        plain = net(g["images"].cuda(), g["sigma"].cuda(), g["labels"].cuda())["x"]
        c = net(g["images"].cuda(), torch.tensor(1.7, dtype=torch.float64).cuda(), g["labels"].cuda(), 1.5)["x"]
    r1, r2 = rel_l2(plain, g["D_plain"]), rel_l2(c, g["D_cfg"])
    b1, b2 = yardstick("D_plain", EVAL_TOL), yardstick("D_cfg", CFG_TOL)
    print("nd XL/2 eval rel-L2 plain", r1, "bound", b1, "cfg", r2, "bound", b2, sorted(rec.attn_fwd))
    assert rec.attn_fwd == {(256, 72, 1)}, rec.attn_fwd
    calls = []
    orig = net.forward

    def spy(x, s, *a, **k):
        calls.append(float(s))
        return orig(x, s, *a, **k)

    net.forward = spy
    with torch.no_grad():
        z = edm_sampler(net, g["latents"].cuda(), g["labels"].cuda(), cfg_scale=1.5, num_steps=int(g["num_steps"]))
    net.forward = orig
    np.testing.assert_allclose(np.array(calls), g["sampler_sigmas"].numpy(), rtol=1e-12)
    rz = rel_l2(z, g["z"])
    print("nd XL/2 3-step sampler rel-L2", rz)
    assert r1 <= b1 and r2 <= b2
    assert z.dtype == torch.float64 and rz <= max(1e-2, b2)


def test_eval_cuda_graph_matches_eager(monkeypatch):
    net, cfg, _ = build_nd()
    net.eval()
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 8, 8, generator=gen).cuda()
    lab = torch.nn.functional.one_hot(torch.tensor([3, 7]), 10).float().cuda()
    sig = torch.tensor(1.7, dtype=torch.float64).cuda()

    def run(graph, xin, cfg_scale):
        monkeypatch.setenv("MDT_CUDA_GRAPH", "1" if graph else "0")
        with torch.no_grad():
            return net(xin, sig, lab, cfg_scale)["x"].clone()

    for cfg_scale in (None, 1.5):
        e = run(False, x, cfg_scale)
        for _ in range(2):  # capture, then replay
            assert torch.equal(run(True, x, cfg_scale), e)
        x2 = x * 0.5 + 0.1
        assert torch.equal(run(True, x2, cfg_scale), run(False, x2, cfg_scale))
    assert len(net._graphs) == 2


def test_train_step_checkpoint_round_trip_in_torch_adamw_layout():
    """`opt` state keyed like torch.optim.AdamW(net.parameters()) of the decoder-less module: pos_embed is position
    0 and owns no state, the first trainable tensor is 1; a resumed TrainStep takes bit-identical steps."""
    from maskdit_b200.maskdit import Precond_models
    from maskdit_b200.train_step import TrainStep
    g = load("nd_s2_train_mask")
    net, cfg, _ = build_nd()
    net.train()
    ema = copy.deepcopy(net).eval()
    ts = TrainStep(net, ema, lr=1e-3, loss_fn=GoldenLoss(g))
    x, y = g["images"].cuda(), g["labels"].cuda()

    def one(t):
        t.loss_fn = GoldenLoss(g)
        return t.step(x, y, 0.5, 0.1)

    one(ts), one(ts)
    buf = io.BytesIO()
    torch.save({"model": net.state_dict(), "ema": ema.state_dict(), "opt": ts.state_dict()}, buf)
    buf.seek(0)
    ck = torch.load(buf, map_location="cuda")
    ref = Precond_models["edm"](8, 4, num_classes=10, model_type="DiT-S/2", use_decoder=False, mae_loss_coef=0.1)
    for p in ref.parameters():
        if p.requires_grad:
            p.grad = torch.zeros_like(p)
    opt = torch.optim.AdamW(ref.parameters())
    opt.step()
    want = opt.state_dict()
    assert set(ck["opt"]["state"]) == set(want["state"]) and min(want["state"]) == 1 and 0 not in ck["opt"]["state"]
    assert ck["opt"]["param_groups"][0]["params"] == want["param_groups"][0]["params"]
    for i, e in want["state"].items():
        assert ck["opt"]["state"][i]["exp_avg"].shape == e["exp_avg"].shape, i
    net2, _, _ = build_nd(seed=5)
    net2.train()
    net2.load_state_dict(ck["model"])
    ema2 = copy.deepcopy(net2).eval()
    ema2.load_state_dict(ck["ema"])
    ts2 = TrainStep(net2, ema2, lr=0.5, loss_fn=GoldenLoss(g))
    ts2.load_state_dict(ck["opt"])
    assert ts2.step_count == 2 and ts2.lr == 1e-3
    l1, l2 = one(ts), one(ts2)
    assert torch.allclose(l1, l2, rtol=1e-6, atol=1e-7)
    for (k, a), (_, b) in zip(net.state_dict().items(), net2.state_dict().items()):
        assert torch.allclose(a, b, rtol=0, atol=1e-6), k
    for (k, a), (_, b) in zip(ema.state_dict().items(), ema2.state_dict().items()):
        assert torch.allclose(a, b, rtol=0, atol=1e-6), k


YAML = """
data: {dataset: imagenet256-latent, category: lmdb, resolution: 16, num_channels: 4, root: none, feat_path: None}
model:
  precond: edm
  model_type: DiT-S/2
  in_size: 16
  in_channels: 4
  num_classes: 1000
  use_decoder: False
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
    r = subprocess.run([sys.executable, *cmd], cwd=cwd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def test_train_resume_then_generate_entry_points(tmp_path):
    cfg = tmp_path / "cfg.yaml"
    cfg.write_text(YAML)
    out = run([os.path.join(ROOT, "train.py"), "--config", str(cfg), "--synthetic", "--max_steps", "4",
               "--results_dir", str(tmp_path / "res")], str(tmp_path))
    assert "Train Loss" in out
    ck = tmp_path / "res" / "checkpoints" / "0000004.pt"
    sd = torch.load(ck, map_location="cpu", weights_only=False)
    assert "model.blocks.0.attn.qkv.weight" in sd["ema"] and not any("decoder" in k for k in sd["ema"])
    assert sd["ema"]["model.final_layer.linear.weight"].shape == (16, 384) and min(sd["opt"]["state"]) == 1
    out = run([os.path.join(ROOT, "train.py"), "--config", str(cfg), "--synthetic", "--max_steps", "2",
               "--results_dir", str(tmp_path / "res")], str(tmp_path))       # resumes from 0000004.pt
    assert "(step=0000006)" in out
    run([os.path.join(ROOT, "generate.py"), "--config", str(cfg), "--ckpt_path", str(ck), "--seeds", "0-3",
         "--num_steps", "6", "--cfg_scale", "1.5", "--results_dir", str(tmp_path / "samples")], str(tmp_path))
    z = np.load(tmp_path / "samples" / "000002.npy")
    assert z.shape == (4, 16, 16) and np.isfinite(z).all()
