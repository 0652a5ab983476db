"""GPU: rectified-flow training and sampling (DESIGN §5) on the H100 kernels.  The network, loss, gradients and
sampler against goldens of the unmodified reference network with the flow objective applied around it
(tests/golden/make_golden_flow.py), the kernels one by one against float64, the flow step front against its fp32
formula, a deterministic flow TrainStep, recomputation, and train.py / generate.py end to end."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from support import EVAL_TOL, FWD_TOL, GRAD_TOL, LOSS_TOL, check_grads, det, load, ops, rel_l2  # noqa: F401

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMPLER_TOL = 1e-2


def flow_net(model_type, R, ncls, dec=True, seed=1):
    from maskdit_b200.maskdit import FlowPrecond
    from oracle import maskdit_oracle as O
    cfg = O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls, use_decoder=dec)
    net = FlowPrecond(img_resolution=R, img_channels=4, num_classes=ncls, model_type=model_type, use_decoder=dec,
                      mae_loss_coef=0.1, pad_cls_token=False)
    net.load_state_dict(O.make_state_dict(cfg, seed), strict=True)
    return net.cuda(), cfg


def golden_loss(g):
    """FlowLoss whose draws are the golden's: the t normal, eps, then the mask noise."""
    from maskdit_b200.loss import FlowLoss

    class L(FlowLoss):
        q = [g["rnd_normal"].reshape(-1, 1, 1, 1).cuda(), g["noise_unit"].cuda()]

        def _randn(self, shape, device):
            return self.q.pop(0)

        def _rand(self, shape, device):
            return g["mask_noise"].cuda()

    return L()


@pytest.mark.parametrize("name, mt, R, ncls, dec", [
    ("flow_s2_train_mask", "DiT-S/2", 8, 10, True),
    ("flow_nd_s2_uncond", "DiT-S/2", 8, 0, False),
    ("flow_xl2_mask", "DiT-XL/2", 32, 1000, True),
])
def test_loss_F_and_grads_vs_reference_golden(name, mt, R, ncls, dec):
    from oracle import maskdit_oracle as O
    g = load(name)
    net, _ = flow_net(mt, R, ncls, dec)
    net.train()
    x = g["images"].cuda()
    lab = g["labels"].cuda() if "labels" in g else None
    ratio, coef = float(g["mask_ratio"]), float(g["mae_coef"])
    loss = golden_loss(g)(net, x, lab, mask_ratio=ratio, mae_loss_coef=coef)
    loss.mean().backward()
    torch.cuda.synchronize()
    r = rel_l2(loss, g["loss"])
    assert r <= LOSS_TOL, (name, loss.tolist(), g["loss"].tolist())
    check_grads(net, g, GRAD_TOL, name)
    t4 = g["t"].reshape(-1, 1, 1, 1)
    xt = ((1 - t4) * g["images"] + t4 * g["noise_unit"]).cuda()
    md = None
    if ratio > 0:
        from maskdit_b200 import ops
        L = net.model.num_patches
        md = ops.mask_indices(g["mask_noise"].cuda(), int(L * (1 - ratio)))
        assert torch.equal(md["mask"].cpu(), O.mask_from_noise(g["mask_noise"], ratio)["mask"])
    with torch.no_grad():
        F = net(xt, g["t"].cuda(), lab, mask_ratio=ratio, mask_dict=md)["x"]
    # v^ is the raw network output, with no c_skip x term to dilute the bf16 error: the bound of the unmasked eval
    # forward; the denoised estimate x^ = x_t - t v^ (the flow's D) is held to the EDM forward bound
    xh = xt - t4.cuda() * F
    print(name, "v^ rel-L2", rel_l2(F, g["F"]), "x^ rel-L2", rel_l2(xh, g["x_hat"]))
    assert rel_l2(F, g["F"]) <= EVAL_TOL, (name, rel_l2(F, g["F"]))
    assert rel_l2(xh, g["x_hat"]) <= FWD_TOL, (name, rel_l2(xh, g["x_hat"]))


def test_sampler_vs_reference_golden():
    from maskdit_b200 import ops
    from maskdit_b200.sampler import flow_sampler
    g = load("flow_s2_sampler")
    net, _ = flow_net("DiT-S/2", 8, 10)
    net.eval()
    n0 = ops.L.LAUNCHES
    z = flow_sampler(net, g["latents"].cuda(), g["labels"].cuda(), cfg_scale=float(g["cfg_scale"]),
                     num_steps=int(g["num_steps"]))
    assert z.dtype == torch.float64 and ops.L.LAUNCHES > n0
    assert rel_l2(z, g["z"]) <= SAMPLER_TOL, rel_l2(z, g["z"])
    # Euler: N evaluations, and the interval gate: CFG only where lo < t <= hi
    calls = []
    orig = type(net).forward

    def spy(self, x, t, labels=None, cfg_scale=None, **kw):
        calls.append((float(t), cfg_scale))
        return orig(self, x, t, labels, cfg_scale, **kw)

    type(net).forward = spy
    try:
        flow_sampler(net, g["latents"].cuda(), g["labels"].cuda(), cfg_scale=1.5, num_steps=4, solver="euler",
                     guidance_interval=(0.3, 0.8))
        assert calls == [(1.0, None), (0.75, 1.5), (0.5, 1.5), (0.25, None)], calls
        calls.clear()
        flow_sampler(net, g["latents"].cuda(), g["labels"].cuda(), num_steps=4)
        assert len(calls) == 7
    finally:
        type(net).forward = orig


# ---- the kernels one by one against float64 ----------------------------------------------------------------------------
def unpatchify64(F, B, C, R, p):
    G = R // p
    return F.double().reshape(B, G, G, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, R, R)


def patchify64(img, p):
    B, C, R, _ = img.shape
    G = R // p
    return img.double().reshape(B, C, G, p, G, p).permute(0, 2, 4, 3, 5, 1).reshape(B, G * G, p * p * C)


def flow_loss64(F, xt, y, eps, t, mask, gl, coef, p):
    """(loss, x_hat, dF) in float64 by autograd."""
    B, C, R, _ = xt.shape
    F64 = F.double().clone().requires_grad_(True)
    v_hat = unpatchify64(F64, B, C, R, p)
    t4 = t.double().reshape(B, 1, 1, 1)
    xh = xt.double() - t4 * v_hat
    e = patchify64((v_hat - (eps.double() - y.double())) ** 2, p).mean(-1)   # [B, L] per-patch means
    if mask is None:
        loss = e.mean(1)
    else:
        m = mask.double()
        loss = (e * (1 - m)).sum(1) / (1 - m).sum(1)
        if coef > 0:
            tgt = patchify64(xt, p)
            tgt = (tgt - tgt.mean(-1, keepdim=True)) / (tgt.var(-1, keepdim=True) + 1e-6) ** 0.5
            mae = ((patchify64(xh, p) - tgt) ** 2).mean(-1)
            nm = m.sum(1)
            loss = loss + coef * torch.where(nm > 0, (mae * m).sum(1) / nm.clamp_min(1), torch.zeros_like(nm))
    (loss * gl.double()).sum().backward()
    return loss.detach(), xh.detach(), F64.grad


def bf16_ulp(x):
    """The spacing of bf16 values (8 significand bits) at |x|."""
    a = x.abs().double().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


@pytest.mark.parametrize("p", [2, 4, 8])
@pytest.mark.parametrize("mode", ["nomask", "mask", "mask_T_eq_L"])
def test_flow_loss_kernel_vs_float64(ops, p, mode):
    B, C, R = 4, 4, 32
    L = (R // p) ** 2
    g = torch.Generator(device="cuda").manual_seed(p)
    F = torch.randn(B, L, p * p * C, device="cuda", generator=g)
    y = torch.randn(B, C, R, R, device="cuda", generator=g)
    eps = torch.randn(B, C, R, R, device="cuda", generator=g)
    t = torch.tensor([1e-4, 0.3, 0.9, 0.9999], device="cuda")          # t near 0 and near 1
    xt = ((1 - t.view(-1, 1, 1, 1)) * y + t.view(-1, 1, 1, 1) * eps).contiguous()
    gl = torch.tensor([0.25, 1.0, 2.0, 0.5], device="cuda")
    mask, coef = None, 0.0
    if mode == "mask":
        mask = (torch.rand(B, L, device="cuda", generator=g) < 0.5).float()
        coef = 0.1
    elif mode == "mask_T_eq_L":
        mask, coef = torch.zeros(B, L, device="cuda"), 0.1
    loss, xh, dF = ops.flow_loss(F, xt, y, eps, t, mask, gl, coef, p, want_xhat=True, want_dF=True)
    l64, xh64, dF64 = flow_loss64(F, xt, y, eps, t, mask, gl, coef, p)
    assert (loss.double() - l64).abs().max().item() <= 1e-3 * l64.abs().max().item()
    assert (xh.double() - xh64).abs().max().item() <= 1e-3 * xh64.abs().max().item()
    err = (dF.double() - dF64).abs()
    bound = bf16_ulp(dF64) + 1e-5 * dF64.abs().max()
    assert bool((err <= bound).all()), (err / bound).max().item()
    lo, _, none = ops.flow_loss(F, xt, y, eps, t, mask, None, coef, p, want_dF=False)
    assert torch.equal(lo, loss) and none is None


@pytest.mark.parametrize("p", [2, 4, 8])
def test_flow_cfg_out_and_timestep_freq_vs_float64(ops, p):
    B, C, R = 3, 4, 32
    L = (R // p) ** 2
    F = torch.randn(2 * B, L, p * p * C, device="cuda")
    v = ops.flow_cfg_out(F, 2 * B, C, R, p)
    assert torch.equal(v.double(), unpatchify64(F, 2 * B, C, R, p))          # a pure rearrangement
    c = ops.flow_cfg_out(F, B, C, R, p, 1.5)
    u64 = unpatchify64(F, 2 * B, C, R, p)
    want = u64[B:] + 1.5 * (u64[:B] - u64[B:])
    assert (c.double() - want).abs().max().item() <= 1e-6 * want.abs().max().item()
    t = torch.tensor([0.0, 1e-4, 0.5, 0.9999, 1.0], device="cuda")
    tf = ops.flow_timestep_freq(t, 256).float().double()
    half = 128
    f = torch.exp(-np.log(10000.0) * torch.arange(half, dtype=torch.float64) / half).cuda()
    a = t.double()[:, None] * f[None]
    want = torch.cat([torch.cos(a), torch.sin(a)], 1)
    assert bool(((tf - want).abs() <= bf16_ulp(want) + 1e-6).all())


def test_flow_step_front_bitwise(ops):
    B, C, R, nc = 5, 4, 16, 10
    g = torch.Generator(device="cuda").manual_seed(3)
    moments = torch.randn(B, 2 * C, R, R, device="cuda", generator=g)
    eps = torch.randn(B, C, R, R, device="cuda", generator=g)
    rnd = torch.tensor([-6.0, -1.0, 0.0, 0.7, 6.0], device="cuda")
    noise = torch.randn(B, C, R, R, device="cuda", generator=g)
    labels = torch.eye(nc, device="cuda")[:B].contiguous()
    drop_u = torch.tensor([0.05, 0.5, 0.09, 0.99, 0.2], device="cuda")
    lab_e = labels.clone()
    y_e, _, _ = ops.step_front(moments, eps, rnd, noise, lab_e, drop_u, 0.1, 0.18215, -1.2, 1.2)
    lab_f = labels.clone()
    y, xt, t = ops.flow_step_front(moments, eps, rnd, noise, lab_f, drop_u, 0.1, 0.18215, 0.25, 1.5)
    assert torch.equal(y, y_e) and torch.equal(lab_f, lab_e)            # latent and label dropout are the EDM front's
    a = rnd * 1.5 + 0.25
    t_ref = 1.0 / (1.0 + torch.exp(-a))
    assert ((t - t_ref).abs() <= 1.2e-7 * t_ref).all(), (t - t_ref)
    t4 = t.view(-1, 1, 1, 1)
    assert torch.equal(xt, (1.0 - t4) * y + t4 * noise)                 # op by op, no contraction


# ---- the training step --------------------------------------------------------------------------------------------------
def _flow_steps(n=3, recompute=None, seed=0):
    from maskdit_b200.loss import FlowLoss
    from maskdit_b200.train_step import TrainStep
    net, _ = flow_net("DiT-S/2", 32, 1000)
    net.train()
    ts = TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, loss_fn=FlowLoss(), recompute_blocks=recompute)
    gen = torch.Generator().manual_seed(seed)
    moments = torch.randn(4, 8, 32, 32, generator=gen).cuda()
    lab = torch.eye(1000)[torch.randint(0, 1000, (4,), generator=gen)].cuda()
    torch.manual_seed(seed)
    losses = [ts.step(moments, lab.clone(), 0.5, 0.1, moments=True, class_dropout_prob=0.1).clone()
              for _ in range(n)]
    out = [*losses, ts.st.grad.clone(), ts.st.w32.clone(), ts.ema_st.w32.clone()]
    assert ts.recompute_blocks == (recompute or 0)
    return out


def test_flow_train_step_deterministic_and_recompute(det):
    a = _flow_steps()
    b = _flow_steps()
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), i
    assert all(torch.isfinite(v).all() for v in a)
    r = _flow_steps(recompute=12 + 8)                                   # every block recomputed
    for i, (x, y) in enumerate(zip(a, r)):
        assert torch.equal(x, y), i


# ---- the entry points ---------------------------------------------------------------------------------------------------
YAML = """
data: {dataset: imagenet256-latent, category: lmdb, resolution: 16, num_channels: 4, root: none, feat_path: None}
model:
  precond: flow
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


def run(cmd, cwd, ok=True):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, *cmd], cwd=cwd, env=env, capture_output=True, text=True, timeout=600)
    assert (r.returncode == 0) == ok, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout + r.stderr


def test_train_validate_then_generate_flow(tmp_path):
    cfg = tmp_path / "cfg.yaml"
    cfg.write_text(YAML)
    out = run([os.path.join(ROOT, "train.py"), "--config", str(cfg), "--synthetic", "--max_steps", "4",
               "--val_every", "2", "--val_count", "3", "--val_levels", "2", "--results_dir", str(tmp_path / "res")],
              str(tmp_path))
    assert "Train Loss" in out and "Val Loss (flow)" in out, out
    ck = tmp_path / "res" / "checkpoints" / "0000004.pt"
    assert ck.exists()
    out = run([os.path.join(ROOT, "generate.py"), "--config", str(cfg), "--ckpt_path", str(ck), "--seeds", "0-3",
               "--num_steps", "4", "--cfg_scale", "1.5", "--results_dir", str(tmp_path / "samples")], str(tmp_path))
    z = np.load(tmp_path / "samples" / "000002.npy")
    assert z.shape == (4, 16, 16) and np.isfinite(z).all()
    out = run([os.path.join(ROOT, "generate.py"), "--config", str(cfg), "--ckpt_path", str(ck), "--seeds", "0",
               "--num_steps", "4", "--S_churn", "10", "--results_dir", str(tmp_path / "s2")], str(tmp_path), ok=False)
    assert "--S_churn" in out
    out = run([os.path.join(ROOT, "val_loss.py"), "--config", str(cfg), "--ckpt", str(ck), "--synthetic", "--count",
               "3", "--levels", "2"], str(tmp_path))
    assert "flow loss" in out and " t " in out, out


def test_validation_identical_across_batches(ops):
    from maskdit_b200 import validate
    net, _ = flow_net("DiT-S/2", 8, 10)
    net.eval()
    held = validate.HeldOut.synthetic(5, 8, 4, 10)
    a = validate.validate(net, held, levels=3, batch=15)
    b = validate.validate(net, held, levels=3, batch=4)
    assert torch.equal(a["per_item"], b["per_item"]) and a["objective"] == "flow"
    np.testing.assert_allclose(a["t"], validate.t_levels(3))
