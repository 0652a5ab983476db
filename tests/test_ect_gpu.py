"""GPU: Easy Consistency Tuning (DESIGN §5) on the H100 kernels.  The loss, gradients, D_t and the consistency sampler
against goldens of the unmodified reference network with the ECT objective applied around it
(tests/golden/make_golden_ect.py), both kernels against float64 (r = 0 rows, t near sigma_min and 80, the smallest
final-stage gap), the step front against its fp32 formula, a deterministic, recompute-invariant ECT TrainStep that
takes the same bits graphed and eager across a stage boundary, resume, train.py / generate.py end to end, and a toy
run where tuning turns an EDM network's one-step output into samples of the data's modes."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from support import EVAL_TOL, GRAD_TOL, LOSS_TOL, check_grads, det, load, ops, oracle_net, rel_l2  # noqa: F401

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMPLER_TOL = 1e-2


def golden_loss(g, stage):
    """ECTLoss whose draws are the golden's: the t normal, eps, then the mask noise."""
    from maskdit_b200.loss import ECTLoss

    class L(ECTLoss):
        draws = [g["rnd_normal"].reshape(-1, 1, 1, 1).cuda(), g["noise_unit"].cuda()]

        def _randn(self, shape, device):
            return self.draws.pop(0)

        def _rand(self, shape, device):
            return g["mask_noise"].cuda()

    f = L(stage_steps=1)
    f.stage = stage
    return f


@pytest.mark.parametrize("name, mt, R, ncls, dec", [
    ("ect_s2_train_mask", "DiT-S/2", 8, 10, True),
    ("ect_nd_s2_uncond", "DiT-S/2", 8, 0, False),
    ("ect_xl2_mask", "DiT-XL/2", 32, 1000, True),
])
def test_loss_D_and_grads_vs_reference_golden(ops, name, mt, R, ncls, dec):
    g = load(name)
    net = oracle_net(mt, R, ncls, dec)
    x = g["images"].cuda()
    lab = g["labels"].cuda() if "labels" in g else None
    ratio, coef = float(g["mask_ratio"]), float(g["mae_coef"])
    f = golden_loss(g, int(g["stage"]))
    loss = f(net, x, lab, mask_ratio=ratio, mae_loss_coef=coef)
    loss.mean().backward()
    torch.cuda.synchronize()
    assert torch.equal(f.last_edm_loss, loss)
    r = rel_l2(loss, g["loss"])
    print(name, "loss rel", r, loss.tolist(), g["loss"].tolist())
    assert r <= LOSS_TOL, (name, loss.tolist(), g["loss"].tolist())
    # the decoder-less case misses 1.5e-2 on one tensor: t_embedder.mlp.0.bias at 1.56e-2 (the gradient seed is
    # proportional to D_t - D_r, where the two forwards' bf16 noise weighs more than in an EDM step; DESIGN §5)
    check_grads(net, g, 2e-2 if name == "ect_nd_s2_uncond" else GRAD_TOL, name)
    # D_t: the student forward with the golden's mask, through the loss kernel's optional output
    md = ops.mask_indices(g["mask_noise"].cuda(), int(net.model.num_patches * (1 - ratio))) if ratio > 0 else None
    t, rr = g["t"].cuda(), g["r"].cuda()
    t4, r4 = t.view(-1, 1, 1, 1), rr.view(-1, 1, 1, 1)
    eps = g["noise_unit"].cuda()
    xt, xr = (x + t4 * eps).contiguous(), (x + r4 * eps).contiguous()
    _, _, labn = net._norm_inputs(x, t, lab)
    with torch.no_grad():
        Ft, _ = net._engine.forward(xt, t, labn, md, save=False)
        Fr, _ = net._engine.forward(xr, torch.where(rr > 0, rr, t).contiguous(), labn, md, save=False)
    c = 0.00054 * (x[0].numel()) ** 0.5
    lo, D, _ = ops.ect_loss(Ft, Fr, xt, xr, x, t, rr, md["mask"] if md else None, None, 0.5, c, coef,
                            net.model.patch_size, want_D=True, want_dF=False)
    # at t >> sigma_data D_t is c_out F almost alone, with no c_skip x_t term to dilute the bf16 error (the t = 6.7 row of
    # the S/2 case: 3.7e-3 measured): the bound of the unmasked eval forward, as for the flow objective's raw output
    print(name, "D_t rel-L2", rel_l2(D, g["D_t"]))
    assert rel_l2(D, g["D_t"]) <= EVAL_TOL
    assert rel_l2(lo, g["loss"]) <= LOSS_TOL


def test_sampler_vs_reference_golden(ops):
    from maskdit_b200.sampler import consistency_sampler
    g = load("ect_s2_sampler")
    net = oracle_net("DiT-S/2", 8, 10, True).eval()
    noises = [n.cuda() for n in g["noises"]]
    drawn = []

    def randn_like(x):
        drawn.append(tuple(x.shape))
        return noises[len(drawn) - 1].to(x.dtype)

    n0 = ops.L.LAUNCHES
    z = consistency_sampler(net, g["latents"].cuda(), g["labels"].cuda(), cfg_scale=float(g["cfg_scale"]),
                            randn_like=randn_like, sigmas=tuple(g["sigmas"].tolist()))
    assert z.dtype == torch.float64 and ops.L.LAUNCHES > n0 and len(drawn) == len(g["sigmas"]) - 1
    print("sampler rel-L2", rel_l2(z, g["z"]))
    assert rel_l2(z, g["z"]) <= SAMPLER_TOL
    # one evaluation per level; the interval gate and the clamp to sigma_max are edm_sampler's
    calls = []
    orig = type(net).forward

    def spy(self, x, sigma, labels=None, cfg_scale=None, **kw):
        calls.append((float(sigma), cfg_scale))
        return orig(self, x, sigma, labels, cfg_scale, **kw)

    type(net).forward = spy
    try:
        net.sigma_max = 40.0
        consistency_sampler(net, g["latents"].cuda(), g["labels"].cuda(), cfg_scale=1.5, sigmas=(80.0, 2.0, 0.5),
                            guidance_interval=(1.0, 50.0))
        assert calls == [(40.0, 1.5), (2.0, 1.5), (0.5, None)], calls
    finally:
        type(net).forward = orig
        net.sigma_max = float("inf")


# ---- the kernels one by one against float64 ----------------------------------------------------------------------------
def unpatchify64(F, B, C, R, p):
    G = R // p
    return F.double().reshape(B, G, G, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, R, R)


def patchify64(img, p):
    B, C, R, _ = img.shape
    G = R // p
    return img.double().reshape(B, C, G, p, G, p).permute(0, 2, 4, 3, 5, 1).reshape(B, G * G, p * p * C)


def ect_loss64(Ft, Fr, xt, xr, y, t, r, mask, gl, sd, c, coef, p):
    """(loss, D_t, dF_t) in float64 by autograd."""
    B, C, R, _ = xt.shape
    F64 = Ft.double().clone().requires_grad_(True)
    t4, r4 = t.double().view(-1, 1, 1, 1), r.double().view(-1, 1, 1, 1)
    cs = lambda s: sd * sd / (s * s + sd * sd)                      # noqa: E731
    co = lambda s: s * sd / (s * s + sd * sd).sqrt()                 # noqa: E731
    Dt = cs(t4) * xt.double() + co(t4) * unpatchify64(F64, B, C, R, p)
    Dr = torch.where(r4 > 0, cs(r4) * xr.double() + co(r4) * unpatchify64(Fr, B, C, R, p), y.double())
    se = patchify64((Dt - Dr) ** 2, p).sum(-1)                       # [B, L]
    L = se.shape[1]
    if mask is None:
        S = se.sum(1)
    else:
        keep = 1 - mask.double()
        S = (se * keep).sum(1) * (L / keep.sum(1))
    loss = ((S + c * c).sqrt() - c) / (t.double() - r.double())
    if mask is not None and coef > 0:
        m = mask.double()
        tgt = patchify64(xt, p)
        tgt = (tgt - tgt.mean(-1, keepdim=True)) / (tgt.var(-1, keepdim=True) + 1e-6) ** 0.5
        mae = ((patchify64(Dt, p) - tgt) ** 2).mean(-1)
        nm = m.sum(1)
        loss = loss + coef * torch.where(nm > 0, (mae * m).sum(1) / nm.clamp_min(1), torch.zeros_like(nm))
    (loss * gl.double()).sum().backward()
    return loss.detach(), Dt.detach(), F64.grad


def bf16_ulp(x):
    a = x.abs().double().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


GAP = 2.0 ** -8   # the smallest final-stage gap (t - r) / t tested: q^-(s+1) at q = 2, s = 7 and large t


def kernel_inputs(p, mode, B=6, C=4, R=32):
    """Rows: t near sigma_min with r = 0 and with the smallest gap, r = 0 at t = 0.5, a stage-1 pair at t = 2, t = 80
    with r = 0 and with the smallest gap.  F_r of an r = 0 row is NaN (it must not reach anything); elsewhere
    F_r = F_t + 1e-3 noise, the nearly consistent outputs of a tuned network."""
    from maskdit_b200.loss import ect_r
    L = (R // p) ** 2
    g = torch.Generator(device="cuda").manual_seed(p)
    Ft = torch.randn(B, L, p * p * C, device="cuda", generator=g)
    Fr = Ft + 1e-3 * torch.randn(B, L, p * p * C, device="cuda", generator=g)
    y = torch.randn(B, C, R, R, device="cuda", generator=g) * 0.5
    eps = torch.randn(B, C, R, R, device="cuda", generator=g)
    t = torch.tensor([0.002, 0.002, 0.5, 2.0, 80.0, 80.0], device="cuda")
    r = torch.stack([torch.tensor(0.0), torch.tensor(0.002 * (1 - GAP)), torch.tensor(0.0),
                     ect_r(torch.tensor(2.0), 0.25), torch.tensor(0.0), torch.tensor(80.0 * (1 - GAP))]).float().cuda()
    Fr[r == 0] = float("nan")
    xt = (y + t.view(-1, 1, 1, 1) * eps).contiguous()
    xr = (y + r.view(-1, 1, 1, 1) * eps).contiguous()
    gl = torch.tensor([0.25, 1.0, 2.0, 0.5, 1.5, 1.0], device="cuda")
    mask, coef = None, 0.0
    if mode == "mask":
        mask, coef = (torch.rand(B, L, device="cuda", generator=g) < 0.5).float(), 0.1
    elif mode == "mask_T_eq_L":
        mask, coef = torch.zeros(B, L, device="cuda"), 0.1
    return Ft, Fr, xt, xr, y, t, r, mask, gl, coef, 0.00054 * (C * R * R) ** 0.5


@pytest.mark.parametrize("p", [2, 4, 8])
@pytest.mark.parametrize("mode", ["nomask", "mask", "mask_T_eq_L"])
def test_ect_loss_kernel_vs_float64(ops, p, mode):
    Ft, Fr, xt, xr, y, t, r, mask, gl, coef, c = kernel_inputs(p, mode)
    loss, D, dF = ops.ect_loss(Ft, Fr, xt, xr, y, t, r, mask, gl, 0.5, c, coef, p, want_D=True, want_dF=True)
    l64, D64, dF64 = ect_loss64(Ft, Fr, xt, xr, y, t, r, mask, gl, 0.5, c, coef, p)
    assert bool(torch.isfinite(loss).all()) and bool(torch.isfinite(dF.float()).all())
    rel = ((loss.double() - l64).abs() / l64.abs()).cpu()
    print(p, mode, "per-row loss rel err", rel.tolist(), "loss", l64.tolist())
    assert bool((rel <= 1e-3).all()), rel                     # every row on its own, the smallest gaps included
    assert (D.double() - D64).abs().max().item() <= 1e-6 * D64.abs().max().item()
    err = (dF.double() - dF64).abs()
    # one bf16 ulp, plus the fp32 rounding of D_t and D_r, which at the smallest gap is ~1e-3 of the largest delta
    bound = bf16_ulp(dF64) + 1e-3 * dF64.abs().amax(dim=(1, 2), keepdim=True)
    assert bool((err <= bound).all()), (err / bound).max().item()
    lo, none_D, none = ops.ect_loss(Ft, Fr, xt, xr, y, t, r, mask, None, 0.5, c, coef, p, want_dF=False)
    assert torch.equal(lo, loss) and none is None and none_D is None


def test_smallest_gap_not_swamped_by_rounding(ops):
    """At the smallest final-stage gap, (t - r) / t = 2^-8, delta = D_t - D_r is a small difference of two nearly equal
    outputs, where fp32 rounding of D_t and D_r is largest relative to it.  The kernel's loss must follow float64 there,
    and resolve the part of the loss that the 1e-3 difference between F_t and F_r contributes: its error must stay far
    below the change that difference makes."""
    p = 2
    Ft, Fr, xt, xr, y, t, r, mask, gl, coef, c = kernel_inputs(p, "mask")
    loss, _, _ = ops.ect_loss(Ft, Fr, xt, xr, y, t, r, mask, None, 0.5, c, 0.0, p, want_dF=False)
    l64, _, _ = ect_loss64(Ft, Fr, xt, xr, y, t, r, mask, gl, 0.5, c, 0.0, p)
    Fs = torch.where(torch.isnan(Fr), Fr, Ft)                      # the same outputs: only the levels differ
    s64, _, _ = ect_loss64(Ft, Fs, xt, xr, y, t, r, mask, gl, 0.5, c, 0.0, p)
    for i in (1, 5):                                               # t = 0.002 and t = 80 at the smallest gap
        err = abs(float(loss[i]) - float(l64[i]))
        signal = abs(float(l64[i]) - float(s64[i]))
        print(f"t {float(t[i]):g} gap {float((t[i] - r[i]) / t[i]):.3g}: loss {float(loss[i]):.6g} float64 "
              f"{float(l64[i]):.6g} rel {err / float(l64[i]):.2e}; F_t - F_r moves the loss by {signal:.3g}, "
              f"error / that {err / signal:.2e}")
        assert err <= 1e-3 * float(l64[i])
        assert err <= 0.1 * signal


def test_ect_step_front_bitwise(ops):
    from maskdit_b200.loss import ect_r
    B, C, R, nc = 6, 4, 16, 10
    g = torch.Generator(device="cuda").manual_seed(3)
    moments = torch.randn(B, 2 * C, R, R, device="cuda", generator=g)
    eps = torch.randn(B, C, R, R, device="cuda", generator=g)
    rnd = torch.tensor([-4.0, -1.0, 0.0, 0.7, 1.6, 2.7], device="cuda")
    noise = torch.randn(B, C, R, R, device="cuda", generator=g)
    labels = torch.eye(nc, device="cuda")[:B].contiguous()
    drop_u = torch.tensor([0.05, 0.5, 0.09, 0.99, 0.2, 0.3], device="cuda")
    lab_e = labels.clone()
    y_e, _, _ = ops.step_front(moments, eps, rnd, noise, lab_e, drop_u, 0.1, 0.18215, -1.2, 1.2)
    for qs in (0.5, 2.0 ** -5):
        word = torch.tensor([qs], device="cuda")
        lab = labels.clone()
        y, xt, xr, sr, t, r = ops.ect_step_front(moments, eps, rnd, noise, word, lab, drop_u, 0.1, 0.18215, -1.1, 2.0,
                                                 8.0, 1.0)
        assert torch.equal(y, y_e) and torch.equal(lab, lab_e)       # latent and label dropout are the EDM front's
        t_ref = (rnd * 2.0 + -1.1).exp()
        assert ((t - t_ref).abs() <= 2.4e-7 * t_ref).all(), (t - t_ref)
        r_ref = ect_r(t, word, 8.0, 1.0)
        assert ((r - r_ref).abs() <= 2.4e-7 * t).all(), (r - r_ref)   # expf vs torch.exp in the sigmoid: an ulp
        if qs == 0.5:
            assert bool((r == 0).any()) and bool((r > 0).any())
        t4, r4 = t.view(-1, 1, 1, 1), r.view(-1, 1, 1, 1)
        assert torch.equal(xt, y + t4 * noise) and torch.equal(xr, y + r4 * noise)   # op by op, no contraction
        assert torch.equal(sr, torch.where(r > 0, r, t))


# ---- the training step --------------------------------------------------------------------------------------------------
class FixedDraws:
    """An ECTLoss mix-in whose draws repeat every step (randn in from_moments' order: eps, the t normal, the noise;
    rand: the label dropout, the mask noise), so a captured graph and the eager step see the same values."""

    def _randn(self, shape, device):
        k = (tuple(shape), self._n % 3)
        self._n += 1
        if k not in self._bank:
            g = torch.Generator(device=device).manual_seed(len(self._bank) + 11)
            self._bank[k] = torch.randn(shape, device=device, generator=g)
        return self._bank[k]

    def _rand(self, shape, device):
        k = tuple(shape)
        if k not in self._bank:
            g = torch.Generator(device=device).manual_seed(len(self._bank) + 101)
            self._bank[k] = torch.rand(shape, device=device, generator=g)
        return self._bank[k]


def fixed_loss(stage_steps):
    from maskdit_b200.loss import ECTLoss

    class L(FixedDraws, ECTLoss):
        pass

    f = L(stage_steps=stage_steps)
    f._n, f._bank = 0, {}
    return f


def _ect_steps(n=4, recompute=None, seed=0, graph=False, fixed=False, stage_steps=2, grad_accum=1):
    from maskdit_b200.loss import ECTLoss
    from maskdit_b200.train_step import TrainStep
    net = oracle_net("DiT-S/2", 32, 1000, True)
    loss_fn = fixed_loss(stage_steps) if fixed else ECTLoss(stage_steps=stage_steps)
    ts = TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, loss_fn=loss_fn, recompute_blocks=recompute,
                   graph=graph)
    gen = torch.Generator().manual_seed(seed)
    moments = torch.randn(4, 8, 32, 32, generator=gen).cuda()
    lab = torch.eye(1000)[torch.randint(0, 1000, (4,), generator=gen)].cuda()
    torch.manual_seed(seed)
    losses, stages = [], []
    for _ in range(n):
        losses.append(ts.step(moments, lab.clone(), 0.5, 0.1, moments=True, class_dropout_prob=0.1,
                              grad_accum=grad_accum).clone())
        stages.append(ts.ect_stage)
    out = [*losses, ts.st.grad.clone(), ts.st.w32.clone(), ts.ema_st.w32.clone()]
    assert ts.recompute_blocks == (recompute or 0)
    return out, stages, ts


def assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (i, (x.double() - y.double()).abs().max().item())


def test_ect_train_step_deterministic_and_recompute(det):
    a, stages, ts = _ect_steps()
    assert stages == [0, 0, 1, 1] and ts.ect_origin == 0
    assert all(bool(torch.isfinite(v).all()) for v in a)
    b, _, _ = _ect_steps()
    assert_same(a, b)
    r, _, _ = _ect_steps(recompute=12 + 8)                          # every block recomputed
    assert_same(a, r)
    ga, _, _ = _ect_steps(n=2, grad_accum=2)
    assert all(bool(torch.isfinite(v).all()) for v in ga) and ga[0].shape == (4,)


def test_ect_graph_matches_eager_across_stage_boundary(det):
    eager, stages, _ = _ect_steps(fixed=True)
    graphed, stages_g, ts = _ect_steps(fixed=True, graph=True)
    assert stages == stages_g == [0, 0, 1, 1] and len(ts._graphs) == 1   # one capture serves both stages
    assert_same(eager, graphed)
    # the stage word reaches the replay: with the same draws and weights, stage 1 gives another loss than stage 0
    assert not torch.equal(eager[1], eager[2])


def test_ect_resume_continues_the_stage(det):
    from maskdit_b200.train_step import TrainStep
    straight, stages, _ = _ect_steps(n=4, fixed=True)
    first, _, ts = _ect_steps(n=3, fixed=True)
    sd = ts.state_dict()
    assert sd["ect"] == {"origin": 0, "stage_steps": 2}
    net2 = oracle_net("DiT-S/2", 32, 1000, True)
    net2.load_state_dict(ts.net.state_dict())
    ema2 = copy.deepcopy(net2).eval()
    ema2.load_state_dict(ts.ema.state_dict())
    ts2 = TrainStep(net2, ema2, lr=1e-3, loss_fn=fixed_loss(2))
    ts2.load_state_dict(sd)
    ts2.lr_step_offset = 3 - ts2.step_count                          # train.py: the run step from the checkpoint name
    gen = torch.Generator().manual_seed(0)
    moments = torch.randn(4, 8, 32, 32, generator=gen).cuda()
    lab = torch.eye(1000)[torch.randint(0, 1000, (4,), generator=gen)].cuda()
    torch.manual_seed(0)
    last = ts2.step(moments, lab.clone(), 0.5, 0.1, moments=True, class_dropout_prob=0.1).clone()
    assert ts2.ect_stage == 1 and ts2.ect_origin == 0
    assert torch.equal(last, straight[3]) and torch.equal(ts2.st.w32, straight[5])
    # a state without the tuning origin (an EDM run's optimizer state) starts tuning at the next step: stage 0
    sd.pop("ect")
    ts3 = TrainStep(copy.deepcopy(net2), lr=1e-3, loss_fn=fixed_loss(2))
    ts3.load_state_dict(sd)
    ts3.lr_step_offset = 3 - ts3.step_count
    ts3.step(moments, lab.clone(), 0.5, 0.1, moments=True)
    assert ts3.ect_origin == 3 and ts3.ect_stage == 0


# ---- the entry points ---------------------------------------------------------------------------------------------------
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


def run(cmd, cwd, ok=True):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, *cmd], cwd=cwd, env=env, capture_output=True, text=True, timeout=600)
    assert (r.returncode == 0) == ok, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout + r.stderr


def test_pretrain_tune_resume_then_generate(tmp_path):
    edm = tmp_path / "edm.yaml"
    edm.write_text(YAML)
    run([os.path.join(ROOT, "train.py"), "--config", str(edm), "--synthetic", "--max_steps", "4",
         "--results_dir", str(tmp_path / "pre")], str(tmp_path))
    pre = tmp_path / "pre" / "checkpoints" / "0000004.pt"
    ect = tmp_path / "ect.yaml"
    ect.write_text(YAML.replace("max_num_steps: 4}", "max_num_steps: 4, objective: ect, ect: {stage_steps: 2}}"))
    out = run([os.path.join(ROOT, "train.py"), "--config", str(ect), "--synthetic", "--max_steps", "4",
               "--ckpt_path", str(pre), "--use_strict_load", "False", "--val_every", "2", "--val_count", "3",
               "--val_levels", "2", "--results_dir", str(tmp_path / "ect")], str(tmp_path))
    # tuning starts at the checkpoint's step 4: stage 0 for steps 4-5, stage 1 for steps 6-7
    assert "ECT stage: 0" in out and "ECT stage: 1" in out and "Val Loss" in out, out
    ck = tmp_path / "ect" / "checkpoints" / "0000008.pt"
    sd = torch.load(ck, map_location="cpu", weights_only=False)
    assert sd["opt"]["ect"]["origin"] == 4
    out = run([os.path.join(ROOT, "train.py"), "--config", str(ect), "--synthetic", "--max_steps", "2",
               "--ckpt_path", str(ck), "--results_dir", str(tmp_path / "ect")], str(tmp_path))
    assert "ECT stage: 2" in out, out                               # resumed at step 8: (8 - 4) // 2
    bad = tmp_path / "bad.yaml"
    bad.write_text(YAML.replace("max_num_steps: 4}", "max_num_steps: 4, objective: ect}"))
    out = run([os.path.join(ROOT, "train.py"), "--config", str(bad), "--synthetic", "--max_steps", "1",
               "--results_dir", str(tmp_path / "bad")], str(tmp_path), ok=False)
    assert "stage_steps" in out
    for sig in (["80"], ["80", "0.8"]):
        d = tmp_path / f"s{len(sig)}"
        run([os.path.join(ROOT, "generate.py"), "--config", str(ect), "--ckpt_path", str(ck), "--seeds", "0-3",
             "--cfg_scale", "1.5", "--consistency_sigmas", *sig, "--results_dir", str(d)], str(tmp_path))
        z = np.load(d / "000002.npy")
        assert z.shape == (4, 16, 16) and np.isfinite(z).all()
    out = run([os.path.join(ROOT, "generate.py"), "--config", str(ect), "--ckpt_path", str(ck), "--seeds", "0",
               "--consistency_sigmas", "80", "--S_churn", "10", "--results_dir", str(tmp_path / "x")], str(tmp_path),
              ok=False)
    assert "--S_churn" in out


# ---- a toy run: tuning turns the EDM network's one-step output into samples of the modes ------------------------------
def test_toy_one_step_samples_reach_the_modes(det):
    """DiT-S/2 at R = 8 on a synthetic set where each of 4 classes is two fixed latents +-P_c (per-element rms 0.5,
    sigma_data's).  EDM pretraining gives a denoiser whose one-step output D(80 z) is the class mean, 0, at rms
    distance ~0.5 from the nearest mode; ECT tuning from it, then the EMA's one-step samples, must land several times
    closer.  Measured on an H100 (deterministic mode): EDM one-step distance 0.44, tuned EMA 0.11; the bound is a
    third of the EDM distance."""
    from maskdit_b200.loss import ECTLoss, EDMLoss
    from maskdit_b200.maskdit import Precond_models
    from maskdit_b200.sampler import consistency_sampler
    from maskdit_b200.train_step import TrainStep
    ncls, R, B = 4, 8, 64
    gen = torch.Generator().manual_seed(0)
    P = torch.randn(ncls, 4, R, R, generator=gen)
    P = (P * 0.5 / P.pow(2).mean(dim=(1, 2, 3), keepdim=True).sqrt()).cuda()
    g = torch.Generator(device="cuda").manual_seed(1)

    def batch():
        c = torch.randint(0, ncls, (B,), device="cuda", generator=g)
        s = torch.randint(0, 2, (B,), device="cuda", generator=g).float() * 2 - 1
        return P[c] * s.view(-1, 1, 1, 1), torch.eye(ncls, device="cuda")[c]

    def one_step_distance(model):
        c = torch.arange(256, device="cuda") % ncls
        z = torch.randn(256, 4, R, R, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
        x = consistency_sampler(model, z, torch.eye(ncls, device="cuda")[c], sigmas=(80.0,)).float()
        d = torch.stack([(x - P[c]).pow(2).mean(dim=(1, 2, 3)), (x + P[c]).pow(2).mean(dim=(1, 2, 3))]).amin(0)
        return d.sqrt().mean().item()

    torch.manual_seed(0)
    net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=ncls, model_type="DiT-S/2",
                                use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False).cuda().train()
    ts = TrainStep(net, None, lr=5e-4, loss_fn=EDMLoss())
    for _ in range(400):
        ts.step(*batch(), mask_ratio=0.0, mae_loss_coef=0.0)
    d_edm = one_step_distance(net.eval())
    net.train()
    ema = copy.deepcopy(net).eval()
    ts = TrainStep(net, ema, lr=5e-4, loss_fn=ECTLoss(stage_steps=150), ema_decay=0.99)
    for _ in range(600):
        loss = ts.step(*batch(), mask_ratio=0.0, mae_loss_coef=0.0)
    assert bool(torch.isfinite(loss).all()) and ts.ect_stage == 3
    d_ect = one_step_distance(ema)
    print(f"one-step rms distance to the nearest mode: EDM {d_edm:.4f}, ECT EMA {d_ect:.4f}")
    assert d_edm > 0.3
    assert d_ect < d_edm / 3
