"""GPU: the learned loss weighting u(sigma) (`EDMPrecond(logvar_channels=C)`, EDM2 uncertainty weighting).

1. `logvar(sigma)` and the weighted loss kernel against float64: u, the objective exp(-u) E + u + M, du, and w's
   gradient kernel; the kernel's reference loss is the unweighted kernel's bit for bit.
2. The fused loss on DiT-S/2 with and without the decoder, at mask 0 and 0.5 with MAE 0.1: with w = 0 one TrainStep
   gives the network gradients of a net without the weighting bit for bit (deterministic mode); with w != 0 the network
   gradient is the linear combination of unweighted runs with per-sample gradient seeds; w's gradient against float64.
3. The training step: w moves and the EMA / post-hoc profiles carry it; resume equals an uninterrupted run; grad_norm
   covers w; a skipped step leaves w; grad_accum = 2 equals the whole batch; the CUDA graph equals eager.
4. generate.py samples a checkpoint with logvar_* keys under a config without them."""
import copy
import io
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

C_LV, R, NCLS = 128, 8, 10
_SD = {}


@pytest.fixture
def det():
    """Deterministic mode for the test; the torch flag and the library setting are restored afterwards."""
    from maskdit_b200 import _lib
    L = _lib.lib()
    was, flag = L.mdt_get_deterministic(), torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(flag)
    assert L.mdt_set_deterministic(was) == 0


def _net(C=0, dec=True, w_scale=0.0, seed=3):
    """DiT-S/2 at 8x8 from the oracle's random weights (seed 1); logvar weight w_scale * randn (seed `seed`)."""
    from maskdit_b200.maskdit import EDMPrecond
    from oracle import maskdit_oracle as O
    if dec not in _SD:
        _SD[dec] = O.make_state_dict(O.Cfg(model_type="DiT-S/2", img_resolution=R, num_classes=NCLS,
                                           use_decoder=dec), 1)
    net = EDMPrecond(R, 4, num_classes=NCLS, model_type="DiT-S/2", use_decoder=dec, mae_loss_coef=0.1,
                     logvar_channels=C)
    net.load_state_dict(_SD[dec], strict=False)
    if C and w_scale:
        with torch.no_grad():
            net.logvar_linear.weight.copy_(w_scale * torch.randn(1, C, generator=torch.Generator().manual_seed(seed)))
    return net.cuda().train()


def _phi64(net, sigma):
    """[N, C] float64 features sqrt(2) cos(freqs c + phases), c = ln(sigma) / 4."""
    f = net.logvar_fourier.freqs.detach().double().cpu()
    p = net.logvar_fourier.phases.detach().double().cpu()
    c = torch.log(torch.as_tensor(sigma).double().cpu().reshape(-1, 1)) / 4
    return math.sqrt(2) * torch.cos(f[None] * c + p[None])


def _u64(net, sigma):
    return _phi64(net, sigma) @ net.logvar_linear.weight.detach().double().cpu().reshape(-1)


class FixedLoss:
    """EDMLoss whose draws come from pre-drawn per-sample tensors, handed out in batch order: a whole batch and its
    micro-batches see the same noise, sigma and mask noise."""

    def __new__(cls, Bt, seed=0):
        from maskdit_b200.loss import EDMLoss

        class _L(EDMLoss):
            def __init__(self):
                super().__init__()
                g = torch.Generator().manual_seed(seed)
                self.rnd = torch.randn(Bt, 1, 1, 1, generator=g).cuda()
                self.noise = torch.randn(Bt, 4, R, R, generator=g).cuda()
                self.mnoise = torch.rand(Bt, (R // 2) ** 2, generator=g).cuda()
                self.off = 0

            def _randn(self, shape, device):
                n = shape[0]
                if len(shape) == 4 and shape[1] == 1:
                    return self.rnd[self.off:self.off + n].clone()
                return self.noise[self.off:self.off + n].clone()

            def _rand(self, shape, device):   # the mask draw is the call's last: the next call starts further on
                n = shape[0]
                out = self.mnoise[self.off:self.off + n].clone()
                self.off = (self.off + n) % Bt
                return out

        return _L()


def _data(B, seed=0):
    g = torch.Generator().manual_seed(100 + seed)
    x = (torch.randn(B, 4, R, R, generator=g) * 0.5).cuda()
    lab = torch.eye(NCLS)[torch.randint(0, NCLS, (B,), generator=g)].cuda()
    return x, lab


def _sigma(loss_fn, lo, hi):
    return (loss_fn.rnd[lo:hi] * loss_fn.P_std + loss_fn.P_mean).exp().reshape(-1)


# ---- 1. kernels ---------------------------------------------------------------------------------------------------------
def test_logvar_vs_float64():
    net = _net(C_LV, w_scale=0.05)
    sigma = torch.logspace(math.log10(0.002), math.log10(80.0), 97)
    u = net.logvar(sigma).double().cpu()
    ref = _u64(net, sigma.float())
    err = (u - ref).abs().max().item()
    assert err <= 1e-5, err
    # one value per element, any container
    assert torch.equal(net.logvar([0.5]).cpu(), net.logvar(torch.tensor([0.5])).cpu())


@pytest.mark.parametrize("p,mask_ratio", [(2, 0.0), (2, 0.5), (8, 0.5)], ids=["p2-mask0", "p2-mask50", "p8-mask50"])
def test_weighted_loss_kernel_vs_float64(p, mask_ratio):
    from maskdit_b200 import ops
    torch.manual_seed(0)
    B, Cc, Rr, Cl = 6, 4, 32, 96
    L = (Rr // p) ** 2
    F = torch.randn(B * L, p * p * Cc, device="cuda")
    xin, y = torch.randn(B, Cc, Rr, Rr, device="cuda"), torch.randn(B, Cc, Rr, Rr, device="cuda")
    sigma = torch.exp(torch.randn(B, device="cuda") * 1.2 - 1.2)
    mask = None
    if mask_ratio:
        mask = ops.mask_indices(torch.rand(B, L, device="cuda"), int(L * (1 - mask_ratio)))["mask"]
    freqs = 2 * math.pi * torch.randn(Cl, device="cuda")
    phases = 2 * math.pi * torch.rand(Cl, device="cuda")
    w = 0.2 * torch.randn(Cl, device="cuda")
    gl = torch.rand(B, device="cuda") + 0.5
    mae = 0.1
    obj, loss, u, du, dF = ops.edm_loss_logvar(F, xin, y, sigma, mask, gl, 0.5, mae, p, freqs, phases, w)
    ref_loss, _, ref_dF = ops.edm_loss(F, xin, y, sigma, mask, gl, 0.5, mae, p)
    assert torch.equal(loss, ref_loss)                       # the reference loss: the unweighted kernel's bits
    E, _, _ = ops.edm_loss(F, xin, y, sigma, mask, None, 0.5, 0.0, p, want_dF=False)   # the EDM term alone
    M = loss.double() - E.double()
    phi = math.sqrt(2) * torch.cos(freqs.double()[None] * (torch.log(sigma.double())[:, None] / 4)
                                   + phases.double()[None])
    u64 = phi @ w.double()
    assert (u.double() - u64).abs().max().item() <= 1e-5
    obj64 = torch.exp(-u64) * E.double() + u64 + M
    assert ((obj.double() - obj64).abs() / obj64.abs().clamp_min(1)).max().item() <= 2e-6
    du64 = gl.double() * (1 - torch.exp(-u64) * E.double())
    assert ((du.double() - du64).abs() / (gl.double() * (1 + torch.exp(-u64) * E.double()))).max().item() <= 2e-6
    # w = 0: u = 0 and the gradient seed is the unweighted kernel's bit for bit
    z = torch.zeros_like(w)
    obj0, loss0, u0, du0, dF0 = ops.edm_loss_logvar(F, xin, y, sigma, mask, gl, 0.5, mae, p, freqs, phases, z)
    assert torch.equal(dF0, ref_dF) and torch.equal(loss0, ref_loss) and not u0.any()
    assert torch.equal(obj0, loss0)
    if mask is None:
        # without a mask there is no MAE term: the seed is the unweighted one at gl exp(-u) (up to the exp's rounding)
        _, _, dF_s = ops.edm_loss(F, xin, y, sigma, None, gl * torch.exp(-u), 0.5, mae, p)
        d = (dF.float() - dF_s.float()).abs().max().item()
        assert d <= 1e-2 * dF_s.float().abs().max().item(), d
    # the weight gradient: fixed-order fp64 sum, accumulating
    dw = torch.full((Cl,), 0.25, device="cuda")
    ops.logvar_wgrad(sigma, freqs, phases, du, dw)
    want = 0.25 + phi.T @ du.double()
    scale = phi.abs().T @ du.double().abs() + 0.25
    assert ((dw.double() - want).abs() / scale).max().item() <= 1e-6
    dw2 = dw.clone()
    ops.logvar_wgrad(sigma, freqs, phases, du, dw2)                # a second round adds to the first
    assert ((dw2.double() - (2 * want - 0.25)).abs() / scale).max().item() <= 2e-6
    again = torch.full((Cl,), 0.25, device="cuda")
    ops.logvar_wgrad(sigma, freqs, phases, du, again)
    assert torch.equal(again, dw)


# ---- 2. the fused loss ----------------------------------------------------------------------------------------------
CASES = [(dec, m) for dec in (True, False) for m in (0.0, 0.5)]
IDS = [f"{'dec' if d else 'nodec'}-mask{int(m * 100)}" for d, m in CASES]


class _CaptureE:
    """Wraps ops.edm_loss_logvar: every forward call also records sigma and the EDM term E (the unweighted kernel
    without the MAE term)."""

    def __init__(self, monkeypatch):
        from maskdit_b200 import ops
        self.real, self.calls = ops.edm_loss_logvar, []

        def wrapped(F, xin, y, sigma, mask, gl, sd, mae, p, *a, **k):
            if gl is None:
                E, _, _ = ops.edm_loss(F, xin, y, sigma, mask, None, sd, 0.0, p, want_dF=False)
                self.calls.append((sigma.clone(), E.clone()))
            return self.real(F, xin, y, sigma, mask, gl, sd, mae, p, *a, **k)

        monkeypatch.setattr(ops, "edm_loss_logvar", wrapped)


def _w_grad64(net, calls):
    """(1/B) sum_i (1 - exp(-u_i) E_i) phi(c_i) in float64 over the recorded calls (each call one mean over B)."""
    tot = 0
    for sigma, E in calls:
        phi = _phi64(net, sigma)
        u = phi @ net.logvar_linear.weight.detach().double().cpu().reshape(-1)
        du = (1 - torch.exp(-u) * E.double().cpu()) / sigma.numel()
        tot = tot + phi.T @ du
    return tot


@pytest.mark.parametrize("dec,mask", CASES, ids=IDS)
def test_w_zero_step_gradients_bit_identical(det, monkeypatch, dec, mask):
    from maskdit_b200.train_step import TrainStep
    B = 4
    x, lab = _data(B)
    off, on = _net(0, dec), _net(C_LV, dec)
    ts_off = TrainStep(off, lr=1e-3, loss_fn=FixedLoss(B))
    cap = _CaptureE(monkeypatch)
    ts_on = TrainStep(on, lr=1e-3, loss_fn=FixedLoss(B))
    l_off = ts_off.step(x, lab, mask, 0.1)
    w0 = on.logvar_linear.weight.detach().clone()
    l_on = ts_on.step(x, lab, mask, 0.1)
    n = ts_off.st.n_train
    assert ts_on.st.n_train == n + C_LV
    assert torch.equal(ts_on.st.grad[:n], ts_off.st.grad), "network gradients differ from the unweighted step"
    assert torch.equal(ts_on.edm_loss, l_off) and ts_off.edm_loss is l_off
    assert torch.equal(l_on, l_off)                 # u = 0: the objective is the reference loss
    g = on.logvar_linear.weight.grad.double().cpu().reshape(-1)
    with torch.no_grad():
        on.logvar_linear.weight.copy_(w0)           # the float64 check is of the step's w (= 0)
    want = _w_grad64(on, cap.calls)
    assert ((g - want).abs().max() / want.abs().max()).item() <= 1e-5


def _grads(net):
    return {k: p.grad.detach().double().clone() for k, p in net.named_parameters()
            if p.requires_grad and k.startswith("model.")}


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize("dec,mask", CASES, ids=IDS)
def test_weighted_gradient_is_a_combination_of_unweighted_runs(det, monkeypatch, dec, mask):
    B = 4
    x, lab = _data(B, 1)
    on = _net(C_LV, dec, w_scale=0.3)
    cap = _CaptureE(monkeypatch)

    def run(net, mae):
        lf = FixedLoss(B, seed=2)
        net.zero_grad(set_to_none=True)
        loss = lf(net, x, lab, mask_ratio=mask, mae_loss_coef=mae)
        sigma = _sigma(lf, 0, B)
        return loss, sigma, lf

    obj, sigma, lf = run(on, 0.1)
    obj.mean().backward()
    g_on = _grads(on)
    g_w = on.logvar_linear.weight.grad.double().cpu().reshape(-1)
    u = on.logvar(sigma)
    assert not lf.last_edm_loss.requires_grad
    off = _net(0, dec)
    parts = []
    for mae, gl in ((0.0, torch.exp(-u) / B), (0.1, torch.full((B,), 1.0 / B, device="cuda")),
                    (0.0, torch.full((B,), 1.0 / B, device="cuda"))):
        loss, _, _ = run(off, mae)
        (loss * gl).sum().backward()
        parts.append(_grads(off))
    worst = 0.0
    for k, g in g_on.items():
        want = parts[0][k] + parts[1][k] - parts[2][k]
        # The MAE part is the difference of two runs, each with its own bf16 rounding of the seed: the bound is
        # GRAD_TOL of tests/test_model_gpu.py (rel-L2 1.5e-2) relative to the parts' norms, not to their sum.
        scale = sum(parts[i][k].norm() for i in range(3))
        if scale == 0:
            assert g.norm() == 0, k
            continue
        r = ((g - want).norm() / scale).item()
        worst = max(worst, r)
        assert r <= 1.5e-2, (k, r)
    print(f"worst rel-L2 {worst:.2e}")
    want_w = _w_grad64(on, cap.calls[:1])
    assert ((g_w - want_w).abs().max() / want_w.abs().max()).item() <= 1e-5
    # the unweighted reference loss is the plain kernel's
    loss_mae, _, _ = run(off, 0.1)
    assert torch.equal(lf.last_edm_loss, loss_mae.detach())


# ---- 3. the training step -----------------------------------------------------------------------------------------------
def _ts(net, **kw):
    from maskdit_b200.train_step import TrainStep
    return TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, **kw)


def test_step_trains_w_and_the_averages_carry_it(det):
    net = _net(C_LV)
    ts = _ts(net, phema_sigma_rels=(0.1,), loss_fn=FixedLoss(4))
    x, lab = _data(4)
    for _ in range(3):
        ts.step(x, lab, 0.5, 0.1)
    w = net.logvar_linear.weight.detach()
    assert w.abs().max().item() > 0
    o, n, _ = ts.st.offsets["logvar_linear.weight"]
    ema_w = ts.ema.logvar_linear.weight.detach()
    assert ema_w.abs().max().item() > 0 and not torch.equal(ema_w, w)
    assert torch.equal(ts.ema_st.w32[o:o + n], ema_w.reshape(-1))
    prof = ts.phema_state_dicts()[0]
    assert torch.equal(prof["logvar_linear.weight"].reshape(-1), ts.phema_emas[0][o:o + n].cpu())
    assert prof["logvar_linear.weight"].abs().max().item() > 0
    assert torch.equal(prof["logvar_fourier.freqs"], net.logvar_fourier.freqs.detach().cpu())
    # the objective moves away from the reference loss once w is non-zero
    lo = ts.step(x, lab, 0.5, 0.1)
    assert not torch.equal(lo, ts.edm_loss)


def _state(ts):
    st = ts.st
    return [st.w32.clone(), st.w16.clone(), ts.m.clone(), ts.v.clone(), ts.ema_st.w32.clone()]


def _same(a, b):
    for i, (p, q) in enumerate(zip(a, b)):
        assert torch.equal(p, q), i


def test_resume_equals_uninterrupted(det):
    x, lab = _data(4, 5)
    torch.manual_seed(7)
    net = _net(C_LV)
    ts = _ts(net)
    la = [ts.step(x, lab, 0.5, 0.1).clone() for _ in range(4)]
    a = _state(ts)
    torch.manual_seed(7)
    net = _net(C_LV)
    ts = _ts(net)
    lb = [ts.step(x, lab, 0.5, 0.1).clone() for _ in range(2)]
    buf = io.BytesIO()
    torch.save({"model": net.state_dict(), "ema": ts.ema.state_dict(), "opt": ts.state_dict(),
                "rng": torch.cuda.get_rng_state()}, buf)
    del net, ts
    buf.seek(0)
    ck = torch.load(buf, weights_only=False)
    assert "logvar_linear.weight" in ck["model"] and "logvar_fourier.freqs" in ck["ema"]
    net = _net(C_LV)
    net.load_state_dict(ck["model"])
    ema = copy.deepcopy(net).eval()
    ema.load_state_dict(ck["ema"])
    from maskdit_b200.train_step import TrainStep
    ts2 = TrainStep(net, ema, lr=1e-3)
    ts2.load_state_dict(ck["opt"])
    torch.cuda.set_rng_state(ck["rng"])
    lb += [ts2.step(x, lab, 0.5, 0.1).clone() for _ in range(2)]
    _same(la, lb)
    _same(a, _state(ts2))


def test_grad_norm_covers_w(det):
    net = _net(C_LV, w_scale=0.3)
    ts = _ts(net, max_grad_norm=float("inf"), loss_fn=FixedLoss(4))
    x, lab = _data(4)
    ts.step(x, lab, 0.5, 0.1)
    gw = net.logvar_linear.weight.grad
    assert gw.abs().max().item() > 0
    g = torch.cat([p.grad.reshape(-1) for p in net.parameters() if p.requires_grad]).double()
    want = g.norm().item()
    assert abs(ts.grad_norm.item() - want) <= 2e-7 * want


def test_skipped_step_leaves_w(det):
    net = _net(C_LV, w_scale=0.3)
    ts = _ts(net, skip_nonfinite=True)
    x, lab = _data(4)
    ts.step(x, lab, 0.5, 0.1)
    w = net.logvar_linear.weight.detach().clone()
    m = ts.m.clone()
    bad = x.clone()
    bad[0, 0, 0, 0] = float("nan")
    ts.step(bad, lab, 0.5, 0.1)
    assert ts.skipped_steps.item() == 1
    assert torch.equal(net.logvar_linear.weight.detach(), w) and torch.equal(ts.m, m)


def test_grad_accum_matches_the_whole_batch(det):
    B = 8
    x, lab = _data(B, 2)
    grads, state = [], []
    for ga in (1, 2):
        net = _net(C_LV, w_scale=0.3)
        ts = _ts(net, loss_fn=FixedLoss(B, seed=4))
        lo = ts.step(x, lab, 0.5, 0.1, grad_accum=ga)
        g = ts.st.grad.double() * (0.5 if ga == 2 else 1.0)   # the buffer holds the sum of the rounds' mean gradients
        grads.append(g)
        state.append((lo, ts.edm_loss))
    (lo1, e1), (lo2, e2) = state
    assert torch.equal(e1, e2) and e2.shape == (B,)
    assert torch.equal(lo1, lo2)
    o, n, _ = ts.st.offsets["logvar_linear.weight"]
    gw1, gw2 = grads[0][o:o + n], grads[1][o:o + n]
    assert ((gw1 - gw2).abs().max() / gw1.abs().max()).item() <= 1e-5
    for k, (ok, nk, _) in ts.st.offsets.items():
        if k.startswith("model.") and ok + nk <= ts.st.n_train and grads[0][ok:ok + nk].norm() > 0:
            assert _rel(grads[1][ok:ok + nk], grads[0][ok:ok + nk]) <= 1e-2, k


def test_cuda_graph_matches_eager(det):
    x, lab = _data(4, 3)
    out = []
    for graph in (False, True):
        net = _net(C_LV, w_scale=0.3)
        ts = _ts(net, graph=graph, loss_fn=FixedLoss(4, seed=6))
        losses = []
        for _ in range(3):
            losses += [ts.step(x, lab, 0.5, 0.1).clone(), ts.edm_loss.clone()]
        out.append(losses + _state(ts) + [ts.st.grad.clone()])
    _same(out[0], out[1])
    assert not torch.equal(out[0][0], out[0][1])   # objective and reference loss are different tensors


# ---- 4. generate.py ---------------------------------------------------------------------------------------------------
YAML = """
model:
  precond: edm
  model_type: DiT-S/2
  in_size: 16
  in_channels: 4
  num_classes: 10
  use_decoder: True
  ext_feature_dim: 0
  pad_cls_token: False
  mae_loss_coef: 0.1
"""


def test_generate_ignores_logvar_keys(tmp_path):
    from maskdit_b200.maskdit import EDMPrecond
    from oracle import maskdit_oracle as O
    sd = O.make_state_dict(O.Cfg(model_type="DiT-S/2", img_resolution=16, num_classes=10, use_decoder=True), 2)
    net = EDMPrecond(16, 4, num_classes=10, model_type="DiT-S/2", use_decoder=True, mae_loss_coef=0.1,
                     logvar_channels=64)
    net.load_state_dict(sd, strict=False)
    with torch.no_grad():
        net.logvar_linear.weight.normal_()
    full = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    assert any(k.startswith("logvar_") for k in full)
    plain = {k: v for k, v in full.items() if not k.startswith("logvar_")}
    (tmp_path / "c.yaml").write_text(YAML)
    env = dict(os.environ, PYTHONPATH=ROOT)
    outs = []
    for name, ema in (("full", full), ("plain", plain)):
        torch.save({"ema": ema}, tmp_path / f"{name}.pt")
        r = subprocess.run([sys.executable, os.path.join(ROOT, "generate.py"), "--config", str(tmp_path / "c.yaml"),
                            "--ckpt_path", str(tmp_path / f"{name}.pt"), "--seeds", "0-2", "--num_steps", "4",
                            "--results_dir", str(tmp_path / name)], env=env, capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        outs.append([np.load(tmp_path / name / f"{s:06d}.npy") for s in range(3)])
    for a, b in zip(*outs):
        assert np.array_equal(a, b)
