"""GPU: multistep DPM-Solver++ (DESIGN §5) on the H100 kernels.  `mdt_dpm_update` against op-by-op torch float64, the
sampler driven by the closed-form Gaussian denoiser against the float64 oracle (oracle/dpm_solver_oracle.py), the
goldens of the unmodified reference network inside that oracle (tests/golden/make_golden_dpm.py), a toy network whose
distance to a fine Heun solution falls with the evaluation count, and generate.py --dpm_order end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from support import det, load, ops, oracle_net, rel_l2  # noqa: F401

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMPLER_TOL = 1e-2
MU, S = 0.3, 0.5


def ulp64(x):
    a = x.abs()
    return torch.nextafter(a, torch.full_like(a, float("inf"))) - a


# ---- the kernel against float64 ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("velocity", [False, True])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_dpm_update_vs_float64(ops, velocity, k):
    g = torch.Generator(device="cuda").manual_seed(10 * k + velocity)
    n = 70001                                                       # not a multiple of the block
    x = torch.randn(n, dtype=torch.float64, device="cuda", generator=g) * 3
    F = torch.randn(n, dtype=torch.float32, device="cuda", generator=g)
    h1 = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    h2 = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    a, b0, b1, b2, t = 0.8173, 0.1931, -0.4512, 0.0377, 0.6180339887
    x0 = x.clone()
    d = torch.full_like(x, float("nan"))
    xf = torch.empty(n, dtype=torch.float32, device="cuda")
    ops.dpm_update(F, x, d, a, b0, h1 if k >= 2 else None, b1, h2 if k >= 3 else None, b2, velocity=velocity, t=t,
                   out_f32=xf)
    Fd = F.double()
    D = x0 - Fd * t if velocity else Fd                              # op by op: each torch op rounds on its own
    v = x0 * a
    v = v + D * b0
    if k >= 2:
        v = v + h1 * b1
    if k >= 3:
        v = v + h2 * b2
    assert torch.equal(d, D)
    assert ((x - v).abs() <= 2 * ulp64(v)).all(), (x - v).abs().max().item()
    assert torch.equal(xf, x.float())                                # the fp64 result rounded
    # without the fp32 output the state is the same
    x2 = x0.clone()
    ops.dpm_update(F, x2, d, a, b0, h1 if k >= 2 else None, b1, h2 if k >= 3 else None, b2, velocity=velocity, t=t)
    assert torch.equal(x2, x)


def test_dpm_update_refusals(ops):
    from maskdit_b200._lib import MdtError
    x = torch.zeros(8, dtype=torch.float64, device="cuda")
    F = torch.zeros(8, device="cuda")
    with pytest.raises(MdtError):
        ops.dpm_update(F, x, torch.empty_like(x), float("nan"), 1.0)
    with pytest.raises(MdtError):
        ops.dpm_update(F, x, torch.empty(4, dtype=torch.float64, device="cuda"), 1.0, 1.0)
    with pytest.raises(MdtError):
        ops.dpm_update(F, x, torch.empty_like(x), 1.0, 1.0, h2=torch.zeros_like(x), b2=1.0)


# ---- the sampler against the float64 oracle on Gaussian data -------------------------------------------------------------
class GaussEDM:
    """An EDM 'network' whose D is the closed-form denoiser of N(MU, S^2) data at its fp32 input, returned in fp32."""
    sigma_min, sigma_max = 0.0, float("inf")

    def __init__(self):
        self.calls = []

    def __call__(self, x, sigma, labels=None, cfg_scale=None, feat=None):
        from oracle import dpm_solver_oracle as O
        s = float(sigma)
        self.calls.append(s)
        return {"x": O.gauss_edm_D(x.double(), s, MU, S).float()}


def f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def latents(n=64):
    z = torch.randn(n, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    z[:3] = torch.tensor([1.3, -0.7, 0.2])
    return z


@pytest.mark.parametrize("order", [1, 2, 3])
def test_sampler_matches_oracle_on_gaussian_edm(ops, order):
    from maskdit_b200.sampler import dpm_solver_sampler
    from oracle import dpm_solver_oracle as O
    z = latents()
    net = GaussEDM()
    got = dpm_solver_sampler(net, z.float().cuda(), num_steps=10, order=order)
    assert got.dtype == torch.float64
    lv = O.karras_levels(10)
    assert net.calls == lv[:-1].tolist()                              # one evaluation per positive level
    alpha, sigma = O.edm_alpha_sigma(lv)
    want = O.dpm_solver(lambda x, i: f32(O.gauss_edm_D(f32(x), sigma[i], MU, S)), sigma[0] * f32(z.numpy()), alpha,
                        sigma, order)
    err = np.abs(got.cpu().numpy() - want).max()
    print("EDM order", order, "max |sampler - oracle|", err)
    assert err <= 1e-12


@pytest.mark.parametrize("order", [1, 2, 3])
def test_sampler_matches_oracle_on_gaussian_flow(ops, order):
    from maskdit_b200.sampler import _dpm_solve, flow_grid
    from oracle import dpm_solver_oracle as O
    z = latents()
    lv = flow_grid(10)
    alpha, sigma = O.flow_alpha_sigma(lv)

    def velocity(x, t):                                                # v^ = (x - D) / t at the fp32 input, in fp32
        xd = x.double()
        return ((xd - O.gauss_flow_D(xd, t, MU, S)) / t).float()

    got = _dpm_solve(velocity, z.float().double().cuda(), lv, True, order)

    def D(x, i):                                                       # D = x - t v^ from the fp64 state
        v = f32((f32(x) - O.gauss_flow_D(f32(x), sigma[i], MU, S)) / sigma[i])
        return x - sigma[i] * v

    want = O.dpm_solver(D, f32(z.numpy()), alpha, sigma, order)
    err = np.abs(got.cpu().numpy() - want).max()
    print("flow order", order, "max |sampler - oracle|", err)
    assert err <= 1e-12


# ---- the reference network inside the oracle ----------------------------------------------------------------------------
def test_edm_golden(ops):
    from maskdit_b200.sampler import dpm_solver_sampler
    g = load("dpm_s2_sampler")
    net = oracle_net("DiT-S/2", 8, 10, True).eval()
    calls = []
    orig = type(net).forward

    def spy(self, x, sigma, labels=None, cfg_scale=None, **kw):
        calls.append((float(sigma), cfg_scale))
        return orig(self, x, sigma, labels, cfg_scale, **kw)

    type(net).forward = spy
    try:
        n0 = ops.L.LAUNCHES
        z = dpm_solver_sampler(net, g["latents"].cuda(), g["labels"].cuda(), cfg_scale=float(g["cfg_scale"]),
                               num_steps=int(g["num_steps"]), order=int(g["order"]))
        assert z.dtype == torch.float64 and ops.L.LAUNCHES > n0
        assert calls == [(s, 1.5) for s in g["levels"][:-1].tolist()], calls
        print("EDM golden rel-L2", rel_l2(z, g["z"]))
        assert rel_l2(z, g["z"]) <= SAMPLER_TOL
        # the interval gate: CFG only where lo < sigma <= hi
        calls.clear()
        dpm_solver_sampler(net, g["latents"].cuda(), g["labels"].cuda(), cfg_scale=1.5, num_steps=4,
                           guidance_interval=(0.1, 10.0))
        assert [c for _, c in calls] == [None, 1.5, 1.5, None], calls
    finally:
        type(net).forward = orig


def test_flow_golden(ops):
    from maskdit_b200.maskdit import FlowPrecond
    from maskdit_b200.sampler import dpm_solver_sampler
    from oracle import maskdit_oracle as O
    g = load("dpm_nd_s2_flow")
    net = FlowPrecond(img_resolution=8, img_channels=4, num_classes=0, model_type="DiT-S/2", use_decoder=False,
                      mae_loss_coef=0.1, pad_cls_token=False)
    net.load_state_dict(O.make_state_dict(O.Cfg(model_type="DiT-S/2", img_resolution=8, num_classes=0,
                                                use_decoder=False), 1), strict=True)
    net = net.cuda().eval()
    z = dpm_solver_sampler(net, g["latents"].cuda(), num_steps=int(g["num_steps"]), order=int(g["order"]))
    print("flow golden rel-L2", rel_l2(z, g["z"]))
    assert z.dtype == torch.float64 and rel_l2(z, g["z"]) <= SAMPLER_TOL


# ---- a toy network: the distance to a fine ODE solution falls with the evaluation count --------------------------------
def test_toy_distance_to_ode_solution_falls(det):
    """The toy of tools/dpm_solver_bench.py (DiT-S/2 at R = 8, 400 EDM steps on four classes of two latents each):
    the rms distance to edm_sampler at 256 steps falls over 6 / 12 / 24 evaluations for 2M and 3M."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from dpm_solver_bench import toy_errors, train_toy
    net, z, lab = train_toy()
    e = toy_errors(net, z, lab)
    for k in sorted(e):
        print(k, f"{e[k]:.3e}")
    for o in (2, 3):
        d = [e[(f"dpm_solver_order{o}", n)] for n in (6, 12, 24)]
        assert d[0] > d[1] > d[2], (o, d)


# ---- generate.py --------------------------------------------------------------------------------------------------------
YAML = """
data: {dataset: imagenet256-latent, category: lmdb, resolution: 16, num_channels: 4, root: none, feat_path: None}
model:
  precond: PRECOND
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


@pytest.mark.parametrize("precond", ["edm", "flow"])
def test_generate_dpm_order(tmp_path, precond):
    cfg = tmp_path / "cfg.yaml"
    cfg.write_text(YAML.replace("PRECOND", precond))
    run([os.path.join(ROOT, "train.py"), "--config", str(cfg), "--synthetic", "--max_steps", "4", "--results_dir",
         str(tmp_path / "res")], str(tmp_path))
    ck = tmp_path / "res" / "checkpoints" / "0000004.pt"
    out = run([os.path.join(ROOT, "generate.py"), "--config", str(cfg), "--ckpt_path", str(ck), "--seeds", "0-3",
               "--dpm_order", "3", "--num_steps", "6", "--cfg_scale", "1.5", "--results_dir", str(tmp_path / "s")],
              str(tmp_path))
    assert "wrote 4 latents" in out, out
    z = np.load(tmp_path / "s" / "000002.npy")
    assert z.shape == (4, 16, 16) and np.isfinite(z).all()
