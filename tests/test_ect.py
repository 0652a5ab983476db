"""Easy Consistency Tuning (DESIGN §5): host logic without a GPU.  The r(t, s) map and its clamp against the reference
goldens (tests/golden/ect_*.npz), the draw order, the stage counter, the config block and its refusals, the loss's
refusals and generate.py's --consistency_sigmas validation."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from maskdit_b200 import ops  # noqa: E402
from maskdit_b200.config import build_loss, load_config  # noqa: E402
from maskdit_b200.loss import ECTLoss, EDMLoss, FlowLoss, Losses, ect_r  # noqa: E402
from maskdit_b200.maskdit import EDMPrecond, FlowPrecond  # noqa: E402
from maskdit_b200.sampler import consistency_sampler, consistency_sigmas  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def _small(cls, **kw):
    return cls(8, 4, num_classes=10, model_type="DiT-S/2", use_decoder=True, mae_loss_coef=0.1, **kw)


def test_registry_and_defaults():
    assert Losses["ect"] is ECTLoss
    f = ECTLoss(stage_steps=100)
    assert (f.q, f.k, f.b, f.P_mean, f.P_std, f.sigma_data) == (2.0, 8.0, 1.0, -1.1, 2.0, 0.5)
    assert f.scale_of(0) == 0.5 and f.scale_of(3) == 2.0 ** -4


def test_r_map_and_clamp():
    t = torch.tensor([0.002, 0.05, 0.5, 1.0, 2.0, 5.0, 20.0, 80.0], dtype=torch.float64)
    f = ECTLoss(stage_steps=1)
    prev = None
    for s in range(8):
        r = ect_r(t, f.scale_of(s))
        assert bool((r >= 0).all()) and bool((r < t).all())
        if prev is not None:                     # a later stage never moves r away from t
            assert bool((r >= prev).all())
        prev = r
    # stage 0: 1 - (1 + 8 sigmoid(-t)) / 2 <= 0 for t <= ln 3 (sigmoid(-t) >= 1/8): clamped to the denoising limit
    r0 = ect_r(t, 0.5)
    assert bool((r0[t <= np.log(7.0)] == 0).all()) and bool((r0[t > np.log(7.0)] > 0).all())
    # the gap (t - r) / t tends to q^-(s+1) (1 + k sigmoid(-b t)), which is q^-(s+1) at large t
    s = 7
    gap = (t - ect_r(t, f.scale_of(s))) / t
    want = f.scale_of(s) * (1 + 8 / (1 + torch.exp(t)))
    torch.testing.assert_close(gap, want, rtol=1e-9, atol=0)


def test_r_matches_golden():
    for name in ("ect_s2_train_mask", "ect_nd_s2_uncond", "ect_xl2_mask"):
        g = _gold(name)
        t = torch.from_numpy(g["rnd_normal"]) * 2.0 - 1.1
        np.testing.assert_array_equal(t.exp().numpy(), g["t"])
        r = ect_r(torch.from_numpy(g["t"]), ECTLoss(stage_steps=1).scale_of(int(g["stage"])))
        np.testing.assert_array_equal(r.numpy(), g["r"])
    g = _gold("ect_s2_train_mask")
    assert (g["r"] == 0).any() and (g["r"] > 0).any()      # both branches of the target


class _Stop(Exception):
    pass


def test_from_moments_draw_order(monkeypatch):
    """Draws in EDMLoss.from_moments' order: eps, drop_u (with dropout), the t normal [B,1,1,1], the noise; the stage
    word, k, b and P_mean / P_std reach the step front as set."""
    calls = []

    class L(ECTLoss):
        def _randn(self, shape, device):
            calls.append(("randn", tuple(shape)))
            return torch.full(tuple(shape), float(len(calls)))

        def _rand(self, shape, device):
            calls.append(("rand", tuple(shape)))
            return torch.full(tuple(shape), 0.5)

        def _net(self, net, dev):
            return None

    seen = {}

    def front(moments, eps, rnd, noise, qs, labels, drop_u, p, sf, P_mean, P_std, k, b):
        seen.update(eps=eps, rnd=rnd, noise=noise, qs=qs, drop_u=drop_u, P=(P_mean, P_std), kb=(k, b))
        raise _Stop

    monkeypatch.setattr(ops, "ect_step_front", front)
    B, C, R = 3, 4, 8
    loss = L(stage_steps=10, q=4.0, k=6.0, b=0.5, P_mean=0.25, P_std=0.75)
    loss.stage = 2
    with pytest.raises(_Stop):
        loss.from_moments(None, torch.zeros(B, 2 * C, R, R), torch.zeros(B, 10), class_dropout_prob=0.1)
    assert calls == [("randn", (B, C, R, R)), ("rand", (B, 1)), ("randn", (B, 1, 1, 1)), ("randn", (B, C, R, R))]
    assert seen["rnd"].shape == (B,) and float(seen["rnd"][0]) == 3.0
    assert float(seen["eps"].flatten()[0]) == 1.0 and float(seen["noise"].flatten()[0]) == 4.0
    assert seen["P"] == (0.25, 0.75) and seen["kb"] == (6.0, 0.5)
    assert seen["qs"].dtype == torch.float32 and float(seen["qs"]) == 4.0 ** -3
    word = torch.tensor([0.125])                  # a TrainStep's device word wins over `stage`
    loss.stage_scale = word
    with pytest.raises(_Stop):
        loss.from_moments(None, torch.zeros(B, 2 * C, R, R))
    assert seen["qs"] is word


def test_stage_counter():
    f = ECTLoss(stage_steps=5)
    assert [f.stage_at(s, 100) for s in (100, 104, 105, 109, 110, 131)] == [0, 0, 1, 1, 2, 6]
    # a run resumed at step 107 with the stored origin 100 continues stage 1; a fresh origin would restart at 0
    assert f.stage_at(107, 100) == 1 and f.stage_at(107, 107) == 0


def test_loss_refusals():
    with pytest.raises(ValueError, match="stage_steps"):
        ECTLoss(stage_steps=0)
    with pytest.raises(ValueError, match="stage_steps"):
        ECTLoss(stage_steps=2.5)
    with pytest.raises(ValueError, match="q > 1"):
        ECTLoss(stage_steps=1, q=1.0)
    with pytest.raises(TypeError, match="FlowPrecond"):
        ECTLoss(stage_steps=1)._net(_small(FlowPrecond), torch.device("cpu"))
    with pytest.raises(ValueError, match="learned loss weighting"):
        ECTLoss(stage_steps=1)._net(_small(EDMPrecond, logvar_channels=8), torch.device("cpu"))


YAML = """
model:
  precond: edm
  model_type: DiT-S/2
  in_size: 8
  in_channels: 4
  num_classes: 10
  use_decoder: true
  mae_loss_coef: 0.1
  pad_cls_token: false
train:
  lr: 0.0001
"""


def test_config_block():
    cfg = load_config(YAML)
    assert type(build_loss(cfg)) is EDMLoss                    # no objective: the precond's own
    cfg.train["objective"] = "edm"
    assert type(build_loss(cfg)) is EDMLoss
    cfg.train["objective"] = "ect"
    cfg.train["ect"] = {"stage_steps": 250, "q": 4, "P_std": 1.5}
    f = build_loss(cfg)
    assert type(f) is ECTLoss and (f.stage_steps, f.q, f.k, f.b, f.P_mean, f.P_std) == (250, 4.0, 8.0, 1.0, -1.1, 1.5)
    cfg.model["precond"] = "flow"
    cfg.train.pop("objective"), cfg.train.pop("ect")
    assert type(build_loss(cfg)) is FlowLoss


@pytest.mark.parametrize("edit, what", [
    (lambda c: c.train.update(objective="ect"), "stage_steps"),
    (lambda c: c.train.update(objective="ect", ect={"q": 2}), "stage_steps"),
    (lambda c: c.train.update(objective="ect", ect={"stage_steps": 0}), "stage_steps"),
    (lambda c: c.train.update(objective="ect", ect={"stage_steps": 10, "rho": 7}), "unknown train.ect keys"),
    (lambda c: c.train.update(ect={"stage_steps": 10}), "train.objective: ect"),
    (lambda c: c.train.update(objective="sCM"), "unknown train.objective"),
    (lambda c: (c.train.update(objective="ect", ect={"stage_steps": 10}), c.model.update(precond="flow")),
     "not model.precond: flow"),
    (lambda c: (c.train.update(objective="ect", ect={"stage_steps": 10}), c.model.update(logvar_channels=16)),
     "logvar_channels"),
])
def test_config_refusals(edit, what):
    cfg = load_config(YAML)
    edit(cfg)
    with pytest.raises(ValueError, match=what):
        build_loss(cfg)


def test_consistency_sigmas():
    assert consistency_sigmas([80]) == [80.0]
    assert consistency_sigmas([200, 0.8], sigma_max=80) == [80.0, 0.8]        # clamped as edm_sampler clamps
    for bad in ([], [0.8, 80], [80, 80], [80, 0], [80, -1], [float("nan")], [200, 100]):
        with pytest.raises(ValueError):
            consistency_sigmas(bad, sigma_max=80)
    with pytest.raises(ValueError):
        consistency_sampler(_small(EDMPrecond), torch.zeros(1, 4, 8, 8), sigmas=(0.5, 1.0))


@pytest.mark.parametrize("argv, what", [
    (["--consistency_sigmas", "80", "--S_churn", "10"], "--S_churn"),
    (["--consistency_sigmas", "80", "--solver", "euler"], "--solver"),
    (["--consistency_sigmas", "80", "--discretization", "vp"], "--discretization"),
    (["--consistency_sigmas", "0.8", "80"], "strictly decreasing"),
    (["--consistency_sigmas", "80", "0"], "positive"),
])
def test_generate_switch_validation(argv, what, capsys):
    import generate
    with pytest.raises(SystemExit):
        generate.parse_args(["--config", "x.yaml", *argv])
    assert what in capsys.readouterr().err
    a = generate.parse_args(["--config", "x.yaml", "--consistency_sigmas", "80", "0.8", "--cfg_scale", "1.5"])
    assert a.consistency_sigmas == [80.0, 0.8]


def test_generate_refuses_flow_config(tmp_path):
    import generate
    cfg = tmp_path / "c.yaml"
    cfg.write_text(YAML.replace("precond: edm", "precond: flow"))
    with pytest.raises(SystemExit, match="flow config"):
        generate.main(["--config", str(cfg), "--consistency_sigmas", "80"])


def test_log_line_stage():
    import train
    assert train.log_line(40, 0.5, 2.0, ect_stage=3) == \
        "(step=0000040) Train Loss: 0.5000, Train Steps/Sec: 2.00, ECT stage: 3"
    assert "ECT" not in train.log_line(40, 0.5, 2.0)
