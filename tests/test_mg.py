"""Model guidance (DESIGN §5): host logic without a GPU.  The w = 1 - 1/s map, the config block and every refusal, the
loss's refusals, the log-line field, and that the loss draws exactly what EDMLoss / FlowLoss draw."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from maskdit_b200 import ops  # noqa: E402
from maskdit_b200.config import build_loss, load_config  # noqa: E402
from maskdit_b200.loss import EDMLoss, FlowLoss, Losses, MGLoss, mg_weight  # noqa: E402
from maskdit_b200.maskdit import EDMPrecond, FlowPrecond  # noqa: E402


def _small(cls, **kw):
    kw.setdefault("num_classes", 10)
    return cls(8, 4, model_type="DiT-S/2", use_decoder=True, mae_loss_coef=0.1, **kw)


def test_weight_map():
    assert Losses["mg"] is MGLoss
    assert mg_weight(1) == 0.0 and mg_weight(2) == 0.5 and mg_weight(4.0) == 0.75
    # the fixed point D_c = E_u + (E_c - E_u) / (1 - w) is CFG at s
    for s in (1.0, 1.5, 3.0, 7.5):
        assert math.isclose(1.0 / (1.0 - mg_weight(s)), s, rel_tol=1e-15)
    for bad in (0.99, 0.0, -2.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="scale"):
            mg_weight(bad)
    f = MGLoss(scale=1.5)
    assert (f.w, f.lo, f.hi, f.P_mean, f.P_std, f.sigma_data) == (1 - 1 / 1.5, 0.0, math.inf, None, None, 0.5)
    f = MGLoss(scale=3, interval=(0.3, 5))
    assert (f.lo, f.hi) == (0.3, 5.0)
    for iv in ((1.0, 1.0), (2.0, 1.0), (float("nan"), 1.0)):
        with pytest.raises(ValueError, match="interval"):
            MGLoss(scale=2, interval=iv)


class _Stop(Exception):
    pass


def _record(monkeypatch, front_name):
    seen = {}

    def front(moments, eps, rnd, noise, labels, drop_u, p, sf, P_mean, P_std):
        seen.update(eps=eps, rnd=rnd, noise=noise, drop_u=drop_u, P=(P_mean, P_std))
        raise _Stop

    monkeypatch.setattr(ops, front_name, front)
    return seen


class _Draws:
    def __init__(self, calls):
        self.calls = calls

    def randn(self, shape, device):
        self.calls.append(("randn", tuple(shape)))
        return torch.full(tuple(shape), float(len(self.calls)))

    def rand(self, shape, device):
        self.calls.append(("rand", tuple(shape)))
        return torch.full(tuple(shape), 0.5)


@pytest.mark.parametrize("cls, base, front", [(EDMPrecond, EDMLoss, "step_front"),
                                               (FlowPrecond, FlowLoss, "flow_step_front")])
def test_draws_are_the_plain_losses(monkeypatch, cls, base, front):
    """from_moments and __call__ make the draws of EDMLoss / FlowLoss for the network given, in the same order and
    shapes, with the same P_mean / P_std reaching the step front: MG draws nothing more."""
    monkeypatch.setattr(cls, "_ready", lambda self, dev: None)
    seen = _record(monkeypatch, front)
    net = _small(cls)
    B, C, R = 3, 4, 8
    runs = {}
    for name, loss in (("mg", MGLoss(scale=2.0)), ("plain", base())):
        calls = []
        d = _Draws(calls)
        loss._randn, loss._rand = d.randn, d.rand
        with pytest.raises(_Stop):
            loss.from_moments(net, torch.zeros(B, 2 * C, R, R), torch.zeros(B, 10), class_dropout_prob=0.1)
        runs[name] = (calls, seen["P"], float(seen["rnd"][0]), float(seen["noise"].flatten()[0]))
    assert runs["mg"] == runs["plain"]
    assert runs["mg"][0] == [("randn", (B, C, R, R)), ("rand", (B, 1)), ("randn", (B, 1, 1, 1)),
                             ("randn", (B, C, R, R))]
    # P_mean / P_std given to MGLoss reach the front
    f = MGLoss(scale=2.0, P_mean=0.25, P_std=0.75)
    d = _Draws([])
    f._randn, f._rand = d.randn, d.rand
    with pytest.raises(_Stop):
        f.from_moments(net, torch.zeros(B, 2 * C, R, R), torch.zeros(B, 10))
    assert seen["P"] == (0.25, 0.75)


@pytest.mark.parametrize("cls, base", [(EDMPrecond, EDMLoss), (FlowPrecond, FlowLoss)])
def test_call_draws_are_the_plain_losses(monkeypatch, cls, base):
    """`__call__` draws what EDMLoss / FlowLoss draw, then the mask noise, before any device work."""
    monkeypatch.setattr(cls, "_ready", lambda self, dev: None)

    def stop(*a, **k):
        raise _Stop

    monkeypatch.setattr(ops, "mask_indices", stop)
    net = _small(cls).train()
    B, C, R = 2, 4, 8
    runs = {}
    for name, loss in (("mg", MGLoss(scale=2.0)), ("plain", base())):
        calls = []
        d = _Draws(calls)
        loss._randn, loss._rand = d.randn, d.rand
        with pytest.raises(_Stop):
            loss(net, torch.zeros(B, C, R, R), torch.eye(10)[:B], mask_ratio=0.5, mae_loss_coef=0.1)
        runs[name] = calls
    assert runs["mg"] == runs["plain"]
    assert runs["mg"] == [("randn", (B, 1, 1, 1)), ("randn", (B, C, R, R)), ("rand", (B, 16))]


def test_loss_refusals(monkeypatch):
    monkeypatch.setattr(EDMPrecond, "_ready", lambda self, dev: None)
    x = torch.zeros(2, 4, 8, 8)
    with pytest.raises(ValueError, match="class-conditional"):
        MGLoss(scale=2.0)(_small(EDMPrecond, num_classes=0), x)
    with pytest.raises(ValueError, match="learned loss weighting"):
        MGLoss(scale=2.0)(_small(EDMPrecond, logvar_channels=8), x, torch.eye(10)[:2])


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
  class_dropout_prob: 0.1
train:
  lr: 0.0001
"""


def test_config_block():
    cfg = load_config(YAML)
    cfg.train.update(objective="mg", mg={"scale": 1.5})
    f = build_loss(cfg)
    assert type(f) is MGLoss and f.w == 1 - 1 / 1.5 and (f.lo, f.hi) == (0.0, math.inf)
    cfg.train["mg"] = {"scale": 4, "interval": [0.3, 5.0]}
    f = build_loss(cfg)
    assert f.scale == 4.0 and (f.lo, f.hi) == (0.3, 5.0)
    cfg.model["precond"] = "flow"
    cfg.train["mg"] = {"scale": 2, "interval": [0.1, 0.9]}
    f = build_loss(cfg)
    assert type(f) is MGLoss and (f.lo, f.hi) == (0.1, 0.9)


@pytest.mark.parametrize("edit, what", [
    (lambda c: c.train.update(objective="mg"), "train.mg.scale"),
    (lambda c: c.train.update(objective="mg", mg={"interval": [0.1, 1]}), "train.mg.scale"),
    (lambda c: c.train.update(objective="mg", mg={"scale": 0.5}), "scale"),
    (lambda c: c.train.update(objective="mg", mg={"scale": 2, "w": 0.5}), "unknown train.mg keys"),
    (lambda c: c.train.update(objective="mg", mg={"scale": 2, "interval": [2, 1]}), "interval"),
    (lambda c: c.train.update(objective="mg", mg={"scale": 2, "interval": [1]}), "interval"),
    (lambda c: c.train.update(objective="mg", mg={"scale": 2, "interval": 3}), "interval"),
    (lambda c: c.train.update(mg={"scale": 2}), "train.objective: mg"),
    (lambda c: c.train.update(objective="ect", ect={"stage_steps": 10}, mg={"scale": 2}), "train.objective: mg"),
    (lambda c: (c.train.update(objective="mg", mg={"scale": 2}), c.model.update(num_classes=0)),
     "class-conditional"),
    (lambda c: (c.train.update(objective="mg", mg={"scale": 2}), c.model.update(class_dropout_prob=0)),
     "class_dropout_prob"),
    (lambda c: (c.train.update(objective="mg", mg={"scale": 2}), c.model.pop("class_dropout_prob")),
     "class_dropout_prob"),
    (lambda c: (c.train.update(objective="mg", mg={"scale": 2}), c.model.update(logvar_channels=16)),
     "logvar_channels"),
])
def test_config_refusals(edit, what):
    cfg = load_config(YAML)
    edit(cfg)
    with pytest.raises(ValueError, match=what):
        build_loss(cfg)


def test_log_line_field():
    import train
    assert train.log_line(40, 0.5, 2.0, mg=0.61234) == \
        "(step=0000040) Train Loss: 0.5000, Train Steps/Sec: 2.00, MG Loss: 0.6123"
    assert "MG" not in train.log_line(40, 0.5, 2.0)


def test_entry_points_exported_abi_unchanged():
    from maskdit_b200 import _lib
    syms = _lib.exported_symbols()
    assert "mdt_mg_loss" in syms and "mdt_flow_mg_loss" in syms
    assert _lib.lib().mdt_abi_version() == 2
