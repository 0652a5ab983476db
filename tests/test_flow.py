"""Rectified-flow training and sampling (DESIGN §5): host logic without a GPU.  The t grid, the logit-normal t and
the draw order against the reference goldens (tests/golden/flow_*.npz), the registries and refusals, the validation
levels, and that the EDM instantiations of the kernels that gained a flow variant compile to the same SASS."""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from maskdit_b200 import _lib, ops, validate  # noqa: E402
from maskdit_b200.config import build_net, load_config  # noqa: E402
from maskdit_b200.loss import EDMLoss, FlowLoss, Losses  # noqa: E402
from maskdit_b200.maskdit import EDMPrecond, FlowPrecond, Precond_models  # noqa: E402
from maskdit_b200.sampler import flow_grid, flow_sampler  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def _small(cls, **kw):
    return cls(8, 4, num_classes=10, model_type="DiT-S/2", use_decoder=True, mae_loss_coef=0.1, **kw)


def test_registries():
    assert Precond_models["flow"] is FlowPrecond and Precond_models["edm"] is EDMPrecond
    assert Losses["flow"] is FlowLoss and Losses["edm"] is EDMLoss
    f = FlowLoss()
    assert (f.P_mean, f.P_std) == (0.0, 1.0)


def test_flow_net_shares_the_edm_layout():
    edm, flow = _small(EDMPrecond), _small(FlowPrecond)
    assert list(edm.state_dict()) == list(flow.state_dict())
    assert flow._layout()[0].tensors() == edm._layout()[0].tensors()
    assert flow._cfg().precond == 1 and edm._cfg().precond == 0
    flow.load_state_dict(edm.state_dict())       # checkpoints load across objectives (same keys)
    assert type(flow.__deepcopy__({})) is FlowPrecond


def test_yaml_precond_selects_flow():
    cfg = load_config("""
model:
  precond: flow
  model_type: DiT-S/2
  in_size: 8
  in_channels: 4
  num_classes: 10
  use_decoder: true
  mae_loss_coef: 0.1
  pad_cls_token: false
""")
    net = build_net(cfg)
    assert type(net) is FlowPrecond
    assert isinstance(Losses[cfg.model.precond](), FlowLoss)
    cfg.model["logvar_channels"] = 16
    with pytest.raises(ValueError, match="learned loss weighting"):
        build_net(cfg)


def test_each_loss_refuses_the_other_network():
    with pytest.raises(TypeError, match="Losses\\['flow'\\]"):
        EDMLoss()._net(_small(FlowPrecond), torch.device("cpu"))
    with pytest.raises(TypeError, match="Losses\\['edm'\\]"):
        FlowLoss()._net(_small(EDMPrecond), torch.device("cpu"))


def test_flow_net_refusals():
    net = _small(FlowPrecond)
    with pytest.raises(ValueError, match="autoguidance"):
        net.check_guide(_small(FlowPrecond))
    with pytest.raises(ValueError, match="learned loss weighting"):
        _small(FlowPrecond, logvar_channels=8)
    with pytest.raises(ValueError, match="solver"):
        flow_sampler(net, torch.zeros(1, 4, 8, 8), solver="dpm")


def test_t_grid_matches_golden_sampler():
    g = _gold("flow_s2_sampler")
    N = int(g["num_steps"])
    grid = flow_grid(N)
    assert grid[0] == 1.0 and grid[-1] == 0.0 and len(grid) == N + 1
    np.testing.assert_allclose(np.diff(grid), -1.0 / N, rtol=0, atol=1e-15)
    # Heun with an Euler last step: the evaluation times are t_0, then (t_{k+1}, t_{k+1}) pairs, 2N - 1 in all
    seen = [grid[0]] + [v for k in range(1, N) for v in (grid[k], grid[k])]
    np.testing.assert_array_equal(np.array(seen), g["sampler_t"])
    with pytest.raises(ValueError):
        flow_grid(0)


def test_logit_normal_t_matches_golden():
    for name in ("flow_s2_train_mask", "flow_nd_s2_uncond", "flow_xl2_mask"):
        g = _gold(name)
        rnd = torch.from_numpy(g["rnd_normal"])
        t = 1.0 / (1.0 + torch.exp(-(rnd * 1.0 + 0.0)))
        np.testing.assert_array_equal(t.numpy(), g["t"])


class _Stop(Exception):
    pass


def test_from_moments_draw_order(monkeypatch):
    """Draws in EDMLoss.from_moments' order: eps, drop_u (with dropout), the t normal [B,1,1,1], the noise; the t
    normal reaches the step front as rnd_normal and P_mean / P_std as set."""
    calls = []

    class L(FlowLoss):
        def _randn(self, shape, device):
            calls.append(("randn", tuple(shape)))
            return torch.full(tuple(shape), float(len(calls)))

        def _rand(self, shape, device):
            calls.append(("rand", tuple(shape)))
            return torch.full(tuple(shape), 0.5)

        def _net(self, net, dev):
            return None

    seen = {}

    def front(moments, eps, rnd, noise, labels, drop_u, p, sf, P_mean, P_std):
        seen.update(eps=eps, rnd=rnd, noise=noise, drop_u=drop_u, P=(P_mean, P_std))
        raise _Stop

    monkeypatch.setattr(ops, "flow_step_front", front)
    B, C, R = 3, 4, 8
    with pytest.raises(_Stop):
        L(P_mean=0.25, P_std=0.75).from_moments(None, torch.zeros(B, 2 * C, R, R), torch.zeros(B, 10),
                                                class_dropout_prob=0.1)
    assert calls == [("randn", (B, C, R, R)), ("rand", (B, 1)), ("randn", (B, 1, 1, 1)), ("randn", (B, C, R, R))]
    assert seen["rnd"].shape == (B,) and float(seen["rnd"][0]) == 3.0
    assert float(seen["eps"].flatten()[0]) == 1.0 and float(seen["noise"].flatten()[0]) == 4.0
    assert seen["P"] == (0.25, 0.75)


def test_validation_levels():
    z = validate.level_normals(8)
    t = validate.t_levels(8)
    np.testing.assert_allclose(t, 1.0 / (1.0 + np.exp(-z)), rtol=1e-15)
    assert np.all(np.diff(t) > 0) and abs(t.mean() - 0.5) < 1e-12       # symmetric about the median t = 1/2
    assert validate.t_levels(1).tolist() == [0.5]
    res = validate.summarize(torch.tensor([[1.0, 2.0], [3.0, 4.0]]), 0.0, 1.0, "flow")
    assert res["objective"] == "flow" and "sigma" not in res
    np.testing.assert_allclose(res["t"], validate.t_levels(2))
    assert res["per_level"] == [2.0, 3.0] and res["mean"] == 2.5
    assert "objective" not in validate.summarize(torch.tensor([[1.0, 2.0]]))   # the EDM result is unchanged


def test_flow_val_line():
    import train
    res = {"mean": 1.5, "per_level": [1.0, 2.0], "count": 3, "objective": "flow"}
    assert train.val_line(12, res) == "(step=0000012) Val Loss (flow): 1.50000 [1.00000 2.00000] (3 items, EMA)"


def _gen_args(**kw):
    base = dict(solver=None, discretization=None, schedule=None, scaling=None, S_churn=0, guide_ckpt=None,
                guide_snapshots=None, guidance=None)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw, what", [
    (dict(solver="euler"), "--solver"), (dict(discretization="vp"), "--discretization"),
    (dict(schedule="vp"), "--schedule"), (dict(scaling="vp"), "--scaling"), (dict(S_churn=10), "--S_churn"),
    (dict(guide_ckpt="g.pt", guidance=2.0), "autoguidance"),
])
def test_generate_refuses_edm_switches_for_flow(kw, what):
    import generate
    generate.check_flow_args(_gen_args())              # the plain flow call passes
    with pytest.raises(SystemExit, match=what):
        generate.check_flow_args(_gen_args(**kw))


def _normalised_sass(text):
    import re
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
            continue
        if cur is None:
            continue
        s = " ".join(re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).split())
        if s and not s.startswith(".headerflags"):
            out[cur].append(s)
    names = subprocess.run(["c++filt"], input="\n".join(out), capture_output=True, text=True, check=True).stdout
    return dict(zip(names.splitlines(), out.values()))


def test_edm_instantiations_sass_unchanged():
    """patch_embed (forward and backward), timestep_freq, step_front and edm_loss compile for EDM to the SASS they
    had before the flow variants were added."""
    gold = json.load(open(os.path.join(GOLD, "flow_sass.json")))
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    nvcc, cuobjdump = os.path.join(cuda, "bin", "nvcc"), os.path.join(cuda, "bin", "cuobjdump")
    if not (os.path.exists(nvcc) and os.path.exists(cuobjdump) and shutil.which("c++filt")):
        pytest.skip("needs nvcc, cuobjdump and c++filt")
    if gold["nvcc"] not in subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout:
        pytest.skip(f"the fingerprints are of nvcc {gold['nvcc']}")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("the library is not built")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    fns = _normalised_sass(sass)
    assert len(gold["functions"]) == 9
    for short, want in gold["functions"].items():
        hits = [v for k, v in fns.items() if k.split("mdt::", 1)[-1].startswith(f"{short}(")]
        assert len(hits) == 1, short
        assert len(hits[0]) == want["lines"], (short, len(hits[0]))
        assert hashlib.sha256("\n".join(hits[0]).encode()).hexdigest() == want["sha256"], short
    # the flow instantiations exist next to them
    names = [k.split("mdt::", 1)[-1] for k in fns]
    for flow in ("timestep_freq_kernel<1>(", "flow_loss_kernel<true>(", "flow_loss_kernel<false>(",
                 "flow_step_front_kernel(", "flow_out_kernel("):
        assert sum(n.startswith(flow) for n in names) == 1, flow
