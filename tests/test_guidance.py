"""CPU: the argument checks of guidance by a second network and of the guidance interval (samplers, EDMPrecond,
the C entry point, generate.py's flags), and the snapshot-built guide of generate.py against posthoc_ema.py."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MDT_ERR_ARG = -1
A = 1 << 20   # a 256-byte aligned dummy address: the argument checks never dereference it


def _net(num_classes=10, model_type="DiT-S/2", img_resolution=8, img_channels=4, **kw):
    from maskdit_b200.maskdit import Precond_models
    return Precond_models["edm"](img_resolution, img_channels, num_classes=num_classes, model_type=model_type,
                                 use_decoder=kw.pop("use_decoder", True), mae_loss_coef=0.1, **kw)


@pytest.fixture(scope="module")
def nets():
    return _net(), _net(model_type="DiT-S/4", use_decoder=False)


SAMPLERS = ["edm_sampler", "ablation_sampler"]


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_sampler_rejects_exclusive_and_incomplete_arguments(nets, sampler):
    from maskdit_b200 import sampler as S
    fn = getattr(S, sampler)
    net, guide = nets
    lat = torch.zeros(1, 4, 8, 8)
    bad = [dict(cfg_scale=1.5, guide_net=guide, guidance=2.0),       # CFG and a guide in one call
           dict(guide_net=guide),                                   # a guide without its weight
           dict(guidance=2.0),                                      # a weight without a guide
           dict(guide_net=guide, guidance=float("nan")),
           dict(guide_net=guide, guidance=float("inf"))]
    for kw in bad:
        with pytest.raises(ValueError):
            fn(net, lat, None, num_steps=2, **kw)


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_sampler_rejects_bad_interval(nets, sampler):
    from maskdit_b200 import sampler as S
    fn = getattr(S, sampler)
    net, guide = nets
    lat = torch.zeros(1, 4, 8, 8)
    for iv in ((1.0, 1.0), (2.0, 1.0), (5.0, 0.1)):
        for kw in (dict(cfg_scale=1.5), dict(guide_net=guide, guidance=2.0)):
            with pytest.raises(ValueError, match="sigma_lo < sigma_hi"):
                fn(net, lat, None, num_steps=2, guidance_interval=iv, **kw)
    with pytest.raises(ValueError, match="needs cfg_scale or guide_net"):    # an interval with nothing to limit
        fn(net, lat, None, num_steps=2, guidance_interval=(0.1, 5.0))


@pytest.mark.parametrize("field,value", [("img_resolution", 16), ("img_channels", 3), ("num_classes", 0),
                                         ("num_classes", 7), ("sigma_data", 1.0)])
def test_guide_of_other_geometry_is_refused(nets, field, value):
    from maskdit_b200.sampler import edm_sampler
    net, _ = nets
    kw = dict(num_classes=10, img_resolution=8, img_channels=4)
    kw[field] = value
    guide = _net(model_type="DiT-S/4", **kw)
    with pytest.raises(ValueError, match=field):
        net.check_guide(guide)
    with pytest.raises(ValueError, match=field):      # refused before any device work: these are CPU tensors
        net.forward_guided(torch.zeros(1, 4, 8, 8), torch.ones(1), None, guide, 2.0)
    with pytest.raises(ValueError, match=field):
        edm_sampler(net, torch.zeros(1, 4, 8, 8), None, num_steps=2, guide_net=guide, guidance=2.0)


def test_guide_may_differ_in_depth_width_patch_and_decoder(nets):
    net, guide = nets
    net.check_guide(guide)
    net.check_guide(_net(model_type="DiT-B/2"))
    with pytest.raises(ValueError):
        net.check_guide(torch.nn.Linear(2, 2))
    with pytest.raises(ValueError, match="finite"):
        net.forward_guided(torch.zeros(1, 4, 8, 8), torch.ones(1), None, guide, float("nan"))


def test_c_entry_point_rejects_bad_arguments():
    from maskdit_b200 import _lib
    L = _lib.lib()

    def call(Fm=A, pm=2, Fg=A, pg=4, x=A, s=A, w=1.5, D=A, b=2, c=4, r=16):
        return L.mdt_guided_precond_out(Fm, pm, Fg, pg, x, s, 0.5, w, D, b, c, r, None)

    for kw in (dict(Fm=None), dict(Fg=None), dict(x=None), dict(s=None), dict(D=None), dict(b=0), dict(c=-1),
               dict(r=0), dict(pm=0), dict(pg=-4), dict(pm=3), dict(pg=32), dict(r=18, pm=4), dict(w=float("nan")),
               dict(w=float("inf"))):
        assert call(**kw) == MDT_ERR_ARG, kw


# ---- generate.py ---------------------------------------------------------------------------------------------------------
def _parse(*extra):
    import generate
    return generate.parse_args(["--config", "c.yaml", *extra])


def test_generate_parses_guidance_flags():
    a = _parse("--guide_ckpt", "g.pt", "--guidance", "2.5", "--guidance_interval", "0.3", "5")
    assert (a.guide_ckpt, a.guide_key, a.guide_config, a.guidance, a.guidance_interval) == \
        ("g.pt", "ema", None, 2.5, [0.3, 5.0])
    a = _parse("--guide_ckpt", "g.pt", "--guide_key", "model", "--guide_config", "s4.yaml", "--guidance", "1.8")
    assert (a.guide_key, a.guide_config, a.guidance_interval) == ("model", "s4.yaml", None)
    a = _parse("--guide_snapshots", "phema", "--guide_sigma_rel", "0.05", "--guide_step", "4000", "--guidance", "2")
    assert (a.guide_snapshots, a.guide_sigma_rel, a.guide_step, a.guide_ckpt) == ("phema", 0.05, 4000, None)
    a = _parse("--cfg_scale", "1.5", "--guidance_interval", "0.28", "5.42")
    assert (a.cfg_scale, a.guidance_interval, a.guidance) == (1.5, [0.28, 5.42], None)
    a = _parse()
    assert (a.guide_ckpt, a.guide_snapshots, a.guidance, a.guidance_interval) == (None, None, None, None)


@pytest.mark.parametrize("flags", [
    ["--cfg_scale", "1.5", "--guide_ckpt", "g.pt", "--guidance", "2"],
    ["--cfg_scale", "1.5", "--guide_snapshots", "d", "--guide_sigma_rel", "0.05", "--guidance", "2"],
    ["--guide_ckpt", "g.pt", "--guide_snapshots", "d", "--guide_sigma_rel", "0.05", "--guidance", "2"],
    ["--guide_ckpt", "g.pt"],
    ["--guidance", "2"],
    ["--guide_snapshots", "d", "--guidance", "2"],
    ["--guide_ckpt", "g.pt", "--guide_sigma_rel", "0.05", "--guidance", "2"],
    ["--guide_ckpt", "g.pt", "--guide_step", "10", "--guidance", "2"],
    ["--guide_config", "s4.yaml"],
    ["--guidance_interval", "0.3", "5"],
    ["--cfg_scale", "1.5", "--guidance_interval", "5", "0.3"],
    ["--guide_ckpt", "g.pt", "--guidance", "2", "--guidance_interval", "1", "1"],
    ["--guide_ckpt", "g.pt", "--guide_key", "opt", "--guidance", "2"],
])
def test_generate_refuses_conflicting_flags(flags):
    with pytest.raises(SystemExit):
        _parse(*flags)


def test_generate_loads_guide_checkpoint_keys(tmp_path):
    import generate
    sd = {"model.a": torch.arange(6.0).view(2, 3)}
    torch.save({"ema": sd, "model": {"_orig_mod.model.a": sd["model.a"] + 1}}, tmp_path / "g.pt")
    got = generate.guide_state_dict(_parse("--guide_ckpt", str(tmp_path / "g.pt"), "--guidance", "2"))
    assert torch.equal(got["model.a"], sd["model.a"])
    got = generate.guide_state_dict(_parse("--guide_ckpt", str(tmp_path / "g.pt"), "--guide_key", "model",
                                           "--guidance", "2"))
    assert list(got) == ["model.a"] and torch.equal(got["model.a"], sd["model.a"] + 1)
    torch.save({"ema": sd}, tmp_path / "posthoc.pt")          # posthoc_ema.py writes 'ema' only
    with pytest.raises(SystemExit, match="'model'"):
        generate.guide_state_dict(_parse("--guide_ckpt", str(tmp_path / "posthoc.pt"), "--guide_key", "model",
                                         "--guidance", "2"))


def _write_snapshots(d, keys):
    """Power-function EMA snapshots as train.py writes them (two profiles per file), of a drifting random state."""
    from maskdit_b200 import phema
    d.mkdir()
    g = torch.Generator().manual_seed(0)
    w = {k: torch.randn(v, generator=g) for k, v in keys.items()}
    for step in (100, 200, 300, 400):
        profiles = []
        for s in (0.05, 0.10):
            profiles.append({"sigma_rel": s, "gamma": phema.sigma_rel_to_gamma(s),
                             "ema": {k: v + 0.1 * torch.randn(v.shape, generator=g) for k, v in w.items()}})
        torch.save({"step": step, "origin": 0, "profiles": profiles}, d / f"phema-{step:07d}.pt")


@pytest.mark.parametrize("step", [None, 300])
def test_snapshot_guide_equals_posthoc_ema_output(tmp_path, step):
    import generate
    import posthoc_ema
    net = _net()
    keys = {k: tuple(v.shape) for k, v in net.state_dict().items() if k.startswith(("model.final_layer",
                                                                                     "model.blocks.0."))}
    _write_snapshots(tmp_path / "phema", keys)
    at = [] if step is None else ["--step", str(step)]
    out = posthoc_ema.main(["--snapshots", str(tmp_path / "phema"), "--sigma_rel", "0.08", *at,
                            "--out", str(tmp_path / "ema.pt")])
    want = torch.load(out[0], weights_only=True)["ema"]
    at = [] if step is None else ["--guide_step", str(step)]
    got = generate.guide_state_dict(_parse("--guide_snapshots", str(tmp_path / "phema"), "--guide_sigma_rel", "0.08",
                                           *at, "--guidance", "2"))
    assert list(got) == list(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), k
    net.load_state_dict(got, strict=False)       # the reconstructed tensors fit the guide's parameters
