"""GPU: guidance by a second network (autoguidance) and the guidance interval.

The combine kernel (`mdt_guided_precond_out`) against float64 at every patch pairing, `EDMPrecond.forward_guided`
against the float64 combine of the two networks' own unguided outputs, the guided samplers against a host loop of
unguided calls, the interval's per-evaluation decision, and `generate.py --guide_ckpt` end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

R, C, B, NCLS = 16, 4, 4, 10
SD = 0.5
EPS32 = float(np.finfo(np.float32).eps)
MDT_ERR_ARG = -1


def _net(model_type="DiT-S/2", num_classes=NCLS, use_decoder=True, seed=1):
    from maskdit_b200.maskdit import Precond_models
    torch.manual_seed(seed)
    net = Precond_models["edm"](img_resolution=R, img_channels=C, num_classes=num_classes, model_type=model_type,
                                use_decoder=use_decoder, mae_loss_coef=0.1, pad_cls_token=False)
    with torch.no_grad():   # the zero-initialised tensors (adaLN, final layer) get values, so the output is not c_skip x
        gz = torch.Generator().manual_seed(seed + 100)
        for p in net.parameters():
            if p.requires_grad and float(p.abs().sum()) == 0.0:
                p.copy_(torch.randn(p.shape, generator=gz) * 0.02)
    return net.cuda().eval()


def _labels(num_classes, seed=3):
    if not num_classes:
        return None
    g = torch.Generator().manual_seed(seed)
    return torch.eye(num_classes)[torch.randint(0, num_classes, (B,), generator=g)].cuda()


def _unpatchify64(F, p):
    G = R // p
    return F.double().view(B, G, G, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, R, R)


def _c(sig):
    s = sig.double().view(-1, 1, 1, 1)
    return SD ** 2 / (s ** 2 + SD ** 2), s * SD / (s ** 2 + SD ** 2).sqrt()


# ---- 1. the kernel against float64 -------------------------------------------------------------------------------------
@pytest.mark.parametrize("pm,pg", [(2, 2), (2, 4), (2, 8), (4, 2)])
@pytest.mark.parametrize("w", [0.0, 0.5, 1.5, 3.0])
def test_kernel_matches_float64(pm, pg, w):
    from maskdit_b200 import ops
    g = torch.Generator().manual_seed(pm * 10 + pg)
    Fm = torch.randn(B * (R // pm) ** 2, pm * pm * C, generator=g).cuda()
    Fg = torch.randn(B * (R // pg) ** 2, pg * pg * C, generator=g).cuda()
    x = (torch.randn(B, C, R, R, generator=g) * 3).cuda()
    sig = torch.tensor([0.002, 0.3, 2.5, 80.0]).cuda()
    D = ops.guided_precond_out(Fm, pm, Fg, pg, x, sig, SD, w).double()
    fm, fg = _unpatchify64(Fm, pm), _unpatchify64(Fg, pg)
    cs, co = _c(sig)
    want = cs * x.double() + co * (fg + w * (fm - fg))
    scale = (cs * x.double()).abs() + co * (fg.abs() + abs(w) * (fm.abs() + fg.abs()))
    err = (D - want).abs()
    assert (err <= 16 * EPS32 * scale + 1e-30).all(), float((err / scale).max())


def test_kernel_rejects_bad_arguments():
    from maskdit_b200 import _lib
    L = _lib.lib()
    t = torch.zeros(B * C * R * R, device="cuda")
    a = t.data_ptr()

    def call(Fm=a, pm=2, Fg=a, pg=4, x=a, s=a, w=1.5, D=a, b=B, c=C, r=R):
        return L.mdt_guided_precond_out(Fm, pm, Fg, pg, x, s, SD, w, D, b, c, r, None)

    for kw in (dict(Fm=None), dict(Fg=None), dict(x=None), dict(s=None), dict(D=None), dict(b=0), dict(c=0),
               dict(r=0), dict(pm=0), dict(pg=-2), dict(pm=3), dict(pg=32), dict(r=18, pg=4), dict(w=float("nan")),
               dict(w=float("inf")), dict(w=float("-inf"))):
        assert call(**kw) == MDT_ERR_ARG, kw
    torch.cuda.synchronize()


# ---- 2. forward_guided against the float64 combine of the unguided outputs ------------------------------------------
GUIDES = {"S/4": dict(model_type="DiT-S/4"), "no-decoder": dict(use_decoder=False)}


@pytest.mark.parametrize("ncls", [NCLS, 0])
@pytest.mark.parametrize("guide_kind", list(GUIDES))
def test_forward_guided_matches_float64_combine(monkeypatch, ncls, guide_kind):
    net = _net(num_classes=ncls)
    guide = _net(num_classes=ncls, seed=7, **GUIDES[guide_kind])
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(B, C, R, R, generator=g) * 2).cuda()
    sig = torch.tensor([0.05, 0.7, 4.0, 40.0]).cuda()
    lab = _labels(ncls)
    with torch.no_grad():
        Dm = net(x, sig, lab)["x"].double()
        Dg = guide(x, sig, lab)["x"].double()
        for w in (0.0, 2.0, 3.0):
            got = net.forward_guided(x, sig, lab, guide, w)
            want = Dg + w * (Dm - Dg)
            scale = max(Dm.abs().max(), Dg.abs().max(), x.abs().max())
            err = float((got.double() - want).abs().max())
            assert err <= 8 * EPS32 * (1 + 2 * w) * float(scale), (w, err)
            monkeypatch.setenv("MDT_CUDA_GRAPH", "0")
            eager = net.forward_guided(x, sig, lab, guide, w)
            monkeypatch.delenv("MDT_CUDA_GRAPH")
            assert torch.equal(eager, got), w
    assert any(len(k) == 5 for k in net._graphs)        # the graphed runs above replayed a guided graph


# ---- 3. the guided samplers against a host loop ------------------------------------------------------------------------
def _karras(n, smin=0.002, smax=80.0, rho=7):
    i = np.arange(n, dtype=np.float64)
    t = (smax ** (1 / rho) + i / (n - 1) * (smin ** (1 / rho) - smax ** (1 / rho))) ** rho
    return np.concatenate([t, [0.0]])


def _host_loop(net, guide, w, lat, lab, noises, num_steps, S_churn, solver="heun", combine="float64"):
    """sample.py:30-66 (Heun) / 146-188 with the edm discretization, linear schedule and no scaling (Euler) in float64,
    each D = D_guide + w (D_net - D_guide) combined in float64 from two unguided evaluations, or (combine="kernel")
    taken from `forward_guided`."""
    def D(x, s):
        sg = torch.tensor(s, dtype=torch.float64, device=x.device)
        if combine == "kernel":
            return net.forward_guided(x.float(), sg, lab, guide, w).double()
        dm = net(x.float(), sg, lab)["x"].double()
        dg = guide(x.float(), sg, lab)["x"].double()
        return dg + w * (dm - dg)

    t = _karras(num_steps)
    x_next = lat.double() * t[0]
    for i in range(num_steps):
        t_cur, t_next = float(t[i]), float(t[i + 1])
        gamma = min(S_churn / num_steps, np.sqrt(2) - 1)
        t_hat = t_cur + gamma * t_cur
        x_hat = x_next + np.sqrt(t_hat ** 2 - t_cur ** 2) * noises[i]
        d_cur = (x_hat - D(x_hat, t_hat)) / t_hat
        x_next = x_hat + (t_next - t_hat) * d_cur
        if solver == "heun" and i < num_steps - 1:
            d_prime = (x_next - D(x_next, t_next)) / t_next
            x_next = x_hat + (t_next - t_hat) * (0.5 * d_cur + 0.5 * d_prime)
    return x_next


def _noises(n, seed=11):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(B, C, R, R, generator=g).cuda()
    return lat, [torch.randn(B, C, R, R, generator=g, dtype=torch.float64).cuda() for _ in range(n)]


def _rel(a, b):
    return float((a - b).norm() / b.norm())


# Against the float64 combine: the fp32 combine differs from it in the last bits, and from there the bf16 operands of
# later evaluations round differently.  Measured on an H100: rel-L2 0.9e-3 to 1.8e-3 over the cases below (5 steps,
# w = 2.5), the same for edm and ablation Heun.  Against the loop that takes D from forward_guided, only the fp64
# state updates' rounding (fused kernels against torch expressions) separates the two: measured 0 to 5.1e-17.
LOOP_TOL, KERNEL_LOOP_TOL = 5e-3, 1e-12


@pytest.mark.parametrize("sampler", ["edm", "ablation-heun", "ablation-euler"])
@pytest.mark.parametrize("case", ["cond-S/4", "cond-nodecoder-churn", "uncond-S/4-churn", "uncond-nodecoder"])
def test_guided_sampler_matches_host_loop(sampler, case):
    from maskdit_b200.sampler import ablation_sampler, edm_sampler
    ncls = 0 if case.startswith("uncond") else NCLS
    churn = 20.0 if case.endswith("churn") else 0.0
    gk = GUIDES["S/4" if "S/4" in case else "no-decoder"]
    net, guide = _net(num_classes=ncls), _net(num_classes=ncls, seed=7, **gk)
    lab, n, w = _labels(ncls), 5, 2.5
    lat, noises = _noises(n)
    q = list(noises)
    with torch.no_grad():
        if sampler == "edm":
            z = edm_sampler(net, lat, lab, randn_like=lambda x: q.pop(0), num_steps=n, S_churn=churn,
                            guide_net=guide, guidance=w)
        else:
            z = ablation_sampler(net, lat, lab, randn_like=lambda x: q.pop(0), num_steps=n, S_churn=churn,
                                 solver=sampler.split("-")[1], guide_net=guide, guidance=w)
        solver = "euler" if sampler.endswith("euler") else "heun"
        want = _host_loop(net, guide, w, lat, lab, noises, n, churn, solver)
        same = _host_loop(net, guide, w, lat, lab, noises, n, churn, solver, combine="kernel")
    assert not q and z.dtype == torch.float64
    rel, rel_k = _rel(z, want), _rel(z, same)
    print(f"{sampler} {case}: rel-L2 against the host loop {rel:.2e}, against it with the kernel's combine {rel_k:.2e}")
    assert rel <= LOOP_TOL and rel_k <= KERNEL_LOOP_TOL, (rel, rel_k)


# ---- 4. the guidance interval ----------------------------------------------------------------------------------------------
class _Spy:
    """Records (sigma, kind) of every evaluation the sampler makes: 'plain', 'cfg' or 'guided'."""

    def __init__(self, net):
        self.net, self.calls = net, []
        self._fwd, self._guided = net.forward, net.forward_guided
        net.forward, net.forward_guided = self.forward, self.forward_guided

    def forward(self, x, s, labels=None, cfg_scale=None, **kw):
        self.calls.append((float(s), "plain" if cfg_scale is None else "cfg"))
        return self._fwd(x, s, labels, cfg_scale, **kw)

    def forward_guided(self, x, s, labels, guide, w):
        self.calls.append((float(s), "guided"))
        return self._guided(x, s, labels, guide, w)

    def close(self):
        del self.net.forward, self.net.forward_guided


def _run(net, lat, lab, n, **kw):
    from maskdit_b200.sampler import edm_sampler
    _, noises = _noises(n)
    with torch.no_grad():
        return edm_sampler(net, lat, lab, randn_like=lambda x: noises.pop(0), num_steps=n, **kw)


def test_interval_outside_every_sigma_is_unguided_and_inside_every_sigma_is_unlimited():
    net, guide, lab, n = _net(), _net(seed=7, model_type="DiT-S/4"), _labels(NCLS), 5
    lat, _ = _noises(n)
    plain = _run(net, lat, lab, n)
    for kw in (dict(cfg_scale=1.5), dict(guide_net=guide, guidance=2.0)):
        spy = _Spy(net)
        none = _run(net, lat, lab, n, guidance_interval=(100.0, 200.0), **kw)
        spy.close()
        assert torch.equal(none, plain), kw
        assert {k for _, k in spy.calls} == {"plain"}
        assert torch.equal(_run(net, lat, lab, n, guidance_interval=(0.0, 1000.0), **kw), _run(net, lat, lab, n, **kw))
    assert not torch.equal(_run(net, lat, lab, n, cfg_scale=1.5), plain)


@pytest.mark.parametrize("mode", ["cfg", "guided"])
def test_partial_interval_guides_exactly_the_evaluations_inside(mode):
    from maskdit_b200 import _lib
    net, guide, lab, n = _net(), _net(seed=7, use_decoder=False), _labels(NCLS), 8
    lat, _ = _noises(n)
    t = _karras(n)
    # upper bound between t[2] and t[3], lower between t[5] and t[6]: the two evaluations of steps 2 and 5 fall on
    # different sides of a bound
    lo, hi = (t[5] + t[6]) / 2, (t[2] + t[3]) / 2
    kw = dict(cfg_scale=1.5) if mode == "cfg" else dict(guide_net=guide, guidance=2.0)
    _run(net, lat, lab, n, guidance_interval=(lo, hi), **kw)   # captures the graphs (a capture counts its launches)
    spy = _Spy(net)
    n0 = _lib.LAUNCHES
    _run(net, lat, lab, n, guidance_interval=(lo, hi), **kw)
    launches = _lib.LAUNCHES - n0
    spy.close()
    evals = [s for k in range(n) for s in ((t[k], t[k + 1]) if k < n - 1 else (t[k],))]
    want = ["plain" if not lo < s <= hi else mode for s in evals]
    np.testing.assert_allclose([s for s, _ in spy.calls], evals, rtol=1e-12)
    assert [k for _, k in spy.calls] == want, (spy.calls, lo, hi)
    assert want[4:6] == ["plain", mode] and want[10:12] == [mode, "plain"]     # step 2 and step 5 straddle a bound
    if mode == "guided":   # a guided evaluation adds exactly one guide pass (its launches less its output kernel)
        n0 = _lib.LAUNCHES
        _run(net, lat, lab, n)
        n_plain = _lib.LAUNCHES - n0
        with torch.no_grad():
            guide(lat, torch.ones(B, device="cuda"), lab)
            n0 = _lib.LAUNCHES
            guide(lat, torch.ones(B, device="cuda"), lab)
        guide_pass = _lib.LAUNCHES - n0 - 1
        assert launches - n_plain == want.count("guided") * guide_pass, (launches, n_plain, guide_pass)


def test_guidance_one_is_the_unguided_network_and_runs_no_guide():
    from maskdit_b200 import _lib
    net, guide, lab, n = _net(), _net(seed=7, model_type="DiT-S/4"), _labels(NCLS), 5
    lat, _ = _noises(n)
    _run(net, lat, lab, n)                # captures the graph (a capture counts its launches)
    n0 = _lib.LAUNCHES
    plain = _run(net, lat, lab, n)
    n_plain = _lib.LAUNCHES - n0
    spy = _Spy(net)
    n0 = _lib.LAUNCHES
    z = _run(net, lat, lab, n, guide_net=guide, guidance=1.0)
    n_one = _lib.LAUNCHES - n0
    spy.close()
    assert torch.equal(z, plain)
    assert {k for _, k in spy.calls} == {"plain"} and n_one == n_plain
    assert guide._engine is None          # the guide was never evaluated, so never even laid out on the device


# ---- 5. generate.py --guide_ckpt end to end --------------------------------------------------------------------------------
YAML = """
model:
  precond: edm
  model_type: {model_type}
  in_size: 16
  in_channels: 4
  num_classes: 10
  use_decoder: {use_decoder}
  ext_feature_dim: 0
  pad_cls_token: False
  mae_loss_coef: 0.1
"""


def test_generate_with_guide_ckpt_matches_direct_sampler_call(tmp_path):
    sys.path.insert(0, ROOT)
    import generate
    from maskdit_b200.config import build_net, load_config
    from maskdit_b200.sampler import edm_sampler
    (tmp_path / "net.yaml").write_text(YAML.format(model_type="DiT-S/2", use_decoder=True))
    (tmp_path / "guide.yaml").write_text(YAML.format(model_type="DiT-S/4", use_decoder=False))
    net, guide = _net(), _net(model_type="DiT-S/4", use_decoder=False, seed=7)
    torch.save({"ema": {k: v.cpu() for k, v in net.state_dict().items()}}, tmp_path / "net.pt")
    torch.save({"model": {"_orig_mod." + k: v.cpu() for k, v in guide.state_dict().items()}}, tmp_path / "guide.pt")
    seeds, n, w, iv = [3, 4, 5], 4, 2.0, (0.5, 20.0)
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "generate.py"), "--config", str(tmp_path / "net.yaml"),
                        "--ckpt_path", str(tmp_path / "net.pt"), "--seeds", "3-5", "--num_steps", str(n),
                        "--guide_ckpt", str(tmp_path / "guide.pt"), "--guide_key", "model", "--guide_config",
                        str(tmp_path / "guide.yaml"), "--guidance", str(w), "--guidance_interval", *map(str, iv),
                        "--results_dir", str(tmp_path / "out")], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    dev = torch.device("cuda")
    net2 = build_net(load_config(str(tmp_path / "net.yaml"))).to(dev).eval()
    net2.load_state_dict(net.state_dict())
    guide2 = build_net(load_config(str(tmp_path / "guide.yaml"))).to(dev).eval()
    guide2.load_state_dict(guide.state_dict())
    rnd = generate.StackedRandomGenerator(dev, seeds)
    lat = rnd.randn([len(seeds), C, R, R], device=dev)
    lab = torch.eye(NCLS, device=dev)[rnd.randint(NCLS, size=[len(seeds)], device=dev)]
    with torch.no_grad():
        z = edm_sampler(net2, lat.float(), lab.float(), randn_like=rnd.randn_like, num_steps=n, guide_net=guide2,
                        guidance=w, guidance_interval=iv).float().cpu().numpy()
    for s, zi in zip(seeds, z):
        got = np.load(tmp_path / "out" / f"{s:06d}.npy")
        assert np.array_equal(got, zi), (s, np.abs(got - zi).max())
