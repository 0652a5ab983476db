"""CPU tests of the decoder-less DiT (use_decoder=False, the reference's default, models/maskdit.py:254): a CPU fp32
restatement of its forward (support.nd_dit_forward) against the unmodified reference (tests/golden/make_golden_nodecoder.py), the module's
state-dict contract and the C driver's model-config validation."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import maskdit_oracle as O  # noqa: E402
from support import nd_dit_forward  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def nd(model_type, R, ncls):
    return O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls, use_decoder=False)


def load(name):
    return {k: v for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}


def t(a):
    return torch.from_numpy(np.asarray(a))


@pytest.fixture
def nd_oracle(monkeypatch):
    """The oracle's EDM preconditioning, loss and sampler running the decoder-less forward above."""
    monkeypatch.setattr(O, "dit_forward", nd_dit_forward)
    return O


def module(mt, R, ncls, **kw):
    from maskdit_b200.maskdit import Precond_models
    with torch.device("meta"):
        return Precond_models["edm"](R, 4, num_classes=ncls, model_type=mt, use_decoder=False, **kw)


# ---- oracle vs reference (fp32 tolerances of test_oracle_golden.py) ------------------------------------------------
@pytest.mark.parametrize("name,cfg", [("nd_s2_train_mask", nd("DiT-S/2", 8, 10)),
                                      ("nd_s2_train_nomask", nd("DiT-S/2", 8, 10)),
                                      ("nd_s2_uncond_mask30", nd("DiT-S/2", 32, 0)),
                                      ("nd_xl2_grads", nd("DiT-XL/2", 32, 1000))])
def test_oracle_train_loss_and_grads_match_reference(name, cfg, nd_oracle):
    g = load(name)
    sd = {k: v.requires_grad_(not k.endswith("pos_embed")) for k, v in O.make_state_dict(cfg, 1).items()}
    assert set(sd) == {k[len("gnorm/"):] for k in g if k.startswith("gnorm/")} | {"model.pos_embed"}
    mr = float(g["mask_ratio"])
    md = O.mask_from_noise(t(g["mask_noise"]), mr) if mr > 0 else None
    if md is not None:
        for k in ("mask", "ids_keep", "ids_restore"):
            assert np.array_equal(md[k].numpy(), g[k])
    labels = t(g["labels"]) if "labels" in g else None
    loss, D = O.edm_loss(sd, cfg, t(g["images"]), labels, t(g["rnd_normal"]), t(g["noise_unit"]), md,
                         cfg.mae_loss_coef)
    np.testing.assert_allclose(loss.detach().numpy(), g["loss"], rtol=2e-5, atol=1e-6)
    np.testing.assert_allclose(D.detach().numpy(), g["D"], rtol=1e-4, atol=2e-5)
    loss.mean().backward()
    checked = 0
    for k, v in g.items():
        if k.startswith("grad/"):
            np.testing.assert_allclose(sd[k[5:]].grad.numpy(), v, rtol=2e-3, atol=1e-6, err_msg=k)
            checked += 1
        elif k.startswith("gnorm/"):
            got = sd[k[6:]].grad.double().norm().item()
            assert abs(got - float(v)) <= 2e-4 * (float(v) + 1e-9) + 1e-9, (k, got, float(v))
            checked += 1
        elif k.startswith("gslice/"):
            gg = sd[k[7:]].grad
            np.testing.assert_allclose(gg.reshape(gg.shape[0], -1)[:4, :8].numpy(), v, rtol=2e-3, atol=1e-6)
    assert checked >= 12 * 10 + 10


def test_oracle_masked_output_rows_are_zero_fill():
    """Training with a mask: D at a removed patch is c_skip * x exactly (the network output there is a zero row)."""
    g = load("nd_s2_train_mask")
    sigma = (t(g["rnd_normal"]) * 1.2 - 1.2).exp()
    yn = t(g["images"]) + t(g["noise_unit"]) * sigma
    c_skip = 0.25 / (sigma ** 2 + 0.25)
    removed = t(g["mask"]).bool()
    got = O.patchify(t(g["D"]), 2, 4)[removed]
    want = O.patchify(c_skip * yn, 2, 4)[removed]
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-6, atol=1e-7)


def test_oracle_xl2_eval_cfg_and_short_sampler_match_reference(nd_oracle):
    g = load("nd_xl2_eval")
    cfg = nd("DiT-XL/2", 32, 1000)
    sd = O.make_state_dict(cfg, 1)
    lab = t(g["labels"])
    with torch.no_grad():
        plain = O.edm_precond(sd, cfg, t(g["images"]), t(g["sigma"]), lab, training=False)
        np.testing.assert_allclose(plain.numpy(), g["D_plain"], rtol=1e-3, atol=1e-4)
        c = O.edm_precond(sd, cfg, t(g["images"]), torch.tensor(1.7, dtype=torch.float64), lab, cfg_scale=1.5,
                          training=False)
        np.testing.assert_allclose(c.numpy(), g["D_cfg"], rtol=1e-3, atol=1e-4)
        z, evals = O.edm_sampler(lambda x, s: O.edm_precond(sd, cfg, x, s, lab, cfg_scale=1.5, training=False),
                                 t(g["latents"]), num_steps=int(g["num_steps"]))
    np.testing.assert_allclose(np.array(evals), g["sampler_sigmas"], rtol=1e-12)
    np.testing.assert_allclose(z.numpy(), g["z"], rtol=1e-3, atol=1e-3)


def test_bf16_autocast_yardstick_is_recorded():
    """The reference's own bf16-autocast error on the XL/2 forwards, which bounds the GPU comparisons."""
    g = load("nd_xl2_bf16")
    for k in ("D_train", "D_plain", "D_cfg"):
        assert 0 < float(g[f"bf16_rel_{k}"]) < 5e-2, k


# ---- module contract ------------------------------------------------------------------------------------------------
MODELS = [f"DiT-{a}/{p}" for a in ("H", "XL", "L", "B", "S") for p in (2, 4, 8)]


@pytest.mark.parametrize("mt", MODELS)
def test_state_dict_every_model(mt):
    """For every DiT_models name: state-dict keys, shapes and ORDER equal the reference's (oracle.param_shapes follows
    the reference's registration order and is pinned by make_golden's strict load).  The C driver's layout of these
    modules: test_geometry.py::test_packed_layout_rules_and_workspace."""
    from maskdit_b200.maskdit import DiT_models
    assert mt in DiT_models
    R = 32
    cfg = nd(mt, R, 1000)
    net = module(mt, R, 1000, mae_loss_coef=0.1)
    shapes = {k: tuple(p.shape) for k, p in net.named_parameters()}
    want = O.param_shapes(cfg)
    assert list(shapes) == list(want) and shapes == {k: tuple(v) for k, v in want.items()}
    assert not any("decoder" in k or "mask_token" in k for k in shapes)
    assert [k for k, p in net.named_parameters() if not p.requires_grad] == ["model.pos_embed"]
    assert list(net.state_dict()) == list(want)
    D = cfg.hidden
    assert shapes["model.final_layer.linear.weight"] == (cfg.patch_dim, D)
    assert shapes["model.final_layer.adaLN_modulation.1.weight"] == (2 * D, D)


def test_module_init_and_unconditional_keys():
    from maskdit_b200.maskdit import Precond_models, sincos_2d
    net = Precond_models["edm"](8, 4, num_classes=10, model_type="DiT-S/2", use_decoder=False, mae_loss_coef=0.1)
    sd = net.state_dict()
    for k, v in sd.items():
        should_be_zero = k.endswith(".bias") or "adaLN_modulation" in k or k.startswith("model.final_layer.linear")
        assert (v.abs().sum() == 0).item() == should_be_zero, k
    assert torch.allclose(sd["model.pos_embed"][0], sincos_2d(384, 4))
    m = net.model
    assert m.decoder_layer is None and m.decoder_blocks is None and m.decoder_pos_embed is None and m.mask_token is None
    c = net._cfg()
    assert (c.dec_hidden, c.dec_depth, c.dec_heads) == (0, 0, 0)
    unc = Precond_models["edm"](32, 4, num_classes=0, model_type="DiT-S/2", use_decoder=False)
    assert list(unc.state_dict()) == list(O.param_shapes(nd("DiT-S/2", 32, 0)))


def cfg_args(**over):
    a = dict(img_resolution=32, img_channels=4, patch_size=2, num_classes=1000, hidden=384, depth=12, heads=6,
             mlp_hidden=1536, dec_hidden=0, dec_depth=0, dec_heads=0, dec_mlp_hidden=0, has_mask_token=0,
             sigma_data=0.5)
    a.update(over)
    return a


@pytest.mark.parametrize("over,ok", [
    ({}, True),                                                                   # decoder-less
    (dict(dec_hidden=512, dec_depth=8, dec_heads=16, dec_mlp_hidden=2048), True),  # MaskDiT decoder
    (dict(dec_hidden=512, dec_depth=8, dec_heads=16, dec_mlp_hidden=2048, has_mask_token=1), True),
    (dict(has_mask_token=1), False),                                              # mask token without a decoder
    (dict(dec_depth=8), False),                                                   # dec_hidden = 0, dec_depth > 0
    (dict(dec_hidden=512), False),
    (dict(dec_heads=16), False),
    (dict(dec_mlp_hidden=2048), False),
    (dict(dec_hidden=512, dec_depth=8, dec_heads=16), False),                     # decoder without an MLP width
    (dict(dec_hidden=512, dec_depth=8, dec_mlp_hidden=2048), False),              # decoder without heads
    (dict(dec_hidden=512, dec_depth=-1, dec_heads=16, dec_mlp_hidden=2048), False),
])
def test_model_create_decoder_fields(over, ok):
    from maskdit_b200 import _lib
    L = _lib.lib()
    a = cfg_args(**over)
    mc = _lib.ModelCfg(*[a[f] for f, _ in _lib.ModelCfg._fields_])
    h = ctypes.c_void_p()
    rc = L.mdt_model_create(ctypes.byref(mc), ctypes.byref(h))
    assert (rc == 0) == ok, (over, rc)
    if rc == 0:
        L.mdt_model_destroy(h)


@pytest.mark.parametrize("flag", [dict(learn_sigma=True), dict(pad_cls_token=True), dict(direct_cls_token=True),
                                  dict(ext_feature_dim=16), dict(use_encoder_feat=True)])
def test_remaining_flags_still_raise(flag):
    from maskdit_b200.maskdit import Precond_models
    for use_decoder in (False, True):
        with pytest.raises(NotImplementedError):
            Precond_models["edm"](8, 4, num_classes=10, model_type="DiT-S/2", use_decoder=use_decoder, **flag)
