"""CPU tests of the DiT_models geometries beyond the shipped XL/2 (patch 4 and 8, DiT-B / L / H): the CPU fp32 oracle
against the unmodified reference's goldens of tests/golden/make_golden_geometry.py, which pins those goldens, and the C
driver's model config, packed layout and workspace plan for all 15 names with and without the decoder."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import maskdit_oracle as O  # noqa: E402
from test_nodecoder import nd_dit_forward  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def load(name):
    return {k: v for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}


def t(a):
    return torch.from_numpy(np.asarray(a))


def cfg(model_type, R, ncls, use_decoder=True):
    return O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls, use_decoder=use_decoder)


# name -> oracle config; the decoder-less ones run test_nodecoder.py's restatement of the forward
TRAIN = {
    "geo_s8_mask50": cfg("DiT-S/8", 32, 10),
    "geo_b8_nd_nomask": cfg("DiT-B/8", 32, 10, use_decoder=False),
    "geo_l4_nd_uncond_mask30": cfg("DiT-L/4", 32, 0, use_decoder=False),
    "geo_h2_mask50": cfg("DiT-H/2", 32, 1000),
}


@pytest.mark.parametrize("name", list(TRAIN))
def test_oracle_train_loss_and_grads_match_reference(name, monkeypatch):
    """fp32 vs fp32 at the tolerances of test_oracle_golden.py."""
    c = TRAIN[name]
    if not c.use_decoder:
        monkeypatch.setattr(O, "dit_forward", nd_dit_forward)
    g = load(name)
    sd = {k: v.requires_grad_(not k.endswith("pos_embed")) for k, v in O.make_state_dict(c, 1).items()}
    assert {k[len("gnorm/"):] for k in g if k.startswith("gnorm/")} <= set(sd)
    mr = float(g["mask_ratio"])
    md = O.mask_from_noise(t(g["mask_noise"]), mr) if mr > 0 else None
    if md is not None:
        for k in ("mask", "ids_keep", "ids_restore"):
            assert np.array_equal(md[k].numpy(), g[k])
        assert md["ids_keep"].shape[1] == int(c.num_patches * (1 - mr))
    labels = t(g["labels"]) if "labels" in g else None
    loss, D = O.edm_loss(sd, c, t(g["images"]), labels, t(g["rnd_normal"]), t(g["noise_unit"]), md, c.mae_loss_coef)
    np.testing.assert_allclose(loss.detach().numpy(), g["loss"], rtol=2e-5, atol=1e-6)
    np.testing.assert_allclose(D.detach().numpy(), g["D"], rtol=1e-4, atol=2e-5)
    loss.mean().backward()
    checked = 0
    for k, v in g.items():
        if k.startswith("grad/"):
            gg = sd[k[5:]].grad   # None == zero gradient (the reference's "+ 0 * sum(mask_token)")
            gg = np.zeros_like(v) if gg is None else gg.numpy()
            np.testing.assert_allclose(gg, v, rtol=2e-3, atol=1e-6, err_msg=k)
            checked += 1
        elif k.startswith("gnorm/"):
            got = sd[k[6:]].grad
            got = 0.0 if got is None else got.double().norm().item()
            assert abs(got - float(v)) <= 2e-4 * (float(v) + 1e-9) + 1e-9, (k, got, float(v))
            checked += 1
        elif k.startswith("gslice/"):
            gg = sd[k[7:]].grad
            np.testing.assert_allclose(gg.reshape(gg.shape[0], -1)[:4, :8].numpy(), v, rtol=2e-3, atol=1e-6)
    assert checked >= 12 * 10 + 10


def test_oracle_s8_eval_cfg_and_short_sampler_match_reference():
    g = load("geo_s8_eval")
    c = cfg("DiT-S/8", 32, 10)
    sd = O.make_state_dict(c, 1)
    lab = t(g["labels"])
    with torch.no_grad():
        plain = O.edm_precond(sd, c, t(g["images"]), t(g["sigma"]), lab, training=False)
        np.testing.assert_allclose(plain.numpy(), g["D_plain"], rtol=1e-4, atol=2e-5)
        cf = O.edm_precond(sd, c, t(g["images"]), torch.tensor(1.7, dtype=torch.float64), lab, cfg_scale=1.5,
                           training=False)
        np.testing.assert_allclose(cf.numpy(), g["D_cfg"], rtol=1e-4, atol=2e-5)
        z, evals = O.edm_sampler(lambda x, s: O.edm_precond(sd, c, x, s, lab, cfg_scale=1.5, training=False),
                                 t(g["latents"]), num_steps=int(g["num_steps"]))
    np.testing.assert_allclose(np.array(evals), g["sampler_sigmas"], rtol=1e-12)
    np.testing.assert_allclose(z.numpy(), g["z"], rtol=1e-3, atol=1e-4)


def test_h2_bf16_autocast_yardstick_is_recorded():
    """The reference's own bf16-autocast error on the 32-block DiT-H/2 forward, which bounds the GPU comparison."""
    g = load("geo_h2_bf16")
    assert 0 < float(g["bf16_rel_D_train"]) < 5e-2


# ---- C driver: every model name, with and without the decoder ---------------------------------------------------------
MODELS = [f"DiT-{a}/{p}" for a in ("H", "XL", "L", "B", "S") for p in (2, 4, 8)]


@pytest.mark.parametrize("use_decoder", [True, False])
@pytest.mark.parametrize("mt", MODELS)
def test_model_create_layout_and_workspace_every_model(mt, use_decoder):
    """`mdt_model_create` accepts the model; its packed tensors are FlatStore's layout in the reference's order; the
    modulation width is the Python engine's; the workspace plan grows with the batch and training needs more than
    eval."""
    from maskdit_b200 import _lib
    from maskdit_b200.engine import Engine
    from maskdit_b200.flat import FlatStore
    from maskdit_b200.maskdit import Precond_models
    R = 32
    c = cfg(mt, R, 1000, use_decoder)
    with torch.device("meta"):
        net = Precond_models["edm"](R, 4, num_classes=1000, model_type=mt, use_decoder=use_decoder, mae_loss_coef=0.1)
    shapes = {k: tuple(p.shape) for k, p in net.named_parameters()}
    want = O.param_shapes(c)
    assert shapes == {k: tuple(v) for k, v in want.items()}
    assert any("decoder_blocks" in k for k in shapes) == use_decoder
    st = FlatStore()
    st.plan(shapes)
    eng = Engine(net._cfg(), st)
    D = c.hidden
    dec = (c.dec_hidden, c.dec_depth, c.dec_heads, 4 * c.dec_hidden, 1) if use_decoder else (0, 0, 0, 0, 0)
    L = _lib.lib()
    mc = _lib.ModelCfg(R, 4, c.patch, 1000, D, c.depth, c.heads, 4 * D, *dec, 0.5)
    h = ctypes.c_void_p()
    assert L.mdt_model_create(ctypes.byref(mc), ctypes.byref(h)) == 0
    try:
        n = L.mdt_model_num_tensors(h)
        assert n == len(shapes)
        name, off, num = ctypes.create_string_buffer(160), ctypes.c_longlong(), ctypes.c_longlong()
        for i in range(n):
            assert L.mdt_model_param_info(h, i, name, 160, ctypes.byref(off), ctypes.byref(num)) == 0
            k = name.value.decode()
            assert st.offsets[k][:2] == (off.value, num.value), k
        assert (L.mdt_model_param_count(h, 1), L.mdt_model_param_count(h, 0)) == (st.n_train, st.n_total)
        assert L.mdt_model_mod_width(h) == eng.NA == st.ada_w_range[1]
        T = c.num_patches // 2
        tr, ev = L.mdt_workspace_bytes(h, 8, T, 1), L.mdt_workspace_bytes(h, 8, 0, 0)
        assert tr > ev > 0 and L.mdt_workspace_bytes(h, 16, T, 1) > tr
        assert L.mdt_workspace_bytes(h, 8, c.num_patches, 1) > tr
    finally:
        L.mdt_model_destroy(h)
