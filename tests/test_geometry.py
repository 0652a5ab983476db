"""CPU tests of the DiT_models geometries beyond the shipped XL/2 (patch 4 and 8, DiT-B / L / H): the CPU fp32 oracle
against the unmodified reference's goldens of tests/golden/make_golden_geometry.py, which pins those goldens, and the C
driver's model config, packed layout and workspace plan for all 15 names with and without the decoder."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import maskdit_oracle as O  # noqa: E402
from support import nd_dit_forward  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def load(name):
    return {k: v for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}


def t(a):
    return torch.from_numpy(np.asarray(a))


def cfg(model_type, R, ncls, use_decoder=True):
    return O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls, use_decoder=use_decoder)


# name -> oracle config; the decoder-less ones run support.nd_dit_forward, the restatement of the forward
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
# (model, latent resolution, classes): every name at 32x32 with 1000 classes, then 8x8 and 16x16 with class counts
# that are not multiples of 8, and XL/2 at 64x64 (512 px)
GEOMS = [(mt, 32, 1000) for mt in MODELS] + [("DiT-S/2", 8, 10), ("DiT-B/4", 16, 7), ("DiT-XL/2", 64, 1000)]


@pytest.mark.parametrize("use_decoder", [True, False])
@pytest.mark.parametrize("mt,R,ncls", GEOMS)
def test_packed_layout_rules_and_workspace(mt, R, ncls, use_decoder):
    """`mdt_model_create` accepts the model, and the packed layout FlatStore reads from its handle follows the blob's
    rules against the nn.Module: the module's tensors; adaLN weights contiguous in head order, then their biases in
    the same order, then the other trainable tensors in registration order, then the frozen pos-embeds; 64-element
    aligned, increasing, disjoint.  Each head's modulation column is the Python engine's; the workspace plan grows
    with the batch and the token count, training needs more than eval, and B = 0 is refused."""
    from maskdit_b200._lib import MdtError
    from maskdit_b200.engine import Engine
    from maskdit_b200.maskdit import Precond_models
    c = cfg(mt, R, ncls, use_decoder)
    with torch.device("meta"):
        net = Precond_models["edm"](R, 4, num_classes=ncls, model_type=mt, use_decoder=use_decoder, mae_loss_coef=0.1)
    named = dict(net.named_parameters())
    assert {k: tuple(p.shape) for k, p in named.items()} == {k: tuple(v) for k, v in O.param_shapes(c).items()}
    assert any("decoder_blocks" in k for k in named) == use_decoder
    ce, st = net._layout()
    assert {k: v[1:] for k, v in st.offsets.items()} == {k: (p.numel(), tuple(p.shape)) for k, p in named.items()}
    D, Dd, dec_depth = (c.hidden, c.dec_hidden, c.dec_depth) if use_decoder else (c.hidden, 0, 0)
    heads = [f"model.blocks.{i}" for i in range(c.depth)]
    if use_decoder:
        heads += ["model.decoder_layer"] + [f"model.decoder_blocks.{i}" for i in range(dec_depth)]
    heads.append("model.final_layer")
    ada_w = [f"{h}.adaLN_modulation.1.weight" for h in heads]
    ada_b = [f"{h}.adaLN_modulation.1.bias" for h in heads]
    rest = [k for k, p in named.items() if p.requires_grad and "adaLN_modulation" not in k]
    frozen = [k for k, p in named.items() if not p.requires_grad]
    assert frozen == ["model.pos_embed", "model.decoder_pos_embed"][:1 + use_decoder]
    assert list(st.offsets) == ada_w + ada_b + rest + frozen
    spans = list(st.offsets.values())
    assert spans[0][0] == 0 and all(o % 64 == 0 for o, _, _ in spans)
    assert all(o + n <= o2 for (o, n, _), (o2, _, _) in zip(spans, spans[1:]))
    assert st.offsets[rest[-1]][0] + st.offsets[rest[-1]][1] <= st.n_train <= st.offsets[frozen[0]][0]
    assert st.offsets[frozen[-1]][0] + st.offsets[frozen[-1]][1] <= st.n_total
    if (mt, use_decoder, ncls) == ("DiT-XL/2", True, 1000):
        assert sum(p.numel() for p in named.values() if p.requires_grad) == 730_115_216 <= st.n_train
    # adaLN: ONE [NA, D] weight matrix, then ONE [NA] bias vector; a head's modulation column is its first row
    off_declayer = 6 * D * c.depth
    off_final = off_declayer + (2 * D + 6 * Dd * dec_depth if use_decoder else 0)
    NA = off_final + 2 * (Dd or D)
    for keys, width in ((ada_w, D), (ada_b, 1)):
        cur = st.offsets[keys[0]][0]
        for k in keys:
            assert st.offsets[k][0] == cur, k
            cur += st.offsets[k][1]
        assert cur - st.offsets[keys[0]][0] == NA * width
    assert st.ada_w_range == (0, NA, D) and st.ada_b_range == (NA * D, NA) and ce.NA == NA
    eng = Engine(net._cfg(), st)
    assert (eng.NA, eng.off_final, eng.off_declayer) == (NA, off_final, off_declayer if use_decoder else None)
    assert [s.mod_off for s in eng.enc] == [6 * D * i for i in range(c.depth)]
    assert [s.mod_off for s in eng.dec] == [off_declayer + 2 * D + 6 * Dd * i for i in range(dec_depth)]
    assert ce._L.mdt_model_param_info(ce._h, len(st.offsets), None, 0, None, None) != 0
    T = c.num_patches // 2
    tr, ev = ce.workspace_bytes(8, T, True), ce.workspace_bytes(8, 0, False)
    assert tr > ev > 0 and ce.workspace_bytes(16, T, True) > tr
    assert ce.workspace_bytes(8, c.num_patches, True) > tr
    with pytest.raises(MdtError):
        ce.workspace_bytes(0, T, True)
