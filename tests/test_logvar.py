"""The learned loss weighting u(sigma) (EDM2 uncertainty weighting, `EDMPrecond(logvar_channels=C)`) on the host: the
step driver's layout with `mdt_model_set_logvar`, the module's tensors, the config key, the checkpoint helper, the log
lines, and the SASS of the loss kernels it must leave alone."""
import copy
import hashlib
import json
import math
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from maskdit_b200 import _lib, ops  # noqa: E402
from maskdit_b200.engine import CEngine  # noqa: E402
from maskdit_b200.maskdit import EDMPrecond, eval_state_dict  # noqa: E402

LV = ("logvar_fourier.freqs", "logvar_fourier.phases", "logvar_linear.weight")


def _net(C=0, use_decoder=True, **kw):
    return EDMPrecond(8, 4, num_classes=10, model_type="DiT-S/2", use_decoder=use_decoder, mae_loss_coef=0.1,
                      logvar_channels=C, **kw)


def _handle(net, C=None):
    """A fresh C handle of `net`'s config; C (not None): mdt_model_set_logvar(C) on it before anything else."""
    cfg = net._cfg()
    cfg.logvar_channels = 0
    ce = CEngine(cfg)
    if C is not None:
        ops.check(ce._L.mdt_model_set_logvar(ce._h, C), "mdt_model_set_logvar", 0)
    return ce


@pytest.mark.parametrize("use_decoder", [True, False])
def test_set_logvar_layout(use_decoder):
    net = _net(use_decoder=use_decoder)
    base = _handle(net)
    t0, n_train, n_total = base.tensors(), base.param_count(True), base.param_count(False)
    zero = _handle(net, 0)
    assert list(zero.tensors().items()) == list(t0.items())
    assert (zero.param_count(True), zero.param_count(False), zero.NA) == (n_train, n_total, base.NA)

    lv = _handle(net, 128)
    t1 = lv.tensors()
    assert set(t1) - set(t0) == set(LV) and set(t0) <= set(t1)
    assert lv.NA == base.NA
    # every trainable tensor keeps its offset; the weight ends the trainable region
    for k, (o, n) in t0.items():
        if o < n_train:
            assert t1[k] == (o, n), k
        else:   # frozen position tables move by the weight's 64-element-aligned slot
            assert t1[k] == (o + 128, n), k
    assert t1["logvar_linear.weight"] == (n_train, 128)
    assert lv.param_count(True) == n_train + 128
    frozen = [k for k, (o, _) in t1.items() if o >= n_train + 128]
    tables = ["model.pos_embed"] + (["model.decoder_pos_embed"] if use_decoder else [])
    assert frozen == tables + ["logvar_fourier.freqs", "logvar_fourier.phases"]
    assert t1["logvar_fourier.freqs"] == (n_total + 128, 128)
    assert t1["logvar_fourier.phases"] == (n_total + 256, 128)
    assert lv.param_count(False) == n_total + 384
    # blob order: the logvar weight is the last trainable tensor
    order = sorted(t1, key=lambda k: t1[k][0])
    assert order[order.index("logvar_linear.weight") + 1] == tables[0]
    # channel counts that are not 64-aligned still start every tensor on the boundary
    t3 = _handle(net, 3).tensors()
    assert t3["logvar_linear.weight"] == (n_train, 3) and t3["logvar_fourier.phases"][0] % 64 == 0


def test_set_logvar_refuses():
    net = _net()
    L = _lib.lib()
    for bad in (-1, 257):
        ce = _handle(net)
        assert L.mdt_model_set_logvar(ce._h, bad) == -1
        assert list(ce.tensors()) == list(_handle(net).tensors())   # a refused call leaves the layout
    assert L.mdt_model_set_logvar(None, 8) == -1
    ce = _handle(net)
    assert L.mdt_model_set_logvar(ce._h, 256) == 0
    assert L.mdt_model_set_logvar(ce._h, 16) == 0      # before any workspace the layout can still change
    ce.workspace_bytes(2, 0, True)
    assert L.mdt_model_set_logvar(ce._h, 32) == -1      # the handle has sized a workspace: the layout is final
    assert ce.tensors()["logvar_linear.weight"][1] == 16
    with pytest.raises(ValueError):
        _net(257)
    with pytest.raises(ValueError):
        _net(-1)


@pytest.mark.parametrize("use_decoder", [True, False])
def test_module_tensors_and_positions(use_decoder):
    off, on = _net(use_decoder=use_decoder), _net(128, use_decoder=use_decoder)
    names_off = [k for k, _ in off.named_parameters()]
    names_on = [k for k, _ in on.named_parameters()]
    assert names_on == names_off + list(LV)     # the reference's parameters keep their optimizer indices
    assert list(on.state_dict()) == list(off.state_dict()) + list(LV)
    p = dict(on.named_parameters())
    assert p["logvar_linear.weight"].shape == (1, 128) and p["logvar_linear.weight"].requires_grad
    assert not p["logvar_fourier.freqs"].requires_grad and not p["logvar_fourier.phases"].requires_grad
    assert torch.equal(p["logvar_linear.weight"], torch.zeros(1, 128))
    # the module's tensors are the handle's: the FlatStore builds
    _, st = on._layout()
    assert st.n_train == off._layout()[1].n_train + 128
    assert set(st.offsets) == set(names_on)


def test_fourier_features_are_fixed():
    a, b = _net(64), _net(64)
    g = torch.Generator().manual_seed(0)
    freqs = 2 * math.pi * torch.randn(64, generator=g)
    phases = 2 * math.pi * torch.rand(64, generator=g)
    for net in (a, b):
        assert torch.equal(net.logvar_fourier.freqs.data, freqs)
        assert torch.equal(net.logvar_fourier.phases.data, phases)
    # the draw does not touch torch's global RNG: the network's own initialisation is the same with and without it
    torch.manual_seed(5)
    x = (_net(0).state_dict()["model.blocks.0.attn.qkv.weight"], torch.rand(3))
    torch.manual_seed(5)
    y = (_net(64).state_dict()["model.blocks.0.attn.qkv.weight"], torch.rand(3))
    assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])


def test_deepcopy_carries_the_logvar():
    net = _net(32)
    with torch.no_grad():
        net.logvar_linear.weight.normal_()
        net.logvar_fourier.freqs.add_(1.0)   # as a checkpoint with other features would
    ema = copy.deepcopy(net)
    assert ema.logvar_channels == 32
    for k in LV:
        assert torch.equal(dict(ema.named_parameters())[k], dict(net.named_parameters())[k]), k


_REFERENCE_MODELS = {   # the `model:` sections of the reference's seven YAML files (train, finetune, test)
    "train/imagenet256-latent": dict(in_size=32, mask_ratio=0.5, mask_ratio_fn="constant"),
    "train/imagenet512-latent": dict(in_size=64, mask_ratio=0.5, mask_ratio_fn="constant"),
    "finetune/imagenet256-latent-const": dict(in_size=32, mask_ratio=0.0, mask_ratio_fn="constant"),
    "finetune/imagenet256-latent-cos": dict(in_size=32, mask_ratio=0.5, mask_ratio_fn="cos4"),
    "finetune/imagenet512-latent": dict(in_size=64, mask_ratio=0.0, mask_ratio_fn="constant"),
    "test/maskdit-256": dict(in_size=32, mask_ratio=0.5, cond_mask_ratio=0),
    "test/maskdit-512": dict(in_size=64, mask_ratio=0.5, cond_mask_ratio=0),
}


def _model_yaml(extra):
    m = dict(precond="edm", model_type="DiT-XL/2", in_channels=4, num_classes=1000, use_decoder=True,
             ext_feature_dim=0, pad_cls_token=False, mae_loss_coef=0.1, class_dropout_prob=0.1, **extra)
    return "model:\n" + "".join(f"  {k}: {v}\n" for k, v in m.items())


@pytest.mark.parametrize("name", sorted(_REFERENCE_MODELS))
def test_build_net_logvar_channels_default(name, monkeypatch):
    from maskdit_b200 import maskdit
    from maskdit_b200.config import build_net, load_config
    seen = {}
    monkeypatch.setitem(maskdit.Precond_models, "edm", lambda **kw: seen.update(kw) or kw)
    build_net(load_config(_model_yaml(_REFERENCE_MODELS[name])))
    assert seen["logvar_channels"] == 0 and seen["model_type"] == "DiT-XL/2"
    build_net(load_config(_model_yaml(dict(_REFERENCE_MODELS[name], logvar_channels=128))))
    assert seen["logvar_channels"] == 128


def test_eval_state_dict():
    off, on = _net(), _net(16)
    with torch.no_grad():
        on.logvar_linear.weight.fill_(0.5)
        for p in on.model.parameters():
            p.add_(0.25)
    sd = on.state_dict()
    compiled = {"_orig_mod." + k: v for k, v in sd.items()}
    for src in (sd, compiled):
        got = eval_state_dict(off, src)
        assert list(got) == list(off.state_dict())
        off.load_state_dict(got)                     # strict
        assert all(torch.equal(off.state_dict()[k], sd[k]) for k in got)
        kept = eval_state_dict(on, src)              # a net with the weighting keeps its tensors
        assert list(kept) == list(sd)
    # a checkpoint without the keys passes through unchanged
    plain = off.state_dict()
    assert list(eval_state_dict(off, plain)) == list(plain)


def test_log_and_val_lines():
    import train
    assert train.log_line(40, 0.123456, 2.5) == "(step=0000040) Train Loss: 0.1235, Train Steps/Sec: 2.50"
    assert train.log_line(40, 0.123456, 2.5, weighted=-1.23456) == \
        "(step=0000040) Train Loss: 0.1235, Train Steps/Sec: 2.50, Weighted Loss: -1.2346"
    assert train.log_line(40, 0.123456, 2.5, 0, (0.41237, 1.5), 0.5) == \
        "(step=0000040) Train Loss: 0.1235, Train Steps/Sec: 2.50, Skipped Steps: 0, Grad Norm: 0.4124 (max 1.5), " \
        "Weighted Loss: 0.5000"
    res = {"mean": 1.5, "per_level": [1.0, 2.0], "count": 3}
    assert train.val_line(12, res) == "(step=0000012) Val Loss: 1.50000 [1.00000 2.00000] (3 items, EMA)"
    assert train.val_line(12, res, [-0.5, 0.123456]) == \
        "(step=0000012) Val Loss: 1.50000 [1.00000 2.00000] (3 items, EMA), Logvar: [-0.5000 0.1235]"


def _normalised_sass(text):
    """{demangled function: [instruction lines]} with address comments removed and whitespace collapsed."""
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


def test_plain_loss_kernels_sass_unchanged():
    """The loss kernels without the weighting compile to the same SASS as before it was added."""
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "edm_loss_sass.json")))
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    nvcc, cuobjdump = os.path.join(cuda, "bin", "nvcc"), os.path.join(cuda, "bin", "cuobjdump")
    if not (os.path.exists(nvcc) and os.path.exists(cuobjdump) and shutil.which("c++filt")):
        pytest.skip("needs nvcc, cuobjdump and c++filt")
    ver = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout
    if gold["nvcc"] not in ver:
        pytest.skip(f"the fingerprints are of nvcc {gold['nvcc']}")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("the library is not built")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    fns = _normalised_sass(sass)
    for short, want in gold["functions"].items():
        hits = [v for k, v in fns.items() if k.startswith(f"void mdt::{short}(")]
        assert len(hits) == 1, (short, [k for k in fns if "edm_loss" in k])
        body = hits[0]
        assert len(body) == want["lines"], (short, len(body))
        assert hashlib.sha256("\n".join(body).encode()).hexdigest() == want["sha256"], short
    # the weighted instantiations exist next to them
    assert sum(k.startswith("void mdt::edm_loss_kernel<") and ", true>" in k for k in fns) == 2
