"""CPU tests of the deterministic mode's host side (`mdt_set_deterministic`): the switch, the GEMM plans it selects
and the workspace it adds.  No device is needed: `mdt_gemm_plan` and `mdt_workspace_bytes` launch nothing."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.fixture
def lib():
    """The library with its deterministic setting, SM budget and torch's flag restored after the test."""
    from maskdit_b200 import _lib
    L = _lib.lib()
    det, budget, flag = L.mdt_get_deterministic(), L.mdt_get_sm_budget(), torch.are_deterministic_algorithms_enabled()
    yield L
    torch.use_deterministic_algorithms(flag)
    assert L.mdt_set_deterministic(det) == 0 and L.mdt_set_sm_budget(budget) == 0


def test_set_get_round_trip(lib):
    assert lib.mdt_set_deterministic(0) == 0 and lib.mdt_get_deterministic() == 0
    assert lib.mdt_set_deterministic(1) == 0 and lib.mdt_get_deterministic() == 1
    assert lib.mdt_set_deterministic(7) == 0 and lib.mdt_get_deterministic() == 1
    assert lib.mdt_set_deterministic(0) == 0 and lib.mdt_get_deterministic() == 0


def test_torch_flag_drives_the_setting(lib):
    from maskdit_b200 import _lib
    torch.use_deterministic_algorithms(True)
    assert _lib.sync_deterministic() is True and lib.mdt_get_deterministic() == 1
    torch.use_deterministic_algorithms(False)
    assert _lib.sync_deterministic() is False and lib.mdt_get_deterministic() == 0


# Every accumulating (MDT_EPI_ATOMIC) GEMM of one XL/2 ImageNet-256 training step at batch 256, mask 0.5:
# (M, N, K, a_mn, b_mn).  Encoder rows Me = 256 * 128, decoder rows Md = 256 * 256, modulation width NA = 221 440.
Me, Md, D, H4, Dd, H4d, NA, B = 32768, 65536, 1152, 4608, 512, 2048, 221440, 256
XL2_ACCUMULATING = (
    [(m, n, Me, True, True) for m, n in ((D, H4), (H4, D), (D, D), (3 * D, D))]             # encoder block wgrads
    + [(m, n, Md, True, True) for m, n in ((Dd, H4d), (H4d, Dd), (Dd, Dd), (3 * Dd, Dd))]   # decoder block wgrads
    + [(16, Dd, Md, True, True), (Dd, D, Me, True, True)]                                  # final / decoder layer
    + [(NA, D, B, True, True), (B, D, NA, False, True)]                                    # adaLN wgrad / dgrad
    + [(D, 1000, B, True, True), (D, D, B, True, True), (B, D, D, False, True), (D, 256, B, True, True)]
)


def _plans():
    from maskdit_b200 import _lib
    return [_lib.gemm_plan(M, N, K, a_mn=am, b_mn=bm, epi=_lib.EPI_ATOMIC) for M, N, K, am, bm in XL2_ACCUMULATING]


def test_accumulating_gemm_plans_do_not_depend_on_the_sm_budget(lib):
    """With the setting on, each accumulating GEMM of the XL/2 step runs one k-slice under every SM budget (only the
    grid follows the budget); turning the setting off restores every default plan exactly."""
    assert lib.mdt_set_sm_budget(0) == 0 and lib.mdt_set_deterministic(0) == 0
    before = {b: (lib.mdt_set_sm_budget(b), _plans())[1] for b in (0, 7, 66, 114)}
    assert any(p["splits"] > 1 for p in before[0])          # the default mode does split these
    assert lib.mdt_set_deterministic(1) == 0
    det = {}
    for b in (0, 7, 66, 114):
        assert lib.mdt_set_sm_budget(b) == 0
        det[b] = _plans()
        for p, shape in zip(det[b], XL2_ACCUMULATING):
            assert p["splits"] == 1, (b, shape, p)
            assert p["units"] == p["num_m_tiles"] * p["num_n_tiles"], (b, shape, p)
            if b:
                assert p["grid"] == min(p["units"], b), (b, shape, p)
    keys = ("block_n", "splits", "pair_halves", "narrow_last", "num_m_tiles", "num_n_tiles", "num_kb", "units")
    for b in (7, 66, 114):
        assert [{k: p[k] for k in keys} for p in det[b]] == [{k: p[k] for k in keys} for p in det[0]], b
    assert lib.mdt_set_deterministic(0) == 0
    for b in (0, 7, 66, 114):
        assert lib.mdt_set_sm_budget(b) == 0
        assert _plans() == before[b], b


def test_non_accumulating_gemm_plans_are_unchanged(lib):
    from maskdit_b200 import _lib
    shapes = [((Me, 3 * D, D), {}), ((Me, H4, D), {"b_mn": True, "epi": _lib.EPI_DGELU}),
              ((Me, D, H4), {"epi": _lib.EPI_GATE_RESID}), ((Md, 3 * Dd, Dd), {})]
    assert lib.mdt_set_deterministic(0) == 0
    off = [_lib.gemm_plan(*s, **kw) for s, kw in shapes]
    assert lib.mdt_set_deterministic(1) == 0
    assert [_lib.gemm_plan(*s, **kw) for s, kw in shapes] == off


def test_entry_points_without_scratch_refuse_under_the_setting(lib):
    """Per-kernel entry points whose deterministic variant needs per-block scratch they have no argument for return
    MDT_ERR_UNSUPPORTED instead of reducing in a scheduling-dependent order.  They refuse before any launch, so
    16-byte aligned dummy pointers suffice."""
    UNSUPPORTED = -5
    p = [(i + 1) << 20 for i in range(12)]
    assert lib.mdt_set_deterministic(1) == 0
    # patch-embedding backward: per-block partials of gW / gb
    assert lib.mdt_patch_embed_bwd(p[0], p[1], 0.5, None, p[2], p[3], p[4], 2, 4, 8, 2, 384, 16, None) == UNSUPPORTED
    # gate backward with a bias gradient (a sum over samples)
    assert lib.mdt_gate_bwd(p[0], p[1], p[2], 2304, 16, p[3], p[4], 2304, p[5], 32, 384, None) == UNSUPPORTED
    # fused LN / gate backward with a bias gradient
    assert lib.mdt_ln_modulate_bwd_gate(p[0], p[1], p[2], p[3], p[4], 2304, 16, p[5], 1, p[6], p[7], 2304, p[8], p[9],
                                        2304, p[10], p[11], 2304, p[1] + 4096, 32, 384, None) == UNSUPPORTED
    # mask-token gradient of the unmask backward
    assert lib.mdt_unmask_tokens_bwd(p[0], None, p[1], p[2], p[3], 2, 8, 16, 512, None) == UNSUPPORTED


# mdt_workspace_bytes of the parent revision (before the deterministic mode existed): (B, T, training) -> bytes
WS_DEFAULT = {
    ("DiT-XL/2", True): [55596751616, 99391838976, 1744094976, 52355328],
    ("DiT-XL/2", False): [44216556288, 87913077504, 1388463872, 36274432],
    ("DiT-S/2", True): [1283953408, 1678758656, 40160000, 2526976],
}


@pytest.mark.parametrize("mt,dec", list(WS_DEFAULT))
def test_workspace_bytes_unchanged_with_the_setting_off(lib, mt, dec):
    """Off: exactly the previous workspace sizes.  On: the training workspace grows by the scratch appended after
    every activation; the inference workspace does not change."""
    from maskdit_b200.engine import CEngine
    from maskdit_b200.maskdit import Precond_models
    R, ncls = (32, 1000) if mt == "DiT-XL/2" else (8, 10)
    with torch.device("meta"):
        net = Precond_models["edm"](R, 4, num_classes=ncls, model_type=mt, use_decoder=dec, mae_loss_coef=0.1)
    ce = CEngine(net._cfg())
    L = (R // 2) ** 2
    args = ((256, L // 2, 1), (256, 0, 1), (8, L // 2, 1), (4, 0, 0))
    assert lib.mdt_set_deterministic(0) == 0
    assert [ce.workspace_bytes(*a) for a in args] == WS_DEFAULT[(mt, dec)]
    assert lib.mdt_set_deterministic(1) == 0
    on = [ce.workspace_bytes(*a) for a in args]
    for a, o, d in zip(args, on, WS_DEFAULT[(mt, dec)]):
        assert (o > d) if a[2] else (o == d), (a, o, d)
    assert lib.mdt_set_deterministic(0) == 0
    assert [ce.workspace_bytes(*a) for a in args] == WS_DEFAULT[(mt, dec)]
