"""CPU tests of activation recomputation's host side (`mdt_model_set_recompute`): the training workspace plan at every
recompute count r, for every DiT_models geometry with and without the decoder, masked and unmasked, in both reduction
modes; the range check; and the automatic choice of r (`engine.pick_recompute`).  No device is needed: the model
handle and `mdt_workspace_bytes` launch nothing."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ERR_ARG = -1

# mdt_workspace_bytes before recomputation existed, at 32x32x4 latents, 1000 classes, B = 4:
# [training T = L/2, training T = L, the same two in the deterministic mode, inference T = L]
WS_PARENT = {
    ('DiT-H/2', True): [1059170560, 1924249856, 1059518720, 1924946176, 56867072],
    ('DiT-H/2', False): [881355008, 1744894208, 881703168, 1745590528, 40786176],
    ('DiT-H/4', True): [278922496, 495192320, 280253696, 496523520, 19499264],
    ('DiT-H/4', False): [233725184, 449634560, 235056384, 450965760, 15220992],
    ('DiT-H/8', True): [83877120, 137927936, 89140480, 143191296, 10157312],
    ('DiT-H/8', False): [71834368, 125819648, 77097728, 131083008, 8829696],
    ('DiT-XL/2', True): [875503872, 1559802112, 875817216, 1560428800, 52355328],
    ('DiT-XL/2', False): [697688320, 1380446464, 698001664, 1381073152, 36274432],
    ('DiT-XL/4', True): [230841600, 401916160, 232039680, 403114240, 17543424],
    ('DiT-XL/4', False): [185644288, 356358400, 186842368, 357556480, 13265152],
    ('DiT-XL/8', True): [69690624, 112444672, 74427648, 117181696, 8840448],
    ('DiT-XL/8', False): [57647872, 100336384, 62384896, 105073408, 7512832],
    ('DiT-L/2', True): [713054464, 1237543168, 713332992, 1238100224, 47941888],
    ('DiT-L/2', False): [535238912, 1058187520, 535517440, 1058744576, 31860992],
    ('DiT-L/4', True): [188249344, 319371520, 189314304, 320436480, 15685888],
    ('DiT-L/4', False): [143052032, 273813760, 144116992, 274878720, 11407616],
    ('DiT-L/8', True): [57060608, 89828608, 61271296, 94039296, 7621888],
    ('DiT-L/8', False): [45017856, 77720320, 49228544, 81931008, 6294272],
    ('DiT-B/2', True): [390547712, 592042240, 390756608, 592460032, 39115008],
    ('DiT-B/2', False): [209848576, 412686592, 210057472, 413104384, 23034112],
    ('DiT-B/4', True): [103662848, 154036480, 104461568, 154835200, 11970816],
    ('DiT-B/4', False): [57744640, 108478720, 58543360, 109277440, 7692544],
    ('DiT-B/8', True): [31948032, 44535040, 35106048, 47693056, 5184768],
    ('DiT-B/8', False): [19725056, 32426752, 22883072, 35584768, 3857152],
    ('DiT-S/2', True): [290025728, 388727040, 290130176, 388935936, 27644160],
    ('DiT-S/2', False): [105001216, 206487808, 105105664, 206696704, 11563264],
    ('DiT-S/4', True): [75910400, 100585728, 76309760, 100985088, 8167680],
    ('DiT-S/4', False): [28910848, 54307072, 29310208, 54706432, 3889408],
    ('DiT-S/8', True): [22387968, 28550400, 23966976, 30129408, 3298560],
    ('DiT-S/8', False): [9894656, 16261888, 11473664, 17840896, 1970944],
}
B = 4


@pytest.fixture
def lib():
    from maskdit_b200 import _lib
    L = _lib.lib()
    det = L.mdt_get_deterministic()
    yield L
    assert L.mdt_set_deterministic(det) == 0


def _engine(mt, dec):
    from maskdit_b200.engine import CEngine
    from maskdit_b200.maskdit import Precond_models
    with torch.device("meta"):
        net = Precond_models["edm"](32, 4, num_classes=1000, model_type=mt, use_decoder=dec, mae_loss_coef=0.1)
    return CEngine(net._cfg())


def _r256(n):
    return (n + 255) // 256 * 256


def _block_slices(M, d, heads, h4, tokens):
    """Bytes of one block's training slices in the plan's order: xm1 mean1 rstd1 qkv O lse X1 y1 xm2 mean2 rstd2 a hpre
    X2 y2."""
    return [M * d * 2, M * 4, M * 4, M * 3 * d * 2, M * d * 2, 2 * B * heads * tokens * 4, M * d * 4, M * d * 2,
            M * d * 2, M * 4, M * 4, M * h4 * 2, M * h4 * 2, M * d * 4, M * d * 2]


X2 = 13


def plan_total(c, NA, T, r):
    """The training workspace (default mode) from the slice rule: every slice rounded up to 256 bytes; a recomputed
    block keeps only X2; one recompute slot holds, per slice, the largest recomputed block's (no X2), plus a second
    mean1 / rstd1."""
    D, Dd, L, pd, has_dec = c.hidden, c.dec_hidden, c.num_patches, c.patch_dim, c.dec_hidden > 0
    Kp = -(-c.num_classes // 8) * 8
    Me, Md = B * T, B * L
    head = [Me * D * 4, B * 256 * 2, B * D * 4, B * D * 2, B * D * 4, B * D * 4, B * Kp * 2 + 16, B * Kp * 2 + 16,
            D * Kp * 2 + 16, B * D * 2, B * NA * 4]
    blocks = [_block_slices(Me, D, c.heads, c.mlp_hidden, T)] * c.depth + \
        [_block_slices(Md, Dd, c.dec_heads, c.dec_mlp_hidden, L)] * c.dec_depth
    n = sum(map(_r256, head))
    for g, s in enumerate(blocks):
        n += _r256(s[X2]) if g < r else sum(map(_r256, s))
    if has_dec:
        n += sum(map(_r256, [Me * D * 2, Me * 4, Me * 4, Me * Dd * 4, Md * Dd * 4]))
    Mf, Df = (Md, Dd) if has_dec else (Me, D)
    n += sum(map(_r256, [Mf * Df * 2, Mf * 4, Mf * 4] + ([] if has_dec else [Me * pd * 4])))
    if r:
        big = [max(col) for col in zip(*blocks[:r])]
        n += sum(_r256(v) for i, v in enumerate(big) if i != X2) + 2 * _r256(big[1])
    Md_ = max(Me * D, Md * Dd)
    Mh = max(Me * c.mlp_hidden, Md * c.dec_mlp_hidden)
    bwd = [B * NA * 4, Mf * Df * 2] + ([Md * Dd * 4] if has_dec else []) + \
        [Md_ * 2, Md_ * 2, Mh * 2, Md_ * 2, Md_ * 2, Md_ * 3 * 2] + ([Me * Dd * 2, Me * D * 2] if has_dec else []) + \
        [Me * D * 4, B * NA * 2, B * D * 4, B * D * 4, B * D * 2, B * D * 4, B * D * 4, B * D * 2, D * Kp * 4]
    return n + sum(map(_r256, bwd))


CASES = [(mt, dec, masked) for mt, dec in WS_PARENT for masked in (True, False)]


@pytest.mark.parametrize("mt,dec,masked", CASES)
def test_training_plan_follows_the_slice_rule(lib, mt, dec, masked):
    ce = _engine(mt, dec)
    c, nb = ce.cfg, ce.num_blocks
    T = c.num_patches // 2 if masked else c.num_patches
    parent = WS_PARENT[(mt, dec)]
    assert lib.mdt_set_deterministic(0) == 0
    sizes = [ce.workspace_bytes(B, T, True, r) for r in range(nb + 1)]
    assert sizes[0] == parent[0 if masked else 1]                   # r = 0: the plan of the parent revision
    assert sizes == [plan_total(c, ce.NA, T, r) for r in range(nb + 1)]
    assert sizes[nb] < sizes[0]
    # strictly decreasing in r while the slot does not grow: each further block that fits the slot gives back its slices
    enc = _block_slices(B * T, c.hidden, c.heads, c.mlp_hidden, T)
    dec_ = _block_slices(B * c.num_patches, c.dec_hidden, c.dec_heads, c.dec_mlp_hidden, c.num_patches)
    blocks = [enc] * c.depth + [dec_] * c.dec_depth
    for r in range(1, nb):
        slot = [max(col) for col in zip(*blocks[:r])]
        if all(v <= s for v, s in zip(blocks[r], slot)):
            assert sizes[r + 1] < sizes[r], (r, sizes)
    # the deterministic mode's scratch comes on top, the same at every r
    assert lib.mdt_set_deterministic(1) == 0
    det = [ce.workspace_bytes(B, T, True, r) for r in range(nb + 1)]
    assert det[0] == parent[2 if masked else 3]
    assert [d - s for d, s in zip(det, sizes)] == [det[0] - sizes[0]] * (nb + 1)


@pytest.mark.parametrize("mt,dec", list(WS_PARENT))
def test_inference_plan_ignores_the_count(lib, mt, dec):
    ce = _engine(mt, dec)
    assert lib.mdt_set_deterministic(0) == 0
    for r in (0, 1, ce.num_blocks):
        ce.set_recompute(r)
        assert ce.workspace_bytes(B, 0, False) == WS_PARENT[(mt, dec)][4]
        assert lib.mdt_model_get_recompute(ce._h) == r


def test_out_of_range_counts_are_refused(lib):
    ce = _engine("DiT-S/2", True)
    nb = ce.num_blocks
    assert nb == 12 + 8
    assert lib.mdt_model_get_recompute(ce._h) == 0                  # default
    assert lib.mdt_model_set_recompute(ce._h, nb) == 0
    for bad in (-1, nb + 1, 10 ** 6):
        assert lib.mdt_model_set_recompute(ce._h, bad) == ERR_ARG
        assert lib.mdt_model_get_recompute(ce._h) == nb             # unchanged
    assert lib.mdt_model_set_recompute(None, 0) == ERR_ARG and lib.mdt_model_get_recompute(None) == -1
    nd = _engine("DiT-S/2", False)
    assert nd.num_blocks == 12 and lib.mdt_model_set_recompute(nd._h, 13) == ERR_ARG
    # workspace_bytes at another count leaves the handle's count as it was
    ce.set_recompute(3)
    ce.workspace_bytes(B, 128, True, nb)
    assert lib.mdt_model_get_recompute(ce._h) == 3


def test_launch_count_includes_the_recomputed_forwards(lib):
    ce = _engine("DiT-XL/2", True)
    for masked in (True, False):
        f0, b0 = ce._count(masked)
        f, b = ce._count(masked, 5)
        assert f == f0 and b == b0 + 7 * 5


def test_pick_recompute():
    from maskdit_b200.engine import pick_recompute
    sizes = [100, 110, 80, 60, 70]      # r = 1 adds the slot; later counts can grow again where the slot does
    assert pick_recompute(sizes, 100) == 0
    assert pick_recompute(sizes, 10 ** 12) == 0
    assert pick_recompute(sizes, 99) == 2
    assert pick_recompute(sizes, 80) == 2
    assert pick_recompute(sizes, 75) == 3
    assert pick_recompute(sizes, 60) == 3
    with pytest.raises(torch.OutOfMemoryError, match=r"needs .* GiB even with 3 of 4 blocks recomputed"):
        pick_recompute(sizes, 59)
    GiB = 2 ** 30
    with pytest.raises(torch.OutOfMemoryError, match=r"needs 12\.50 GiB .* 3\.00 GiB of device memory is available"):
        pick_recompute([20 * GiB, 12.5 * GiB], 3 * GiB)


def test_automatic_choice_on_a_real_plan(lib):
    """DiT-XL/2 without the decoder at batch 256, no mask: the full plan is 87.9 GB; the automatic choice is the
    smallest count that fits a 70 GiB budget, and full recomputation fits in a fraction of it."""
    from maskdit_b200.engine import pick_recompute
    ce = _engine("DiT-XL/2", False)
    assert lib.mdt_set_deterministic(0) == 0
    sizes = [ce.workspace_bytes(256, 0, True, r) for r in range(ce.num_blocks + 1)]
    assert sizes[0] == 87913077504
    r = pick_recompute(sizes, 70 * 2 ** 30)
    assert 0 < r < ce.num_blocks and sizes[r] <= 70 * 2 ** 30 < sizes[r - 1]
    assert sizes[-1] < 20 * 2 ** 30
