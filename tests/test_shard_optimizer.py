"""CPU: the sharded optimizer's ownership map (`owned_ranges`), its padded exchange layout, the driver's fp32-read set,
the C entry points' argument checks, the refusals and train.py's switch."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MDT_ERR_ARG = -1
NEW = ("mdt_reduce_scatter_grads", "mdt_allgather", "mdt_model_fp32_read_ranges", "mdt_copy_segments_f32")
A = 1 << 20   # a 256-byte aligned dummy address: the argument checks never dereference it
XL2_N = 730_115_216   # trainable elements of MaskDiT-XL/2 (test_host.py)


def layout(mt, dec=True, logvar=0):
    from maskdit_b200.maskdit import Precond_models
    with torch.device("meta"):
        net = Precond_models["edm"](32, 4, num_classes=1000, model_type=mt, use_decoder=dec, mae_loss_coef=0.1,
                                    logvar_channels=logvar)
    return net._layout()


def sizes():
    _, s2 = layout("DiT-S/2")
    _, xl = layout("DiT-XL/2")
    return [1, 63, 64, 65, 1000, 4095, 4096, 4097, 123_457, 1 << 20, (1 << 20) + 64, s2.n_train, xl.n_train]


@pytest.fixture(scope="module")
def L():
    from maskdit_b200 import _lib
    return _lib.lib()


def test_symbols_exported_and_abi_unchanged(L):
    from maskdit_b200 import _lib
    for name in NEW:
        assert name in _lib.exported_symbols() and hasattr(L, name), name
    assert L.mdt_abi_version() == 2


@pytest.mark.parametrize("n", sizes())
def test_owned_ranges_partition_the_region(n):
    """Disjoint, covering [0, n), 64-aligned starts, and per chunk one equal count for every rank."""
    from maskdit_b200.train_step import ar_chunk_bounds, owned_ranges, shard_piece
    for world in (1, 2, 3, 4, 5, 8, 16):
        for chunks in (1, 2, 4, 7):
            own = owned_ranges(n, world, chunks)
            bounds = ar_chunk_bounds(n, chunks)
            assert len(own) == world and all(len(o) == len(bounds) for o in own)
            got = sorted((a, b) for o in own for a, b in o if b > a)
            assert got[0][0] == 0 and got[-1][1] == n
            for (a0, b0), (a1, b1) in zip(got, got[1:]):
                assert b0 == a1   # disjoint and no gap
            for k, (lo, hi) in enumerate(bounds):
                p = shard_piece(hi - lo, world)
                assert p % 64 == 0 and world * p >= hi - lo and world * (p - 64) < hi - lo
                for r in range(world):
                    a, b = own[r][k]
                    assert lo <= a <= b <= hi
                    assert a == min(hi, lo + r * p) and b - a == min(p, max(0, hi - lo - r * p))
                    assert a % 64 == 0 or a == hi   # piece starts are aligned (chunk starts are 4 KiB aligned)


def test_padded_tail():
    """A chunk that world pieces of 64-multiples do not fill: the last ranks' pieces are shorter or empty, and the
    exchange slot is padded to world equal counts."""
    from maskdit_b200.train_step import owned_ranges, shard_piece
    own = owned_ranges(1000, 4, 1)
    assert shard_piece(1000, 4) == 256
    assert [o[0] for o in own] == [(0, 256), (256, 512), (512, 768), (768, 1000)]
    own = owned_ranges(130, 4, 1)   # 64 each: the fourth rank owns nothing, the third 2 elements
    assert [o[0] for o in own] == [(0, 64), (64, 128), (128, 130), (130, 130)]
    assert owned_ranges(5, 8, 3) == [[(0, 5)]] + [[(5, 5)]] * 7   # below 1024 per chunk: one chunk
    # XL/2 as 8 ranks x 4 chunks: the first three chunks divide evenly, the last pads 8 * 64 - 1 elements at most
    from maskdit_b200.train_step import ar_chunk_bounds
    b = ar_chunk_bounds(XL2_N, 4)
    pads = [8 * shard_piece(hi - lo, 8) - (hi - lo) for lo, hi in b]
    assert pads[:3] == [0, 0, 0] and 0 <= pads[3] < 8 * 64


def test_owned_ranges_argument_errors():
    from maskdit_b200.train_step import owned_ranges
    for bad in ((0, 2, 4), (10, 0, 4), (10, 2, 0), (-5, 2, 4), (10.0, 2, 4), (10, 2.5, 4), (10, True, 4),
                (10, 2, None)):
        with pytest.raises(ValueError):
            owned_ranges(*bad)


@pytest.mark.parametrize("mt,dec,logvar", [("DiT-XL/2", True, 0), ("DiT-XL/2", False, 0), ("DiT-S/2", True, 8)])
def test_fp32_read_set(mt, dec, logvar):
    """The driver's fp32-read set: sorted, disjoint, inside the trainable region, made of whole tensors, and exactly
    the biases, the patch embedder, the mask token and the weighting's w.  A few MB for XL/2."""
    eng, st = layout(mt, dec, logvar)
    read = eng.fp32_read_ranges()
    assert read and all(a < b for a, b in read)
    for (a0, b0), (a1, b1) in zip(read, read[1:]):
        assert b0 < a1
    assert read[-1][1] <= st.n_train
    inside = lambda o, n: any(a <= o and o + n <= b for a, b in read)   # noqa: E731
    want = {k for k in st.offsets if k.endswith(".bias") or k.startswith("model.x_embedder")
            or k in ("model.mask_token", "logvar_linear.weight")}
    for k, (o, n, _) in st.offsets.items():
        if o >= st.n_train:
            continue
        assert inside(o, n) == (k in want), k
    total = sum(b - a for a, b in read)
    if mt == "DiT-XL/2":
        assert total * 4 < 8e6, total   # a few MB against 2.92 GB of masters


def test_fp32_read_ranges_arguments(L):
    assert L.mdt_model_fp32_read_ranges(None, None, 0) == MDT_ERR_ARG
    eng, _ = layout("DiT-S/2")
    assert L.mdt_model_fp32_read_ranges(eng._h, None, -1) == MDT_ERR_ARG
    assert L.mdt_model_fp32_read_ranges(eng._h, None, 4) == MDT_ERR_ARG
    assert L.mdt_model_fp32_read_ranges(eng._h, None, 0) == len(eng.fp32_read_ranges())


def test_collective_and_copy_argument_errors(L):
    for bf in (0, 1):
        assert L.mdt_reduce_scatter_grads(None, A, 64, bf, None) == MDT_ERR_ARG
        assert L.mdt_reduce_scatter_grads(A, None, 64, bf, None) == MDT_ERR_ARG
        assert L.mdt_reduce_scatter_grads(A, A, 0, bf, None) == MDT_ERR_ARG
    for dt in (0, 1, 2):
        assert L.mdt_allgather(None, A, 64, dt, None) == MDT_ERR_ARG
        assert L.mdt_allgather(A, A, -1, dt, None) == MDT_ERR_ARG
    assert L.mdt_allgather(A, A, 64, 3, None) == MDT_ERR_ARG
    assert L.mdt_copy_segments_f32(A, A, A, -1, None) == MDT_ERR_ARG
    assert L.mdt_copy_segments_f32(None, A, A, 1, None) == MDT_ERR_ARG
    assert L.mdt_copy_segments_f32(A, A, A, 1 << 16, None) == MDT_ERR_ARG
    assert L.mdt_copy_segments_f32(None, None, None, 0, None) == 0   # nothing to copy


def test_train_py_flag():
    import train
    ap = train.build_parser()
    parse = lambda *a: ap.parse_known_args(["--config", "c.yaml", *a])[0]   # noqa: E731
    assert parse().shard_optimizer is False
    assert parse("--shard_optimizer").shard_optimizer is True


def test_unsharded_step_has_no_layout():
    from maskdit_b200.train_step import TrainStep
    ts = TrainStep.__new__(TrainStep)
    assert not ts.sharded
    ts.materialize()   # nothing to gather
