"""CPU: the non-finite gradient guard's C ABI argument checks, train.py's switch and the host step bookkeeping."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MDT_ERR_ARG = -1
NEW = ("mdt_nonfinite_check", "mdt_cast_f32_bf16_check", "mdt_adamw_ema_guarded", "mdt_adamw_ema_guarded_g16",
       "mdt_optim_guard_advance")
A = 1 << 20   # a 256-byte aligned dummy address: the argument checks never dereference it


@pytest.fixture(scope="module")
def L():
    from maskdit_b200 import _lib
    return _lib.lib()


def test_symbols_exported_and_abi_unchanged(L):
    from maskdit_b200 import _lib
    for name in NEW:
        assert name in _lib.exported_symbols() and hasattr(L, name), name
    assert L.mdt_abi_version() == 2


def test_check_entries_reject_bad_arguments(L):
    assert L.mdt_nonfinite_check(None, 4, A, None) == MDT_ERR_ARG
    assert L.mdt_nonfinite_check(A, 4, None, None) == MDT_ERR_ARG
    assert L.mdt_nonfinite_check(A, 0, A, None) == MDT_ERR_ARG
    assert L.mdt_nonfinite_check(A, -3, A, None) == MDT_ERR_ARG
    assert L.mdt_nonfinite_check(A + 4, 4, A, None) == MDT_ERR_ARG        # not 16-byte aligned
    assert L.mdt_cast_f32_bf16_check(None, A, 4, A, None) == MDT_ERR_ARG
    assert L.mdt_cast_f32_bf16_check(A, None, 4, A, None) == MDT_ERR_ARG
    assert L.mdt_cast_f32_bf16_check(A, A, 4, None, None) == MDT_ERR_ARG
    assert L.mdt_cast_f32_bf16_check(A, A, 0, A, None) == MDT_ERR_ARG
    assert L.mdt_cast_f32_bf16_check(A + 8, A, 4, A, None) == MDT_ERR_ARG
    assert L.mdt_cast_f32_bf16_check(A, A + 2, 4, A, None) == MDT_ERR_ARG
    assert L.mdt_optim_guard_advance(None, A, None) == MDT_ERR_ARG
    assert L.mdt_optim_guard_advance(A, None, None) == MDT_ERR_ARG
    assert L.mdt_optim_guard_advance(A, A + 4, None) == MDT_ERR_ARG         # counts: int64, 8-byte aligned


@pytest.mark.parametrize("name", ["mdt_adamw_ema_guarded", "mdt_adamw_ema_guarded_g16"])
def test_guarded_adamw_rejects_bad_arguments(L, name):
    fn = getattr(L, name)

    def call(w=A, g=A, m=A, v=A, ema=A, w16=A, n=64, flag=A, counts=A, max_blocks=0):
        return fn(w, g, m, v, ema, w16, n, 1e-4, 0.9, 0.999, 1e-8, 0.0, 0.9999, 1.0, flag, counts, max_blocks, None)

    for bad in (dict(w=None), dict(g=None), dict(m=None), dict(v=None), dict(flag=None), dict(counts=None),
                dict(n=0), dict(n=-4), dict(n=66), dict(w=A + 8), dict(m=A + 4), dict(v=A + 8), dict(ema=A + 8),
                dict(w16=A + 2), dict(counts=A + 4), dict(flag=A + 2)):
        assert call(**bad) == MDT_ERR_ARG, bad
    if name.endswith("g16"):
        assert call(g=A + 2) == MDT_ERR_ARG      # a bf16 gradient needs 8-byte alignment only
    else:
        assert call(g=A + 8) == MDT_ERR_ARG


def test_train_py_maps_no_amp_to_the_guard():
    import train
    ap = train.build_parser()
    assert train.skip_nonfinite(ap.parse_known_args(["--config", "c.yaml"])[0]) is True
    assert train.skip_nonfinite(ap.parse_known_args(["--config", "c.yaml", "--no_amp"])[0]) is False


class _Net:
    """Two parameters, the first frozen (as pos_embed): optimizer state is keyed by position in parameters()."""

    def __init__(self):
        self.p = [("pos", torch.nn.Parameter(torch.zeros(2), requires_grad=False)),
                  ("w", torch.nn.Parameter(torch.zeros(2, 4)))]

    def named_parameters(self):
        return iter(self.p)


def _host_step(skip_nonfinite):
    """A TrainStep with host tensors in place of its device buffers: the bookkeeping only, no launch."""
    from types import SimpleNamespace

    from maskdit_b200.train_step import TrainStep
    ts = TrainStep.__new__(TrainStep)
    ts.net = _Net()
    ts.st = SimpleNamespace(offsets={"w": (0, 8, (2, 4))})
    ts.m, ts.v = torch.arange(8.0), torch.arange(8.0) + 1
    ts.lr, ts.betas, ts.eps, ts.wd = 1e-4, (0.9, 0.999), 1e-8, 0.0
    ts.step_count, ts.lr_step_offset = 0, 0
    ts.skip_nonfinite = skip_nonfinite
    ts._flag = torch.zeros(1) if skip_nonfinite else None
    ts._counts = torch.zeros(2, dtype=torch.int64) if skip_nonfinite else None
    return ts


def test_step_bookkeeping_across_a_skip_and_a_resume():
    """Four attempted steps, one skipped: the lr schedule has advanced four times, Adam three.  The checkpoint stores
    Adam's count; after a resume at run step 4, lr continues from 4 (lr_step_offset, as train.py sets it) and Adam from
    3 (the device counter)."""
    from maskdit_b200.train_step import lr_at
    ts = _host_step(True)
    ts.step_count = 4                       # what four calls of step() leave, whatever the flags
    ts._counts[0], ts._counts[1] = 3, 1     # what the device counters hold after one skip
    assert ts.applied_steps() == 3 and int(ts.skipped_steps) == 1
    sd = ts.state_dict()
    assert sd["param_groups"][0]["step"] == 3 and float(sd["state"][1]["step"]) == 3.0 and 0 not in sd["state"]
    ts2 = _host_step(True)
    ts2.load_state_dict(sd)
    assert ts2.step_count == 3 and ts2._counts.tolist() == [3, 0] and torch.equal(ts2.m, ts.m)
    run_step = 4
    ts2.lr_step_offset = run_step - ts2.step_count
    # the next step's lr is the one the uninterrupted run uses for its fifth step; its Adam step is counts[0] + 1 = 4
    for gb, ramp in ((256, 0.5), (256, 0.0), (8, 1.0)):
        assert lr_at(ts2.step_count + ts2.lr_step_offset, 1e-4, gb, ramp) == lr_at(run_step, 1e-4, gb, ramp)
    # without the guard the step count is Adam's, as before
    ts3 = _host_step(False)
    ts3.step_count = 4
    assert ts3.applied_steps() == 4 and ts3.skipped_steps is None
    assert ts3.state_dict()["param_groups"][0]["step"] == 4
    ts4 = _host_step(False)
    ts4.load_state_dict(sd)
    assert ts4.step_count == 3
