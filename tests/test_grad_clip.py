"""CPU: gradient-norm clipping's C ABI entries and argument checks, the bound's validation, train.py's switch and its
log line."""
import math
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MDT_ERR_ARG = -1
NEW = ("mdt_grad_sumsq_scratch", "mdt_grad_sumsq", "mdt_grad_clip_coef", "mdt_adamw_ema_coef", "mdt_adamw_ema_coef_g16",
       "mdt_adamw_ema_guarded_coef", "mdt_adamw_ema_guarded_coef_g16")
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


def test_sumsq_scratch_depends_on_n_only(L):
    """One slot per block of the norm pass's grid: 4 elements per thread, 256 threads, at most 16 blocks per SM of a
    132-SM H100."""
    assert L.mdt_grad_sumsq_scratch(0) == MDT_ERR_ARG and L.mdt_grad_sumsq_scratch(-4) == MDT_ERR_ARG
    assert L.mdt_grad_sumsq_scratch(1) == 1 and L.mdt_grad_sumsq_scratch(1024) == 1
    assert L.mdt_grad_sumsq_scratch(1027) == 1 and L.mdt_grad_sumsq_scratch(1028) == 2   # a 3-element tail: no block
    assert L.mdt_grad_sumsq_scratch(1_000_003) == 977
    assert L.mdt_grad_sumsq_scratch(730_115_216) == 132 * 16
    counts = [L.mdt_grad_sumsq_scratch(n) for n in (5, 4099, 10 ** 6, 10 ** 7, 10 ** 9)]
    assert counts == sorted(counts)   # a buffer sized for the whole gradient serves every chunk of it


def test_sumsq_rejects_bad_arguments(L):
    def call(g=A, n=64, bf16=0, scratch=A, out=A, flag=0):
        return L.mdt_grad_sumsq(g, n, bf16, scratch, out, flag, None)

    for bad in (dict(g=None), dict(scratch=None), dict(out=None), dict(n=0), dict(n=-1), dict(g=A + 8),
                dict(g=A + 4, bf16=1), dict(scratch=A + 4), dict(out=A + 4), dict(flag=A + 2)):
        assert call(**bad) == MDT_ERR_ARG, bad


def test_clip_coef_rejects_bad_arguments(L):
    def call(sumsq=A, k=1, gs=0.5, c=1.0, norm=A, coef=A + 4, flag=0):
        return L.mdt_grad_clip_coef(sumsq, k, gs, c, norm, coef, flag, None)

    for bad in (dict(sumsq=None), dict(norm=None), dict(coef=None), dict(k=0), dict(k=-2), dict(gs=0.0),
                dict(gs=-1.0), dict(gs=math.nan), dict(c=0.0), dict(c=-1.0), dict(c=math.nan), dict(c=-math.inf),
                dict(sumsq=A + 4), dict(norm=A + 2), dict(coef=A + 1), dict(flag=A + 2)):
        assert call(**bad) == MDT_ERR_ARG, bad


@pytest.mark.parametrize("name", ["mdt_adamw_ema_coef", "mdt_adamw_ema_coef_g16"])
def test_coef_adamw_rejects_bad_arguments(L, name):
    fn = getattr(L, name)

    def call(w=A, g=A, m=A, v=A, ema=A, w16=A, n=64, step=1, coef=A):
        return fn(w, g, m, v, ema, w16, n, 1e-4, 0.9, 0.999, 1e-8, 0.0, step, 0.9999, 1.0, coef, 0, None)

    for bad in (dict(coef=None), dict(coef=A + 2), dict(w=None), dict(n=66), dict(step=0), dict(m=A + 4),
                dict(w16=A + 2)):
        assert call(**bad) == MDT_ERR_ARG, bad


@pytest.mark.parametrize("name", ["mdt_adamw_ema_guarded_coef", "mdt_adamw_ema_guarded_coef_g16"])
def test_guarded_coef_adamw_rejects_bad_arguments(L, name):
    fn = getattr(L, name)

    def call(w=A, g=A, m=A, v=A, ema=A, w16=A, n=64, coef=A, flag=A, counts=A):
        return fn(w, g, m, v, ema, w16, n, 1e-4, 0.9, 0.999, 1e-8, 0.0, 0.9999, 1.0, coef, flag, counts, 0, None)

    for bad in (dict(coef=None), dict(coef=A + 1), dict(flag=None), dict(counts=None), dict(counts=A + 4),
                dict(n=0), dict(v=A + 8)):
        assert call(**bad) == MDT_ERR_ARG, bad


def test_bound_validation():
    from maskdit_b200.train_step import check_max_grad_norm
    assert check_max_grad_norm(None) is None
    assert check_max_grad_norm(1) == 1.0 and check_max_grad_norm("0.5") == 0.5
    assert check_max_grad_norm(float("inf")) == math.inf and check_max_grad_norm("inf") == math.inf
    assert check_max_grad_norm(1e-30) == 1e-30
    for bad in (0, 0.0, -0.0, -1.0, float("nan"), "nan", -math.inf):
        with pytest.raises(ValueError):
            check_max_grad_norm(bad)


def test_train_py_flag():
    import train
    ap = train.build_parser()
    parse = lambda *a: ap.parse_known_args(["--config", "c.yaml", *a])[0]   # noqa: E731
    assert parse().max_grad_norm is None
    assert parse("--max_grad_norm", "1.0").max_grad_norm == 1.0
    assert parse("--max_grad_norm", "inf").max_grad_norm == math.inf
    for bad in ("0", "-1", "nan"):
        with pytest.raises(SystemExit):
            parse("--max_grad_norm", bad)


def test_log_line_without_the_flag_is_unchanged():
    """The reference's format (train.py:247), then the guard's count; the norm only when measured."""
    import train
    assert train.log_line(40, 0.123456, 2.5) == "(step=0000040) Train Loss: 0.1235, Train Steps/Sec: 2.50"
    assert train.log_line(40, 0.123456, 2.5, 3) == \
        "(step=0000040) Train Loss: 0.1235, Train Steps/Sec: 2.50, Skipped Steps: 3"
    assert train.log_line(40, 0.123456, 2.5, 0, (0.41237, 1.5)) == \
        "(step=0000040) Train Loss: 0.1235, Train Steps/Sec: 2.50, Skipped Steps: 0, Grad Norm: 0.4124 (max 1.5)"


def test_grad_norm_is_none_when_off():
    from maskdit_b200.train_step import TrainStep
    ts = TrainStep.__new__(TrainStep)
    ts.max_grad_norm = None
    assert ts.grad_norm is None and not ts._clips()
    ts.max_grad_norm = math.inf
    assert not ts._clips()
    ts.max_grad_norm = 1.0
    assert ts._clips()
