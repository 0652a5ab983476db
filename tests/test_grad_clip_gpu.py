"""GPU: gradient-norm clipping (`TrainStep(max_grad_norm=)`, torch.nn.utils.clip_grad_norm_ on the device).

1. The norm pass (`mdt_grad_sumsq` + `mdt_grad_clip_coef`) against float64 torch: fp32 and bf16 buffers, scalar tails,
   all-reduce chunk slices, the XL/2 gradient size, magnitudes whose fp32 squares overflow; bit-repeatable under any SM
   budget and in both modes; its fused non-finite check.
2. The AdamW entries that read the coefficient: bit-identical to the plain ones at coef 1, float64 AdamW at coef < 1.
3. The world-1 step: c = inf and a bound above the norm change nothing; a bound below it equals torch's AdamW after
   clip_grad_norm_; grad_accum; the guard; no host synchronisation in the added calls.
4. Rank 0 of two emulated ranks: the norm of the summed exchange buffer, and every chunk's pass using the final
   coefficient.
5. train.py end to end.
"""
import copy
import ctypes
import gc
import math
import os
import re
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

bf16 = torch.bfloat16
NAN, INF = float("nan"), float("inf")
XL2_TRAINABLE = 730_115_216   # DiT-XL/2 with the decoder: elements of the flat gradient


@pytest.fixture(scope="module")
def ops():
    from maskdit_b200 import ops as o
    return o


@pytest.fixture
def det():
    """Deterministic mode on for the test; the torch flag and the SM budget are restored afterwards."""
    from maskdit_b200 import _lib
    flag = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(flag)
    _lib.sync_deterministic()
    assert _lib.lib().mdt_set_sm_budget(0) == 0


def _ulp32(x64):
    a = torch.as_tensor(x64, dtype=torch.float64).abs().float()
    return (torch.nextafter(a, torch.full_like(a, INF)) - a).double()


def _norm(ops, g, grad_scale=1.0, flag=None):
    """(norm, sum of squares) of g through the two new entries; c = inf, so coef must be 1."""
    scratch = ops.grad_sumsq_scratch(g.numel(), g.device)
    s = torch.zeros(1, dtype=torch.float64, device=g.device)
    out = torch.zeros(2, device=g.device)
    ops.grad_sumsq(g, s, scratch, flag=flag)
    ops.grad_clip_coef(s, grad_scale, INF, out[:1], out[1:])
    assert out[1].item() == 1.0
    return out[0], s


def _ref_norm(g, step=1 << 26):
    """float64 norm of g, in slices so that a 730 M-element buffer needs no 5.8 GB float64 copy."""
    acc = 0.0
    for lo in range(0, g.numel(), step):
        acc += float(torch.linalg.vector_norm(g[lo:lo + step].double()) ** 2)
    return math.sqrt(acc)


def _assert_norm(got, ref, what):
    err = abs(got.double().item() - ref)
    assert err <= _ulp32(ref).item(), (what, got.item(), ref, err / _ulp32(ref).item())


def _values(n, seed, lo=-2.0, hi=2.0):
    """sign * 10**u, u uniform in [lo, hi)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    e = torch.rand(n, device="cuda", generator=g) * (hi - lo) + lo
    s = torch.randint(0, 2, (n,), device="cuda", generator=g).float() * 2 - 1
    return s * torch.pow(10.0, e)


# ---- 1. the norm pass ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, bf16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("n", [4, 1020, 1_000_003])
def test_norm_vs_float64(ops, dtype, n):
    for seed, (lo, hi) in enumerate([(-2, 2), (-30, 30), (15, 30), (-30, -20)]):
        g = _values(n, seed, lo, hi).to(dtype)
        assert torch.isfinite(g).all()
        got, _ = _norm(ops, g)
        _assert_norm(got, _ref_norm(g), (dtype, n, lo, hi))
        gs = 1 / 6   # the norm of the averaged gradient: 3 ranks x grad_accum 2
        got, _ = _norm(ops, g, grad_scale=gs)
        _assert_norm(got, _ref_norm(g) * gs, (dtype, n, "scaled"))


@pytest.mark.parametrize("dtype", [torch.float32, bf16], ids=["fp32", "bf16"])
def test_norm_of_chunk_slices(ops, dtype):
    """The exchange chunks of TrainStep (4 KiB aligned starts, a ragged last chunk): each slice's sum of squares, and the
    slots summed by the coefficient kernel give the whole buffer's norm."""
    from maskdit_b200.train_step import ar_chunk_bounds
    n = 4 * 1024 * 3 + 4099
    g = _values(n, 7, -20, 20).to(dtype)
    bounds = ar_chunk_bounds(n, 4)
    assert len(bounds) == 4 and (bounds[-1][1] - bounds[-1][0]) % 4
    scratch = ops.grad_sumsq_scratch(n, "cuda")
    slots = torch.zeros(len(bounds), dtype=torch.float64, device="cuda")
    for k, (lo, hi) in enumerate(bounds):
        ops.grad_sumsq(g[lo:hi], slots[k:k + 1], scratch)   # one scratch for every call on the stream
        got, _ = _norm(ops, g[lo:hi])
        _assert_norm(got, _ref_norm(g[lo:hi]), (dtype, lo, hi))
    out = torch.zeros(2, device="cuda")
    ops.grad_clip_coef(slots, 0.25, INF, out[:1], out[1:])
    _assert_norm(out[0], _ref_norm(g) * 0.25, (dtype, "all chunks"))


@pytest.mark.parametrize("dtype", [torch.float32, bf16], ids=["fp32", "bf16"])
def test_norm_at_xl2_size(ops, dtype):
    g = _values(XL2_TRAINABLE, 3, -3, 1).to(dtype)
    got, _ = _norm(ops, g)
    _assert_norm(got, _ref_norm(g), (dtype, "XL/2"))
    del g
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dtype", [torch.float32, bf16], ids=["fp32", "bf16"])
def test_norm_repeats_bit_for_bit(ops, dtype):
    """Same bits on repeated calls, with 32 SMs budgeted and with the whole device, deterministic mode on and off."""
    from maskdit_b200 import _lib
    L = ops.lib()
    g = _values(5_000_003, 11, -10, 10).to(dtype)
    seen = set()
    try:
        for deterministic in (False, True):
            assert L.mdt_set_deterministic(int(deterministic)) == 0
            for budget in (0, 32, 0):
                assert L.mdt_set_sm_budget(budget) == 0
                for _ in range(3):
                    _, s = _norm(ops, g)
                    seen.add(s.item().hex())
    finally:
        assert L.mdt_set_sm_budget(0) == 0
        _lib.sync_deterministic()
    assert len(seen) == 1, seen


@pytest.mark.parametrize("dtype", [torch.float32, bf16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("n", [4, 1_000_003])
def test_nonfinite_element_sets_flag_and_norm(ops, dtype, n):
    g = _values(n, 5).to(dtype)
    for pos in sorted({0, n // 2, n - 1}):
        for val in (NAN, INF, -INF):
            keep = g[pos].clone()
            g[pos] = val
            flag = torch.zeros(1, device="cuda")
            got, _ = _norm(ops, g, flag=flag)
            assert flag.item() == 1.0 and not math.isfinite(got.item()), (n, pos, val)
            g[pos] = keep
    flag = torch.zeros(1, device="cuda")
    got, _ = _norm(ops, g, flag=flag)
    assert flag.item() == 0.0 and math.isfinite(got.item())
    flag.fill_(1.0)   # the check only ever sets the flag
    _norm(ops, g, flag=flag)
    assert flag.item() == 1.0


def test_coefficient_formula_and_overflowing_norm(ops):
    """coef is torch's clamp(reciprocal(norm + 1e-6) * c, max=1) bit for bit; a norm beyond fp32 from finite sums sets
    the flag under a finite bound only."""
    for s, gs, c in ((4.0, 1.0, 1.0), (4.0, 1.0, 3.0), (2.5e7, 0.5, 0.7), (1e-20, 1.0, 1e-12), (9.0, 1 / 3, 0.1)):
        slots = torch.tensor([s * 0.25, s * 0.75], dtype=torch.float64, device="cuda")
        out, flag = torch.zeros(2, device="cuda"), torch.zeros(1, device="cuda")
        ops.grad_clip_coef(slots, gs, c, out[:1], out[1:], flag=flag)
        norm = torch.tensor(gs * math.sqrt(s), dtype=torch.float64).float()
        assert out[0].cpu().view(torch.int32) == norm.view(torch.int32), (s, gs)
        want = torch.clamp(torch.reciprocal(out[:1].cpu() + 1e-6) * c, max=1.0)
        assert out[1].cpu().view(torch.int32) == want.view(torch.int32), (s, gs, c, out[1].item(), want.item())
        assert flag.item() == 0.0
    for slots in ([1e78], [1e308, 1e308]):   # sqrt beyond fp32's range; a sum beyond fp64's
        for c, flagged in ((1.0, 1.0), (INF, 0.0)):
            out, flag = torch.zeros(2, device="cuda"), torch.zeros(1, device="cuda")
            ops.grad_clip_coef(torch.tensor(slots, dtype=torch.float64, device="cuda"), 1.0, c, out[:1], out[1:],
                               flag=flag)
            assert out[0].item() == INF and flag.item() == flagged, (slots, c)
            assert out[1].item() == (0.0 if c == 1.0 else 1.0)


# ---- 2. AdamW with the coefficient ---------------------------------------------------------------------------------------
def _dp():
    import test_dp_step_gpu as dp
    return dp


@pytest.mark.parametrize("guarded", [False, True], ids=["plain", "guarded"])
@pytest.mark.parametrize("fp32_grad", [False, True], ids=["g16", "g32"])
def test_coef_one_is_bit_identical(ops, guarded, fp32_grad):
    dp = _dp()
    n = 1_000_004
    wd, gs, _, _ = dp.CFGS["wd-half-ema"]
    w0, ema0, grads = dp._state(n, seed=21)
    outs = []
    for use_coef in (False, True):
        s = {"w": w0.cuda(), "m": torch.zeros(n, device="cuda"), "v": torch.zeros(n, device="cuda"),
             "ema": ema0.cuda(), "w16": torch.zeros(n, dtype=bf16, device="cuda")}
        coef = torch.ones(1, device="cuda") if use_coef else None
        flag, counts = torch.zeros(1, device="cuda"), torch.zeros(2, dtype=torch.int64, device="cuda")
        for step, g in zip(dp.STEPS, grads):
            g = g.cuda().float() if fp32_grad else g.cuda()
            if guarded:
                counts[0] = step - 1
                ops.adamw_ema_guarded(s["w"], g, s["m"], s["v"], s["ema"], s["w16"], n, dp.LR, flag, counts,
                                      weight_decay=wd, grad_scale=gs, max_blocks=3, coef=coef)
            else:
                ops.adamw_ema(s["w"], g, s["m"], s["v"], s["ema"], s["w16"], n, dp.LR, step, weight_decay=wd,
                              grad_scale=gs, coef=coef)
        outs.append(s)
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


@pytest.mark.parametrize("guarded", [False, True], ids=["plain", "guarded"])
@pytest.mark.parametrize("fp32_grad", [False, True], ids=["g16", "g32"])
def test_coef_below_one_vs_float64(ops, guarded, fp32_grad):
    """At the tolerance of the plain kernel's float64 test (test_dp_step_gpu.py::test_adamw_g16_vs_float64)."""
    from oracle import maskdit_oracle as O
    dp = _dp()
    n = 2_500_004
    wd, gs, _, _ = dp.CFGS["wd-half-ema"]
    w0, ema0, grads = dp._state(n, seed=22)
    coefs = [0.37, 0.9, 1.0, 0.05, 0.61, 0.2]
    s = {"w": w0.cuda(), "m": torch.zeros(n, device="cuda"), "v": torch.zeros(n, device="cuda"), "ema": ema0.cuda()}
    flag, counts = torch.zeros(1, device="cuda"), torch.zeros(2, dtype=torch.int64, device="cuda")
    for step, g, c in zip(dp.STEPS, grads, coefs):
        g = g.cuda().float() if fp32_grad else g.cuda()
        coef = torch.tensor([c], device="cuda")
        if guarded:
            counts[0] = step - 1
            ops.adamw_ema_guarded(s["w"], g, s["m"], s["v"], s["ema"], None, n, dp.LR, flag, counts,
                                  weight_decay=wd, grad_scale=gs, coef=coef)
        else:
            ops.adamw_ema(s["w"], g, s["m"], s["v"], s["ema"], None, n, dp.LR, step, weight_decay=wd, grad_scale=gs,
                          coef=coef)
    got = {k: t.cpu() for k, t in s.items()}
    f32 = dp.f32
    sc = dict(lr=f32(dp.LR), b1=f32(0.9), b2=f32(0.999), eps=f32(1e-8), wd=f32(wd), ema_decay=f32(0.9999))
    w, m, v, e = w0.double(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), ema0.double()
    for step, g, c in zip(dp.STEPS, grads, coefs):
        O.adamw_ema_step(w, g.double() * gs * f32(c), m, v, e, step, **sc)
    slack = 1e-5 * dp.LR * len(dp.STEPS)
    for name, ref in (("w", w), ("ema", e)):
        err = (got[name].double() - ref).abs()
        assert (err <= 8 * dp._ulp32(ref) + slack).all(), (name, err.max().item())
    for name, ref in (("m", m), ("v", v)):
        rel = (got[name].double() - ref).abs().max().item() / ref.abs().max().item()
        assert rel <= 1e-5, (name, rel)


# ---- 3. the world-1 step -------------------------------------------------------------------------------------------------
ENV = ("MDT_GRAD_AR", "MDT_COLLECTIVE", "MDT_AR_CHUNKS", "MDT_TRAIN_GRAPH")


@pytest.fixture
def clean_env(monkeypatch):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)


def _g():
    import test_nonfinite_guard_gpu as g
    return g


def _trainstep(max_grad_norm, **kw):
    from maskdit_b200.train_step import TrainStep
    net = _g()._net("S/2")
    return TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, weight_decay=0.01, global_batch=4,
                     max_grad_norm=max_grad_norm, **kw)


def _state(ts):
    s = _g()._opt_state(ts)
    for i, e in enumerate(ts.phema_emas):
        s[f"phema{i}"] = e.clone()
    return s


def _run(ts, data, ga=1):
    losses = [_g()._step(ts, b, ga) for b in data]
    torch.cuda.synchronize()
    return losses


def _free():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("guard", [False, True], ids=["plain", "guard"])
def test_world1_inf_and_loose_bound_change_nothing(det, clean_env, guard):
    data = _g()._batches("S/2", 3)
    kw = dict(skip_nonfinite=guard, phema_sigma_rels=(0.05, 0.10))
    ts = _trainstep(None, **kw)
    loss_off = _run(ts, data)
    off = _state(ts)
    del ts
    _free()
    norms = {}
    for c in (INF, 1e6):
        ts = _trainstep(c, **kw)
        loss = _run(ts, data)
        norms[c] = ts.grad_norm.item()
        got = _state(ts)
        for k in off:
            assert torch.equal(off[k], got[k]), (c, k)
        for a, b in zip(loss_off, loss):
            assert torch.equal(a, b), c
        if guard:
            assert ts._counts.tolist() == [3, 0]
        del ts
        _free()
    assert norms[INF] == norms[1e6] and 0 < norms[INF] < 1e6


@pytest.mark.parametrize("ga", [1, 2])
def test_world1_clipped_step_equals_torch(clean_env, ga):
    """A bound below the norm: `grad_norm` is clip_grad_norm_'s total norm of the p.grad views (x 1/grad_accum), and
    weights and moments equal torch.optim.AdamW after clip_grad_norm_ on a float64 copy."""
    dp = _dp()
    f32 = dp.f32
    data = _g()._batches("S/2", 1)
    ts = _trainstep(1e-3)
    n = ts.st.n_train
    params = [(k, p) for k, p in ts.net.named_parameters() if p.requires_grad]
    ref = [p.detach().double().clone().requires_grad_(True) for _, p in params]
    _run(ts, data, ga)
    got = ts.grad_norm.item()
    for r, (_, p) in zip(ref, params):
        r.grad = p.grad.double() / ga   # the views into the flat gradient the step just accumulated
    total = torch.nn.utils.clip_grad_norm_(ref, ts.max_grad_norm).item()
    _assert_norm(ts.grad_norm, total, ("grad_accum", ga))
    _assert_norm(ts.grad_norm, _ref_norm(ts.st.grad[:n]) / ga, ("flat", ga))
    assert ts.max_grad_norm < got, (got, "the bound must clip")
    opt = torch.optim.AdamW(ref, lr=f32(ts.lr), betas=(f32(0.9), f32(0.999)), eps=f32(1e-8), weight_decay=f32(0.01))
    opt.step()
    worst = {}
    for r, (k, p) in zip(ref, params):
        lo, cnt, _ = ts.st.offsets[k]
        st = opt.state[r]
        for name, a, b in (("w", ts.st.w32[lo:lo + cnt], r.detach().reshape(-1)),
                           ("m", ts.m[lo:lo + cnt], st["exp_avg"].reshape(-1)),
                           ("v", ts.v[lo:lo + cnt], st["exp_avg_sq"].reshape(-1))):
            err = (a.double() - b).abs()
            bound = 8 * dp._ulp32(b) + (1e-5 * ts.lr if name == "w" else 1e-5 * b.abs().max().item())
            worst[name] = max(worst.get(name, 0.0), (err / bound).max().item())
            assert (err <= bound).all(), (ga, k, name, err.max().item())
    print(f"grad_accum {ga}: norm {got:.6g} clipped to {ts.max_grad_norm}; worst error / bound {worst}")
    del ts, opt, ref
    _free()


def test_world1_guard_skips_a_nonfinite_step(clean_env):
    data = _g()._batches("S/2", 3)
    ts = _trainstep(0.5, skip_nonfinite=True)
    _run(ts, data[:1])
    assert math.isfinite(ts.grad_norm.item()) and ts._counts.tolist() == [1, 0]
    before = _g()._opt_state(ts)
    _run(ts, [_g()._poison(data[1])])
    assert not math.isfinite(ts.grad_norm.item()) and int(ts.skipped_steps) == 1
    _g()._assert_skip(before, _g()._opt_state(ts), ts.ema_decay)
    _run(ts, data[2:])
    assert math.isfinite(ts.grad_norm.item()) and ts._counts.tolist() == [2, 1]
    del ts
    _free()


def test_added_calls_do_not_synchronise(clean_env):
    """The norm pass, the coefficient and the coefficient-reading optimizer pass under sync debug mode 'error'."""
    from maskdit_b200 import ops
    data = _g()._batches("S/2", 2)
    for guard in (False, True):
        ts = _trainstep(0.5, skip_nonfinite=guard)
        _run(ts, data[:1])
        n = ts.st.n_train
        torch.cuda.set_sync_debug_mode("error")
        try:
            ops.grad_sumsq(ts.st.grad[:n], ts._gn_slots[:1], ts._gn_scratch, flag=ts._flag)
            ts._grad_norm_coef(1)
            ts._step_range(0, n)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        del ts
        _free()


# ---- 4. rank 0 of two emulated ranks ----------------------------------------------------------------------------------------
class TwoIdenticalRanks:
    """`GradComm` stand-in on rank 0 of two ranks holding the same gradient: the real one-rank `mdt_allreduce_grads`,
    then the buffer doubled (the exact two-rank sum).  The guard's flag word is summed with a clear peer flag."""

    def __init__(self, ts, comm, log):
        self.ts, self.comm, self.log = ts, comm, log

    def all_reduce(self, t):
        from maskdit_b200 import ops
        self.log.append(ops.lib().mdt_allreduce_grads(self.comm, t.data_ptr(), t.numel(), int(t.dtype == bf16),
                                                      ops.stream_ptr()))
        if self.ts._flag is None or t.data_ptr() != self.ts._flag.data_ptr():
            t.mul_(2)

    def close(self):
        pass


def make_rank0_of_two(ts, comm, log, ar_chunks):
    ts.world = 2
    ts.comm = TwoIdenticalRanks(ts, comm, log)
    if ts.grad_dtype == "bf16":
        ts.g16 = torch.empty(ts.st.n_train, dtype=bf16, device="cuda")
    ts.ar_chunks = ar_chunks


@pytest.fixture(scope="module")
def comm(ops):
    L = ops.lib()
    uid = ctypes.create_string_buffer(128)
    assert L.mdt_nccl_unique_id(uid) == 0
    c = ctypes.c_void_p()
    assert L.mdt_nccl_comm_create(bytes(uid.raw), 0, 1, 0, ctypes.byref(c)) == 0 and c.value
    yield c
    assert L.mdt_nccl_comm_destroy(c) == 0


def _world2(max_grad_norm, grad_dtype, chunks, comm, log, **kw):
    ts = _trainstep(max_grad_norm, grad_dtype=grad_dtype, **kw)
    ts.global_batch = 8
    make_rank0_of_two(ts, comm, log, chunks)
    return ts


WORLD2 = [("bf16", 1), ("bf16", 4), ("fp32", 1), ("fp32", 4)]


@pytest.mark.parametrize("grad_dtype,chunks", WORLD2, ids=[f"{d}-{c}" for d, c in WORLD2])
def test_world2_inf_changes_nothing(det, clean_env, comm, grad_dtype, chunks):
    data = _g()._batches("S/2", 2)
    log = []
    states = []
    for c in (None, INF):
        ts = _world2(c, grad_dtype, chunks, comm, log, skip_nonfinite=True)
        _run(ts, data)
        states.append(_state(ts))
        if c is not None:
            buf = ts.g16 if ts.g16 is not None else ts.st.grad[:ts.st.n_train]
            _assert_norm(ts.grad_norm, _ref_norm(buf) / 2, (grad_dtype, chunks))
        del ts
        _free()
    for k in states[0]:
        assert torch.equal(states[0][k], states[1][k]), (grad_dtype, chunks, k)
    assert log and all(rc == 0 for rc in log), log


@pytest.mark.parametrize("ga", [1, 2])
@pytest.mark.parametrize("grad_dtype,chunks", WORLD2, ids=[f"{d}-{c}" for d, c in WORLD2])
def test_world2_every_chunk_uses_the_final_coefficient(clean_env, comm, ops, grad_dtype, chunks, ga):
    """The norm is the float64 norm of the summed buffer x 1/(2 grad_accum), and one AdamW pass over the whole summed
    buffer with that step's coefficient reproduces every chunk's update bit for bit: a pass that ran before the last
    chunk's norm was known would have read the previous step's coefficient (0 before the first step)."""
    data = _g()._batches("S/2", 3)
    log = []
    ts = _world2(1e-3, grad_dtype, chunks, comm, log)
    n = ts.st.n_train
    coefs = []
    for step, b in enumerate(data, 1):
        pre = {"w": ts.st.w32[:n].clone(), "m": ts.m.clone(), "v": ts.v.clone(), "ema": ts.ema_st.w32[:n].clone()}
        _run(ts, [b], ga)
        buf = ts.g16 if ts.g16 is not None else ts.st.grad[:n]
        _assert_norm(ts.grad_norm, _ref_norm(buf) / (2 * ga), (grad_dtype, chunks, ga, step))
        coef = ts._gn[1:].clone()
        assert 0 < coef.item() < 1, coef.item()
        want = torch.clamp(torch.reciprocal(ts._gn[:1] + 1e-6) * ts.max_grad_norm, max=1.0)
        assert torch.equal(coef, want)
        coefs.append(coef.item())
        w16 = torch.empty(n, dtype=bf16, device="cuda")
        ops.adamw_ema(pre["w"], buf, pre["m"], pre["v"], pre["ema"], w16, n, ts._lr_now, ts.step_count, ts.betas[0],
                      ts.betas[1], ts.eps, ts.wd, ts.ema_decay, 1.0 / (2 * ga), coef=coef)
        torch.cuda.synchronize()
        for name, got, exp in (("w32", ts.st.w32[:n], pre["w"]), ("m", ts.m, pre["m"]), ("v", ts.v, pre["v"]),
                               ("ema", ts.ema_st.w32[:n], pre["ema"]), ("w16", ts.st.w16[:n], w16)):
            assert torch.equal(got, exp), (grad_dtype, chunks, ga, step, name)
    assert len(set(coefs)) == len(coefs), coefs
    assert log and all(rc == 0 for rc in log), log
    del ts
    _free()


# ---- 5. train.py end to end -------------------------------------------------------------------------------------------------
LINE = re.compile(r"^\(step=\d{7}\) Train Loss: -?\d+\.\d{4}, Train Steps/Sec: \d+\.\d{2}, Skipped Steps: \d+"
                  r"(, Grad Norm: \S+ \(max \S+\))?$")


@pytest.mark.parametrize("bound", [None, "1.0", "inf"])
def test_train_py_logs_the_norm(tmp_path, monkeypatch, capsys, bound):
    import train
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", *ENV):
        monkeypatch.delenv(k, raising=False)
    cfg = tmp_path / "cfg.yaml"
    cfg.write_text(_g().YAML.replace("max_num_steps: 4", "max_num_steps: 6").replace("ckpt_every: 4", "ckpt_every: 6"))
    argv = ["train.py", "--config", str(cfg), "--synthetic", "--max_steps", "6", "--results_dir", str(tmp_path / "r")]
    monkeypatch.setattr(sys, "argv", argv + (["--max_grad_norm", bound] if bound else []))
    train.main()
    out = capsys.readouterr().out
    lines = [ln for ln in out.splitlines() if "Train Loss" in ln]
    assert len(lines) == 3, out
    for ln in lines:
        assert LINE.match(ln), ln
        assert ("Grad Norm: " in ln) == (bound is not None), ln
        if bound:
            mean, mx = (float(v) for v in re.search(r"Grad Norm: (\S+) \(max (\S+)\)", ln).groups())
            assert 0 < mean <= mx * (1 + 1e-3) and math.isfinite(mx), ln
