"""GPU: the non-finite gradient guard (`TrainStep(skip_nonfinite=True)`, GradScaler's inf-skip of the reference).

1. The check kernel and the checking bf16 cast: which values they flag, at which positions, over which sizes.
2. The guarded AdamW entries: bit-identical to the unguarded ones with the flag clear; only the EMA moves with it set.
3. Exact skip: under the deterministic mode a run that skips a poisoned batch equals, bit for bit, a run that never saw
   it (world 1, CUDA graph, gradient accumulation, and rank 0 of two emulated ranks in the exchange modes).
4. Consensus: the other rank's flag makes this rank skip (a real two-process run needs two GPUs).
5. Resume after a skip equals an uninterrupted run; the checkpoint carries Adam's applied step count.
6. train.py end to end with a loader that yields one NaN batch, with and without --no_amp.
"""
import copy
import ctypes
import gc
import io
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

bf16 = torch.bfloat16
NAN, INF = float("nan"), float("inf")


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


def _flag():
    return torch.zeros(1, device="cuda")


# ---- 1. check kernels ----------------------------------------------------------------------------------------------------
SIZES = [4, 5, 7, 1024, 4099, 1_000_003]


def _positions(n):
    return sorted({0, n // 2, n - 1})


def _check_size(ops, buf, n):
    """buf[:n] is finite on entry and on exit."""
    x = buf[:n]
    for pos in _positions(n):
        for val in (NAN, INF, -INF):
            keep = x[pos].clone()
            x[pos] = val
            f = _flag()
            ops.nonfinite_check(x, f)
            out = torch.empty(n, dtype=bf16, device="cuda")
            f16 = _flag()
            ops.cast_bf16_check(x, f16, out=out)
            assert f.item() == 1.0 and f16.item() == 1.0, (n, pos, val)
            assert torch.equal(out.view(torch.int16), ops.cast_bf16(x).view(torch.int16)), (n, pos, val)
            x[pos] = keep
    f = _flag()
    ops.nonfinite_check(x, f)
    assert f.item() == 0.0, n


def test_check_flags_nonfinite_at_every_position(ops):
    buf = torch.randn(max(SIZES), device="cuda")
    for n in SIZES:
        _check_size(ops, buf, n)


def test_check_finite_extremes_and_accumulation(ops):
    ext = torch.tensor([3.4e38, -3.4e38, 3.4028235e38, 1e-45, -1e-45, 1e-40, -0.0, 0.0], device="cuda")
    x = ext.repeat(1001)[:8003].contiguous()   # 8003: a 3-element tail after the float4 groups
    f = _flag()
    ops.nonfinite_check(x, f)
    assert f.item() == 0.0
    # the checking cast flags what it STORES: within bf16's range nothing, beyond it the rounded inf
    inrange = torch.tensor([3.3895e38, -3.3895e38, 1e-45, 1e-40, -0.0, 0.0, 9.2e-41, 1.0], device="cuda").repeat(9)
    f16 = _flag()
    out = ops.cast_bf16_check(inrange, f16)
    assert f16.item() == 0.0 and torch.isfinite(out.float()).all()
    assert torch.equal(out.view(torch.int16), ops.cast_bf16(inrange).view(torch.int16))
    f16 = _flag()
    out = ops.cast_bf16_check(x, f16)
    assert f16.item() == 1.0 and torch.equal(out.view(torch.int16), ops.cast_bf16(x).view(torch.int16))
    # flags accumulate: a clean call after a flagged one leaves the flag set
    bad = torch.zeros(64, device="cuda")
    bad[63] = NAN
    f = _flag()
    ops.nonfinite_check(bad, f)
    ops.nonfinite_check(torch.zeros(64, device="cuda"), f)
    assert f.item() == 1.0
    f16 = _flag()
    ops.cast_bf16_check(bad, f16)
    ops.cast_bf16_check(torch.zeros(64, device="cuda"), f16)
    assert f16.item() == 1.0


def test_check_chunk_tails(ops):
    """The all-reduce chunks of TrainStep: a NaN in the last element of a chunk is seen by that chunk's call, one just
    past its end is not."""
    from maskdit_b200.train_step import ar_chunk_bounds
    n = 4 * 1024 * 3 + 4099
    x = torch.randn(n, device="cuda")
    bounds = ar_chunk_bounds(n, 4)
    assert len(bounds) > 1 and (bounds[-1][1] - bounds[-1][0]) % 4
    for k, (lo, hi) in enumerate(bounds):
        x[hi - 1] = NAN
        f = _flag()
        ops.nonfinite_check(x[lo:hi], f)
        assert f.item() == 1.0, (lo, hi)
        if k + 1 < len(bounds):
            nlo, nhi = bounds[k + 1]
            f = _flag()
            ops.nonfinite_check(x[nlo:nhi], f)
            assert f.item() == 0.0, (nlo, nhi)
        x[hi - 1] = 0.5


def test_check_at_xl2_size(ops):
    """The XL/2 trainable-parameter count (one read of 2.92 GB): first, middle, last element."""
    from maskdit_b200.maskdit import Precond_models
    with torch.device("meta"):
        net = Precond_models["edm"](32, 4, num_classes=1000, model_type="DiT-XL/2", use_decoder=True,
                                    mae_loss_coef=0.1, pad_cls_token=False)
    n = sum(p.numel() for p in net.parameters() if p.requires_grad)
    assert n > 700_000_000
    x = torch.full((n,), 0.25, device="cuda")
    out = torch.empty(n, dtype=bf16, device="cuda")
    for pos in (0, n // 2 + 1, n - 1):
        for val in (NAN, INF, -INF):
            x[pos] = val
            f, f16 = _flag(), _flag()
            ops.nonfinite_check(x, f)
            ops.cast_bf16_check(x, f16, out=out)
            assert f.item() == 1.0 and f16.item() == 1.0, (pos, val)
            x[pos] = 0.25
    f, f16 = _flag(), _flag()
    ops.nonfinite_check(x, f)
    ops.cast_bf16_check(x, f16, out=out)
    assert f.item() == 0.0 and f16.item() == 0.0
    assert torch.equal(out.view(torch.int16), ops.cast_bf16(x).view(torch.int16))


# ---- 2. guarded AdamW ------------------------------------------------------------------------------------------------------
def _dp():
    import test_dp_step_gpu as dp
    return dp


@pytest.mark.parametrize("fp32_grad", [False, True])
@pytest.mark.parametrize("max_blocks", [0, 3])
@pytest.mark.parametrize("cfg", ["wd0-half-ema-w16", "wd-16th-w16", "wd-half-ema", "wd0-16th-bare"])
def test_guarded_adamw_flag_clear_is_bit_identical(ops, cfg, max_blocks, fp32_grad):
    dp = _dp()
    n = 1_000_004
    wd, gs, with_ema, with_w16 = dp.CFGS[cfg]
    w0, ema0, grads = dp._state(n, seed=11)
    ref = dp._run_kernel(ops, w0, ema0, grads, wd, gs, with_ema, with_w16, max_blocks=max_blocks,
                         fp32_grad=fp32_grad)
    out = {"w": w0.cuda(), "m": torch.zeros(n, device="cuda"), "v": torch.zeros(n, device="cuda"),
           "ema": ema0.cuda() if with_ema else None,
           "w16": torch.zeros(n, dtype=bf16, device="cuda") if with_w16 else None}
    flag, counts = _flag(), torch.zeros(2, dtype=torch.int64, device="cuda")
    for step, g in zip(dp.STEPS, grads):
        g = g.cuda().float() if fp32_grad else g.cuda()
        counts[0] = step - 1
        ops.adamw_ema_guarded(out["w"], g, out["m"], out["v"], out["ema"], out["w16"], n, dp.LR, flag, counts,
                              weight_decay=wd, grad_scale=gs, max_blocks=max_blocks)
        ops.optim_guard_advance(flag, counts)
        assert counts.tolist() == [step, 0]
    for k, t in ref.items():
        if t is not None:
            assert torch.equal(out[k], t), (cfg, k)


@pytest.mark.parametrize("fp32_grad", [False, True])
def test_guarded_adamw_flag_set_moves_only_the_ema(ops, fp32_grad):
    dp = _dp()
    n = 1_000_004
    gen = torch.Generator().manual_seed(3)
    w = torch.randn(n, generator=gen).cuda()
    ema = (w.cpu() + 0.01 * torch.randn(n, generator=gen)).cuda()
    m, v = (torch.randn(n, generator=gen) * 1e-3).cuda(), (torch.rand(n, generator=gen) * 1e-6).cuda()
    w16 = w.to(bf16)
    g = torch.randn(n, generator=gen).cuda()
    g[5] = NAN
    g = g if fp32_grad else g.to(bf16)
    flag, counts = torch.ones(1, device="cuda"), torch.tensor([7, 2], dtype=torch.int64, device="cuda")
    state = dict(w=w, m=m, v=v, w16=w16, counts=counts)
    before = {k: t.clone() for k, t in state.items()}
    before["ema"] = ema.clone()
    ops.adamw_ema_guarded(w, g, m, v, ema, w16, n, dp.LR, flag, counts, weight_decay=0.03, grad_scale=0.5,
                          max_blocks=3)
    torch.cuda.synchronize()
    for k, t in state.items():
        assert torch.equal(t, before[k]), k
    d = dp.f32(0.9999)
    want = d * before["ema"].double() + (1 - d) * before["w"].double()
    err = (ema.double() - want).abs()
    assert (err <= dp._ulp32(want)).all(), err.max().item()
    ops.optim_guard_advance(flag, counts)
    assert counts.tolist() == [7, 3]


# ---- the emulated second rank ----------------------------------------------------------------------------------------------
class Peer:
    """What the other rank contributes to the summed flag word."""

    def __init__(self, flag=0.0):
        self.flag = flag


class RankZeroOfTwo:
    """`GradComm` stand-in on rank 0 of two ranks: runs the real one-rank `mdt_allreduce_grads`, then adds the other
    rank's contribution (the same gradient, or the peer's flag word).  Records the statuses for the fixture to check."""

    def __init__(self, ts, comm, peer, log):
        self.ts, self.comm, self.peer, self.log = ts, comm, peer, log

    def all_reduce(self, t):
        from maskdit_b200 import ops
        L = ops.lib()
        self.log.append(L.mdt_allreduce_grads(self.comm, t.data_ptr(), t.numel(), int(t.dtype == bf16),
                                              ops.stream_ptr()))
        if t.data_ptr() == self.ts._flag.data_ptr():
            t.add_(self.peer.flag)
            return
        t.mul_(2)

    def close(self):
        pass


@pytest.fixture(scope="module")
def comm(ops):
    """A one-rank communicator."""
    L = ops.lib()
    uid = ctypes.create_string_buffer(128)
    assert L.mdt_nccl_unique_id(uid) == 0
    c = ctypes.c_void_p()
    assert L.mdt_nccl_comm_create(bytes(uid.raw), 0, 1, 0, ctypes.byref(c)) == 0 and c.value
    yield c
    assert L.mdt_nccl_comm_destroy(c) == 0


@pytest.fixture
def rank0_of_two(comm):
    """make(ts, peer, ar_chunks): turn a world-1 TrainStep into rank 0 of a two-rank job; the statuses are checked at
    the end."""
    logs = []

    def make(ts, peer, ar_chunks):
        log = []
        logs.append(log)
        ts.world = 2
        ts.comm = RankZeroOfTwo(ts, comm, peer, log)
        if ts.grad_dtype == "bf16":
            ts.g16 = torch.empty(ts.st.n_train, dtype=bf16, device="cuda")
        ts.ar_chunks = ar_chunks
        return ts

    yield make
    for log in logs:
        assert all(rc == 0 for rc in log), log


# ---- 3. exact skip -----------------------------------------------------------------------------------------------------------
MODELS = {"S/2": ("DiT-S/2", 32, 1000, 4), "XL/2": ("DiT-XL/2", 32, 1000, 8)}
MODES = {
    "world1": dict(),
    "graph": dict(graph=True),
    "accum2": dict(grad_accum=2),
    "bf16-chunked": dict(world2=True, grad_dtype="bf16", ar_chunks=4),
    "fp32-one-chunk": dict(world2=True, grad_dtype="fp32", ar_chunks=1),
    "fp32-chunked": dict(world2=True, grad_dtype="fp32", ar_chunks=4),
}
ENV = ("MDT_GRAD_AR", "MDT_COLLECTIVE", "MDT_AR_CHUNKS", "MDT_TRAIN_GRAPH")


def _net(model):
    from maskdit_b200.maskdit import Precond_models
    mt, R, ncls, _ = MODELS[model]
    torch.manual_seed(1)
    with torch.device("cuda"):
        net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=ncls, model_type=mt,
                                    use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False)
        gz = torch.Generator(device="cuda").manual_seed(2)
        with torch.no_grad():   # the zero-initialised tensors (adaLN, final layer) get values: every gradient is live
            for p in net.parameters():
                if p.requires_grad and float(p.abs().sum()) == 0.0:
                    p.copy_(torch.randn(p.shape, generator=gz, device="cuda") * 0.02)
    return net.train()


def _batches(model, k):
    """k batches of VAE moments and one-hot labels; batch i is drawn with its own seed."""
    _, R, ncls, B = MODELS[model]
    out = []
    for i in range(k):
        g = torch.Generator().manual_seed(100 + i)
        mom = torch.cat([torch.randn(B, 4, R, R, generator=g), torch.randn(B, 4, R, R, generator=g) - 2], 1)
        lab = torch.nn.functional.one_hot(torch.randint(0, ncls, (B,), generator=g), ncls).float()
        out.append((mom.cuda(), lab.cuda(), 1000 + i))
    return out


def _poison(batch):
    mom, lab, seed = batch
    mom = mom.clone()
    mom[0, 0, 3, 5] = NAN   # one NaN in the moments' mean
    return mom, lab, seed


def _trainstep(model, mode, rank0_of_two=None, peer=None, lr_rampup_kimg=0.0):
    from maskdit_b200.train_step import TrainStep
    kw = dict(MODES[mode])
    world2, ga = kw.pop("world2", False), kw.pop("grad_accum", 1)
    chunks = kw.pop("ar_chunks", 4)
    net = _net(model)
    B = MODELS[model][3]
    ts = TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, weight_decay=0.01, global_batch=B * (2 if world2 else 1),
                   lr_rampup_kimg=lr_rampup_kimg, reference_lr_schedule=True, skip_nonfinite=True, **kw)
    if world2:
        rank0_of_two(ts, peer or Peer(), chunks)
    return ts, ga


def _step(ts, batch, ga):
    mom, lab, seed = batch
    torch.manual_seed(seed)   # the step's draws (sigma, noise, latent eps, mask noise, label dropout) belong to the batch
    return ts.step(mom, lab, 0.5, 0.1, grad_accum=ga, moments=True, class_dropout_prob=0.1)


def _opt_state(ts):
    n = ts.st.n_train
    return {"w32": ts.st.w32[:n].clone(), "w16": ts.st.w16[:n].clone(), "m": ts.m.clone(), "v": ts.v.clone(),
            "ema": ts.ema_st.w32[:n].clone()}


def _assert_skip(before, after, ema_decay):
    for k in ("w32", "w16", "m", "v"):
        assert torch.equal(before[k], after[k]), k
    from test_dp_step_gpu import _ulp32, f32
    d = f32(ema_decay)
    step = 1 << 26   # float64 temporaries in slices: XL/2 has 675 M trainable elements
    for lo in range(0, before["ema"].numel(), step):
        e0, w0, e1 = (before["ema"][lo:lo + step].double(), before["w32"][lo:lo + step].double(),
                      after["ema"][lo:lo + step].double())
        want = d * e0 + (1 - d) * w0
        err = (e1 - want).abs()
        # 1 ulp of the result, plus the rounding of either product (the fused multiply-add rounds one of them):
        # trained weights include elements where d*ema and (1-d)*w nearly cancel, and there a product's rounding is
        # many ulps of the result
        bound = _ulp32(want) + _ulp32(d * e0) + _ulp32((1 - d) * w0)
        assert (err <= bound).all(), (lo, (err / bound).max().item())


def _exact_skip(model, mode, rank0_of_two):
    data = _batches(model, 4)
    bad = _poison(data[2])
    # run A: four steps, the third batch poisoned
    ts, ga = _trainstep(model, mode, rank0_of_two)
    for b in data[:2]:
        _step(ts, b, ga)
    before = _opt_state(ts)
    loss = _step(ts, bad, ga)
    torch.cuda.synchronize()
    assert not torch.isfinite(loss).all()
    _assert_skip(before, _opt_state(ts), ts.ema_decay)
    _step(ts, data[3], ga)
    a = _opt_state(ts)
    a_counts, a_steps = ts._counts.tolist(), ts.step_count
    del ts
    gc.collect()
    torch.cuda.empty_cache()
    # run B: the same batches without the poisoned one
    ts, ga = _trainstep(model, mode, rank0_of_two)
    for b in (data[0], data[1], data[3]):
        _step(ts, b, ga)
    b_ = _opt_state(ts)
    b_counts = ts._counts.tolist()
    assert a_counts == [3, 1] and b_counts == [3, 0] and a_steps == 4 and ts.step_count == 3
    assert ts.applied_steps() == 3
    for k in ("w32", "w16", "m", "v"):
        assert torch.equal(a[k], b_[k]), (model, mode, k)
    for k in ("w32", "ema"):
        assert torch.isfinite(a[k]).all(), k
    del ts
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("mode", list(MODES))
def test_exact_skip_s2(det, rank0_of_two, monkeypatch, mode):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    _exact_skip("S/2", mode, rank0_of_two)


@pytest.mark.parametrize("mode", ["world1", "bf16-chunked"])
def test_exact_skip_xl2(det, rank0_of_two, monkeypatch, mode):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    _exact_skip("XL/2", mode, rank0_of_two)


# ---- 4. consensus ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["bf16-chunked", "fp32-chunked", "fp32-one-chunk"])
def test_other_rank_nonfinite_makes_this_rank_skip(det, rank0_of_two, monkeypatch, mode):
    """This rank's gradients are finite, the other rank's are not: every rank checks its local values and one flag word
    is summed over the ranks, so the other rank's flag makes this rank skip too."""
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    data = _batches("S/2", 2)
    p = Peer()
    ts, ga = _trainstep("S/2", mode, rank0_of_two, p)
    _step(ts, data[0], ga)
    before = _opt_state(ts)
    p.flag = 1.0
    loss = _step(ts, data[1], ga)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    _assert_skip(before, _opt_state(ts), ts.ema_decay)
    assert ts._counts.tolist() == [1, 1] and int(ts.skipped_steps) == 1
    p.flag = 0.0
    _step(ts, data[0], ga)
    assert ts._counts.tolist() == [2, 1]
    assert not torch.equal(before["w32"], ts.st.w32[:ts.st.n_train])


def _two_process_worker():
    """torchrun --nproc-per-node 2: rank 1's batch is poisoned; both ranks must skip and stay identical."""
    import torch.distributed as dist
    from maskdit_b200.train_step import TrainStep
    rank = int(os.environ["RANK"])
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    torch.use_deterministic_algorithms(True)
    net = _net("S/2")
    ts = TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, skip_nonfinite=True, global_batch=8)
    data = _batches("S/2", 2)
    _step(ts, data[0], 1)
    before = _opt_state(ts)
    _step(ts, _poison(data[1]) if rank == 1 else data[1], 1)
    torch.cuda.synchronize()
    after = _opt_state(ts)
    _assert_skip(before, after, ts.ema_decay)
    counts = ts._counts.clone()
    allc = [torch.zeros_like(counts) for _ in range(2)]
    dist.all_gather(allc, counts)
    assert all(c.tolist() == [1, 1] for c in allc), allc
    ts.close()
    dist.destroy_process_group()
    print(f"rank {rank}: skipped in consensus")


def test_two_process_consensus(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29517", os.path.abspath(__file__)],
                       cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("skipped in consensus") == 2


# ---- 5. resume ---------------------------------------------------------------------------------------------------------------
def test_resume_after_a_skip_equals_uninterrupted(det):
    """Four steps (the second poisoned) in one go == two steps, a checkpoint, a fresh TrainStep and two more steps.
    The lr ramps over the four steps, so the resumed run's lr must follow the run's step counter (lr_step_offset, as
    train.py sets it) while Adam follows the applied count."""
    from maskdit_b200.train_step import TrainStep
    data = _batches("S/2", 4)
    data[1] = _poison(data[1])
    ramp = 4 * 4 / 1000   # 4 steps of batch 4

    def fresh():
        net = _net("S/2")
        return TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, global_batch=4, lr_rampup_kimg=ramp,
                         reference_lr_schedule=True, skip_nonfinite=True)

    ts = fresh()
    lrs_a = []
    for b in data:
        _step(ts, b, 1)
        lrs_a.append(ts._lr_now)
    a = _opt_state(ts)
    assert ts.applied_steps() == 3
    del ts
    gc.collect()
    ts = fresh()
    lrs_b = []
    for b in data[:2]:
        _step(ts, b, 1)
        lrs_b.append(ts._lr_now)
    sd = ts.state_dict()
    assert sd["param_groups"][0]["step"] == 1 and all(float(e["step"]) == 1.0 for e in sd["state"].values())
    buf = io.BytesIO()
    torch.save({"model": ts.net.state_dict(), "ema": ts.ema.state_dict(), "opt": sd}, buf)
    del ts
    gc.collect()
    torch.cuda.empty_cache()
    buf.seek(0)
    ck = torch.load(buf, weights_only=False)
    net = _net("S/2")
    net.load_state_dict(ck["model"])
    ema = copy.deepcopy(net).eval()
    ema.load_state_dict(ck["ema"])
    ts2 = TrainStep(net, ema, lr=1e-3, global_batch=4, lr_rampup_kimg=ramp, reference_lr_schedule=True,
                    skip_nonfinite=True)
    ts2.load_state_dict(ck["opt"])
    assert ts2.applied_steps() == 1 and int(ts2.skipped_steps) == 0
    ts2.lr_step_offset = 2 - ts2.step_count   # the run's step counter at the checkpoint minus Adam's count
    for b in data[2:]:
        _step(ts2, b, 1)
        lrs_b.append(ts2._lr_now)
    assert lrs_a == lrs_b and lrs_a[0] == 0.0 and len(set(lrs_a)) == 4, lrs_a
    assert ts2.applied_steps() == 3
    b_ = _opt_state(ts2)
    for k in a:
        assert torch.equal(a[k], b_[k]), k


# ---- 6. train.py end to end --------------------------------------------------------------------------------------------------
YAML = """
data: {dataset: imagenet256-latent, category: lmdb, resolution: 16, num_channels: 4, root: none, feat_path: None}
model:
  precond: edm
  model_type: DiT-S/2
  in_size: 16
  in_channels: 4
  num_classes: 1000
  use_decoder: True
  ext_feature_dim: 0
  pad_cls_token: False
  mask_ratio: 0.5
  mask_ratio_fn: constant
  mask_ratio_min: 0
  mae_loss_coef: 0.1
  class_dropout_prob: 0.1
train: {tf32: False, amp: True, batchsize: 8, grad_accum: 1, epochs: 1, lr: 0.0001, lr_rampup_kimg: 0, xflip: False,
        max_num_steps: 4}
log: {log_every: 2, ckpt_every: 4, tag: t}
"""


@pytest.mark.parametrize("no_amp", [False, True])
def test_train_py_skips_a_nan_batch(tmp_path, monkeypatch, capsys, no_amp):
    import train
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", *ENV):
        monkeypatch.delenv(k, raising=False)
    real = train.synthetic_loader

    def poisoned(cfg, batch, device, seed):   # the third batch carries one NaN
        for i, (mom, lab) in enumerate(real(cfg, batch, device, seed)):
            if i == 2:
                mom = mom.clone()
                mom[0, 0, 0, 0] = NAN
            yield mom, lab

    monkeypatch.setattr(train, "synthetic_loader", poisoned)
    cfg = tmp_path / "cfg.yaml"
    cfg.write_text(YAML)
    argv = ["train.py", "--config", str(cfg), "--synthetic", "--max_steps", "4", "--results_dir", str(tmp_path / "r")]
    monkeypatch.setattr(sys, "argv", argv + (["--no_amp"] if no_amp else []))
    train.main()
    out = capsys.readouterr().out
    lines = [ln for ln in out.splitlines() if "Train Loss" in ln]
    assert len(lines) == 2, out
    sd = torch.load(tmp_path / "r" / "checkpoints" / "0000004.pt", map_location="cpu", weights_only=False)
    finite = all(torch.isfinite(v).all() for k, v in sd["model"].items() if v.is_floating_point())
    if no_amp:
        assert "Skipped" not in out and not finite, out
    else:
        assert lines[0].endswith("Skipped Steps: 0") and lines[1].endswith("Skipped Steps: 1"), lines
        assert finite and all(torch.isfinite(v).all() for v in sd["ema"].values() if v.is_floating_point())
        assert sd["opt"]["param_groups"][0]["step"] == 3


if __name__ == "__main__":
    _two_process_worker()
