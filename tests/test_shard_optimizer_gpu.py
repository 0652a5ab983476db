"""GPU: the sharded optimizer (`TrainStep(shard_optimizer=True)`) against the replicated step, on one H100.

`Ranks` stands in for the communicator of rank 0 of `world` ranks that all hold the same gradient.  It runs the real
one-rank NCCL collective, then supplies the other ranks' part: the all-reduce and the reduce-scatter multiply by
`world` (the exact sum of `world` equal values, a power of two), and the all-gather fills the other ranks' pieces from
a replicated twin `TrainStep` that steps the same batches on the same GPU as rank 0 of the same world.  Without a twin
the all-gather leaves the other ranks' pieces as they are.  Two TrainSteps give the same gradients only under the
deterministic mode, so every comparison with a twin runs in it."""
import copy
import gc
import os
import subprocess
import sys

import pytest
import torch

from support import NAN, batches, bf16, comm, det, f32, poison, step_batch, ulp32  # noqa: F401

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Ranks:
    """`GradComm` stand-in on rank 0 of `world` ranks; `rcs` collects the statuses of the real one-rank calls."""

    def __init__(self, ts, comm, world, twin):
        self.ts, self.comm, self.world, self.twin = ts, comm, world, twin
        self.rank = 0
        self.rcs = []
        self.gathering = None   # (local piece, chunk) of the TrainStep's `_gather_chunk` in progress

    def all_reduce(self, t):
        from maskdit_b200 import ops
        self.rcs.append(ops.lib().mdt_allreduce_grads(self.comm, t.data_ptr(), t.numel(), int(t.dtype == bf16),
                                                      ops.stream_ptr()))
        t.mul_(self.world)

    def reduce_scatter(self, t, count):
        from maskdit_b200 import ops
        self.rcs.append(ops.lib().mdt_reduce_scatter_grads(self.comm, t.data_ptr(), count, int(t.dtype == bf16),
                                                           ops.stream_ptr()))
        t[:count].mul_(self.world)

    def all_gather(self, t, count):
        from maskdit_b200 import ops
        from maskdit_b200.train_step import _GATHER_DTYPES
        self.rcs.append(ops.lib().mdt_allgather(self.comm, t.data_ptr(), count, _GATHER_DTYPES[t.dtype],
                                                ops.stream_ptr()))
        if self.twin is not None:
            self._peers(t, count)

    def close(self):
        pass

    # -- the other ranks' pieces, from the twin -------------------------------------------------------------------
    def _peers(self, t, count):
        ts, tw, sh, W = self.ts, self.twin, self.ts._sh, self.world

        def within(base):
            a = t.data_ptr() - base.data_ptr()
            return 0 <= a < base.numel() * base.element_size()

        def fill(k, full):   # chunk k's pieces of the other ranks from the twin's full-layout buffer
            lo, hi = sh.bounds[k]
            p = sh.pieces[k]
            for rr in range(1, W):
                a, b = min(hi, lo + rr * p), min(hi, lo + (rr + 1) * p)
                t[rr * p:rr * p + b - a].copy_(full[a:b])

        if self.gathering is not None:
            piece, k = self.gathering
            self.gathering = None
            for mine, full in [(ts.m, tw.m), (ts.v, tw.v), (ts.st.w32, tw.st.w32), (ts.ema_st.w32, tw.ema_st.w32),
                               *zip(ts.phema_emas, tw.phema_emas)]:
                a = piece.data_ptr() - mine.data_ptr()
                if 0 <= a < mine.numel() * 4:
                    return fill(k, full)
            raise AssertionError("gather of an unknown buffer")
        if within(ts.st.w16):
            lo = (t.data_ptr() - ts.st.w16.data_ptr()) // 2
            t[count:].copy_(tw.st.w16[lo + count:lo + W * count])
        elif within(ts.xbuf):   # the shadow of a padded chunk, staged in its exchange slot
            off = (t.data_ptr() - ts.xbuf.data_ptr()) // ts.xbuf.element_size()
            fill(sh.xoff.index(off), tw.st.w16)
        elif t.data_ptr() == ts._rset.data_ptr():
            P = sh.rset_piece
            for rr in range(1, W):
                for g, o, c in sh.read_segs[rr]:
                    t[rr * P + o:rr * P + o + c].copy_(tw.st.w32[g:g + c])
        elif within(ts._gn_slots):
            from maskdit_b200 import ops
            k = (t.data_ptr() - ts._gn_slots.data_ptr()) // 8 // W
            lo, hi = sh.bounds[k]
            p = sh.pieces[k]
            g = tw.g16 if tw.g16 is not None else tw.st.grad
            for rr in range(1, W):
                a, b = min(hi, lo + rr * p), min(hi, lo + (rr + 1) * p)
                if b > a:
                    ops.grad_sumsq(g[a:b], t[rr:rr + 1], ts._gn_scratch)
                else:
                    t[rr:rr + 1].zero_()
        else:
            raise AssertionError("all-gather of an unknown buffer")


def as_rank0(ts, comm, world, ar_chunks, shard, twin=None):
    """Turn a world-1 TrainStep into rank 0 of `world` ranks, sharded or replicated."""
    ts.world, ts.rank, ts.ar_chunks, ts.shard_optimizer = world, 0, ar_chunks, shard
    ts.comm = Ranks(ts, comm, world, twin)
    if shard:
        ts._shard_setup()
        gather = ts._gather_chunk

        def traced(k, piece, out):
            ts.comm.gathering = (piece, k)
            gather(k, piece, out)
        ts._gather_chunk = traced
    elif ts.grad_dtype == "bf16":
        ts.g16 = torch.empty(ts.st.n_train, dtype=bf16, device="cuda")
    return ts


def make_net(dec=True, logvar=0, precond="edm", seed=1):
    from maskdit_b200.maskdit import Precond_models
    torch.manual_seed(seed)
    kw = {"logvar_channels": logvar} if logvar else {}
    with torch.device("cuda"):
        net = Precond_models[precond](img_resolution=32, img_channels=4, num_classes=1000, model_type="DiT-S/2",
                                      use_decoder=dec, mae_loss_coef=0.1, pad_cls_token=False, **kw)
        gz = torch.Generator(device="cuda").manual_seed(seed + 1)
        with torch.no_grad():   # the zero-initialised tensors get values: every gradient is live
            for p in net.parameters():
                if p.requires_grad and float(p.abs().sum()) == 0.0:
                    p.copy_(torch.randn(p.shape, generator=gz, device="cuda") * 0.02)
    return net.train()


def pair(comm, world, chunks, dec=True, logvar=0, precond="edm", **kw):
    """(sharded rank 0 of world, its replicated twin) from the same network."""
    from maskdit_b200.train_step import TrainStep
    net = make_net(dec, logvar, precond)
    net2 = copy.deepcopy(net)
    args = dict(lr=1e-3, ema_decay=0.99, phema_sigma_rels=(0.05, 0.10), **kw)
    twin = as_rank0(TrainStep(net2, copy.deepcopy(net2).eval(), **args), comm, world, chunks, False)
    ts = as_rank0(TrainStep(net, copy.deepcopy(net).eval(), **args), comm, world, chunks, True, twin)
    return ts, twin


def owned_mask(ts, with_read=True):
    n = ts.st.n_train
    keep = torch.zeros(n, dtype=torch.bool, device="cuda")
    for a, b in ts._sh.own:
        keep[a:b] = True
    if with_read:
        for a, b in ts._sh.read:
            keep[a:b] = True
    return keep


def assert_matches_twin(ts, twin, what=""):
    """w16 everywhere, w32 on the owned pieces and the fp32-read set, and m, v, the EMA and the profiles on the owned
    pieces: bit for bit."""
    sh, n = ts._sh, ts.st.n_train
    assert torch.equal(ts.st.w16[:n], twin.st.w16[:n]), what
    keep = owned_mask(ts)
    assert torch.equal(ts.st.w32[:n][keep], twin.st.w32[:n][keep]), what
    for k, (a, b) in enumerate(sh.own):
        s = sh.loff[k]
        pairs = [(ts.m, twin.m), (ts.v, twin.v), *zip(ts.phema_emas, twin.phema_emas)]
        for mine, full in pairs:
            assert torch.equal(mine[s:s + b - a], full[a:b]), (what, k)
        assert torch.equal(ts.ema_st.w32[a:b], twin.ema_st.w32[a:b]), (what, k)


def run_pair(ts, twin, data, ga=1, check=True):
    for i, b in enumerate(data):
        la = step_batch(twin, b, ga)
        lb = step_batch(ts, b, ga)
        torch.cuda.synchronize()
        assert torch.equal(la.view(torch.int32), lb.view(torch.int32)), i   # bitwise: a poisoned step's NaN too
        if check:
            assert_matches_twin(ts, twin, f"step {i}")


def statuses_ok(*tss):
    for t in tss:
        assert t.comm.rcs and all(rc == 0 for rc in t.comm.rcs), t.comm.rcs


# ---- 1. bit identity --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dec", [True, False], ids=["maskdit", "nodecoder"])
@pytest.mark.parametrize("world,grad,chunks", [(2, "bf16", 1), (2, "fp32", 4), (4, "bf16", 4), (4, "fp32", 1),
                                                 (3, "bf16", 4)])
def test_sharded_step_equals_replicated(comm, det, dec, world, grad, chunks):
    ts, twin = pair(comm, world, chunks, dec=dec, grad_dtype=grad)
    assert ts.xbuf.dtype == (bf16 if grad == "bf16" else torch.float32)
    n = ts.st.n_train
    assert ts.m.numel() == sum(ts._sh.pieces) and ts.m.numel() <= n // world + 64 * len(ts._sh.bounds)
    run_pair(ts, twin, batches("S/2", 3))
    ts.materialize()
    assert torch.equal(ts.st.w32, twin.st.w32) and torch.equal(ts.ema_st.w32, twin.ema_st.w32)
    assert "sharded" in ts.describe_collective()
    statuses_ok(ts, twin)


@pytest.mark.parametrize("variant", ["skip_nonfinite", "grad_accum", "logvar"])
def test_sharded_step_variants(comm, det, variant):
    kw = {"skip_nonfinite": True} if variant == "skip_nonfinite" else {}
    ts, twin = pair(comm, 4, 4, logvar=8 if variant == "logvar" else 0, **kw)
    data = batches("S/2", 3)
    if variant == "skip_nonfinite":
        data[1] = poison(data[1])
    run_pair(ts, twin, data, ga=2 if variant == "grad_accum" else 1)
    if variant == "skip_nonfinite":
        assert int(ts.skipped_steps) == int(twin.skipped_steps) == 1
    statuses_ok(ts, twin)


def test_sharded_step_is_reproducible(comm, det):
    """Two sharded runs from the same start give the same bits."""
    outs = []
    for _ in range(2):
        ts, twin = pair(comm, 2, 4)
        run_pair(ts, twin, batches("S/2", 2), check=False)
        ts.materialize()
        outs.append((ts.st.w32.clone(), ts.m.clone(), ts.phema_emas[1].clone()))
        del ts, twin
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ---- 2. clipping ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world,chunks", [(2, 4), (4, 1)])
def test_sharded_clipping(comm, det, world, chunks):
    ts, twin = pair(comm, world, chunks, max_grad_norm=0.05)
    for i, b in enumerate(batches("S/2", 3)):
        step_batch(twin, b)
        step_batch(ts, b)
        torch.cuda.synchronize()
        a, c = float(ts.grad_norm), float(twin.grad_norm)
        assert abs(a - c) <= float(ulp32(c)), (i, a, c)
        if a != c:   # the weights follow the norm: compare from the twin's state on
            return
        assert_matches_twin(ts, twin, f"step {i}")
    statuses_ok(ts, twin)


# ---- 3. the stale masters are never read -------------------------------------------------------------------------------
@pytest.mark.parametrize("what", ["maskdit", "nodecoder", "flow", "ect", "logvar"])
def test_stale_masters_are_never_read(comm, det, what):
    from maskdit_b200.loss import ECTLoss, FlowLoss
    ts, twin = pair(comm, 4, 4, dec=what != "nodecoder", logvar=8 if what == "logvar" else 0,
                    precond="flow" if what == "flow" else "edm")
    if what in ("flow", "ect"):   # each TrainStep its own loss object (ECT's stage word belongs to one step object)
        make = FlowLoss if what == "flow" else (lambda: ECTLoss(stage_steps=2))
        ts.loss_fn, twin.loss_fn = make(), make()
    stale = ~owned_mask(ts)
    assert stale.any()
    for i, b in enumerate(batches("S/2", 3)):
        la = step_batch(twin, b)
        ts.st.w32[:ts.st.n_train][stale] = NAN
        ts.st.mark_shadow_fresh(ts.net._params())   # the write is not a weight change: keep the shadow
        lb = step_batch(ts, b)
        torch.cuda.synchronize()
        assert torch.isfinite(lb).all() and torch.equal(la, lb), i
        assert_matches_twin(ts, twin, f"{what} step {i}")
    statuses_ok(ts, twin)


# ---- 4. checkpoints -----------------------------------------------------------------------------------------------------
def test_state_dict_and_snapshot_equal_replicated(comm, det):
    ts, twin = pair(comm, 4, 4)
    run_pair(ts, twin, batches("S/2", 2), check=False)
    a, b = ts.state_dict(), twin.state_dict()
    assert a.keys() == b.keys() and a["param_groups"] == b["param_groups"]
    assert a["state"].keys() == b["state"].keys()
    for i in a["state"]:
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(a["state"][i][k].cpu(), b["state"][i][k].cpu()), (i, k)
    for x, y in zip(a["phema"]["emas"], b["phema"]["emas"]):
        assert torch.equal(x, y)
    sa, sb = ts.phema_snapshot(), twin.phema_snapshot()
    assert sa["step"] == sb["step"] and sa["origin"] == sb["origin"]
    for pa, pb in zip(sa["profiles"], sb["profiles"]):
        assert pa["ema"].keys() == pb["ema"].keys()
        for k in pa["ema"]:
            assert torch.equal(pa["ema"][k].cpu(), pb["ema"][k].cpu()), k
    ts.materialize()
    for x, y in [(ts.net.state_dict(), twin.net.state_dict()), (ts.ema.state_dict(), twin.ema.state_dict())]:
        for k in x:
            assert torch.equal(x[k], y[k]), k
    statuses_ok(ts, twin)


def _resume(state, comm, world, shard, twin_next):
    """A fresh TrainStep (rank 0 of world) loaded from `state`, one step, compared with the twin's next step (which
    also supplies the other ranks' pieces when sharded)."""
    from maskdit_b200.train_step import TrainStep
    net = make_net(seed=7)          # other weights: the load must replace them
    net.load_state_dict(state["model"])
    ema = copy.deepcopy(net).eval()
    ema.load_state_dict(state["ema"])
    ts = TrainStep(net, ema, lr=1e-3, ema_decay=0.99, phema_sigma_rels=(0.05, 0.10))
    b, twin = twin_next
    as_rank0(ts, comm, world, 4, shard, twin if shard else None)
    ts.load_state_dict(state["opt"])
    step_batch(ts, b)
    torch.cuda.synchronize()
    ts.materialize()
    assert torch.equal(ts.st.w32, twin.st.w32) and torch.equal(ts.st.w16, twin.st.w16)
    assert torch.equal(ts.ema_st.w32, twin.ema_st.w32)
    full = [ts._full(t) for t in (ts.m, ts.v, *ts.phema_emas)]
    for x, y in zip(full, [twin.m, twin.v, *twin.phema_emas]):
        assert torch.equal(x, y.cpu())


def _state(ts):
    ts.materialize()
    return {"model": copy.deepcopy(ts.net.state_dict()), "ema": copy.deepcopy(ts.ema.state_dict()),
            "opt": ts.state_dict()}


def test_checkpoint_round_trips(comm, det):
    """Saved as rank 0 of 2 sharded and loaded replicated; saved replicated and loaded as rank 0 of 4 sharded.  With
    power-of-two worlds the exchanged gradient (world equal values summed, times 1/world) is the same at every world,
    so both continue bit for bit with the twin."""
    ts, twin = pair(comm, 2, 4)
    data = batches("S/2", 4)
    run_pair(ts, twin, data[:2], check=False)
    sharded, replicated = _state(ts), _state(twin)
    step_batch(twin, data[2])
    torch.cuda.synchronize()
    _resume(sharded, comm, 2, False, (data[2], twin))
    _resume(replicated, comm, 4, True, (data[2], twin))


# ---- 5. memory at production size ---------------------------------------------------------------------------------------
def _xl2_peak(comm, use_decoder, shard, mask, phema):
    """Peak allocated bytes of two XL/2 steps at batch 256 as rank 0 of 8 (sharded or replicated; no twin), and the
    recompute count the step picked."""
    from maskdit_b200.maskdit import Precond_models
    from maskdit_b200.train_step import TrainStep
    gc.collect()   # the earlier tests' steps (a stand-in and its TrainStep refer to each other)
    torch.cuda.empty_cache()
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = Precond_models["edm"](img_resolution=32, img_channels=4, num_classes=1000, model_type="DiT-XL/2",
                                    use_decoder=use_decoder, mae_loss_coef=0.1, pad_cls_token=False).train()
    ts = TrainStep(net, copy.deepcopy(net).eval(), lr=1e-4, phema_sigma_rels=phema)
    as_rank0(ts, comm, 8, 4, shard)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator().manual_seed(5)
    mom = torch.cat([torch.randn(256, 4, 32, 32, generator=g), torch.randn(256, 4, 32, 32, generator=g) - 2], 1).cuda()
    lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (256,), generator=g), 1000).float().cuda()
    for _ in range(2):
        loss = ts.step(mom, lab, mask, 0.1, moments=True, class_dropout_prob=0.1)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    out = torch.cuda.max_memory_allocated(), ts.recompute_blocks
    del ts, net, loss
    gc.collect()
    torch.cuda.empty_cache()
    return out


def test_xl2_memory_at_batch_256(comm):
    n = 730_115_216
    accounted = 7 / 8 * 4 * n * 4   # m, v and two profiles: 7/8 of each stays on the other ranks
    rep, r_rep = _xl2_peak(comm, True, False, 0.5, (0.05, 0.10))
    sh, r_sh = _xl2_peak(comm, True, True, 0.5, (0.05, 0.10))
    print(f"MaskDiT-XL/2 b256 mask 0.5, two profiles, rank 0 of 8: peak {rep / 1e9:.2f} GB replicated "
          f"(recompute {r_rep}), {sh / 1e9:.2f} GB sharded (recompute {r_sh}); saved {(rep - sh) / 1e9:.2f} GB of "
          f"{accounted / 1e9:.2f} accounted")
    assert rep - sh >= 0.9 * accounted
    rep, r_rep = _xl2_peak(comm, False, False, 0.0, ())
    sh, r_sh = _xl2_peak(comm, False, True, 0.0, ())
    print(f"DiT-XL/2 b256 unmasked, rank 0 of 8: {r_rep} blocks recomputed replicated, {r_sh} sharded; peak "
          f"{rep / 1e9:.2f} / {sh / 1e9:.2f} GB")
    assert r_sh < r_rep


# ---- 6. two real GPUs ----------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_sharded_equal_replicated():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29633", os.path.join(ROOT, "tools", "shard_equivalence.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "SHARD_EQUIV_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
