"""GPU, one device, one process: the data-parallel training step's own machinery.

(a) The fused AdamW + EMA + bf16-shadow kernel with a bf16 gradient (the buffer a bf16 all-reduce produces) against
    float64, over sizes that wrap its capped grid, capped grids, weight decay, gradient scales, zero gradients, the
    optional EMA / shadow outputs and a late step; and its elementwise identities (bf16 vs fp32 operand, chunked vs one
    pass, any grid cap).
(b) The NCCL entry points of the C ABI on a one-rank communicator (plain and CTA-confined): a one-rank SUM is the
    identity, argument errors are statuses.
(c) `TrainStep`'s world > 1 exchange run in process as rank 0 of two ranks holding the same gradient
    (`support.make_rank0_of_two`): which element ranges are exchanged, on which stream, under which SM budget, that
    nothing writes a range after its exchange started, and that the optimizer pass is exactly one AdamW pass over the
    summed buffer.
(d) What a C caller that overlaps its own exchange with the backward relies on: `mdt_backward`'s `on_ready` reports
    each block's range once it is final, and a backward under `mdt_set_sm_budget` computes the plain gradient.
"""
import copy
import ctypes
import os
import sys
from dataclasses import dataclass

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from support import (CFGS, LR, STEPS, adamw_inputs, clean_env, comm, f32, one_rank_comm, ops,  # noqa: E402,F401
                     rank0_of_two, run_adamw, ulp32)

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
MDT_ERR_ARG = -1


@pytest.fixture
def sm_budget(ops):
    yield ops.lib()
    assert ops.lib().mdt_set_sm_budget(0) == 0


# ---- (a) bf16-gradient AdamW -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", list(CFGS))
@pytest.mark.parametrize("n", [4, 1020, 2_500_004])
def test_adamw_g16_vs_float64(ops, n, cfg):
    """n = 2 500 004 is 625 001 float4 groups: the grid (capped at 132 x 8 blocks of 256 threads = 270 336 groups per
    pass) wraps more than twice, and max_blocks 1 / 3 make it wrap thousands of times."""
    from oracle import maskdit_oracle as O
    wd, gs, with_ema, with_w16 = CFGS[cfg]
    w0, ema0, grads = adamw_inputs(n, seed=n)
    runs = {mb: run_adamw(ops, w0, ema0, grads, wd, gs, with_ema, with_w16, max_blocks=mb) for mb in (0, 1, 3)}
    for mb in (1, 3):   # the grid-stride loop visits every element once, whatever the grid
        for k, t in runs[0].items():
            if t is not None:
                assert torch.equal(runs[mb][k], t), (mb, k)
    got = {k: (t.cpu() if t is not None else None) for k, t in runs[0].items()}

    # The float64 reference takes the scalars as the kernel receives them (float32 through the C ABI, as apex
    # FusedAdam's).  With the decimal betas instead, the stored v differs by 1.3e-5 relative: 1 - float(0.999) is
    # 0.000999987, not 0.001 (the bias correction uses the same beta2, so the update itself does not move).
    sc = dict(lr=f32(LR), b1=f32(0.9), b2=f32(0.999), eps=f32(1e-8), wd=f32(wd), ema_decay=f32(0.9999))
    w, m, v = w0.double(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    e = ema0.double() if with_ema else None
    for step, g in zip(STEPS, grads):
        O.adamw_ema_step(w, g.double() * gs, m, v, e, step, **sc)
    slack = 1e-5 * LR * len(STEPS)
    worst = {}
    for name, ref in (("w", w), ("ema", e)):
        if ref is None:
            assert got[name] is None
            continue
        err, ulp = (got[name].double() - ref).abs(), ulp32(ref)
        bound = 8 * ulp + slack
        big = 8 * ulp >= slack   # elements whose bound is mostly the ulp term
        worst[name] = (f"{(err / bound).max().item():.2f} of bound, {(err[big] / ulp[big]).max().item():.2f} ulp "
                       f"where 8 ulp >= slack")
        assert (err <= bound).all(), (name, err.max().item(), ((err - bound).argmax().item()))
    for name, ref in (("m", m), ("v", v)):
        rel = (got[name].double() - ref).abs().max().item() / ref.abs().max().item()
        worst[name] = f"{rel:.2e} rel"
        assert rel <= 1e-5, (name, rel)
    z0, z1 = n // 3, n // 3 + max(n // 10, 1)
    assert (got["m"][z0:z1] == 0).all() and (got["v"][z0:z1] == 0).all()   # zero gradients: only the decay moves w
    if with_w16:
        assert torch.equal(got["w16"], got["w"].to(bf16))
    print(f"ADAMW_G16 n={n} {cfg}: " + ", ".join(f"{k} {s}" for k, s in worst.items()))


@pytest.mark.parametrize("n", [1020, 2_500_004])
def test_adamw_elementwise_identities(ops, n):
    """Bit for bit: the bf16-operand kernel == the fp32 kernel on the widened gradient, and one pass over [0, n) ==
    passes over the all-reduce chunks (what TrainStep's pipelined chunk steps rely on)."""
    from maskdit_b200.train_step import ar_chunk_bounds
    w0, ema0, grads = adamw_inputs(n, seed=n + 1)
    for cfg in ("wd0-half-ema-w16", "wd-16th-w16"):
        wd, gs, _, _ = CFGS[cfg]
        a = run_adamw(ops, w0, ema0, grads, wd, gs, True, True)
        b = run_adamw(ops, w0, ema0, grads, wd, gs, True, True, fp32_grad=True)
        c = run_adamw(ops, w0, ema0, grads, wd, gs, True, True, chunks=ar_chunk_bounds(n, 4))
        for k in a:
            assert torch.equal(a[k], b[k]), (cfg, k, "g16 vs fp32 operand")
            assert torch.equal(a[k], c[k]), (cfg, k, "chunked vs one pass")


# ---- (b) NCCL through the C ABI --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def comms(ops, comm):
    """One-rank communicators: full width (ncclCommInitRank) and confined to 4 CTAs (ncclCommInitRankConfig)."""
    c4 = one_rank_comm(ops.lib(), 4)
    yield {0: comm, 4: c4}
    assert ops.lib().mdt_nccl_comm_destroy(c4) == 0


def test_nccl_one_rank_allreduce_is_identity(ops, comms):
    L = ops.lib()
    n, off = 1_000_003, 64
    s = torch.cuda.Stream()
    for max_ctas, comm in comms.items():
        for dtype in (torch.float32, bf16):
            buf = torch.randn(n + off, device="cuda").to(dtype)
            before = buf.clone()
            sl = buf[off:]
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                rc = L.mdt_allreduce_grads(comm, sl.data_ptr(), n, int(dtype == bf16), s.cuda_stream)
            assert rc == 0, (max_ctas, dtype, rc)
            s.synchronize()
            assert torch.equal(buf, before), (max_ctas, dtype)
    uid = ctypes.create_string_buffer(128)
    assert L.mdt_nccl_unique_id(uid) == 0
    c = ctypes.c_void_p()
    key = bytes(uid.raw)
    assert L.mdt_nccl_comm_create(key, 0, 0, 0, ctypes.byref(c)) == MDT_ERR_ARG       # world 0
    assert L.mdt_nccl_comm_create(key, 1, 1, 0, ctypes.byref(c)) == MDT_ERR_ARG       # rank >= world
    assert L.mdt_nccl_comm_create(key, 2, 1, 4, ctypes.byref(c)) == MDT_ERR_ARG
    x = torch.zeros(64, device="cuda")
    assert L.mdt_allreduce_grads(comms[0], x.data_ptr(), 0, 0, None) == MDT_ERR_ARG
    assert L.mdt_allreduce_grads(comms[0], x.data_ptr(), -5, 0, None) == MDT_ERR_ARG
    assert L.mdt_allreduce_grads(None, x.data_ptr(), 64, 0, None) == MDT_ERR_ARG
    assert L.mdt_nccl_comm_destroy(None) == MDT_ERR_ARG


# ---- (c) TrainStep as rank 0 of two identical ranks ---------------------------------------------------------------------
@dataclass
class Call:
    lo: int
    hi: int
    dtype: torch.dtype
    stream: int
    budget: int
    snap: torch.Tensor


R, NCLS, B = 32, 1000, 4


def _draws():
    from maskdit_b200.loss import EDMLoss
    g = torch.Generator().manual_seed(0)
    images = (torch.randn(B, 4, R, R, generator=g) * 0.5).cuda()
    labels = torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), generator=g), NCLS).float().cuda()
    rnd, noise = torch.randn(B, 1, 1, 1, generator=g).cuda(), torch.randn(B, 4, R, R, generator=g).cuda()
    mnoise = torch.rand(B, (R // 2) ** 2, generator=g).cuda()

    class Draws(EDMLoss):
        """Fixed draws; a call on b < B rows (a gradient-accumulation round) gets the next b-row slice."""

        def __init__(self):
            super().__init__()
            self.k = self.j = 0

        def _randn(self, shape, device):
            b = shape[0]
            r = (self.k // 2) % (B // b)
            t = (rnd, noise)[self.k % 2][r * b:(r + 1) * b]
            self.k += 1
            assert tuple(t.shape) == tuple(shape)
            return t

        def _rand(self, shape, device):
            b = shape[0]
            r = self.j % (B // b)
            self.j += 1
            return mnoise[r * b:(r + 1) * b]

    return images, labels, Draws


def _net(use_decoder):
    from maskdit_b200.maskdit import Precond_models
    torch.manual_seed(1)
    net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=NCLS, model_type="DiT-S/2",
                                use_decoder=use_decoder, mae_loss_coef=0.1, pad_cls_token=False)
    with torch.no_grad():   # the zero-initialised tensors (adaLN, final layer) get values, so every gradient is live
        gz = torch.Generator().manual_seed(2)
        for p in net.parameters():
            if p.requires_grad and float(p.abs().sum()) == 0.0:
                p.copy_(torch.randn(p.shape, generator=gz) * 0.02)
    return net.cuda().train()


MODES = {
    "bf16-flat": dict(grad_dtype="bf16", ar_chunks=1),
    "bf16-chunked": dict(grad_dtype="bf16", ar_chunks=4),
    "fp32-flat": dict(grad_dtype="fp32", ar_chunks=1),
    "fp32-chunked": dict(grad_dtype="fp32", ar_chunks=4),
    "bf16-chunked-graph": dict(grad_dtype="bf16", ar_chunks=4, graph=True),
    "bf16-chunked-accum2": dict(grad_dtype="bf16", ar_chunks=4, grad_accum=2),
    "fp32-flat-lr-schedule": dict(grad_dtype="fp32", ar_chunks=1, reference_lr_schedule=True),
    "nodecoder-bf16-chunked": dict(grad_dtype="bf16", ar_chunks=4, use_decoder=False),
    "nodecoder-fp32-chunked": dict(grad_dtype="fp32", ar_chunks=4, use_decoder=False),
}


def _block_ranges_backward_order(net, st):
    m = net.model
    dec = [f"model.decoder_blocks.{i}." for i in range(len(m.decoder_blocks or []))]
    enc = [f"model.blocks.{i}." for i in range(len(m.blocks))]
    return [st.prefix_range(p) for p in reversed(dec)] + [st.prefix_range(p) for p in reversed(enc)]


@pytest.mark.parametrize("mode", list(MODES))
def test_train_step_world2_exchange(ops, rank0_of_two, sm_budget, clean_env, mode):
    from maskdit_b200.train_step import TrainStep, ar_chunk_bounds
    kw = dict(MODES[mode])
    use_decoder, ga = kw.pop("use_decoder", True), kw.pop("grad_accum", 1)
    chunks = kw.pop("ar_chunks")
    bf = kw["grad_dtype"] == "bf16"
    images, labels, Draws = _draws()
    net = _net(use_decoder)
    ema = copy.deepcopy(net).eval()
    ts = TrainStep(net, ema, lr=LR, weight_decay=0.01, loss_fn=Draws(), global_batch=2 * B, **kw)
    assert ts.overlap is False
    log = []
    rank0_of_two(ts, chunks, record=lambda *a: log.append(Call(*a)))
    st, n, L = ts.st, ts.st.n_train, sm_budget
    for step in (1, 2, 3):
        pre = {"w": st.w32[:n].clone(), "m": ts.m.clone(), "v": ts.v.clone(), "ema": ts.ema_st.w32[:n].clone()}
        log.clear()
        ts.step(images, labels, 0.5, 0.1, grad_accum=ga)
        torch.cuda.synchronize()
        what = f"{mode} step {step}"
        assert L.mdt_get_sm_budget() == 0, what
        assert log, what
        # 1. coverage: the chunks, in order, tiling [0, n_train) exactly once
        spans = [(c.lo, c.hi) for c in log]
        assert spans[0][0] == 0 and spans[-1][1] == n, (what, spans[:2], spans[-2:])
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:])), (what, spans)
        assert spans == ar_chunk_bounds(n, chunks), (what, spans)
        assert all(c.dtype == (bf16 if bf else torch.float32) for c in log), what
        # 2. finality: nothing writes a range after its exchange started
        for c in log:
            final = st.grad[c.lo:c.hi]
            ok = torch.equal(c.snap, final.to(bf16)) if bf else torch.equal(c.snap * 2, final)
            assert ok, (what, "range written after its exchange started", c.lo, c.hi)
        # 3. the exchange buffer holds the two-rank sum
        if bf:
            assert torch.equal(ts.g16, st.grad.to(bf16) * 2), what
        # 4. streams and SM budget: every exchange on the side stream, the whole device's grids
        for c in log:
            assert c.stream == ts.side.cuda_stream, (what, c.lo)
            assert c.budget == 0, (what, c.lo, c.budget)
        # 5. the optimizer: exactly one AdamW pass over the summed buffer
        if mode == "fp32-flat-lr-schedule" and step == 1:
            assert ts._lr_now == 0.0
        w16 = torch.empty(n, dtype=bf16, device="cuda")
        ops.adamw_ema(pre["w"], ts.g16 if bf else st.grad, pre["m"], pre["v"], pre["ema"], w16, n, ts._lr_now,
                      ts.step_count, ts.betas[0], ts.betas[1], ts.eps, ts.wd, ts.ema_decay, 1.0 / (2 * ga))
        torch.cuda.synchronize()
        for name, got, want in (("w32", st.w32[:n], pre["w"]), ("m", ts.m, pre["m"]), ("v", ts.v, pre["v"]),
                                ("ema", ts.ema_st.w32[:n], pre["ema"]), ("w16", st.w16[:n], w16)):
            assert torch.equal(got, want), (what, name, "optimizer pass differs from one AdamW pass over the sum")
    ts.close()


# ---- (d) what a C caller overlapping its own exchange relies on ---------------------------------------------------------
@pytest.mark.parametrize("use_decoder", [True, False], ids=["maskdit", "nodecoder"])
def test_backward_on_ready_reports_each_block_once_final(ops, use_decoder):
    """`mdt_backward`'s `on_ready(user, lo, hi)` reports each block's gradient range once, in backward order (decoder
    blocks, then encoder blocks), and nothing writes a range after it was reported: a clone enqueued from the callback
    on the backward's stream equals the final gradient."""
    net = _net(use_decoder)
    st = net.prepare()
    st.ensure_grad().zero_()
    ce, Lt = net._engine, net.model.num_patches
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(B, 4, R, R, generator=g) * 0.5).cuda()
    sigma = (torch.rand(B, generator=g) + 0.5).cuda()
    labels = torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), generator=g), NCLS).float().cuda()
    mask = ops.mask_indices(torch.rand(B, Lt, generator=g).cuda(), Lt // 2)
    dF = (torch.randn(B * Lt, ce.cfg.patch_dim, generator=g) * 0.1).to(bf16).cuda()
    _, ctx = ce.forward(x, sigma, labels, mask, True)
    seen = []

    def on_ready(user, lo, hi):   # runs inside mdt_backward: records, never raises
        seen.append((lo, hi, st.grad[lo:hi].clone()))

    cb, p = ops.L.GRAD_READY_FN(on_ready), ops.ptr
    rc = ce._L.mdt_backward(ce._h, p(st.w32), p(st.w16), p(st.grad), p(ctx["x_in"]), p(ctx["sigma"]),
                            p(ctx["ids_keep"]), p(ctx["ids_restore"]), p(dF), ctx["B"], ctx["T"], p(ctx["ws"]),
                            ctx["nbytes"], cb, None, ops.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0
    assert [(lo, hi) for lo, hi, _ in seen] == _block_ranges_backward_order(net, st)
    for lo, hi, snap in seen:
        assert snap.abs().max().item() > 0, (lo, hi)
        assert torch.equal(snap, st.grad[lo:hi]), ("range written after it was reported final", lo, hi)


@pytest.mark.parametrize("use_decoder", [True, False], ids=["maskdit", "nodecoder"])
def test_backward_under_sm_budget_matches_plain_step(ops, sm_budget, use_decoder):
    """A step whose persistent GEMM grids are sized for 8 SMs fewer than the device has (`mdt_set_sm_budget`, which a
    C caller sets to leave SMs to an exchange running next to the backward) computes the same gradient as a plain one:
    every block tensor within 5e-5 of its scale, the conditioning path within 1e-2 (default-mode order noise)."""
    from maskdit_b200.train_step import TrainStep
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grads = {}
    for budget in (sms - 8, 0):
        images, labels, Draws = _draws()
        ts = TrainStep(_net(use_decoder), None, lr=LR, loss_fn=Draws())
        assert sm_budget.mdt_set_sm_budget(budget) == 0
        ts.step(images, labels, 0.5, 0.1)
        torch.cuda.synchronize()
        assert sm_budget.mdt_get_sm_budget() == budget
        grads[budget] = (ts.st, ts.st.grad.clone())
    (st, budgeted), (ref_st, ref) = grads[sms - 8], grads[0]
    assert ref_st.offsets == st.offsets
    worst = 0.0
    for k, (o, cnt, _) in st.offsets.items():
        if o + cnt > st.n_train:
            continue
        a, b = budgeted[o:o + cnt], ref[o:o + cnt]
        scale = b.abs().max().item()
        err = (a - b).abs().max().item() / scale if scale > 0 else a.abs().max().item()
        cond = any(t in k for t in ("adaLN_modulation", "t_embedder", "y_embedder"))
        worst = max(worst, 0.0 if cond else err)
        assert err <= (1e-2 if cond else 5e-5), (use_decoder, k, err)
    print(f"use_decoder={use_decoder}: budgeted backward vs plain step, worst block-tensor deviation {worst:.2e}")
