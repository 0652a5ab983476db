"""GPU: activation recomputation (`TrainStep(recompute_blocks=...)`, `mdt_model_set_recompute`).

Under `torch.use_deterministic_algorithms(True)` a step at any recompute count gives the bits of r = 0 (loss, gradient,
weights, bf16 shadow, moments, EMA): the re-run forward kernels neither split K nor use atomics.  In the default mode a
fully recomputed step meets the reference goldens at the usual bounds.  mdt_backward refuses a workspace laid out for
another count.  And the decoder-less DiT-XL/2 trains at batch 256 without masking on one 80 GB card, choosing the count
itself, with the gradients of 2 x 128 gradient accumulation."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from support import (LOSS_TOL, GoldenLoss, assert_same, check_grads, det_steps, lib, load,  # noqa: E402,F401
                     oracle_net, rel_l2)

pytestmark = pytest.mark.gpu


# (case, depth, depth + dec_depth): the steps of support.det_steps on existing goldens' shapes
CASES = {
    "s2_mask50": (dict(mt="DiT-S/2", R=8, ncls=10, dec=True, B=2, mask=0.5, golden="s2_train_mask", n=2), 12, 20),
    "xl2_c1": (dict(mt="DiT-XL/2", R=32, ncls=1000, dec=True, B=2, mask=0.5, golden="xl2_c1_grads", n=1), 28, 36),
    "s2_nodecoder_nomask": (dict(mt="DiT-S/2", R=8, ncls=10, dec=False, B=2, mask=0.0, golden="nd_s2_train_nomask",
                                 n=2), 12, 12),
    "s2_uncond_mask30": (dict(mt="DiT-S/2", R=32, ncls=0, dec=True, B=3, mask=0.3, golden="s2_uncond_mask30", n=2),
                         12, 20),
    "s2_nodecoder_uncond_mask30": (dict(mt="DiT-S/2", R=32, ncls=0, dec=False, B=3, mask=0.3,
                                        golden="nd_s2_uncond_mask30", n=2), 12, 12),
    "s2_grad_accum2": (dict(mt="DiT-S/2", R=8, ncls=10, dec=True, B=4, mask=0.5, grad_accum=2, n=2), 12, 20),
    "s2_graph": (dict(mt="DiT-S/2", R=8, ncls=10, dec=True, B=2, mask=0.5, golden="s2_train_mask", n=2, graph=True),
                 12, 20),
}


@pytest.mark.parametrize("case", list(CASES))
def test_recomputed_steps_are_bit_identical(lib, case):
    kw, depth, nb = CASES[case]
    kw = dict(kw)
    if kw.get("golden"):
        kw["golden"] = load(kw["golden"])
    base = det_steps(**kw, recompute_blocks=0)
    for r in sorted({1, depth, nb}):
        assert_same(base, det_steps(**kw, recompute_blocks=r))


@pytest.mark.parametrize("name,mt,R,ncls,dec", [("s2_train_mask", "DiT-S/2", 8, 10, True),
                                                ("xl2_c1_grads", "DiT-XL/2", 32, 1000, True),
                                                ("nd_xl2_grads", "DiT-XL/2", 32, 1000, False)])
def test_full_recompute_vs_reference_golden(lib, name, mt, R, ncls, dec):
    """Default mode, every block recomputed: loss and gradients within the bounds of the r = 0 golden tests."""
    torch.use_deterministic_algorithms(False)
    g = load(name)
    net = oracle_net(mt, R, ncls, dec)
    net.prepare()
    ce = net._engine
    ce.recompute = ce.num_blocks
    lf = GoldenLoss(g)
    loss = lf(net, g["images"].cuda(), g["labels"].cuda(), mask_ratio=float(g["mask_ratio"]), mae_loss_coef=0.1)
    assert ce.recompute_blocks == ce.num_blocks
    assert torch.allclose(loss.cpu(), g["loss"], rtol=LOSS_TOL), (loss, g["loss"])
    loss.mean().backward()
    check_grads(net, g, what=f"{name} full recompute")


def _raw_backward(ce, ctx, dF):
    """mdt_backward at the handle's current count (CEngine.backward would set the context's count first)."""
    from maskdit_b200 import ops
    st, p = ce.store, ops.ptr
    return ce._L.mdt_backward(ce._h, p(st.w32), p(st.w16), p(st.grad), p(ctx["x_in"]), p(ctx["sigma"]),
                              p(ctx["ids_keep"]), p(ctx["ids_restore"]), p(dF), ctx["B"], ctx["T"], p(ctx["ws"]),
                              ctx["nbytes"], ops.L.GRAD_READY_FN(), None, ops.stream_ptr())


def test_backward_refuses_a_workspace_of_another_count(lib):
    torch.use_deterministic_algorithms(False)
    net = oracle_net("DiT-S/2", 8, 10, True)
    st = net.prepare()
    st.ensure_grad().zero_()
    ce = net._engine
    gen = torch.Generator().manual_seed(3)
    x = (torch.randn(2, 4, 8, 8, generator=gen) * 0.5).cuda()
    sigma = (torch.rand(2, generator=gen) + 0.5).cuda()
    lab = torch.eye(10)[:2].cuda()
    dF = (torch.randn(2 * 16, 16, generator=gen) * 0.1).to(torch.bfloat16).cuda()
    for fwd_r, bwd_rs in ((0, (1, 2, 20)), (1, (0, 2)), (20, (0, 19))):
        ce.recompute = fwd_r
        _, ctx = ce.forward(x, sigma, lab, None, True)
        assert ctx["recompute"] == fwd_r
        for r in bwd_rs:
            ce.set_recompute(r)
            assert _raw_backward(ce, ctx, dF) == -1, (fwd_r, r)
        ce.set_recompute(fwd_r)
        assert _raw_backward(ce, ctx, dF) == 0, fwd_r
    # at r > 0 a workspace other than the last saving forward's is refused as well
    ce.recompute = 2
    _, ctx_a = ce.forward(x, sigma, lab, None, True)
    _, ctx_b = ce.forward(x, sigma, lab, None, True)
    assert _raw_backward(ce, ctx_a, dF) == -1 and _raw_backward(ce, ctx_b, dF) == 0
    torch.cuda.synchronize()


class _SameDraws:
    """EDMLoss whose (sigma, noise) draws are consecutive row slices of fixed tensors: one batch of B and two
    micro-batches of B/2 see the same randoms for the same samples."""

    def __new__(cls, rnd, nz):
        from maskdit_b200.loss import EDMLoss

        class _L(EDMLoss):
            off, k = 0, 0

            def _randn(self, shape, device):
                n = shape[0]
                t = (rnd if self.k % 2 == 0 else nz)[self.off:self.off + n]
                self.k += 1
                if self.k % 2 == 0:
                    self.off += n
                return t.reshape(shape).contiguous()

        return _L()


def test_nodecoder_xl2_batch256_unmasked_fits_one_card(lib):
    """DiT-XL/2 without the decoder, no mask, batch 256: 87.9 GB of workspace at r = 0.  TrainStep picks r > 0 itself,
    the step is finite and stays within the card, and its gradient equals that of 2 x 128 accumulation at r = 0 within
    the default mode's summation-order noise."""
    from maskdit_b200.train_step import TrainStep
    torch.use_deterministic_algorithms(False)
    torch.cuda.empty_cache()          # the workspace needs the blocks earlier tests left in the caching allocator
    total = torch.cuda.get_device_properties(0).total_memory
    net = oracle_net("DiT-XL/2", 32, 1000, False)
    ts = TrainStep(net, None, lr=0.0)
    B = 256
    gen = torch.Generator().manual_seed(11)
    x = (torch.randn(B, 4, 32, 32, generator=gen) * 0.5).cuda()
    lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=gen), 1000).float().cuda()
    rnd, nz = torch.randn(B, 1, 1, 1, generator=gen).cuda(), torch.randn(B, 4, 32, 32, generator=gen).cuda()
    assert ts.recompute_blocks == 0
    torch.cuda.reset_peak_memory_stats()
    ts.loss_fn = _SameDraws(rnd, nz)
    loss = ts.step(x, lab, 0.0, 0.1)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    r = ts.recompute_blocks
    print(f"batch 256: recompute_blocks {r}, peak allocated {peak / 2**30:.1f} GiB of {total / 2**30:.1f} GiB")
    assert 0 < r <= 28
    assert torch.isfinite(loss).all()
    assert peak < total
    g_full = ts.st.grad.clone()
    ts.loss_fn = _SameDraws(rnd, nz)
    loss2 = ts.step(x, lab, 0.0, 0.1, grad_accum=2)
    assert ts.recompute_blocks == 0   # a micro-batch of 128 fits without recomputation
    g_acc = ts.st.grad.clone() / 2    # the sum of two micro-batch mean-loss gradients
    assert torch.allclose(loss, loss2, rtol=1e-4), (loss - loss2).abs().max()
    worst = (0.0, "")
    for k, (o, n, _) in ts.st.offsets.items():
        if o + n > ts.st.n_train:
            continue
        e = rel_l2(g_full[o:o + n], g_acc[o:o + n])
        worst = max(worst, (e, k))
        assert e <= 1e-2, (k, e)
    print("batch 256 recomputed vs 2 x 128 accumulated: worst gradient rel-L2", worst)
    del ts, net, g_full, g_acc
    torch.cuda.empty_cache()
