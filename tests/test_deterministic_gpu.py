"""GPU: the deterministic mode (`torch.use_deterministic_algorithms(True)` -> `mdt_set_deterministic(1)`).

Kernel level: every reducing kernel against float64 torch at DESIGN §5's per-kernel tolerance (1e-3 of the output
scale), at shapes with many contributions per address, and bit-identical over three launches and over SM budgets.
Step level: TrainStep runs repeat bit for bit (loss, gradient, weights, bf16 shadow, moments, EMA), also across a
checkpoint round trip, CUDA-graph replay and SM budgets; the reference goldens hold under the mode."""
import copy
import ctypes
import io
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from support import GoldenLoss, assert_same, det_steps, lib, load, oracle_net, step_state  # noqa: E402,F401

pytestmark = pytest.mark.gpu


def _s():
    return torch.cuda.current_stream().cuda_stream


def _close(got, want, what):
    """DESIGN §5 per-kernel bound: max |error| <= 1e-3 of the float64 reference's scale."""
    got, want = got.double().cpu(), want.double().cpu()
    scale = want.abs().max().item() + 1e-30
    err = (got - want).abs().max().item() / scale
    assert err <= 1e-3, (what, err)
    return err


def _repeat(fn, n=3):
    """fn() -> tuple of output tensors, run n times: every run must give the same bits."""
    outs = [tuple(t.clone() for t in fn()) for _ in range(n)]
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a, b)
    return outs[0]


# ---- kernels -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,ld", [(1152, 1152), (1157, 1158)])
def test_colsum_ordered(lib, N, ld):
    from maskdit_b200 import ops
    assert lib.mdt_set_deterministic(1) == 0
    g = torch.Generator(device="cuda").manual_seed(0)
    M = 32768
    x32 = torch.randn(M, ld, device="cuda", generator=g) + 0.3
    x16 = x32.to(torch.bfloat16)
    init = torch.randn(N, device="cuda", generator=g)

    def run():
        o16, o32 = init.clone(), init.clone()
        ops.check(lib.mdt_colsum_bf16(x16.data_ptr(), M, N, ld, o16.data_ptr(), _s()), "colsum_bf16")
        ops.check(lib.mdt_colsum_f32(x32.data_ptr(), M, N, ld, o32.data_ptr(), _s()), "colsum_f32")
        return o16, o32

    o16, o32 = _repeat(run)
    _close(o16, init.double() + x16[:, :N].double().sum(0), "bf16")
    _close(o32, init.double() + x32[:, :N].double().sum(0), "f32")


def _ln_ref(dxm, x, scale, T):
    """float64 LN-modulate backward: g, dshift, dscale per sample."""
    xd = x.double()
    mu, var = xd.mean(1, keepdim=True), xd.var(1, unbiased=False, keepdim=True)
    rs = (var + 1e-6).rsqrt()
    xh = (xd - mu) * rs
    d = dxm.double()
    dy = d * (1 + scale.double().repeat_interleave(T, 0))
    g = rs * (dy - dy.mean(1, keepdim=True) - xh * (dy * xh).mean(1, keepdim=True))
    B = x.shape[0] // T
    return g, d.view(B, T, -1).sum(1), (d * xh).view(B, T, -1).sum(1), mu.float().flatten(), rs.float().flatten()


@pytest.mark.parametrize("T", [128, 179])
def test_ln_and_gate_backward(lib, T):
    """The fused LN + gate backward (one block per sample: T rows, also T not a multiple of the 4-row batch or of 32)
    and the standalone LN and gate backwards over 32 768+ rows at D = 1152."""
    from maskdit_b200 import ops
    assert lib.mdt_set_deterministic(1) == 0
    D, B = 1152, 32768 // 128
    M = B * T
    gen = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(M, D, device="cuda", generator=gen) * 2 + 0.5
    dxm = torch.randn(M, D, device="cuda", generator=gen).to(torch.bfloat16)
    scale = torch.randn(B, D, device="cuda", generator=gen) * 0.1
    y = torch.randn(M, D, device="cuda", generator=gen).to(torch.bfloat16)
    gate = torch.randn(B, D, device="cuda", generator=gen)
    g0 = torch.randn(M, D, device="cuda", generator=gen)
    gref, dsh_ref, dsc_ref, mu, rs = _ln_ref(dxm, x, scale, T)
    gref = gref + g0.double()

    def fused():
        g, dsh, dsc = g0.clone(), torch.zeros(B, D, device="cuda"), torch.zeros(B, D, device="cuda")
        dgate, dy = torch.zeros(B, D, device="cuda"), torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
        ops.check(lib.mdt_ln_modulate_bwd_gate(dxm.data_ptr(), x.data_ptr(), mu.data_ptr(), rs.data_ptr(),
                                               scale.data_ptr(), D, T, g.data_ptr(), 1, dsh.data_ptr(), dsc.data_ptr(),
                                               D, y.data_ptr(), gate.data_ptr(), D, dy.data_ptr(), dgate.data_ptr(), D,
                                               None, M, D, _s()), "ln_bwd_gate")
        return g, dsh, dsc, dgate, dy

    g, dsh, dsc, dgate, dy = _repeat(fused)
    _close(g, gref, "g")
    _close(dsh, dsh_ref, "dshift")
    _close(dsc, dsc_ref, "dscale")
    _close(dgate, (g.double() * y.double()).view(B, T, D).sum(1), "dgate")
    q = g.double() * gate.double().repeat_interleave(T, 0)
    # bf16 output: DESIGN §5's bound is one bf16 ulp of each element
    assert ((dy.double() - q).abs() <= q.abs() * 2.0 ** -7 + 1e-30).all()

    def standalone():
        g, dsh, dsc = g0.clone(), torch.zeros(B, D, device="cuda"), torch.zeros(B, D, device="cuda")
        ops.check(lib.mdt_ln_modulate_bwd(dxm.data_ptr(), x.data_ptr(), mu.data_ptr(), rs.data_ptr(), scale.data_ptr(),
                                          D, T, g.data_ptr(), 1, dsh.data_ptr(), dsc.data_ptr(), D, M, D, _s()),
                  "ln_modulate_bwd")
        dgate, dy = torch.zeros(B, D, device="cuda"), torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
        ops.check(lib.mdt_gate_bwd(g0.data_ptr(), y.data_ptr(), gate.data_ptr(), D, T, dy.data_ptr(), dgate.data_ptr(),
                                   D, None, M, D, _s()), "gate_bwd")
        return g, dsh, dsc, dgate

    g2, dsh2, dsc2, dgate2 = _repeat(standalone)
    _close(g2, gref, "g standalone")
    _close(dsh2, dsh_ref, "dshift standalone")
    _close(dsc2, dsc_ref, "dscale standalone")
    _close(dgate2, (g0.double() * y.double()).view(B, T, D).sum(1), "dgate standalone")


GEMMS = {
    # name: (M, N, K, a_mn, b_mn)
    "adaLN dgrad": (256, 1152, 221440, False, True),
    "encoder proj wgrad": (1152, 1152, 32768, True, True),
    "class table wgrad (ragged N)": (1152, 1000, 256, True, True),
    "final layer wgrad": (16, 512, 65536, True, True),
}


@pytest.mark.parametrize("name", list(GEMMS))
def test_accumulating_gemm_bits_under_sm_budgets(lib, name):
    from maskdit_b200 import ops
    M, N, K, a_mn, b_mn = GEMMS[name]
    gen = torch.Generator(device="cuda").manual_seed(2)
    A = (torch.randn(K, M, device="cuda", generator=gen) if a_mn else
         torch.randn(M, K, device="cuda", generator=gen)).to(torch.bfloat16)
    Bm = (torch.randn(K, N, device="cuda", generator=gen) if b_mn else
          torch.randn(N, K, device="cuda", generator=gen)).to(torch.bfloat16)
    init = torch.randn(M, N, device="cuda", generator=gen)
    ref = init.double() + (A.double().t() if a_mn else A.double()) @ (Bm.double() if b_mn else Bm.double().t())
    assert lib.mdt_set_deterministic(1) == 0
    outs = []
    for budget in (0, 66, 7):
        assert lib.mdt_set_sm_budget(budget) == 0

        def run():
            out = init.clone()
            ops.gemm(A, Bm, M, N, K, a_mn=a_mn, b_mn=b_mn, epi=ops.EPI_ATOMIC, out=out)
            return (out,)

        outs.append(_repeat(run)[0])
    assert lib.mdt_set_sm_budget(0) == 0
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    _close(outs[0], ref, name)


def test_dgelu_column_sum(lib):
    """The fc1 bias gradient of the DGELU dgrad: an ordered column sum of the stored bf16 output under the mode."""
    from maskdit_b200 import ops
    M, N, K = 32768, 4608, 1152
    gen = torch.Generator(device="cuda").manual_seed(3)
    dY = torch.randn(M, K, device="cuda", generator=gen).to(torch.bfloat16)
    W = (torch.randn(N, K, device="cuda", generator=gen) * 0.03).to(torch.bfloat16)
    hpre = torch.randn(M, N, device="cuda", generator=gen).to(torch.bfloat16)
    init = torch.randn(N, device="cuda", generator=gen)
    Wt = W.t().contiguous()   # [K, N]: the MN-major operand the dgrad reads
    assert lib.mdt_set_deterministic(1) == 0
    outs = []
    for budget in (0, 66, 7):
        assert lib.mdt_set_sm_budget(budget) == 0

        def run():
            out, cs = torch.empty(M, N, dtype=torch.bfloat16, device="cuda"), init.clone()
            ops.gemm(dY, Wt, M, N, K, b_mn=True, epi=ops.EPI_DGELU, out=out, aux=hpre, ld_aux=N, colsum=cs)
            return out, cs

        outs.append(_repeat(run))
    assert lib.mdt_set_sm_budget(0) == 0
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0]) and torch.equal(o[1], outs[0][1])
    _close(outs[0][1], init.double() + outs[0][0].double().sum(0), "colsum")


# ---- steps -------------------------------------------------------------------------------------------------------------
CASES = {
    "s2_mask50": dict(mt="DiT-S/2", R=8, ncls=10, dec=True, B=2, mask=0.5, golden="s2_train_mask"),
    "s2_nodecoder_uncond_mask30": dict(mt="DiT-S/2", R=32, ncls=0, dec=False, B=3, mask=0.3,
                                       golden="nd_s2_uncond_mask30"),
    "xl2_b8_mask50": dict(mt="DiT-XL/2", R=32, ncls=1000, dec=True, B=8, mask=0.5),
    "xl2_b8_mask0": dict(mt="DiT-XL/2", R=32, ncls=1000, dec=True, B=8, mask=0.0),
    "s2_grad_accum2": dict(mt="DiT-S/2", R=8, ncls=10, dec=True, B=4, mask=0.5, grad_accum=2),
}


@pytest.mark.parametrize("case", list(CASES))
def test_train_steps_repeat_bit_for_bit(lib, case):
    kw = dict(CASES[case])
    if kw.get("golden"):
        kw["golden"] = load(kw["golden"])
    assert_same(det_steps(**kw), det_steps(**kw))


def test_graph_replay_and_sm_budget_give_the_same_bits(lib):
    g = load("s2_train_mask")
    base = det_steps("DiT-S/2", 8, 10, True, 2, 0.5, golden=g)
    assert_same(base, det_steps("DiT-S/2", 8, 10, True, 2, 0.5, golden=g, graph=True))
    assert_same(base, det_steps("DiT-S/2", 8, 10, True, 2, 0.5, golden=g, budget=66))
    xl = det_steps("DiT-XL/2", 32, 1000, True, 8, 0.5, n=1)
    assert_same(xl, det_steps("DiT-XL/2", 32, 1000, True, 8, 0.5, n=1, budget=66))


def test_resume_equals_uninterrupted(lib):
    """Four steps in one go == two steps, a torch.save / torch.load of {model, ema, opt} and the CUDA RNG state into
    fresh objects, then two more steps: identical weights, EMA, moments and losses."""
    from maskdit_b200.train_step import TrainStep
    torch.use_deterministic_algorithms(True)
    gen = torch.Generator().manual_seed(5)
    x = (torch.randn(4, 4, 8, 8, generator=gen) * 0.5).cuda()
    lab = torch.eye(10)[torch.randint(0, 10, (4,), generator=gen)].cuda()

    def fresh():
        net = oracle_net("DiT-S/2", 8, 10, True)
        return net, TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3)

    torch.manual_seed(7)
    net, ts = fresh()
    la = [ts.step(x, lab, 0.5, 0.1).clone() for _ in range(4)]
    a = step_state(ts, la)[len(la) + 1:]   # w32, w16, m, v, ema (the gradient buffer is the last step's either way)
    torch.manual_seed(7)
    net, ts = fresh()
    lb = [ts.step(x, lab, 0.5, 0.1).clone() for _ in range(2)]
    buf = io.BytesIO()
    torch.save({"model": net.state_dict(), "ema": ts.ema.state_dict(), "opt": ts.state_dict(),
                "rng": torch.cuda.get_rng_state()}, buf)
    del net, ts
    torch.cuda.empty_cache()
    buf.seek(0)
    ck = torch.load(buf, weights_only=False)
    net = oracle_net("DiT-S/2", 8, 10, True)
    net.load_state_dict(ck["model"])
    ema = copy.deepcopy(net).eval()
    ema.load_state_dict(ck["ema"])
    ts2 = TrainStep(net, ema, lr=1e-3)
    ts2.load_state_dict(ck["opt"])
    torch.cuda.set_rng_state(ck["rng"])
    lb += [ts2.step(x, lab, 0.5, 0.1).clone() for _ in range(2)]
    assert_same(la, lb)
    assert_same(a, step_state(ts2, lb)[len(lb) + 1:])


def test_default_and_deterministic_gradients_differ_by_order_noise_only(lib):
    """One XL/2 backward (golden xl2_c1_grads inputs) in both modes: the gradients differ within the order noise the
    default mode's fp32 atomics produce between two of its own runs (DESIGN §5)."""
    g = load("xl2_c1_grads")
    net = oracle_net("DiT-XL/2", 32, 1000, True)
    st = net.prepare()
    grads = []
    for det in (False, True, False):
        torch.use_deterministic_algorithms(det)
        st.ensure_grad().zero_()
        GoldenLoss(g)(net, g["images"].cuda(), g["labels"].cuda(), mask_ratio=0.5, mae_loss_coef=0.1).mean().backward()
        grads.append(st.grad.clone())
    torch.use_deterministic_algorithms(False)
    worst = {}
    for k, (o, n, _) in st.offsets.items():
        if o + n > st.n_train:
            continue
        ref = grads[0][o:o + n]
        scale = ref.abs().max().item() + 1e-30
        cond = any(t in k for t in ("adaLN_modulation", "t_embedder", "y_embedder"))
        noise = (grads[2][o:o + n] - ref).abs().max().item() / scale      # default against default
        err = (grads[1][o:o + n] - ref).abs().max().item() / scale        # deterministic against default
        # the bounds check_c_driver_matches_engine uses for the default mode's order noise
        assert err <= (1e-2 if cond else 5e-5), (k, err, noise)
        worst[k] = (err, noise)
    k = max(worst, key=lambda k: worst[k][0])
    print("default vs deterministic: worst", k, worst[k])


def test_sampler_repeats_bit_for_bit(lib):
    from maskdit_b200.sampler import edm_sampler
    torch.use_deterministic_algorithms(True)
    net = oracle_net("DiT-XL/2", 32, 1000, True).eval()
    gen = torch.Generator().manual_seed(9)
    lat = torch.randn(4, 4, 32, 32, generator=gen).cuda()
    lab = torch.eye(1000)[torch.randint(0, 1000, (4,), generator=gen)].cuda()
    with torch.no_grad():
        a = edm_sampler(net, lat, lab, cfg_scale=1.5, num_steps=3)
        b = edm_sampler(net, lat, lab, cfg_scale=1.5, num_steps=3)
    assert torch.equal(a, b)


# ---- reference goldens under the mode, at the existing tests' bounds ------------------------------------------------------
GOLDEN_TESTS = {
    "xl2_c1_grads": ("test_model_gpu_extra", "test_xl2_r32_loss_and_all_grads_vs_reference_golden", ()),
    "s2_train_mask": ("test_model_gpu", "test_train_loss_and_grads_vs_reference_golden", ("s2_train_mask",)),
    "nd_xl2_grads": ("test_nodecoder_gpu", "test_loss_D_and_grads_vs_reference_golden", ("nd_xl2_grads",)),
    "geo_h2_mask50": ("test_geometry_gpu", "test_loss_D_and_grads_vs_reference_golden", ("geo_h2_mask50",)),
    "geo_s8_mask50": ("test_geometry_gpu", "test_loss_D_and_grads_vs_reference_golden", ("geo_s8_mask50",)),
}


@pytest.mark.parametrize("name", list(GOLDEN_TESTS))
def test_reference_goldens_under_the_mode(lib, name):
    import importlib
    mod, fn, args = GOLDEN_TESTS[name]
    torch.use_deterministic_algorithms(True)
    getattr(importlib.import_module(mod), fn)(*args)
    assert lib.mdt_get_deterministic() == 1
