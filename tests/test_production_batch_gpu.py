"""GPU: the XL/2 training step at production batch.

The benchmarked workload is DiT-XL/2 with the decoder at 256 px, mask 0.5, batch 256 per GPU (M_e = 32 768 encoder
rows, M_d = 65 536 decoder rows); at 512 px the batch is 64 per card (the same row counts at T = 512, L = 1024).  The
model-level goldens validate batch 2 (M = 256 token rows).  This file carries that validation to production batch in
three cases: (a) XL/2 + decoder at 32 x 32 latents, B 256; (b) XL/2 + decoder at 64 x 64 latents, B 64; (c) the
decoder-less XL/2 at 32 x 32 latents, B 256.

1. Every distinct `mdt_gemm_bf16` launch of one training step (forward + `mdt_backward`, as csrc/driver.cu issues them)
   at its real size, with bf16 operands, against a float64 matmul of the same values.  The list is proven complete by
   the library's own launch profile of a real step.  The accumulating launches (wgrads split into k-slices, the
   stream-K adaLN and timestep dgrads) run from a non-zero output in the default mode and in the deterministic mode.
2. The full batch through `CEngine.forward(save=True)` (every block recomputed) + `CEngine.backward` against the same
   rows run as chunks of B = 2 at r = 0: every output row and per-row loss bit for bit, every gradient tensor against
   the sum of the chunk gradients; and the unmasked eval forward at the sampler's batch (64 with CFG: 128 rows) against
   batch-2 runs bit for bit.  The GEMMs of the production plans are validated by part 1 and the batch-2 runs by the
   small-batch goldens, so this reaches every other kernel at production batch: the attention grids, LN / gate
   backwards, patch-embedding and mask-token partials, column sums, recomputation and the conditioning path.

Bounds are the per-kernel ones of test_kernels_gpu.py (part 1) and DESIGN.md §5 (part 2).  The file keeps its device
memory well below a shared card's: no r = 0 workspace at B = 256, float64 references built in blocks."""
import collections
import ctypes
import gc
import os
import sys
import time
import types

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
f64, bf16 = torch.float64, torch.bfloat16

MT, NCLS, MASK_RATIO, CHUNK = "DiT-XL/2", 1000, 0.5, 2
# name -> (use_decoder, latent resolution, batch per GPU)
CASES = {"a": (True, 32, 256), "b": (True, 64, 64), "c": (False, 32, 256)}
EVAL_B = 64                       # the sampler's batch; with CFG the network runs 2 * EVAL_B rows
# deterministic mode, max-abs of each gradient tensor's scale (DESIGN.md §5): block tensors, whose wgrads contract the
# 32 768 / 65 536 token rows in one k-slice (measured 1.3e-4), and the conditioning path (measured 5.9e-7)
DET_BLOCK_GRAD_TOL, DET_COND_GRAD_TOL = 3e-4, 1e-5
BLOCK_GRAD_TOL, COND_GRAD_TOL = 5e-5, 1e-2   # default mode: check_c_driver_matches_engine's bounds
COND = ("adaLN_modulation", "t_embedder", "y_embedder")
EPI_STORE, EPI_GELU, EPI_GATE_RESID, EPI_DGELU, EPI_ATOMIC = range(5)
EPI_NAME = {EPI_STORE: "store", EPI_GELU: "gelu", EPI_GATE_RESID: "gate_resid", EPI_DGELU: "dgelu",
            EPI_ATOMIC: "atomic"}


@pytest.fixture
def lib():
    """The library; the torch flag, the library setting and the SM budget are restored afterwards."""
    from maskdit_b200 import _lib
    Lb = _lib.lib()
    det, budget, flag = Lb.mdt_get_deterministic(), Lb.mdt_get_sm_budget(), torch.are_deterministic_algorithms_enabled()
    assert Lb.mdt_set_sm_budget(0) == 0
    yield Lb
    torch.use_deterministic_algorithms(flag)
    assert Lb.mdt_set_deterministic(det) == 0 and Lb.mdt_set_sm_budget(budget) == 0


@pytest.fixture(scope="module", autouse=True)
def _report():
    """Wall time and peak allocated device memory of the whole file."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    torch.cuda.synchronize()
    print(f"\n{os.path.basename(__file__)}: wall {time.time() - t0:.0f} s, peak allocated "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB on {torch.cuda.get_device_name()}")


def _net(dec, R):
    """The training network with test_model_gpu.build()'s weights (the oracle's seeded state dict, every tensor the
    reference zero-inits randomised)."""
    from maskdit_b200.maskdit import Precond_models
    from oracle import maskdit_oracle as O
    cfg = O.Cfg(model_type=MT, img_resolution=R, num_classes=NCLS, use_decoder=dec)
    net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=NCLS, model_type=MT, use_decoder=dec,
                                mae_loss_coef=0.1, pad_cls_token=False)
    net.load_state_dict(O.make_state_dict(cfg, 1), strict=True)
    return net.cuda().train()


@pytest.fixture(scope="module", params=sorted(CASES))
def case(request):
    """One production case: the network, its step driver and flat store, and seeded inputs of one training step
    (labels with about 10 % dropped rows, sigma drawn as in training, a 0.5 mask, a random bf16 dF)."""
    from maskdit_b200 import ops
    from maskdit_b200.engine import Engine
    dec, R, B = CASES[request.param]
    gc.collect()
    torch.cuda.empty_cache()
    net = _net(dec, R)
    st = net.prepare()
    cfg = net._cfg()
    L, pd = cfg.num_patches, cfg.patch_dim
    T = int(L * (1 - MASK_RATIO))
    gen = torch.Generator().manual_seed(1000 + R + B + dec)
    y = torch.randn(B, 4, R, R, generator=gen) * 0.5
    labels = F.one_hot(torch.randint(0, NCLS, (B,), generator=gen), NCLS).float()
    labels[torch.rand(B, generator=gen) < 0.1] = 0
    sigma = (torch.randn(B, generator=gen) * 1.2 - 1.2).exp()
    x = y + torch.randn(B, 4, R, R, generator=gen) * sigma.view(-1, 1, 1, 1)
    noise = torch.rand(B, L, generator=gen)
    dF = (torch.randn(B * L, pd, generator=gen) * 0.1).to(bf16)
    c = types.SimpleNamespace(name=request.param, net=net, ce=net._engine, st=st, cfg=cfg, spec=Engine(cfg, st),
                              B=B, T=T, L=L, pd=pd, y=y.cuda(), x=x.cuda(), labels=labels.cuda(), sigma=sigma.cuda(),
                              dF=dF.cuda())
    c.md = ops.mask_indices(noise.cuda(), T)
    yield c
    c.__dict__.clear()
    del net, st
    gc.collect()
    torch.cuda.empty_cache()


# ---- 1. every GEMM launch of the step against float64 -----------------------------------------------------------------
def _gemm(name, M, N, K, *, a_mn=False, b_mn=False, epi=EPI_STORE, out32=True, bias=False, resid=False, aux=False,
          gate=None, colsum=False):
    """One mdt_gemm_bf16 launch as the step driver issues it; `gate` = (first column in the [B, NA] modulation buffer,
    ld_gate, rows_per_group)."""
    key = (M, N, K, a_mn, b_mn, epi, out32, bias, resid, aux, gate[1:] if gate else None, colsum)
    return types.SimpleNamespace(name=name, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, epi=epi, out32=out32, bias=bias,
                                 resid=resid, aux=aux, gate=gate, colsum=colsum, key=key)


def _wgrad(name, n_out, k_in, tokens):
    return _gemm(name, n_out, k_in, tokens, a_mn=True, b_mn=True, epi=EPI_ATOMIC)


def step_gemms(cfg, NA, mod_off, B, T):
    """Every mdt_gemm_bf16 launch of one masked training step with every block recomputed (`mdt_forward(save = 1)` +
    `mdt_backward`, csrc/driver.cu), repeats included: each block's GEMMs once per block, a recomputed block's four
    forward GEMMs a second time in the backward.  `mod_off(tag, i)`: column of block i's modulation in the [B, NA]
    buffer."""
    D, Dd, L, pd, nc = cfg.hidden, cfg.dec_hidden, cfg.num_patches, cfg.patch_dim, cfg.num_classes
    Me, Md = B * T, B * L
    Kp = (nc + 7) // 8 * 8

    def block_fwd(tag, i, M, d, h4, rows):
        o = mod_off(tag, i)
        return [_gemm(f"{tag} qkv", M, 3 * d, d, out32=False, bias=True),
                _gemm(f"{tag} proj", M, d, d, epi=EPI_GATE_RESID, bias=True, resid=True, aux=True,
                      gate=(o + 2 * d, NA, rows)),
                _gemm(f"{tag} fc1", M, h4, d, epi=EPI_GELU, out32=False, bias=True, aux=True),
                _gemm(f"{tag} fc2", M, d, h4, epi=EPI_GATE_RESID, bias=True, resid=True, aux=True,
                      gate=(o + 5 * d, NA, rows))]

    def block_bwd(tag, M, d, h4):
        return [_gemm(f"{tag} fc2 dgrad", M, h4, d, b_mn=True, epi=EPI_DGELU, out32=False, aux=True, colsum=True),
                _wgrad(f"{tag} fc2 wgrad", d, h4, M),
                _gemm(f"{tag} fc1 dgrad", M, d, h4, b_mn=True, out32=False),
                _wgrad(f"{tag} fc1 wgrad", h4, d, M),
                _gemm(f"{tag} proj dgrad", M, d, d, b_mn=True, out32=False),
                _wgrad(f"{tag} proj wgrad", d, d, M),
                _gemm(f"{tag} qkv dgrad", M, d, 3 * d, b_mn=True, out32=False),
                _wgrad(f"{tag} qkv wgrad", 3 * d, d, M)]

    stacks = [("enc", cfg.depth, Me, D, cfg.mlp_hidden, T)]
    if Dd:
        stacks.append(("dec", cfg.dec_depth, Md, Dd, cfg.dec_mlp_hidden, L))
    out = [_gemm("t_embedder.mlp.0", B, D, 256, bias=True), _gemm("t_embedder.mlp.2", B, D, D, bias=True)]
    if nc:
        out.append(_gemm("y_embedder", B, D, Kp, resid=True))
    out.append(_gemm("adaLN (all heads)", B, NA, D, bias=True))
    for tag, n, M, d, h4, rows in stacks:
        if tag == "dec":
            out.append(_gemm("decoder_layer", Me, Dd, D, bias=True))
        for i in range(n):
            out += block_fwd(tag, i, M, d, h4, rows)
    Mf, Df = (Md, Dd) if Dd else (Me, D)
    out.append(_gemm("final_layer", Mf, pd, Df, bias=True))
    # backward: final layer, decoder blocks, decoder layer, encoder blocks (each recomputed block's forward re-run
    # inside), then the adaLN projections and the conditioning MLPs
    out += [_wgrad("final_layer wgrad", pd, Df, Mf), _gemm("final_layer dgrad", Mf, Df, pd, b_mn=True, out32=False)]
    for tag, n, M, d, h4, rows in reversed(stacks):
        for i in reversed(range(n)):
            out += block_fwd(tag, i, M, d, h4, rows) + block_bwd(tag, M, d, h4)
        if tag == "dec":
            out += [_wgrad("decoder_layer wgrad", Dd, D, Me),
                    _gemm("decoder_layer dgrad", Me, D, Dd, b_mn=True, out32=False)]
    out += [_wgrad("adaLN wgrad", NA, D, B),
            _gemm("adaLN dgrad", B, D, NA, b_mn=True, epi=EPI_ATOMIC)]
    if nc:
        out.append(_wgrad("y_embedder wgrad", D, Kp, B))
    out += [_wgrad("t_embedder.mlp.2 wgrad", D, D, B),
            _gemm("t_embedder.mlp.2 dgrad", B, D, D, b_mn=True, epi=EPI_ATOMIC),
            _wgrad("t_embedder.mlp.0 wgrad", D, 256, B)]
    return out


def _profiled_step_flops(Lb, c):
    """2 M N K of every mdt_gemm_bf16 launch of one real step of case `c` (every block recomputed), read from the
    library's launch profile."""
    ce = c.ce
    ce.recompute = ce.num_blocks
    Lb.mdt_gemm_profile_enable(1)
    try:
        Fo, ctx = ce.forward(c.x, c.sigma, c.labels, c.md, True)
        assert ctx["recompute"] == ce.num_blocks
        c.st.ensure_grad().zero_()
        ce.backward(ctx, c.dF)
        torch.cuda.synchronize()
    finally:
        Lb.mdt_gemm_profile_enable(0)
        ce.recompute = None
    del Fo, ctx
    n = Lb.mdt_gemm_profile_read(None, None, 0)
    fl = (ctypes.c_double * n)()
    assert Lb.mdt_gemm_profile_read(None, fl, n) == n
    return [int(v) for v in fl]


def _rb(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(bf16)


class _Err:
    """Worst |got - want| and largest |want| of one output, gathered over row blocks."""

    def __init__(self, tol):
        self.tol, self.err, self.scale = tol, 0.0, 0.0

    def add(self, got, want):
        got = got.double()
        assert torch.isfinite(got).all(), "non-finite output"
        self.err = max(self.err, (got - want).abs().max().item())
        self.scale = max(self.scale, want.abs().max().item())

    @property
    def ratio(self):
        return self.err / (self.tol * (self.scale + 1e-30))


def _dgelu(h):
    hr = h.detach().requires_grad_(True)
    F.gelu(hr, approximate="tanh").sum().backward()
    return hr.grad


def check_launch(ops, Lb, g, seed, me_md):
    """Launch `g` at its real size on seeded bf16 operands (gate: column slices of a [B, NA] buffer, ld_gate = NA) and
    compare with float64 in row blocks: 1e-3 of the output scale for fp32 outputs, one bf16 ulp (2^-8) for bf16
    outputs, 2^-7 for the GELU / dGELU outputs.  Accumulating launches start from a non-zero output and run in the
    default mode (k-slices on this device) and in the deterministic mode (one slice, repeated bit for bit); so does the
    dGELU's fused column sum.  Returns (k-slices in the default mode, {output: worst error / bound})."""
    from maskdit_b200 import _lib
    torch.manual_seed(seed)
    M, N, K = g.M, g.N, g.K
    A = _rb(K, M) if g.a_mn else _rb(M, K)
    Bw = _rb(K, N, scale=K ** -0.5) if g.b_mn else _rb(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device="cuda") if g.bias else None
    resid = torch.randn(M, N, device="cuda") if g.resid else None
    gate, gbuf = None, None
    if g.gate:
        col, ld, rows = g.gate
        assert M % rows == 0 and col + N <= ld
        gbuf = torch.randn(M // rows, ld, device="cuda")
        gate = gbuf[:, col:]
    hpre = _rb(M, N) if g.epi == EPI_DGELU else None
    out0 = torch.randn(M, N, device="cuda") * 0.5 if g.epi == EPI_ATOMIC else None
    cs0 = torch.randn(N, device="cuda") if g.colsum else None
    odt = torch.float32 if g.out32 else bf16

    def run():
        out = out0.clone() if out0 is not None else torch.full((M, N), float("nan"), device="cuda", dtype=odt)
        aux = None
        if g.epi in (EPI_GELU, EPI_GATE_RESID):
            aux = torch.full((M, N), float("nan"), device="cuda", dtype=bf16)
        elif g.epi == EPI_DGELU:
            aux = hpre
        cs = cs0.clone() if cs0 is not None else None
        ops.gemm(A, Bw, M, N, K, a_mn=g.a_mn, b_mn=g.b_mn, epi=g.epi, out=out, bias=bias,
                 aux=aux, ld_aux=N if aux is not None else 0, resid=resid, ld_resid=N if resid is not None else 0,
                 gate=gate, ld_gate=g.gate[1] if g.gate else 0, rows_per_group=g.gate[2] if g.gate else 1,
                 colsum=cs)
        return out, (aux if g.epi in (EPI_GELU, EPI_GATE_RESID) else None), cs

    split = g.epi == EPI_ATOMIC or g.colsum   # launches whose result depends on the library mode
    runs = {}
    assert Lb.mdt_set_deterministic(0) == 0
    splits = _lib.gemm_plan(M, N, K, a_mn=g.a_mn, b_mn=g.b_mn, epi=g.epi)["splits"] if g.epi == EPI_ATOMIC else 1
    if g.epi == EPI_ATOMIC and K in me_md:
        # the token-contracting wgrads: test_host.py pins more than one k-slice for them (132 SMs); so on this device
        assert splits > 1, (g.name, M, N, K, splits)
    runs["default"] = run()
    if split:
        assert Lb.mdt_set_deterministic(1) == 0
        try:
            if g.epi == EPI_ATOMIC:
                assert _lib.gemm_plan(M, N, K, a_mn=g.a_mn, b_mn=g.b_mn, epi=g.epi)["splits"] == 1
            runs["deterministic"] = run()
            again = run()
        finally:
            assert Lb.mdt_set_deterministic(0) == 0
        for a, b in zip(runs["deterministic"], again):
            if a is not None:
                assert torch.equal(a, b), f"{g.name}: the deterministic mode does not repeat bit for bit"
        del again
    torch.cuda.synchronize()

    tol_out = 2 ** -7 if g.epi in (EPI_GELU, EPI_DGELU) else (1e-3 if g.out32 else 2 ** -8)
    errs = {m: {"out": _Err(tol_out)} for m in runs}
    for m in runs:
        if g.epi in (EPI_GELU, EPI_GATE_RESID):
            errs[m]["aux"] = _Err(2 ** -8)
        if g.colsum:
            errs[m]["colsum"] = _Err(1e-4)
    csum = {m: cs0.double().clone() for m in runs} if g.colsum else None
    rows = max(64, min(M, (1 << 24) // N))
    kc = max(64, min(8192, (1 << 24) // rows) // 64 * 64)
    for r0 in range(0, M, rows):
        r1 = min(M, r0 + rows)
        acc = torch.zeros(r1 - r0, N, dtype=f64, device="cuda")
        for k0 in range(0, K, kc):
            k1 = min(K, k0 + kc)
            a = A[k0:k1, r0:r1].t() if g.a_mn else A[r0:r1, k0:k1]
            b = Bw[k0:k1] if g.b_mn else Bw[:, k0:k1].t()
            acc += a.double() @ b.double()
        if bias is not None:
            acc += bias.double()
        for m, (out, aux, _) in runs.items():
            e = errs[m]
            o = out[r0:r1]
            if g.epi == EPI_STORE:
                e["out"].add(o, acc + resid[r0:r1].double() if resid is not None else acc)
            elif g.epi == EPI_GELU:
                e["aux"].add(aux[r0:r1], acc)
                e["out"].add(o, F.gelu(aux[r0:r1].double(), approximate="tanh"))
            elif g.epi == EPI_GATE_RESID:
                e["aux"].add(aux[r0:r1], acc)
                gr = gbuf[r0 // g.gate[2]:(r1 - 1) // g.gate[2] + 1, g.gate[0]:g.gate[0] + N].double()
                gr = gr.repeat_interleave(g.gate[2], 0)[r0 % g.gate[2]:][:r1 - r0]
                e["out"].add(o, resid[r0:r1].double() + gr * acc)
            elif g.epi == EPI_DGELU:
                e["out"].add(o, acc * _dgelu(hpre[r0:r1].double()))
                csum[m] += o.double().sum(0)
            else:
                e["out"].add(o, out0[r0:r1].double() + acc)
        del acc
    if g.colsum:
        for m, (_, _, cs) in runs.items():
            errs[m]["colsum"].add(cs, csum[m])
    report = {}
    for m, d in errs.items():
        for what, e in d.items():
            report[f"{what}" if m == "default" else f"{what} ({m})"] = e.ratio
            assert e.err <= e.tol * e.scale, \
                f"{g.name} [{m}] {what}: max_abs {e.err:.4g} > {e.tol:.3g} * scale {e.scale:.4g}"
    del runs, A, Bw, resid, gbuf, hpre, out0
    return splits, report


def test_every_gemm_launch_of_the_step_vs_float64(case, lib):
    """The launch list of `step_gemms` is the step driver's: the multiset of 2 M N K over one real step's launches
    (the library's launch profile) equals the list's, so a GEMM the driver gains later fails here until it is listed.
    Then every distinct launch against float64 at its real size, with the k-slice counts of this device's plans."""
    from maskdit_b200 import ops
    torch.use_deterministic_algorithms(False)
    c = case
    spec = c.spec

    def mod_off(tag, i):
        return (spec.enc if tag == "enc" else spec.dec)[i].mod_off

    gemms = step_gemms(c.cfg, c.ce.NA, mod_off, c.B, c.T)
    seen = _profiled_step_flops(lib, c)
    want = collections.Counter(2 * g.M * g.N * g.K for g in gemms)
    got = collections.Counter(seen)
    assert got == want, (f"case {c.name}: launches the list misses {dict(got - want)}, "
                         f"listed but not launched {dict(want - got)}")
    distinct = {}
    for g in gemms:
        distinct.setdefault(g.key, g)
    me_md = (c.B * c.T, c.B * c.L)
    print(f"\ncase {c.name}: {len(seen)} launches in one step, {len(distinct)} distinct, "
          f"{torch.cuda.get_device_properties(0).multi_processor_count} SMs")
    worst = 0.0
    for i, g in enumerate(distinct.values()):
        splits, rep = check_launch(ops, lib, g, 7000 + i, me_md)
        worst = max([worst, *rep.values()])
        print(f"  {g.name:24s} M {g.M:6d} N {g.N:6d} K {g.K:6d} {EPI_NAME[g.epi]:10s} "
              f"{'fp32' if g.out32 else 'bf16'} k-slices {splits:2d}  err/bound " +
              ", ".join(f"{k} {v:.3f}" for k, v in rep.items()))
        torch.cuda.empty_cache()
    print(f"case {c.name}: worst error / bound {worst:.3f}")


# ---- 2. every row and every gradient at production batch against chunks of 2 -------------------------------------
def _loss(ops, c, Fo, rows):
    """Per-row loss of `mdt_edm_loss` for the samples `rows` (EDM + MAE terms)."""
    n = rows.stop - rows.start
    return ops.edm_loss(Fo, c.x[rows], c.y[rows], c.sigma[rows], c.md["mask"][rows].contiguous(),
                        torch.ones(n, device="cuda"), 0.5, 0.1, c.cfg.patch, want_dF=False)[0]


@pytest.mark.parametrize("mode", ["deterministic", "default"])
def test_rows_and_gradients_vs_chunks_of_2(case, lib, mode):
    """The full batch with every block recomputed against the same rows as chunks of B = 2 at r = 0 (each chunk with
    its rows of ids_keep / ids_restore and of dF): every row of F and of the per-row loss bit for bit (the forward never
    splits K), and every trainable gradient tensor against the sum of the chunk gradients.  The backward is linear in
    dF, so no loss scaling enters.  Deterministic mode: the per-sample quantities are computed in an order fixed by the
    per-sample shape, so only the fp32 order of the cross-sample sums differs: max-abs <= 1e-5 of each tensor's scale
    on the conditioning path, 3e-4 on the block tensors (their one-slice wgrads accumulate 512 / 1024 k-blocks in one
    fp32 chain at the full batch).  Default mode: the bounds of check_c_driver_matches_engine (5e-5 block tensors, 1e-2 on the
    conditioning path, whose sums are re-rounded to bf16)."""
    from maskdit_b200 import ops
    torch.use_deterministic_algorithms(mode == "deterministic")
    c = case
    ce, st, B, L, pd = c.ce, c.st, c.B, c.L, c.pd
    ce.recompute = ce.num_blocks
    try:
        Fo, ctx = ce.forward(c.x, c.sigma, c.labels, c.md, True)
        assert ctx["recompute"] == ce.num_blocks
        st.ensure_grad().zero_()
        ce.backward(ctx, c.dF)
        del ctx
        g_full = st.grad.clone()
        loss = _loss(ops, c, Fo, slice(0, B))
        assert torch.isfinite(loss).all() and torch.isfinite(g_full).all()
        ce.recompute = 0
        st.grad.zero_()
        Fo3 = Fo.view(B, L, pd)
        bad_rows, bad_loss = [], []
        for i in range(0, B, CHUNK):
            rows = slice(i, i + CHUNK)
            mdc = {k: v[rows].contiguous() for k, v in c.md.items()}
            Fc, ctxc = ce.forward(c.x[rows].contiguous(), c.sigma[rows].contiguous(), c.labels[rows].contiguous(),
                                  mdc, True)
            assert ctxc["recompute"] == 0
            if not torch.equal(Fc.view(CHUNK, L, pd), Fo3[rows]):
                bad_rows.append(i)
            if not torch.equal(_loss(ops, c, Fc, rows), loss[rows]):
                bad_loss.append(i)
            ce.backward(ctxc, c.dF[i * L:(i + CHUNK) * L].contiguous())
            del Fc, ctxc
        torch.cuda.synchronize()
    finally:
        ce.recompute = None
    assert not bad_rows, f"case {c.name} [{mode}]: F rows differ from the batch-{CHUNK} runs at samples {bad_rows}"
    assert not bad_loss, f"case {c.name} [{mode}]: per-row loss differs from the batch-{CHUNK} runs at {bad_loss}"
    g_sum = st.grad
    worst = {"block": (0.0, ""), "conditioning": (0.0, "")}
    fails, n = [], 0
    for k, (o, cnt, _) in st.offsets.items():
        if o + cnt > st.n_train:
            continue
        a, b = g_full[o:o + cnt], g_sum[o:o + cnt]
        scale = a.abs().max().item()
        assert scale > 0, (k, "zero gradient")
        err = (a - b).abs().max().item() / scale
        cls = "conditioning" if any(t in k for t in COND) else "block"
        worst[cls] = max(worst[cls], (err, k))
        if mode == "deterministic":
            tol = DET_COND_GRAD_TOL if cls == "conditioning" else DET_BLOCK_GRAD_TOL
        else:
            tol = COND_GRAD_TOL if cls == "conditioning" else BLOCK_GRAD_TOL
        if err > tol:
            fails.append((k, err, tol))
        n += 1
    assert n > 200
    print(f"\ncase {c.name} [{mode}]: {B // CHUNK} chunks, F and loss rows bit-equal; gradient max-abs / scale, worst: "
          + ", ".join(f"{cls} {e:.3g} ({k})" for cls, (e, k) in worst.items()))
    assert not fails, f"case {c.name} [{mode}]: gradient tensors beyond their bound: {fails[:10]}"
    del g_full, Fo, loss
    st.grad.zero_()
    torch.cuda.empty_cache()


def test_eval_rows_vs_batch_2(case, lib):
    """The unmasked eval forward (`save=False`) at the sampler's production batch: 64 samples with CFG, i.e. the
    conditional and the unconditional half in one 128-row batch.  Every row equals a batch-2 run bit for bit."""
    torch.use_deterministic_algorithms(False)
    c = case
    ce, L, pd = c.ce, c.L, c.pd
    n = min(EVAL_B, c.B)
    x2 = torch.cat([c.x[:n], c.x[:n]]).contiguous()
    s2 = torch.cat([c.sigma[:n], c.sigma[:n]]).contiguous()
    y2 = torch.cat([c.labels[:n], torch.zeros_like(c.labels[:n])]).contiguous()
    Fo, _ = ce.forward(x2, s2, y2, None, False)
    Fo = Fo.view(2 * n, L, pd)
    bad = []
    for i in range(0, 2 * n, CHUNK):
        Fc, _ = ce.forward(x2[i:i + CHUNK].contiguous(), s2[i:i + CHUNK].contiguous(), y2[i:i + CHUNK].contiguous(),
                           None, False)
        if not torch.equal(Fc.view(CHUNK, L, pd), Fo[i:i + CHUNK]):
            bad.append(i)
    assert torch.isfinite(Fo).all()
    assert not bad, f"case {c.name}: eval rows differ from the batch-{CHUNK} runs at samples {bad}"
    print(f"\ncase {c.name}: eval forward at {2 * n} rows bit-equal to {n} batch-{CHUNK} runs")
    del Fo
    torch.cuda.empty_cache()
