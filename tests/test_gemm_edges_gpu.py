"""The GEMM's unit edges against torch fp32 on the same bf16 inputs, at the tolerances of test_kernels_gpu.py.  Each
128-row unit is computed as two 64-row halves, one per consumer warpgroup: ragged M that leaves the bottom half empty
or partial, paired half-width column tiles over an odd number of m-panels, MN-major A, an in-place residual, gate
groups that change inside a half, the fused column sum at a ragged N, and run-to-run bit equality."""
import pytest
import torch
import torch.nn.functional as F

from support import ops  # noqa: F401

pytestmark = pytest.mark.gpu

EPIS = ("store16", "store32_resid", "gelu", "gate_resid", "dgelu", "atomic")


def close(got, ref, tol, what=""):
    got, ref = got.float(), ref.float()
    scale = ref.abs().max().item() + 1e-12
    err = (got - ref).abs().max().item()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    assert err <= tol * scale, f"{what}: max_abs {err:.4g} > {tol} * scale {scale:.4g}"


def rb(*shape, scale=1.0, g=None):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def run(ops, epi, M, N, K, *, rpg=128, seed=0, b_mn=False, in_place=False):
    """One launch of epilogue `epi` on seeded inputs; returns (outputs, references) as dicts of tensors."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = rb(M, K, g=g)
    B = rb(K, N, scale=K ** -0.5, g=g) if b_mn else rb(N, K, scale=K ** -0.5, g=g)
    acc = A.float() @ (B.float() if b_mn else B.float().t())
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    kw = dict(b_mn=b_mn)
    if epi == "store16":
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        ops.gemm(A, B, M, N, K, out=out, bias=bias, **kw)
        return {"out": out}, {"out": (acc + bias, 2 ** -8)}
    if epi == "store32_resid":
        R = torch.randn(M, N, device="cuda", generator=g)
        out = R.clone() if in_place else torch.empty(M, N, device="cuda")
        ops.gemm(A, B, M, N, K, out=out, bias=bias, resid=out if in_place else R, ld_resid=N, **kw)
        return {"out": out}, {"out": (acc + bias + R, 1e-3)}
    if epi == "gelu":
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        aux = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        ops.gemm(A, B, M, N, K, out=out, bias=bias, epi=ops.EPI_GELU, aux=aux, ld_aux=N, **kw)
        return {"out": out, "aux": aux}, {"aux": (acc + bias, 2 ** -8),
                                          "out": (F.gelu(aux.float(), approximate="tanh"), 2 ** -7)}
    if epi == "gate_resid":
        R = torch.randn(M, N, device="cuda", generator=g)
        gate = torch.randn((M + rpg - 1) // rpg, N, device="cuda", generator=g)
        out = R.clone() if in_place else torch.empty(M, N, device="cuda")
        aux = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        ops.gemm(A, B, M, N, K, out=out, bias=bias, epi=ops.EPI_GATE_RESID, aux=aux, ld_aux=N,
                 resid=out if in_place else R, ld_resid=N, gate=gate, ld_gate=N, rows_per_group=rpg, **kw)
        gate_rows = gate[torch.arange(M, device="cuda") // rpg]
        return {"out": out, "aux": aux}, {"aux": (acc + bias, 2 ** -8), "out": (R + gate_rows * (acc + bias), 1e-3)}
    if epi == "dgelu":
        h = rb(M, N, g=g)
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        cs = torch.full((N,), 0.5, device="cuda")
        ops.gemm(A, B, M, N, K, out=out, epi=ops.EPI_DGELU, aux=h, ld_aux=N, colsum=cs, **kw)
        hf = h.float().requires_grad_(True)
        F.gelu(hf, approximate="tanh").sum().backward()
        return {"out": out, "colsum": cs - 0.5}, {"out": (acc * hf.grad, 2 ** -7),
                                                  "colsum": (out.float().sum(0), 1e-4)}
    assert epi == "atomic"
    out = torch.full((M, N), 0.25, device="cuda")
    ops.gemm(A, B, M, N, K, out=out, epi=ops.EPI_ATOMIC, **kw)
    return {"out": out}, {"out": (acc + 0.25, 1e-3)}


def check(got, want, what):
    for k, (ref, tol) in want.items():
        close(got[k], ref, tol, f"{what} {k}")


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("rem", [1, 37, 64, 65, 100])
def test_ragged_m_every_epilogue(ops, epi, rem):
    """M % 128 = rem: the last unit's bottom half is empty (rem <= 64) or partly present (rem > 64)."""
    M, N, K = 3 * 128 + rem, 1152, 192
    got, want = run(ops, epi, M, N, K, seed=rem, b_mn=epi in ("dgelu", "atomic"))
    check(got, want, f"{epi} M={M}")


@pytest.mark.parametrize("N", [1152, 3456])
@pytest.mark.parametrize("panels,rem", [(5, 0), (5, 37), (7, 100)])
def test_paired_half_tiles_odd_panels(ops, N, panels, rem):
    """N = 4.5 / 13.5 column tiles: the half-width last tiles of two m-panels form one unit; odd panel count."""
    M = (panels - 1) * 128 + (rem or 128)
    for epi in ("store16", "gate_resid"):
        got, want = run(ops, epi, M, N, 256, seed=N + M)
        check(got, want, f"{epi} M={M} N={N}")


@pytest.mark.parametrize("M", [9 * 128 + 40, 9 * 128 + 104])
def test_wgrad_mn_major_a_ragged_m(ops, M):
    """MN-major A (one {64 mn, 64 k} box per half), k-sliced red.add, M % 128 with an empty / partial bottom half."""
    N, K = 1000, 2048
    g = torch.Generator(device="cuda").manual_seed(M)
    A, B = rb(K, M, g=g), rb(K, N, g=g)
    out = torch.zeros(M, N, device="cuda")
    ops.gemm(A, B, M, N, K, a_mn=True, b_mn=True, out=out, epi=ops.EPI_ATOMIC)
    close(out, A.float().t() @ B.float(), 1e-3, f"wgrad M={M}")


@pytest.mark.parametrize("epi", ["gate_resid", "store32_resid"])
def test_in_place_residual(ops, epi):
    """`out` aliases `resid` (eval-mode block forward): every element is read before it is overwritten."""
    got, want = run(ops, epi, 4 * 128 + 65, 1152, 384, seed=7, in_place=True)
    check(got, want, f"{epi} in place")


@pytest.mark.parametrize("rpg", [100, 179])
def test_gate_group_boundary_inside_half(ops, rpg):
    got, want = run(ops, "gate_resid", 6 * 128 + 37, 1152, 192, rpg=rpg, seed=rpg)
    check(got, want, f"gate rows_per_group={rpg}")


@pytest.mark.parametrize("M,N", [(3 * 128 + 65, 1000), (2 * 128 + 37, 1000), (5 * 128 + 100, 200)])
def test_dgelu_colsum_ragged_n(ops, M, N):
    got, want = run(ops, "dgelu", M, N, 320, seed=M + N, b_mn=True)
    check(got, want, f"dgelu M={M} N={N}")


@pytest.fixture
def sm_budget(ops):
    L = ops.lib()
    yield L
    assert L.mdt_set_sm_budget(0) == 0


@pytest.mark.parametrize("budget", [1, 7, 124])
def test_sm_budget_every_epilogue(ops, sm_budget, budget):
    """A persistent grid narrowed by `mdt_set_sm_budget` (the backward next to the overlapped gradient exchange) deals
    the same tiles to fewer CTAs: paired half tiles, ragged M.  A tile's arithmetic does not depend on which CTA runs
    it, so every non-accumulating output is bit-identical to the full-width run; the accumulating epilogue's k-slice
    count follows the budget, so it is held to the reference."""
    M, N, K = 5 * 128 + 37, 1152, 256
    for epi in EPIS:
        b_mn = epi in ("dgelu", "atomic")
        full, _ = run(ops, epi, M, N, K, seed=budget, b_mn=b_mn)
        assert sm_budget.mdt_set_sm_budget(budget) == 0
        got, want = run(ops, epi, M, N, K, seed=budget, b_mn=b_mn)
        assert sm_budget.mdt_set_sm_budget(0) == 0
        check(got, want, f"{epi} budget={budget}")
        for k in got:
            if epi != "atomic" and k != "colsum":    # fp32 red.add: summation order varies
                assert torch.equal(got[k], full[k]), f"{epi} {k} differs under budget {budget}"


@pytest.mark.parametrize("epi", [e for e in EPIS if e != "atomic"])
def test_two_runs_bit_identical(ops, epi):
    M, N, K = 9 * 128 + 65, 3456, 1152
    a, _ = run(ops, epi, M, N, K, seed=11, b_mn=epi == "dgelu")
    b, _ = run(ops, epi, M, N, K, seed=11, b_mn=epi == "dgelu")
    for k in a:
        if k == "colsum":  # fp32 red.add across units: order varies between runs
            continue
        assert torch.equal(a[k], b[k]), f"{epi} {k} differs between two runs"
