"""Per-kernel parity (GPU) at the shapes of the DiT_models geometries beyond the shipped XL/2: patch 4 and 8 (pd and
cpp up to 256), DiT-H's head_dim 80, the LayerNorm widths of DiT-B / L / H (768 / 1024 / 1280) and the token counts
of the small-grid models (T = 8, 16, 32, 44).  Each kernel is compared with a plain float64 torch reference of the
same op fed the same (bf16-rounded where the kernel reads bf16) inputs.

Tolerances are those of test_kernels_gpu.py: fp32-accumulate kernels 1e-3 relative to the output scale (1e-4 / 1e-5
where the kernel is a short fp32 sum), bf16-output kernels 1 bf16 ulp (2^-8) relative, the attention 2^-7; pure
data movement is bit-exact."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
f64 = torch.float64


@pytest.fixture(scope="module")
def ops():
    from maskdit_b200 import ops as o
    return o


def dev():
    return torch.device("cuda")


def close(got, ref, tol, what=""):
    got, ref = got.double(), ref.double()
    scale = ref.abs().max().item() + 1e-30
    err = (got - ref).abs().max().item()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    assert err <= tol * scale, f"{what}: max_abs {err:.4g} > {tol} * scale {scale:.4g}"


def rb(*shape, scale=1.0):
    return (torch.randn(*shape, device=dev()) * scale).to(torch.bfloat16)


def patchify(x, p):
    """[B, C, R, R] -> [B, L, p*p*C], element order (ph, pw, c) as DiT.unpatchify."""
    B, C, R, _ = x.shape
    G = R // p
    return x.reshape(B, C, G, p, G, p).permute(0, 2, 4, 3, 5, 1).reshape(B, G * G, p * p * C)


def unpatchify(F_, p, C):
    B, L, _ = F_.shape
    G = int(round(L ** 0.5))
    return F_.reshape(B, G, G, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, G * p, G * p)


def precond(sigma):
    s4 = sigma.to(f64).view(-1, 1, 1, 1)
    return 0.25 / (s4 ** 2 + 0.25), s4 * 0.5 / (s4 ** 2 + 0.25).sqrt(), (s4 ** 2 + 0.25) / (s4 * 0.5) ** 2


# ---- EDM loss + gradient seed -----------------------------------------------------------------------------------------
# (p, R): L = (R / p)^2 = 16, 64 and 1024 tokens: below, at and above one 256-thread pass of the per-sample block
EDM_GEOMS = [(p, R) for p in (2, 4, 8) for R in (4 * p, 8 * p, 32 * p)]


@pytest.mark.parametrize("p,R", EDM_GEOMS)
@pytest.mark.parametrize("variant", ["nomask", "mask", "mask_mae"])
def test_edm_loss_and_grad(ops, p, R, variant):
    torch.manual_seed(20 + p + R)
    B, C = 3, 4
    L, pd = (R // p) ** 2, p * p * C
    masked, mae = variant != "nomask", 0.1 if variant == "mask_mae" else 0.0
    Fo = torch.randn(B, L, pd, device=dev())
    xin, y = torch.randn(B, C, R, R, device=dev()), torch.randn(B, C, R, R, device=dev()) * 0.5
    sigma = torch.tensor([0.05, 1.3, 7.0], device=dev())
    gl = torch.rand(B, device=dev()) + 0.5
    mask = None
    if masked:
        mask = ops.mask_indices(torch.rand(B, L, device=dev()), L // 2)["mask"]
        mask[0] = 0.0
        mask[0, L // 3] = 1.0           # sample 0: exactly one masked token (MAE mean over one patch)
    loss, Dx, dF = ops.edm_loss(Fo, xin, y, sigma, mask, gl, 0.5, mae, p, want_D=True)

    Fr = Fo.to(f64).requires_grad_(True)
    c_skip, c_out, w = precond(sigma)
    xd, yd = xin.to(f64), y.to(f64)
    D = c_skip * xd + c_out * unpatchify(Fr, p, C)
    per_patch = patchify(w * (D - yd) ** 2, p).mean(-1)          # [B, L]
    if masked:
        m = mask.to(f64)
        ref = (per_patch * (1 - m)).sum(1) / (1 - m).sum(1)
        if mae:
            tgt = patchify(xd, p)
            tgt = (tgt - tgt.mean(-1, keepdim=True)) / (tgt.var(-1, keepdim=True) + 1e-6) ** 0.5
            ref = ref + mae * (((patchify(D, p) - tgt) ** 2).mean(-1) * m).sum(1) / m.sum(1)
    else:
        ref = per_patch.mean(1)
    close(loss, ref, 1e-4, "loss")
    close(Dx, D, 1e-5, "D")
    (ref * gl.to(f64)).sum().backward()
    close(dF, Fr.grad, 2 ** -7, "dF")
    if masked and not mae:   # without the MAE term a masked token's gradient seed is exactly zero
        assert (dF.view(B, L, pd)[mask.bool()] == 0).all()


@pytest.mark.parametrize("p,R", [(4, 32), (4, 16), (8, 64), (8, 32)])
def test_precond_out_fwd_bwd_and_cfg(ops, p, R):
    torch.manual_seed(30 + p + R)
    B, C = 3, 4
    L, pd = (R // p) ** 2, p * p * C
    Fo = torch.randn(B, L, pd, device=dev())
    xin = torch.randn(B, C, R, R, device=dev())
    sigma = torch.tensor([0.02, 0.9, 40.0], device=dev())
    c_skip, c_out, _ = precond(sigma)
    D = c_skip * xin.to(f64) + c_out * unpatchify(Fo.to(f64), p, C)
    close(ops.edm_precond_out(Fo, xin, sigma, 0.5, p), D, 1e-5, "precond_out")
    gD = torch.randn_like(xin)
    close(ops.edm_precond_out_bwd(gD, sigma, 0.5, p).view(B, L, pd), patchify(c_out * gD.to(f64), p), 2 ** -8,
          "precond_out_bwd")
    F2 = torch.randn(2 * B, L, pd, device=dev())
    F2d = F2.to(f64)
    comb = F2d[B:] + 1.5 * (F2d[:B] - F2d[B:])
    close(ops.cfg_precond_out(F2, xin, sigma, 0.5, 1.5, p), c_skip * xin.to(f64) + c_out * unpatchify(comb, p, C),
          1e-5, "cfg_precond_out")


# ---- patch embedding -------------------------------------------------------------------------------------------------
# (p, R, kept): 179 of 256 tokens at patch 4 (forward 32-token blocks and backward 128-token blocks, ragged last one),
# 44 of 64 and 179 of 256 at patch 8 (cpp 256: 32-token backward blocks)
@pytest.mark.parametrize("p,R,kept", [(4, 64, 179), (8, 64, 44), (8, 128, 179)])
@pytest.mark.parametrize("D", [384, 1280])
@pytest.mark.parametrize("masked", [True, False])
def test_patch_embed_fwd_bwd(ops, p, R, kept, D, masked):
    torch.manual_seed(40 + p + D)
    B, C = 2, 4
    L, cpp = (R // p) ** 2, C * p * p
    x = torch.randn(B, C, R, R, device=dev())
    sigma = torch.tensor([0.3, 6.0], device=dev())
    W = torch.randn(D, C, p, p, device=dev()) * 0.2
    bias = torch.randn(D, device=dev())
    pos = torch.randn(L, D, device=dev())
    ids = torch.stack([torch.randperm(L, device=dev())[:kept] for _ in range(B)]) if masked else None
    out = ops.patch_embed(x, sigma, 0.5, W.reshape(D, -1).contiguous(), bias, pos, ids, p, D)
    c_in = 1 / (0.25 + sigma.to(f64) ** 2).sqrt()
    # conv weight [D, C, p, p] flattens (c, ph, pw): patches in the same order
    G = R // p
    pt = (x.to(f64) * c_in.view(-1, 1, 1, 1)).reshape(B, C, G, p, G, p).permute(0, 2, 4, 1, 3, 5).reshape(B, L, cpp)
    if masked:
        pt = torch.gather(pt, 1, ids.unsqueeze(-1).expand(-1, -1, cpp))
    Wd = W.to(f64).reshape(D, cpp)
    ref = pt @ Wd.t() + bias.to(f64) + (pos.to(f64)[ids] if masked else pos.to(f64))
    close(out, ref, 1e-5, "patch_embed")
    g = torch.randn_like(out)
    gW = torch.zeros(D, cpp, device=dev())
    gb = torch.zeros(D, device=dev())
    ops.patch_embed_bwd(x, sigma, 0.5, ids, g, gW, gb, p)
    gd = g.to(f64).reshape(-1, D)
    close(gW, gd.t() @ pt.reshape(-1, cpp), 1e-3, "patch_embed gW")
    close(gb, gd.sum(0), 1e-3, "patch_embed gb")


def test_patch_embed_rejects_cpp_over_384(ops):
    """cpp = 16 * 16 * 4 = 1024 exceeds the 48 KB patch block of both kernels: a clean error, not a launch failure."""
    from maskdit_b200._lib import MdtError
    x = torch.randn(1, 4, 32, 32, device=dev())
    W, bias, pos = torch.randn(64, 1024, device=dev()), torch.randn(64, device=dev()), torch.randn(4, 64, device=dev())
    sigma = torch.ones(1, device=dev())
    with pytest.raises(MdtError, match="unsupported"):
        ops.patch_embed(x, sigma, 0.5, W, bias, pos, None, 16, 64)
    with pytest.raises(MdtError, match="unsupported"):
        ops.patch_embed_bwd(x, sigma, 0.5, None, torch.randn(1, 4, 64, device=dev()), W.clone(), bias.clone(), 16)


# ---- attention -------------------------------------------------------------------------------------------------------
def attn_ref(qkv, B, T, H, dh):
    q, k, v = qkv.view(B, T, 3, H, dh).permute(2, 0, 3, 1, 4).unbind(0)
    s = q @ k.transpose(-1, -2) * dh ** -0.5
    return (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * T, H * dh), torch.logsumexp(s, -1)


def run_attention(ops, qkv, B, T, H, dh):
    out, lse = ops.attention_fwd(qkv, B, T, H, dh)
    impl_fwd = ops.lib().mdt_attention_last_impl(0)
    qr = qkv.to(f64).requires_grad_(True)
    ref, ref_lse = attn_ref(qr, B, T, H, dh)
    close(out, ref, 2 ** -7, "attention fwd")
    close(lse[0], ref_lse, 1e-3, "lse")
    dout = rb(B * T, H * dh)
    (ref * dout.to(f64)).sum().backward()
    dqkv = ops.attention_bwd(qkv, out, dout, lse, B, T, H, dh)
    impl_bwd = ops.lib().mdt_attention_last_impl(1)
    # dq, dk and dv each against its own scale: an error in the smallest cannot hide under the largest
    got, want = dqkv.view(B * T, 3, H * dh), qr.grad.view(B * T, 3, H * dh)
    for i, name in enumerate("qkv"):
        close(got[:, i], want[:, i], 2 ** -7, f"attention bwd d{name}")
    return impl_fwd, impl_bwd


# head_dim 80 (DiT-H, 16 heads): no wgmma instance, so every T runs the mma.sync kernels; head_dim 64 at the token
# counts of S/8 (16), B/8 at 256 px latents (32) and L/4 with 30 % masking (44)
@pytest.mark.parametrize("B,T,H,dh", [(3, 8, 16, 80), (2, 16, 16, 80), (2, 32, 16, 80), (2, 128, 16, 80),
                                      (1, 200, 4, 80), (2, 256, 16, 80),
                                      (3, 16, 6, 64), (2, 32, 12, 64), (2, 44, 16, 64)])
def test_attention_small_T_and_head_dim_80(ops, B, T, H, dh):
    torch.manual_seed(50 + T + dh)
    impl = run_attention(ops, rb(B * T, 3 * H * dh), B, T, H, dh)
    print("attention impl", (B, T, H, dh), impl)
    assert impl == (0, 0), impl


@pytest.mark.parametrize("B,T,H,dh,family", [(2, 128, 16, 72, 1), (1, 200, 4, 80, 0)])
def test_attention_large_logits(ops, B, T, H, dh, family):
    """q and k scaled so the scaled scores span about +-50: the online softmax's running max and rescaling must match
    torch.softmax, on one shape of each kernel family (wgmma, mma.sync)."""
    torch.manual_seed(60 + dh)
    qkv = torch.randn(B, T, 3, H, dh, device=dev())
    s = qkv[:, :, 0].transpose(1, 2) @ qkv[:, :, 1].permute(0, 2, 3, 1) * dh ** -0.5
    qkv[:, :, :2] *= (50.0 / s.abs().max()).sqrt()
    qkv = qkv.reshape(B * T, 3 * H * dh).to(torch.bfloat16)
    q, k = qkv.to(f64).view(B, T, 3, H, dh)[:, :, 0].transpose(1, 2), qkv.to(f64).view(B, T, 3, H, dh)[:, :, 1]
    smax = (q @ k.permute(0, 2, 3, 1) * dh ** -0.5).abs().max().item()
    assert 40 < smax < 60, smax
    impl = run_attention(ops, qkv, B, T, H, dh)
    assert impl == (family, family), impl


# ---- LayerNorm + modulate, gate backward -----------------------------------------------------------------------------
# T = 130, 179 and 192: backward blocks of gcd(T, 32) = 2, 1 and 32 rows of one sample in the default mode
@pytest.mark.parametrize("D", [768, 1024, 1152, 1280])
@pytest.mark.parametrize("T", [8, 16, 32, 44, 128, 130, 179, 192])
def test_ln_modulate_and_gate_kernels(ops, D, T):
    torch.manual_seed(70 + D + T)
    B = 3
    M = B * T
    x = torch.randn(M, D, device=dev()) * 2 + 0.3
    mod = torch.randn(B, 3 * D, device=dev()) * 0.5
    shift, scale, gate = mod[:, :D], mod[:, D:2 * D], mod[:, 2 * D:]
    out, mean, rstd = ops.ln_modulate(x, shift, scale, 3 * D, T, M, D)
    xr = x.to(f64).requires_grad_(True)
    mr = mod.to(f64).requires_grad_(True)
    ln = torch.nn.functional.layer_norm(xr, (D,), eps=1e-6).view(B, T, D)
    ref = (ln * (1 + mr[:, None, D:2 * D]) + mr[:, None, :D]).view(M, D)
    close(out, ref, 2 ** -8, "ln_modulate")
    close(mean, x.to(f64).mean(1), 1e-5, "mean")
    close(rstd, 1 / (x.to(f64).var(1, unbiased=False) + 1e-6).sqrt(), 1e-5, "rstd")
    dxmod = rb(M, D)
    (ref * dxmod.to(f64)).sum().backward()
    # ln_modulate_bwd, accumulating into g
    g0 = torch.randn(M, D, device=dev())
    g = g0.clone()
    dmod = torch.zeros(B, 3 * D, device=dev())
    ops.ln_modulate_bwd(dxmod, x, mean, rstd, scale, 3 * D, T, g, True, dmod[:, :D], dmod[:, D:], 3 * D, M, D)
    close(g.to(f64) - g0.to(f64), xr.grad, 1e-3, "ln bwd dx")
    close(dmod[:, :D], mr.grad[:, :D], 1e-3, "dshift")
    close(dmod[:, D:2 * D], mr.grad[:, D:2 * D], 1e-3, "dscale")
    # gate backward of the branch y -> gate * y, reading the finished residual gradient
    y = rb(M, D)
    gd = g.to(f64).view(B, T, D)
    ref_dy = (gd * gate.to(f64)[:, None, :]).reshape(M, D)
    ref_dgate = (gd * y.to(f64).view(B, T, D)).sum(1)
    dgate, dbias = torch.zeros(B, D, device=dev()), torch.zeros(D, device=dev())
    dy = ops.gate_bwd(g, y, gate, 3 * D, T, dgate, D, dbias, M, D)
    close(dy, ref_dy, 2 ** -8, "gate_bwd dy")
    close(dgate, ref_dgate, 1e-4, "gate_bwd dgate")
    close(dbias, ref_dy.sum(0), 1e-4, "gate_bwd dbias")
    # fused LN backward + gate backward: same g, dshift, dscale, dy, dgate, dbias
    gf = g0.clone()
    dmf, dbf = torch.zeros(B, 3 * D, device=dev()), torch.zeros(D, device=dev())
    dyf = ops.ln_modulate_bwd_gate(dxmod, x, mean, rstd, scale, 3 * D, T, gf, True, dmf[:, :D], dmf[:, D:], 3 * D,
                                   M, D, gate_next=(y, gate, 3 * D, dmf[:, 2 * D:], 3 * D, dbf))
    close(gf.to(f64) - g0.to(f64), xr.grad, 1e-3, "fused ln bwd dx")
    close(dmf[:, :D], mr.grad[:, :D], 1e-3, "fused dshift")
    close(dmf[:, D:2 * D], mr.grad[:, D:2 * D], 1e-3, "fused dscale")
    close(dyf, ref_dy, 2 ** -8, "fused dy")
    close(dmf[:, 2 * D:], ref_dgate, 1e-4, "fused dgate")
    close(dbf, ref_dy.sum(0), 1e-4, "fused dbias")


# ---- decoder-less output scatter / gather ----------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 256])
@pytest.mark.parametrize("T,L", [(8, 16), (44, 64)])
def test_unmask_null_table_and_gather_rows(ops, D, T, L):
    """The decoder-less DiT's kept-row scatter into zeros (D = pd) and its backward gathers."""
    torch.manual_seed(80 + D + T)
    B = 3
    md = ops.mask_indices(torch.rand(B, L, device=dev()), T)
    u = torch.randn(B, T, D, device=dev())
    out = ops.unmask_tokens(u, None, None, md["ids_restore"], B, T, L, D)
    ref = u.new_zeros(B, L, D).scatter(1, md["ids_keep"].unsqueeze(-1).expand(-1, -1, D), u)
    assert torch.equal(out, ref)
    g = torch.randn(B, L, D, device=dev())
    kept = torch.gather(g, 1, md["ids_keep"].unsqueeze(-1).expand(-1, -1, D))
    du = ops.unmask_tokens_bwd(g, md["ids_restore"], None, B, T, L, D)
    close(du.view(B, T, D), kept, 2 ** -8, "unmask_tokens_bwd du")
    g16 = g.to(torch.bfloat16)
    rows = ops.gather_rows_bf16(g16.view(B * L, D), md["ids_keep"], B, T, L, D)
    assert torch.equal(rows.view(B, T, D), torch.gather(g16, 1, md["ids_keep"].unsqueeze(-1).expand(-1, -1, D)))
