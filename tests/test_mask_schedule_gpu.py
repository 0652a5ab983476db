"""GPU: the kept-token counts a mask-ratio schedule visits.

`train.py` takes the mask ratio from `mask_ratio_fn` at every step, so under the finetune recipe's `cos4` schedule the
kept-token count T = int(L * (1 - r)) changes almost every step: every count from L / 2 to L, and in the last steps
T = L with masking on (r < 1e-16, `ids_keep` a full permutation).  This file checks the kernels and the training step at
those counts: the attention at every T of the 256-px range and its kernel family, the LN / gate kernels and the gate
GEMM with `rows_per_group = T` on a strided modulation buffer in both library modes, the loss with no removed token,
the driver's step at schedule T against the float64 oracle, a bit-reproducible run whose T changes between steps
(CUDA-graph cache, recomputation) and `train.py` under `cos4`.

Bounds are those of test_geometry_kernels_gpu.py (kernels against float64) and test_model_gpu.py (model level)."""
import copy
import math
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from support import (FWD_TOL, GRAD_TOL, LOSS_TOL, GoldenLoss, ImplRecorder, assert_same, lib,  # noqa: E402,F401
                     oracle_net, ops, rel_l2, step_state)

pytestmark = pytest.mark.gpu
f64 = torch.float64

# DiT-S/2 on 32 x 32 latents: L = 256 tokens, encoder head_dim 64, decoder head_dim 32
MT, R, NCLS, B = "DiT-S/2", 32, 10, 2
L = (R // 2) ** 2
R_FULL = 1e-17   # a ratio the schedule reaches in its last steps: masking on, int(L * (1 - r)) == L


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


def ratio(T):
    """A mask ratio whose kept-token count is T (exact: L is a power of two); T = L keeps masking on."""
    r = (L - T) / L if T < L else R_FULL
    assert int(L * (1 - r)) == T
    return r


def draws(seed):
    """Images, labels and every random draw of one loss call, in GoldenLoss's layout."""
    gen = torch.Generator().manual_seed(seed)
    return {"images": torch.randn(B, 4, R, R, generator=gen) * 0.5,
            "labels": torch.eye(NCLS)[torch.randint(0, NCLS, (B,), generator=gen)],
            "rnd_normal": torch.randn(B, 1, 1, 1, generator=gen),
            "noise_unit": torch.randn(B, 4, R, R, generator=gen),
            "mask_noise": torch.rand(B, L, generator=gen)}


# ---- attention -------------------------------------------------------------------------------------------------------
def check_attention(ops, B_, T, H, dh, seed):
    torch.manual_seed(seed)
    qkv = rb(B_ * T, 3 * H * dh)
    out, lse = ops.attention_fwd(qkv, B_, T, H, dh)
    impl_fwd = ops.lib().mdt_attention_last_impl(0)
    qr = qkv.to(f64).requires_grad_(True)
    q, k, v = qr.view(B_, T, 3, H, dh).permute(2, 0, 3, 1, 4).unbind(0)
    s = q @ k.transpose(-1, -2) * dh ** -0.5
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B_ * T, H * dh)
    close(out, ref, 2 ** -7, f"T={T} attention fwd")
    close(lse[0], torch.logsumexp(s, -1), 1e-3, f"T={T} lse")
    dout = rb(B_ * T, H * dh)
    (ref * dout.to(f64)).sum().backward()
    dqkv = ops.attention_bwd(qkv, out, dout, lse, B_, T, H, dh)
    impl_bwd = ops.lib().mdt_attention_last_impl(1)
    got, want = dqkv.view(B_ * T, 3, H * dh), qr.grad.view(B_ * T, 3, H * dh)
    for i, name in enumerate("qkv"):
        close(got[:, i], want[:, i], 2 ** -7, f"T={T} attention bwd d{name}")
    fam = 1 if T % 64 == 0 and dh in (32, 64, 72) else 0
    assert (impl_fwd, impl_bwd) == (fam, fam), (T, dh, impl_fwd, impl_bwd)


def test_attention_over_the_256px_schedule_range(ops):
    """Every kept-token count cos4 visits at 256 px, at the XL encoder's shape (wgmma at 128, 192 and 256, mma.sync
    elsewhere, incl. one valid key in the last tile and 63), then the decoder's shape at the unmasked L of 256 and
    512 px."""
    for T in range(128, 257):
        check_attention(ops, 2, T, 16, 72, seed=T)
    for T in (256, 1024):
        check_attention(ops, 2, T, 16, 32, seed=T + 1)


# ---- LN-modulate, gate backward and the gate-residual GEMM with rows_per_group = T -----------------------------------
SCHED_T = [129, 130, 132, 136, 144, 192, 255, 256]   # backward blocks of gcd(T, 32) = 1, 2, 4, 8, 16, 32, 1, 32 rows


@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
def test_block_kernels_at_schedule_T(lib, ops, det):
    """As the step driver calls them: the modulation is the column slices of one block in a [B, NA] buffer (ld = NA),
    one group of T rows per sample.  Under the deterministic mode the standalone entry points take no bias gradient
    (they have no scratch for its per-sample rows)."""
    assert lib.mdt_set_deterministic(int(det)) == 0
    D = 1152
    NA, o = 18 * D, 6 * D            # the second of three blocks' modulations
    for T in SCHED_T:
        torch.manual_seed(90 + T)
        M = B * T
        x = torch.randn(M, D, device=dev()) * 2 + 0.3
        mod = torch.randn(B, NA, device=dev()) * 0.5
        shift, scale, gate = mod[:, o:o + D], mod[:, o + D:o + 2 * D], mod[:, o + 2 * D:o + 3 * D]
        out, mean, rstd = ops.ln_modulate(x, shift, scale, NA, T, M, D)
        xr = x.to(f64).requires_grad_(True)
        mr = mod.to(f64).requires_grad_(True)
        ln = torch.nn.functional.layer_norm(xr, (D,), eps=1e-6).view(B, T, D)
        ref = (ln * (1 + mr[:, None, o + D:o + 2 * D]) + mr[:, None, o:o + D]).view(M, D)
        close(out, ref, 2 ** -8, f"T={T} ln_modulate")
        close(mean, x.to(f64).mean(1), 1e-5, f"T={T} mean")
        close(rstd, 1 / (x.to(f64).var(1, unbiased=False) + 1e-6).sqrt(), 1e-5, f"T={T} rstd")
        dxmod = rb(M, D)
        (ref * dxmod.to(f64)).sum().backward()
        g0 = torch.randn(M, D, device=dev())
        g = g0.clone()
        dmod = torch.zeros(B, NA, device=dev())
        ops.ln_modulate_bwd(dxmod, x, mean, rstd, scale, NA, T, g, True, dmod[:, o:o + D], dmod[:, o + D:], NA, M, D)
        close(g.to(f64) - g0.to(f64), xr.grad, 1e-3, f"T={T} ln bwd dx")
        close(dmod[:, o:o + D], mr.grad[:, o:o + D], 1e-3, f"T={T} dshift")
        close(dmod[:, o + D:o + 2 * D], mr.grad[:, o + D:o + 2 * D], 1e-3, f"T={T} dscale")
        y = rb(M, D)
        gd = g.to(f64).view(B, T, D)
        ref_dy = (gd * gate.to(f64)[:, None, :]).reshape(M, D)
        ref_dgate = (gd * y.to(f64).view(B, T, D)).sum(1)
        dgate = torch.zeros(B, NA, device=dev())
        dbias = None if det else torch.zeros(D, device=dev())
        dy = ops.gate_bwd(g, y, gate, NA, T, dgate[:, o + 2 * D:], NA, dbias, M, D)
        close(dy, ref_dy, 2 ** -8, f"T={T} gate_bwd dy")
        close(dgate[:, o + 2 * D:o + 3 * D], ref_dgate, 1e-4, f"T={T} gate_bwd dgate")
        if dbias is not None:
            close(dbias, ref_dy.sum(0), 1e-4, f"T={T} gate_bwd dbias")
        gf = g0.clone()
        dmf = torch.zeros(B, NA, device=dev())
        dbf = None if det else torch.zeros(D, device=dev())
        dyf = ops.ln_modulate_bwd_gate(dxmod, x, mean, rstd, scale, NA, T, gf, True, dmf[:, o:o + D], dmf[:, o + D:],
                                       NA, M, D, gate_next=(y, gate, NA, dmf[:, o + 2 * D:], NA, dbf))
        close(gf.to(f64) - g0.to(f64), xr.grad, 1e-3, f"T={T} fused ln bwd dx")
        close(dmf[:, o:o + D], mr.grad[:, o:o + D], 1e-3, f"T={T} fused dshift")
        close(dmf[:, o + D:o + 2 * D], mr.grad[:, o + D:o + 2 * D], 1e-3, f"T={T} fused dscale")
        close(dyf, ref_dy, 2 ** -8, f"T={T} fused dy")
        close(dmf[:, o + 2 * D:o + 3 * D], ref_dgate, 1e-4, f"T={T} fused dgate")
        if dbf is not None:
            close(dbf, ref_dy.sum(0), 1e-4, f"T={T} fused dbias")
        # the attention projection's gate-residual GEMM: out = X + gate[row // T] * (O W^T + b), y = O W^T + b (bf16)
        K = D
        A, W = rb(M, K), rb(D, K, scale=0.05)
        bias = torch.randn(D, device=dev())
        resid = torch.randn(M, D, device=dev())
        acc = A.to(f64) @ W.to(f64).t() + bias.to(f64)
        outg = torch.empty(M, D, device=dev())
        aux = torch.empty(M, D, device=dev(), dtype=torch.bfloat16)
        ops.gemm(A, W, M, D, K, out=outg, bias=bias, epi=ops.EPI_GATE_RESID, aux=aux, ld_aux=D, resid=resid,
                 ld_resid=D, gate=gate, ld_gate=NA, rows_per_group=T)
        close(aux, acc, 2 ** -8, f"T={T} gate_resid y")
        close(outg, resid.to(f64) + gate.to(f64).repeat_interleave(T, 0) * acc, 1e-3, f"T={T} gate_resid out")


# ---- loss with no removed token --------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [2, 8])
def test_edm_loss_with_no_removed_token(ops, p):
    """T = L with masking on: the mask is all zero.  The reference's mae_loss divides by mask.sum(1) = 0 there (NaN);
    this kernel drops the MAE term, so the loss is the EDM term over every token - the unmasked loss - and the gradient
    seed is the EDM one, bit for bit what the same call with mae_coef = 0 gives."""
    torch.manual_seed(100 + p)
    B_, C, Rp = 3, 4, 16 * p
    Lp, pd = (Rp // p) ** 2, p * p * C
    Fo = torch.randn(B_, Lp, pd, device=dev())
    xin, y = torch.randn(B_, C, Rp, Rp, device=dev()), torch.randn(B_, C, Rp, Rp, device=dev()) * 0.5
    sigma = torch.tensor([0.05, 1.3, 7.0], device=dev())
    gl = torch.rand(B_, device=dev()) + 0.5
    mask = ops.mask_indices(torch.rand(B_, Lp, device=dev()), Lp)["mask"]
    assert not mask.any()
    loss, _, dF = ops.edm_loss(Fo, xin, y, sigma, mask, gl, 0.5, 0.1, p)
    loss0, _, dF0 = ops.edm_loss(Fo, xin, y, sigma, mask, gl, 0.5, 0.0, p)
    assert torch.isfinite(loss).all() and torch.isfinite(dF.float()).all()
    Fr = Fo.to(f64).requires_grad_(True)
    s4 = sigma.to(f64).view(-1, 1, 1, 1)
    c_skip, c_out, w = 0.25 / (s4 ** 2 + 0.25), s4 * 0.5 / (s4 ** 2 + 0.25).sqrt(), (s4 ** 2 + 0.25) / (s4 * 0.5) ** 2
    G = Rp // p
    D = c_skip * xin.to(f64) + c_out * Fr.reshape(B_, G, G, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(B_, C, Rp, Rp)
    l = w * (D - y.to(f64)) ** 2
    per_patch = l.reshape(B_, C, G, p, G, p).mean((1, 3, 5)).reshape(B_, Lp)
    unmask = 1 - mask.to(f64)
    ref = (per_patch * unmask).sum(1) / unmask.sum(1)          # EDM-only masked loss ...
    assert torch.allclose(ref, l.mean((1, 2, 3)), rtol=1e-12)   # ... which is the unmasked loss
    close(loss, ref, 1e-4, "loss")
    (ref * gl.to(f64)).sum().backward()
    close(dF, Fr.grad, 2 ** -7, "dF")
    assert torch.equal(loss, loss0) and torch.equal(dF, dF0)


# ---- the step driver at schedule T against the float64 oracle --------------------------------------------------------
_SD64 = {}


def _oracle_sd():
    from oracle import maskdit_oracle as O
    if not _SD64:
        _SD64.update(O.make_state_dict(O.Cfg(model_type=MT, img_resolution=R, num_classes=NCLS), 1, dtype=f64))
    return {k: v.clone().requires_grad_(not k.endswith("pos_embed")) for k, v in _SD64.items()}


@pytest.mark.parametrize("T", [64, 128, 129, 192, 193, 255, 256])
def test_driver_step_at_schedule_T_vs_float64_oracle(lib, T):
    """Loss and every parameter gradient of one masked step against the float64 oracle on the same draws; the
    attention family of the encoder (head_dim 64 at T) and of the decoder (head_dim 32 at L).  At T = L the oracle
    runs without its MAE term (NaN there) and the mask token's gradient is exactly zero; the network output equals the
    unmasked forward's within the forward bound (a full permutation only reorders the attention sums)."""
    from oracle import maskdit_oracle as O
    torch.use_deterministic_algorithms(False)
    g = draws(200 + T)
    r = ratio(T)
    net = oracle_net(MT, R, NCLS, True)
    lf = GoldenLoss(g)
    x, lab = g["images"].cuda(), g["labels"].cuda()
    with ImplRecorder() as rec:
        loss = lf(net, x, lab, mask_ratio=r, mae_loss_coef=0.1)
        loss.mean().backward()
        torch.cuda.synchronize()
    md = O.mask_from_noise(g["mask_noise"], r)
    assert md["ids_keep"].shape[1] == T
    for k in ("mask", "ids_keep", "ids_restore"):
        assert torch.equal(lf.last_mask_dict[k].cpu(), md[k]), k
    fam = int(T % 64 == 0)
    assert rec.attn_fwd == {(T, 64, fam), (L, 32, 1)}, rec.attn_fwd
    assert rec.attn_bwd == {(T, 64, fam), (L, 32, 1)}, rec.attn_bwd

    cfg = O.Cfg(model_type=MT, img_resolution=R, num_classes=NCLS)
    sdr = _oracle_sd()
    mae = 0.1 if T < L else 0.0
    ref, _ = O.edm_loss(sdr, cfg, g["images"].to(f64), g["labels"].to(f64), g["rnd_normal"].to(f64),
                        g["noise_unit"].to(f64), md, mae)
    assert torch.isfinite(ref).all()
    assert torch.allclose(loss.cpu().to(f64), ref.detach(), rtol=LOSS_TOL), (T, loss, ref)
    ref.mean().backward()
    worst, n = (0.0, ""), 0
    for k, p in net.named_parameters():
        if not p.requires_grad:
            continue
        want = sdr[k].grad
        if T == L and k == "model.mask_token":
            assert want is None or not want.any()
            assert not p.grad.any(), "mask token gradient with no masked token"
            continue
        e = rel_l2(p.grad, want)
        worst = max(worst, (e, k))
        assert e <= GRAD_TOL, (T, k, e)
        n += 1
    assert n > 200
    print(f"T={T}: loss {loss.tolist()} vs {ref.tolist()}, worst gradient rel-L2 {worst}")

    if T == L:
        with torch.no_grad():
            sigma = (g["rnd_normal"].cuda() * 1.2 - 1.2).exp()
            xf, sig, lb = net._norm_inputs(x + g["noise_unit"].cuda() * sigma, sigma, lab)
            F_masked, _ = net._engine.forward(xf, sig, lb, lf.last_mask_dict, save=False)
            F_full, _ = net._engine.forward(xf, sig, lb, None, save=False)
        e = rel_l2(F_masked, F_full)
        print("T = L masked vs unmasked forward rel-L2", e)
        assert e <= FWD_TOL


# ---- a run whose T changes between steps repeats bit for bit ---------------------------------------------------------
# 128 and 192 are captured, 128 is replayed, 255 evicts 128, 192 is replayed, 256 (masked) evicts 192, 64 evicts 255
T_SEQ = [128, 192, 128, 255, 192, 256, 64]


def test_T_changing_run_repeats_bit_for_bit(lib):
    """Under the deterministic mode one TrainStep goes through a sequence of kept-token counts eagerly, from CUDA graphs
    (at most 2 kept), recomputing one block and recomputing every block: loss, gradient, weights, bf16 shadow,
    moments and EMA agree bit for bit after every step."""
    from maskdit_b200.train_step import TrainStep
    torch.use_deterministic_algorithms(True)
    g = draws(7)
    x, lab = g["images"].cuda(), g["labels"].cuda()
    runs = {}
    for name, kw in (("eager", {}), ("graph", dict(graph=True)), ("recompute 1", dict(recompute_blocks=1)),
                     ("recompute all", dict(recompute_blocks=20))):
        net = oracle_net(MT, R, NCLS, True)
        runs[name] = TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, loss_fn=GoldenLoss(g), **kw)
    graphs = runs["graph"]._graphs
    for i, T in enumerate(T_SEQ):
        base = None
        for name, ts in runs.items():
            st = step_state(ts, [ts.step(x, lab, ratio(T), 0.1).clone()])
            if base is None:
                base = st
                assert torch.isfinite(st[0]).all()
                continue
            try:
                assert_same(base, st)
            except AssertionError as e:
                raise AssertionError(f"step {i} (T = {T}): {name} differs from eager: {e}") from None
            del st
        assert len(graphs) <= 2 and T in [k[2] for k in graphs], (T, list(graphs))
        del base
    assert runs["recompute 1"].recompute_blocks == 1 and runs["recompute all"].recompute_blocks == 20
    for ts in runs.values():
        ts.close()
    del runs
    torch.cuda.empty_cache()


# ---- train.py under cos4 ---------------------------------------------------------------------------------------------
YAML = """
data: {dataset: imagenet256-latent, category: lmdb, resolution: 32, num_channels: 4, root: none, feat_path: None}
model:
  precond: edm
  model_type: DiT-S/2
  in_size: 32
  in_channels: 4
  num_classes: 10
  use_decoder: True
  ext_feature_dim: 0
  pad_cls_token: False
  mask_ratio: 0.5
  mask_ratio_fn: cos4
  mask_ratio_min: 0
  mae_loss_coef: 0.1
  class_dropout_prob: 0.1
train: {tf32: False, amp: True, batchsize: 4, grad_accum: 1, epochs: 1, lr: 0.0001, lr_rampup_kimg: 0, xflip: False,
        max_num_steps: 6}
log: {log_every: 2, ckpt_every: 1000, tag: t}
"""


def test_train_py_under_cos4(tmp_path):
    """Seven steps at T = 128, 144, 184, 224, 248, 255 and 256 (masked) with the training step replayed from CUDA
    graphs: every logged loss is finite."""
    from maskdit_b200.config import mask_ratio_schedule
    f = mask_ratio_schedule("cos4", 0.5, 0.0)
    assert [int(L * (1 - f(s / 6))) for s in range(7)] == [128, 144, 184, 224, 248, 255, 256] and f(1.0) > 0
    cfg = tmp_path / "cfg.yaml"
    cfg.write_text(YAML)
    env = dict(os.environ, PYTHONPATH=ROOT, MDT_TRAIN_GRAPH="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "train.py"), "--config", str(cfg), "--synthetic",
                        "--results_dir", str(tmp_path / "res")], cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    losses = [float(v) for v in re.findall(r"Train Loss: (\S+),", r.stdout)]
    assert len(losses) == 3 and all(math.isfinite(v) for v in losses), r.stdout[-2000:]
