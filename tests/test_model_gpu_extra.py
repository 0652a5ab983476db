"""GPU: further reference goldens on the CUDA path — another geometry (DiT-B/4: patch 4, 12 heads of 64, three of
four patches masked) and the stochastic (S_churn > 0) sampler."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from test_model_gpu import (CFG_TOL, EVAL_TOL, FWD_TOL, GRAD_TOL, LOSS_TOL, GoldenLoss, ImplRecorder, build,  # noqa: E402
                            check_c_driver_matches_engine, check_grads, load, rel_l2)

pytestmark = pytest.mark.gpu


def test_b4_patch4_mask75_loss_and_grads_vs_reference_golden():
    g = load("b4_train_mask75")
    net, cfg, _ = build("DiT-B/4", 16, 7)
    net.train()
    lf = GoldenLoss(g)
    loss = lf(net, g["images"].cuda(), g["labels"].cuda(), mask_ratio=0.75, mae_loss_coef=0.1)
    for k in ("mask", "ids_keep", "ids_restore"):
        assert torch.equal(lf.last_mask_dict[k].cpu(), g[k]), k
    assert torch.allclose(loss.cpu(), g["loss"], rtol=LOSS_TOL), (loss, g["loss"])
    loss.mean().backward()
    check_grads(net, g, what="B/4")


def test_sampler_with_churn_vs_reference_golden():
    from maskdit_b200.sampler import edm_sampler
    g = load("s2_sampler_churn")
    net, cfg, _ = build()
    net.eval()
    noises = [n.cuda() for n in g["noises"]]
    calls = []
    orig = net.forward

    def spy(x, s, *a, **k):
        calls.append(float(s))
        return orig(x, s, *a, **k)

    net.forward = spy
    with torch.no_grad():
        z = edm_sampler(net, g["latents"].cuda(), g["labels"].cuda(), randn_like=lambda x: noises.pop(0),
                        num_steps=int(g["num_steps"]), S_churn=float(g["S_churn"]), S_min=float(g["S_min"]),
                        S_max=float(g["S_max"]), S_noise=float(g["S_noise"]))
    net.forward = orig
    assert len(calls) == 15 and not noises
    np.testing.assert_allclose(np.array(calls), g["sampler_sigmas"].numpy(), rtol=1e-12)
    assert z.dtype == torch.float64 and rel_l2(z, g["z"]) <= 2e-2


# ---- reference goldens that reach the production kernels (256-wide wgmma GEMM tiles, flash attention) -----------------
def _train_case(name, R, mask_ratio=0.5):
    g = load(name)
    net, cfg, _ = build("DiT-XL/2", R, 1000)
    net.train()
    lf = GoldenLoss(g)
    with ImplRecorder() as rec:
        loss = lf(net, g["images"].cuda(), g["labels"].cuda(), mask_ratio=mask_ratio, mae_loss_coef=0.1)
        for k in ("mask", "ids_keep", "ids_restore"):
            assert torch.equal(lf.last_mask_dict[k].cpu(), g[k]), k
        loss.mean().backward()
    print(name, "loss", loss.tolist(), "ref", g["loss"].tolist(), "gemm", sorted(rec.gemm_cfgs), "attn fwd",
          sorted(rec.attn_fwd), "bwd", sorted(rec.attn_bwd))
    assert torch.allclose(loss.cpu(), g["loss"], rtol=LOSS_TOL), (loss, g["loss"])
    check_grads(net, g, what=name)
    return rec


def test_xl2_r32_loss_and_all_grads_vs_reference_golden():
    """BASELINE config 1/2 geometry (XL/2, 32x32x4, mask 0.5) at batch 2 WITH gradients: 256 encoder token rows ->
    the 256-wide GEMM instances incl. wgrad/dgrad, the encoder attention (T=128, head_dim 72) and the decoder
    attention (T=256, head_dim 32) — end to end against the unmodified reference's autograd."""
    rec = _train_case("xl2_c1_grads", 32)
    assert 2561 in rec.gemm_cfgs, rec.gemm_cfgs                     # BLOCK_N 256
    assert rec.attn_fwd == {(128, 72, 1), (256, 32, 1)}, rec.attn_fwd
    assert rec.attn_bwd == {(128, 72, 1), (256, 32, 1)}, rec.attn_bwd


def test_xl2_r64_loss_and_all_grads_vs_reference_golden():
    """BASELINE config 4 geometry (XL/2, 64x64x4 latents: T=512 kept tokens of head_dim 72, L=1024 decoder tokens of
    head_dim 32): the attention kernels forward + backward at the long sequences, end to end against the reference."""
    rec = _train_case("xl2_r64_grads", 64)
    assert rec.attn_fwd == {(512, 72, 1), (1024, 32, 1)}, rec.attn_fwd
    assert rec.attn_bwd == {(512, 72, 1), (1024, 32, 1)}, rec.attn_bwd


def test_xl2_eval_cfg_forward_and_short_sampler_vs_reference_golden():
    """BASELINE config 5's network evaluation (XL/2 unmasked: 256 tokens, 16 heads of 72; CFG = one pass at 2B)."""
    from maskdit_b200.sampler import edm_sampler
    g = load("xl2_eval")
    net, cfg, _ = build("DiT-XL/2", 32, 1000)
    net.eval()
    with torch.no_grad(), ImplRecorder() as rec:
        plain = net(g["images"].cuda(), g["sigma"].cuda(), g["labels"].cuda())["x"]
        c = net(g["images"].cuda(), torch.tensor(1.7, dtype=torch.float64).cuda(), g["labels"].cuda(), 1.5)["x"]
    r1, r2 = rel_l2(plain, g["D_plain"]), rel_l2(c, g["D_cfg"])
    print("XL/2 eval rel-L2 plain", r1, "cfg", r2, sorted(rec.attn_fwd))
    assert rec.attn_fwd == {(256, 72, 1), (256, 32, 1)}, rec.attn_fwd
    with torch.no_grad():
        z = edm_sampler(net, g["latents"].cuda(), g["labels"].cuda(), cfg_scale=1.5, num_steps=int(g["num_steps"]))
    rz = rel_l2(z, g["z"])
    print("XL/2 3-step sampler rel-L2", rz)
    assert r1 <= EVAL_TOL and r2 <= CFG_TOL
    assert z.dtype == torch.float64 and rz <= 1e-2


def test_train_step_cuda_graph_matches_eager():
    """TrainStep(graph=True) (zero-grad + loss forward + backward replayed from a CUDA graph) takes the same steps as
    the eager TrainStep: identical loss bit for bit, weights equal up to the order noise of the wgrad atomics."""
    import copy
    from maskdit_b200.train_step import TrainStep
    g = load("s2_train_mask")
    outs = []
    for graph in (False, True):
        net, cfg, _ = build()
        net.train()
        ema = copy.deepcopy(net).eval()
        ts = TrainStep(net, ema, lr=1e-3, loss_fn=GoldenLoss(g), graph=graph)
        losses = [ts.step(g["images"].cuda(), g["labels"].cuda(), 0.5, 0.1).clone() for _ in range(3)]
        outs.append((losses, {k: v.clone() for k, v in net.state_dict().items()}))
    (l0, w0), (l1, w1) = outs
    assert torch.equal(l0[0], l1[0])
    for a, b in zip(l0, l1):
        assert torch.allclose(a, b, rtol=1e-4), (a, b)
    for k in w0:
        assert torch.allclose(w0[k], w1[k], rtol=0, atol=2e-3 * 3), k  # 3 Adam steps of lr 1e-3, sign-like


# ---- round 2: step front, ablation sampler, gradient accumulation, optimizer-state layouts -------------------------------
def test_step_front_kernel_vs_reference_golden():
    from maskdit_b200 import ops
    g = load("step_front")
    lab = g["labels"].cuda().clone()
    y, yn, sigma = ops.step_front(g["moments"].cuda(), g["eps"].cuda(), g["rnd_normal"].cuda(), g["noise_unit"].cuda(),
                                  lab, g["drop_u"].cuda(), float(g["drop_prob"]))
    assert torch.equal(lab.cpu(), g["labels_out"])                      # dropped rows: exact
    assert torch.allclose(y.cpu(), g["y"], rtol=1e-5, atol=1e-6)        # expf vs torch.exp: a few ulp
    assert torch.allclose(sigma.cpu(), g["sigma"], rtol=1e-5)
    assert torch.allclose(yn.cpu(), g["yn"], rtol=1e-5, atol=1e-5)
    y2, _, _ = ops.step_front(g["moments"].cuda(), g["eps"].cuda(), g["rnd_normal"].cuda(), g["noise_unit"].cuda())
    assert torch.equal(y2, y)                                            # no labels / no dropout variant


def test_loss_from_moments_equals_loss_on_sampled_latent():
    """EDMLoss.from_moments (fused step front) == EDMLoss.__call__ on the latent the reference's utils.sample gives
    for the same draws, incl. the label dropout."""
    from maskdit_b200.loss import EDMLoss
    g = load("step_front")
    net, cfg, _ = build()
    net.train()
    mn = torch.rand(6, 16, generator=torch.Generator().manual_seed(3)).cuda()

    class Draws(EDMLoss):
        def __init__(self, seq):
            super().__init__()
            self.seq = list(seq)

        def _randn(self, shape, device):
            t = self.seq.pop(0)
            assert tuple(t.shape) == tuple(shape), (t.shape, shape)
            return t

        def _rand(self, shape, device):
            return g["drop_u"].cuda().reshape(-1, 1) if tuple(shape) == (6, 1) else mn

    a = Draws([g["eps"].cuda(), g["rnd_normal"].cuda().reshape(6, 1, 1, 1), g["noise_unit"].cuda()])
    la = a.from_moments(net, g["moments"].cuda(), g["labels"].cuda().clone(), mask_ratio=0.5, mae_loss_coef=0.1,
                        class_dropout_prob=float(g["drop_prob"]))
    b = Draws([g["rnd_normal"].cuda().reshape(6, 1, 1, 1), g["noise_unit"].cuda()])
    lb = b(net, g["y"].cuda(), g["labels_out"].cuda(), mask_ratio=0.5, mae_loss_coef=0.1)
    assert torch.allclose(la, lb, rtol=2e-3), (la, lb)   # expf vs torch.exp ulps in y, amplified by bf16 rounding


def test_ablation_sampler_vs_reference_golden():
    from maskdit_b200.sampler import ablation_sampler
    g = load("s2_ablation")
    net, cfg, _ = build()
    net.eval()
    lab = g["labels"].cuda()
    for ci in range(int(g["n"])):
        kw = eval(str(g[f"kw{ci}"]))  # noqa: S307 - our own fixture
        noises = [n.cuda() for n in g[f"noises{ci}"]]
        calls = []
        orig = net.forward

        def spy(x, s, *a, **k):
            calls.append(float(s))
            return orig(x, s, *a, **k)

        net.forward = spy
        with torch.no_grad():
            z = ablation_sampler(net, g[f"latents{ci}"].cuda(), lab, cfg_scale=1.5 if ci % 2 == 0 else None,
                                 randn_like=lambda x: noises.pop(0), num_steps=5, **kw)
        net.forward = orig
        assert not noises and z.dtype == torch.float64
        np.testing.assert_allclose(np.array(calls), g[f"sigmas{ci}"].numpy(), rtol=1e-9, err_msg=str(kw))
        r = rel_l2(z, g[f"z{ci}"])
        print("ablation", kw["discretization"], kw["schedule"], kw["scaling"], kw["solver"], "rel-L2", r)
        assert r <= 2e-2, (kw, r)


def test_grad_accum_equals_one_big_batch_and_lr_schedule():
    """train.py:211-227: two micro-batch rounds == one step on the concatenated batch (mean of means, equal sizes);
    reference lr schedule: the first update of a run uses lr 0 (train.py:223 with the pre-increment counter)."""
    import copy
    from maskdit_b200.train_step import TrainStep
    g = load("s2_train_mask")
    x, y = g["images"].cuda(), g["labels"].cuda()

    def fresh(**kw):
        net, _, _ = build()
        net.train()
        return net, TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, loss_fn=GoldenLoss(g), **kw)

    # the same two samples as two micro-batches of one: hand every round its slice of the batch-2 golden draws
    from maskdit_b200.loss import EDMLoss

    class Sliced(EDMLoss):
        def __init__(self):
            super().__init__()
            self.round, self.k = -1, 0

        def __call__(self, *a, **k):
            self.round += 1
            self.k = 0
            return super().__call__(*a, **k)

        def _randn(self, shape, device):
            t = (g["rnd_normal"], g["noise_unit"])[self.k].cuda()[self.round:self.round + 1]
            self.k += 1
            assert tuple(t.shape) == tuple(shape)
            return t

        def _rand(self, shape, device):
            return g["mask_noise"].cuda()[self.round:self.round + 1]

    net1, ts1 = fresh()
    ts1.step(x, y, 0.5, 0.1)
    g1 = ts1.st.grad.clone()
    net2, ts2 = fresh()
    ts2.loss_fn = Sliced()
    ts2.step(x, y, 0.5, 0.1, grad_accum=2)
    g2 = ts2.st.grad.clone() * 0.5            # the kernel folds 1/rounds into the optimizer; the buffer holds the sum
    assert rel_l2(g2, g1) < 2e-3, rel_l2(g2, g1)
    for (k, a), (_, b) in zip(net1.state_dict().items(), net2.state_dict().items()):
        assert torch.allclose(a, b, rtol=0, atol=2.5e-3), k
    net3, ts3 = fresh(reference_lr_schedule=True, lr_rampup_kimg=0.0, global_batch=2)
    w0 = {k: v.clone() for k, v in net3.state_dict().items()}
    ts3.step(x, y, 0.5, 0.1)
    assert all(torch.equal(w0[k], v) for k, v in net3.state_dict().items())      # lr = 0 at train_steps = 0
    ts3.step(x, y, 0.5, 0.1)
    assert any(not torch.equal(w0[k], v) for k, v in net3.state_dict().items())


def test_optimizer_state_layouts_and_namespace_checkpoint(tmp_path):
    """ADVICE r1: (i) `opt` in the layout torch.optim.AdamW(model.parameters()) / apex FusedAdam emit (indices over ALL
    parameters, frozen pos-embeds = 0 and 1 without state; apex keeps `step` in the param_group), (ii) checkpoints whose
    `args` is an argparse.Namespace (reference train.py:259-265) load in train.py / generate.py (weights_only=False)."""
    import argparse
    import copy
    from maskdit_b200.train_step import TrainStep
    g = load("s2_train_mask")
    net, cfg, sd0 = build()
    net.train()
    ts = TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, loss_fn=GoldenLoss(g))
    ts.step(g["images"].cuda(), g["labels"].cuda(), 0.5, 0.1)
    own = ts.state_dict()
    names = [k for k, _ in net.named_parameters()]
    assert min(own["state"]) == 2 and names[0].endswith("pos_embed") and own["param_groups"][0]["params"] == list(
        range(len(names)))
    # (b) a real torch.optim.AdamW over the same parameters produces a loadable dict
    cpu_params = [torch.nn.Parameter(p.detach().cpu().clone(), requires_grad=p.requires_grad) for p in net.parameters()]
    opt = torch.optim.AdamW(cpu_params, lr=3e-4, weight_decay=0)
    for p in cpu_params:
        if p.requires_grad:
            p.grad = torch.randn_like(p)
    opt.step()
    tsd = opt.state_dict()
    assert min(tsd["state"]) == 2
    net2, _, _ = build()
    ts2 = TrainStep(net2.train(), None, lr=1.0)
    ts2.load_state_dict(tsd)
    assert ts2.step_count == 1 and ts2.lr == 3e-4
    k = names[5]
    lo, n, shape = ts2.st.offsets[k]
    assert torch.equal(ts2.m[lo:lo + n].view(shape).cpu(), tsd["state"][5]["exp_avg"])
    # (c) apex layout: no per-parameter step
    apex = {"state": {i: {kk: vv for kk, vv in e.items() if kk != "step"} for i, e in tsd["state"].items()},
            "param_groups": [dict(tsd["param_groups"][0], step=7)]}
    ts2.load_state_dict(apex)
    assert ts2.step_count == 7
    # (ii) Namespace args
    ck = tmp_path / "0000001.pt"
    torch.save({"model": net.state_dict(), "ema": net.state_dict(), "opt": own,
                "args": argparse.Namespace(config="x.yaml", global_seed=0)}, ck)
    loaded = torch.load(ck, map_location="cuda", weights_only=False)
    assert isinstance(loaded["args"], argparse.Namespace)
    ts2.load_state_dict(loaded["opt"])
    assert ts2.step_count == 1


# ---- round 2: the C++ step driver (mdt_forward / mdt_backward) against the kernel-by-kernel Python engine ----------------
@pytest.mark.parametrize("case", ["s2_train_mask", "s2_train_nomask", "xl2_c1_grads"])
def test_c_driver_matches_python_engine(case):
    """`mdt_forward` == `Engine.forward` bit for bit; backward within the fp32-atomics order noise
    (test_model_gpu.py::check_c_driver_matches_engine); the workspace contract."""
    g = load(case)
    xl = case.startswith("xl2")
    net, cfg, _ = build("DiT-XL/2", 32, 1000) if xl else build()
    net.train()
    sigma = (g["rnd_normal"].cuda() * 1.2 - 1.2).exp().reshape(-1).contiguous()
    x = (g["images"].cuda() + g["noise_unit"].cuda() * sigma.view(-1, 1, 1, 1)).contiguous()
    lab = g["labels"].cuda().contiguous()
    md = {k: g[k].cuda() for k in ("mask", "ids_keep", "ids_restore")} if "ids_keep" in g else None
    ce, ctx_c, Fc = check_c_driver_matches_engine(net, x, sigma, lab, md, case)
    st = net.flat_store()
    # the workspace contract: mdt_workspace_bytes is what mdt_forward checks against
    B, T = x.shape[0], (md["ids_keep"].shape[1] if md else cfg.num_patches)
    assert ctx_c["nbytes"] == ce.workspace_bytes(B, T, True) > ce.workspace_bytes(B, T, False)
    from maskdit_b200._lib import MdtError
    with pytest.raises(MdtError):       # a workspace that is too small is refused, not overrun
        ops_ = __import__("maskdit_b200.ops", fromlist=["x"])
        small = torch.empty(1024, dtype=torch.uint8, device="cuda")
        ops_.check(ce._L.mdt_forward(ce._h, st.w32.data_ptr(), st.w16.data_ptr(), x.data_ptr(), sigma.data_ptr(),
                                     lab.data_ptr(), 0, 0, B, 0, 0, small.data_ptr(), 1024, Fc.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream), "mdt_forward", 0)


# ---- the sampler tail — SD-VAE decode on the wgmma GEMM + fused im2col (sample.py:275,287) ----------------
def test_vae_decode_vs_reference_golden():
    """`AutoencoderKLDecoder.decode` vs the unmodified reference Decoder + post_quant_conv (autoencoder.py:306-453) on the
    stand-in weights: 8x8 latents -> 64x64 images (every layer type: conv_in, ResnetBlocks with and without nin_shortcut,
    the AttnBlock, three upsampling convolutions, norm_out + conv_out), then the 8-bit conversion of sample.py:287."""
    from maskdit_b200 import ops
    from maskdit_b200.vae import AutoencoderKLDecoder
    from oracle import vae_oracle as VO
    g = load("vae_decode")
    vae = AutoencoderKLDecoder()
    vae.load_state_dict(VO.make_vae_state_dict(3), strict=True)
    vae = vae.cuda().eval()
    img = vae.decode(g["z"].cuda())
    assert img.shape == g["images"].shape and torch.isfinite(img).all()
    r = rel_l2(img, g["images"])
    print("VAE decode rel-L2 vs the reference's fp32 output:", r)
    assert r <= 1e-2, r                                   # measured 5.5e-3: ~30 bf16-operand convolutions
    u8 = ops.to_uint8_nhwc(img.contiguous()).cpu()
    diff = (u8.int() - g["u8"].int()).abs()
    print("8-bit image: mean |diff|", diff.float().mean().item(), "max", diff.max().item())
    assert diff.float().mean().item() <= 1.5
    # deterministic (no atomics anywhere on the path): a second run, and a run with chunked im2col operands (several GEMM
    # launches per convolution), give the same image bit for bit
    assert torch.equal(vae.decode(g["z"].cuda()), img)
    vae.max_rows = 2048
    assert torch.equal(vae.decode(g["z"].cuda()), img)
    with pytest.raises(NotImplementedError):
        vae(g["z"].cuda(), "encode")


def test_unconditional_odd_token_count_vs_reference_golden():
    """Edge geometry against the unmodified reference: class-UNconditional network (num_classes = 0: no label embedder,
    labels None) with 30 % masking -> 179 kept tokens per sample, batch 3: token counts that are not multiples of 128
    (the mma.sync attention kernels, asserted), ragged GEMM M (537 / 768 rows), loss and every gradient."""
    g = load("s2_uncond_mask30")
    net, cfg, _ = build("DiT-S/2", 32, 0)
    net.train()
    lf = GoldenLoss(g)
    with ImplRecorder() as rec:
        loss = lf(net, g["images"].cuda(), None, mask_ratio=0.3, mae_loss_coef=0.1)
        for k in ("mask", "ids_keep", "ids_restore"):
            assert torch.equal(lf.last_mask_dict[k].cpu(), g[k]), k
        loss.mean().backward()
    assert lf.last_mask_dict["ids_keep"].shape == (3, 179)
    assert torch.allclose(loss.cpu(), g["loss"], rtol=LOSS_TOL), (loss, g["loss"])
    check_grads(net, g, what="unconditional, T=179")
    assert (179, 64, 0) in rec.attn_fwd and (179, 64, 0) in rec.attn_bwd, (rec.attn_fwd, rec.attn_bwd)
    assert (256, 32, 1) in rec.attn_fwd            # the decoder still runs all 256 tokens on the wgmma kernels


def test_full_size_config4_properties():
    """BASELINE config 4 at the largest per-GPU batch an 80 GB H100 holds (XL/2, 64x64x4 latents, mask 0.5, batch 64:
    512 kept / 1024 decoder tokens per sample, a 54 GB workspace) through the loss interface without recomputation:
    the mask path invariants hold for every row and one backward leaves finite gradients everywhere.  Every row and
    every gradient of this step against batch-2 runs: tests/test_production_batch_gpu.py."""
    from maskdit_b200.loss import EDMLoss
    import gc
    gc.collect()
    torch.cuda.empty_cache()          # the 54 GB workspace needs the blocks earlier tests left in the caching allocator
    torch.manual_seed(0)
    net, cfg, _ = build("DiT-XL/2", 64, 1000)
    net.train()
    B, L = 64, 1024
    g = torch.Generator().manual_seed(6)
    images = (torch.randn(B, 4, 64, 64, generator=g) * 0.5).cuda()
    labels = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float().cuda()
    rnd, nz, mn = torch.randn(B, 1, 1, 1, generator=g).cuda(), torch.randn(B, 4, 64, 64, generator=g).cuda(), \
        torch.rand(B, L, generator=g).cuda()

    class Lz(EDMLoss):
        def __init__(self, n):
            super().__init__()
            self.q, self.n = [rnd[:n], nz[:n]], n

        def _randn(self, shape, device):
            return self.q.pop(0).contiguous()

        def _rand(self, shape, device):
            return mn[:self.n].contiguous()

    lf = Lz(B)
    full = lf(net, images, labels, mask_ratio=0.5, mae_loss_coef=0.1)
    md = lf.last_mask_dict
    assert torch.isfinite(full).all()
    assert torch.equal(md["mask"].sum(1), torch.full((B,), 512.0, device="cuda"))
    assert torch.equal(torch.gather(md["ids_restore"], 1, md["ids_keep"]), torch.arange(512, device="cuda").expand(B, -1))
    full.mean().backward()
    st = net.flat_store()
    assert torch.isfinite(st.grad).all() and float(st.grad.abs().sum()) > 0
    del lf, md
    torch.cuda.empty_cache()
