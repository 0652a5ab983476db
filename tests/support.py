"""Shared support of the test suites: fixtures, float64 and golden helpers, the kernel- and step-reference helpers of
more than one suite, and the stand-in that runs a world-1 `TrainStep` as rank 0 of two ranks.

A test module imports the fixtures it uses by name (`from support import ops  # noqa: F401`): pytest finds fixtures
in a module's namespace.  Nothing here needs a GPU to import."""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
bf16 = torch.bfloat16
NAN = float("nan")


# ---- fixtures -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
    from maskdit_b200 import ops as o
    return o


@pytest.fixture
def lib():
    """The library, entered with the whole device's grids; the torch flag, the library setting and the SM budget are
    restored afterwards."""
    from maskdit_b200 import _lib
    L = _lib.lib()
    det, budget, flag = L.mdt_get_deterministic(), L.mdt_get_sm_budget(), torch.are_deterministic_algorithms_enabled()
    assert L.mdt_set_sm_budget(0) == 0
    yield L
    torch.use_deterministic_algorithms(flag)
    assert L.mdt_set_deterministic(det) == 0 and L.mdt_set_sm_budget(budget) == 0


@pytest.fixture
def det():
    """Deterministic mode on for the test; the torch flag and the library setting are restored afterwards, and the SM
    budget is reset to the whole device."""
    from maskdit_b200 import _lib
    L = _lib.lib()
    was, flag = L.mdt_get_deterministic(), torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(flag)
    assert L.mdt_set_deterministic(was) == 0
    assert L.mdt_set_sm_budget(0) == 0


@pytest.fixture
def clean_env(monkeypatch):
    """None of the environment variables that select the gradient exchange or the training graph."""
    for k in ("MDT_GRAD_AR", "MDT_COLLECTIVE", "MDT_AR_CHUNKS", "MDT_TRAIN_GRAPH"):
        monkeypatch.delenv(k, raising=False)


def one_rank_comm(L, max_ctas=0):
    """A one-rank NCCL communicator of the C ABI; max_ctas > 0 confines it to that many CTAs (ncclCommInitRankConfig)."""
    uid = ctypes.create_string_buffer(128)
    rc = L.mdt_nccl_unique_id(uid)
    assert rc == 0, f"mdt_nccl_unique_id: status {rc} (-3: libnccl.so.2 not resolved)"
    comm = ctypes.c_void_p()
    rc = L.mdt_nccl_comm_create(bytes(uid.raw), 0, 1, max_ctas, ctypes.byref(comm))
    assert rc == 0 and comm.value, f"mdt_nccl_comm_create(max_ctas={max_ctas}): status {rc}"
    return comm


@pytest.fixture(scope="module")
def comm():
    """A one-rank communicator, full width."""
    from maskdit_b200 import _lib
    c = one_rank_comm(_lib.lib())
    yield c
    assert _lib.lib().mdt_nccl_comm_destroy(c) == 0


@pytest.fixture
def rank0_of_two(comm):
    """make(ts, ar_chunks, peer_flag=0.0, record=None): `make_rank0_of_two` on the module's communicator.  At the end
    of the test every stand-in must have exchanged, and every `mdt_allreduce_grads` status must be 0."""
    statuses = []

    def make(ts, ar_chunks, peer_flag=0.0, record=None):
        make_rank0_of_two(ts, comm, ar_chunks, peer_flag, record)
        statuses.append(ts.comm.rcs)   # the list only: the TrainStep can be freed before the end of the test
        return ts

    yield make
    for rcs in statuses:
        assert rcs and all(rc == 0 for rc in rcs), rcs


# ---- rank 0 of two ranks ------------------------------------------------------------------------------------------------
class TwoRanks:
    """`GradComm` stand-in on rank 0 of two ranks that hold the same gradient: runs the real one-rank
    `mdt_allreduce_grads` (statuses in `rcs`), then adds the other rank's contribution: a gradient buffer is doubled
    (the exact two-rank sum), the guard's flag word gets `peer_flag`.  `record(lo, hi, dtype, stream, sm_budget, snap)`,
    when given, is called for every gradient range with a copy of the range taken before its exchange."""

    def __init__(self, ts, comm, peer_flag, record):
        self.ts, self.comm, self.peer_flag, self.record = ts, comm, peer_flag, record
        self.rcs = []

    def all_reduce(self, t):
        from maskdit_b200 import ops
        L = ops.lib()
        flag = self.ts._flag is not None and t.data_ptr() == self.ts._flag.data_ptr()
        snap = t.clone() if self.record and not flag else None   # on the current stream: in stream order
        self.rcs.append(L.mdt_allreduce_grads(self.comm, t.data_ptr(), t.numel(), int(t.dtype == bf16),
                                              ops.stream_ptr()))
        if flag:
            t.add_(self.peer_flag)
            return
        if self.record:
            base = self.ts.g16 if t.dtype == bf16 else self.ts.st.grad
            lo = (t.data_ptr() - base.data_ptr()) // t.element_size()
            self.record(lo, lo + t.numel(), t.dtype, torch.cuda.current_stream().cuda_stream, L.mdt_get_sm_budget(),
                        snap)
        t.mul_(2)

    def close(self):
        pass   # the communicator belongs to the module's fixture


def make_rank0_of_two(ts, comm, ar_chunks, peer_flag=0.0, record=None):
    """Turn a world-1 TrainStep into rank 0 of a two-rank job (tools/dp_equivalence.py flips the same fields back)."""
    ts.world = 2
    ts.comm = TwoRanks(ts, comm, peer_flag, record)
    if ts.grad_dtype == "bf16":
        ts.g16 = torch.empty(ts.st.n_train, dtype=bf16, device="cuda")
    ts.ar_chunks = ar_chunks
    return ts


# ---- float64 and the reference goldens -----------------------------------------------------------------------------------
def f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def ulp32(x64):
    a = torch.as_tensor(x64, dtype=torch.float64).abs().float()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def load(name):
    return {k: (torch.from_numpy(np.asarray(v)) if v.dtype.kind in "fiub" else v)
            for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}


def rel_l2(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def build(model_type="DiT-S/2", R=8, ncls=10, seed=1):
    from maskdit_b200.maskdit import Precond_models
    from oracle import maskdit_oracle as O
    cfg = O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls)
    net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=ncls, model_type=model_type,
                                use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False)
    sd = O.make_state_dict(cfg, seed)
    net.load_state_dict(sd, strict=True)
    return net.cuda(), cfg, sd


# the model-level bounds of a bf16-operand implementation against an fp32 reference: test_model_gpu.py's docstring
FWD_TOL, GRAD_TOL, LOSS_TOL = 3e-3, 1.5e-2, 5e-3   # rel-L2 outputs / rel-L2 gradients / relative loss
EVAL_TOL, CFG_TOL = 6e-3, 1e-2   # unmasked eval forward / CFG-combined output (see the yardstick in DESIGN.md §5)


def check_grads(net, g, tol=GRAD_TOL, what=""):
    """Every parameter-gradient norm, the stored full gradients and the stored 4x8 slices against the reference's."""
    worst, n = (0.0, ""), 0
    for k, p in net.named_parameters():
        key = f"gnorm/{k}"
        if key not in g:
            continue
        gn, ref = p.grad.double().norm().item(), float(g[key])
        assert abs(gn - ref) <= tol * ref + 1e-7, (k, gn, ref)
        n += 1
        if f"grad/{k}" in g and ref > 0:
            r = rel_l2(p.grad, g[f"grad/{k}"])
            worst = max(worst, (r, k))
            assert r <= tol, (k, r)
        if f"gslice/{k}" in g and ref > 0:
            sl = p.grad.reshape(p.grad.shape[0], -1)[:4, :8]
            want = g[f"gslice/{k}"]
            # a 32-element slice: compare against the scale of the whole tensor (rms), bf16 backward noise
            rms = ref / max(p.grad.numel(), 1) ** 0.5
            assert (sl.cpu().double() - want.double()).abs().max().item() <= 8 * tol * rms + 1e-9, k
    assert n > 100
    print(what, "worst grad rel-L2", worst, "over", n, "tensors")


def check_c_driver_matches_engine(net, x, sigma, lab, md, what="", dF_same_grads=None):
    """The C++ step driver (`mdt_forward` / `mdt_backward`: one ctypes call each, one workspace) of the training-mode
    `net` against the kernel-by-kernel Python `Engine` on the same flat store.  The forward agrees BIT FOR BIT, with and
    without saved activations: same kernels, same order, same operands.  The backward accumulates wgrads with fp32
    atomics (run-to-run order noise), so the gradients of a random dF agree to 5e-5 of each tensor's scale (1e-2 on the
    conditioning path, see below).  `dF_same_grads(dF)`, when given, is a second dF for which the driver must give the
    same gradients.  Returns the driver, its context of the saving forward and its F."""
    from maskdit_b200.engine import CEngine, Engine
    st = net.prepare()
    ce, pe = net._engine, Engine(net._cfg(), st)
    assert isinstance(ce, CEngine)
    for save in (False, True):
        Fc, ctx_c = ce.forward(x, sigma, lab, md, save)
        Fp, ctx_p = pe.forward(x, sigma, lab, md, save)
        assert torch.equal(Fc, Fp), (save, (Fc - Fp).abs().max())
    dF = (torch.randn_like(Fc) * 0.1).to(torch.bfloat16)

    def grads(engine, ctx, dF_):
        st.ensure_grad().zero_()
        engine.backward(ctx, dF_)
        return st.grad.clone()

    got = [grads(ce, ctx_c, dF)]
    gp = grads(pe, ctx_p, dF)
    if dF_same_grads is not None:
        got.append(grads(ce, ctx_c, dF_same_grads(dF)))
    worst = 0.0
    for k, (o, n, _) in st.offsets.items():
        if o + n > st.n_train:
            continue
        b = gp[o:o + n]
        scale = b.abs().max().item() + 1e-30
        # Order noise of the fp32 atomics: 1e-7 .. 1e-5 on the block tensors.  On the conditioning path the noisy sums
        # are re-rounded to bf16 several times before GEMMs that contract over only B = 2 rows (dmod -> bf16 -> adaLN
        # wgrad; dsc -> dc (bf16) -> dth -> dpre (bf16) -> t_embedder wgrad): one flipped bf16 rounding moves an element
        # by 2^-8, measured up to 2e-3 of a tensor's scale between two runs of the SAME engine - not a code difference.
        cond = any(t in k for t in ("adaLN_modulation", "t_embedder", "y_embedder"))
        for g in got:
            err = (g[o:o + n] - b).abs().max().item() / scale
            worst = max(worst, err)
            assert err <= (1e-2 if cond else 5e-5), (k, err)
    print(what, "C driver vs Python engine: forward bit-equal, worst gradient deviation", worst)
    return ce, ctx_c, Fc


class ImplRecorder:
    """Which GEMM instances (BLOCK_N*10 + CTAs per tile) and which attention kernel families served the calls made
    inside the `with` block — read from the library's own logs (mdt_gemm_configs_seen / mdt_attention_impl_log), so the
    C++ step driver's internal launches are covered as well as per-kernel calls from Python."""

    def __enter__(self):
        from maskdit_b200 import ops
        self.L = ops.lib()
        self.L.mdt_gemm_configs_seen(1)
        self.L.mdt_attention_impl_log(None, 0)
        self.gemm_cfgs, self.attn_fwd, self.attn_bwd = set(), set(), set()
        return self

    def __exit__(self, *exc):
        bits = self.L.mdt_gemm_configs_seen(1)
        names = [1281, 1282, 1921, 1922, 2561, 2562]
        self.gemm_cfgs = {names[i] for i in range(6) if bits >> i & 1}
        buf = (ctypes.c_int * 4096)()
        n = self.L.mdt_attention_impl_log(buf, 1024)
        for i in range(n):
            which, T, dh, impl = buf[4 * i:4 * i + 4]
            (self.attn_bwd if which else self.attn_fwd).add((T, dh, impl))


class GoldenLoss:
    """EDMLoss with the golden random draws injected in the reference's draw order."""

    def __new__(cls, g):
        from maskdit_b200.loss import EDMLoss

        class _L(EDMLoss):
            def __init__(self):
                super().__init__()
                self.q_randn = [g["rnd_normal"].cuda(), g["noise_unit"].cuda()]
                self.q_rand = [g["mask_noise"].cuda()] if "mask_noise" in g else []

                self.n_randn = 0

            def _randn(self, shape, device):   # draws cycle (sigma, noise, sigma, noise, ...): reusable across steps
                t = self.q_randn[self.n_randn % 2]
                self.n_randn += 1
                assert tuple(t.shape) == tuple(shape)
                return t

            def _rand(self, shape, device):
                return self.q_rand[0]

        return _L()


def nd_dit_forward(sd, cfg, x, t, y, mask_dict=None, training=True):
    """DiT.forward without the decoder (models/maskdit.py:511-557 with use_decoder=False), built from the oracle's
    pieces: embedding + mask_out_token, the encoder blocks, FinalLayer on the encoder width, and for masked training
    the kept rows scattered into zeros (:551-553).  The decoder model is left to `maskdit_oracle.dit_forward`."""
    from oracle import maskdit_oracle as O
    assert not cfg.use_decoder
    D, P, B = cfg.hidden, cfg.patch, x.shape[0]
    patches = x.reshape(B, cfg.img_channels, cfg.grid, P, cfg.grid, P).permute(0, 2, 4, 1, 3, 5).reshape(
        B, cfg.num_patches, -1)
    h = F.linear(patches, sd["model.x_embedder.proj.weight"].reshape(D, -1), sd["model.x_embedder.proj.bias"]) + \
        sd["model.pos_embed"]
    masked = mask_dict is not None and training
    if masked:
        h = torch.gather(h, 1, mask_dict["ids_keep"].unsqueeze(-1).expand(-1, -1, D))
    te = F.linear(O.timestep_embedding(t, 256), sd["model.t_embedder.mlp.0.weight"], sd["model.t_embedder.mlp.0.bias"])
    c = F.linear(F.silu(te), sd["model.t_embedder.mlp.2.weight"], sd["model.t_embedder.mlp.2.bias"])
    if cfg.num_classes:
        c = c + F.linear(y, sd["model.y_embedder.embedding_table.weight"])
    for i in range(cfg.depth):
        h = O._block(sd, f"model.blocks.{i}", h, c, cfg.heads)
    sh, sc = F.linear(F.silu(c), sd["model.final_layer.adaLN_modulation.1.weight"],
                      sd["model.final_layer.adaLN_modulation.1.bias"]).chunk(2, dim=1)
    out = F.linear(O._modulate(O._ln(h), sh, sc), sd["model.final_layer.linear.weight"],
                   sd["model.final_layer.linear.bias"])
    if masked:
        full = out.new_zeros(B, cfg.num_patches, out.shape[-1])
        out = full.scatter(1, mask_dict["ids_keep"].unsqueeze(-1).expand(-1, -1, out.shape[-1]), out)
    return O.unpatchify(out, P, cfg.img_channels)


# ---- the fused AdamW + EMA kernel against float64 ------------------------------------------------------------------------
STEPS = (1, 2, 3, 4, 5, 1000)   # five consecutive steps, then one where the bias corrections are far from 1
LR = 1e-3
# weight decay, gradient scale, EMA given, bf16 shadow given
CFGS = {"wd0-half-ema-w16": (0.0, 1 / 2, True, True), "wd-16th-w16": (0.03, 1 / 16, False, True),
        "wd-half-ema": (0.03, 1 / 2, True, False), "wd0-16th-bare": (0.0, 1 / 16, False, False)}


def adamw_inputs(n, seed):
    """Seeded fp32 start state and one bf16 gradient per step, each with a slice of exact zeros."""
    gen = torch.Generator().manual_seed(seed)
    w = torch.randn(n, generator=gen)
    ema = w + 0.01 * torch.randn(n, generator=gen)
    z0, z1 = n // 3, n // 3 + max(n // 10, 1)
    grads = []
    for k in range(len(STEPS)):
        g = (torch.randn(n, generator=gen) * 10.0 ** (-1 - k % 3)).to(bf16)
        g[z0:z1] = 0
        grads.append(g)
    return w, ema, grads


def run_adamw(ops, w, ema, grads, wd, gs, with_ema, with_w16, max_blocks=0, fp32_grad=False, chunks=None):
    n = w.numel()
    out = {"w": w.cuda(), "m": torch.zeros(n, device="cuda"), "v": torch.zeros(n, device="cuda"),
           "ema": ema.cuda() if with_ema else None,
           "w16": torch.zeros(n, dtype=bf16, device="cuda") if with_w16 else None}
    for step, g in zip(STEPS, grads):
        g = g.cuda()
        if fp32_grad:
            g = g.float()
        for lo, hi in chunks or [(0, n)]:
            sl = {k: (v[lo:hi] if v is not None else None) for k, v in out.items()}
            ops.adamw_ema(sl["w"], g[lo:hi], sl["m"], sl["v"], sl["ema"], sl["w16"], hi - lo, LR, step,
                          weight_decay=wd, grad_scale=gs, max_blocks=max_blocks)
    torch.cuda.synchronize()
    return out


# ---- deterministic-mode steps from the oracle's weights ------------------------------------------------------------------
_SD = {}


def oracle_net(mt, R, ncls, dec):
    """A fresh training network from a cached oracle state dict (seed 1)."""
    from maskdit_b200.maskdit import Precond_models
    from oracle import maskdit_oracle as O
    key = (mt, R, ncls, dec)
    if key not in _SD:
        _SD[key] = O.make_state_dict(O.Cfg(model_type=mt, img_resolution=R, num_classes=ncls, use_decoder=dec), 1)
    net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=ncls, model_type=mt, use_decoder=dec,
                                mae_loss_coef=0.1, pad_cls_token=False)
    net.load_state_dict(_SD[key], strict=True)
    return net.cuda().train()


def step_state(ts, losses):
    st = ts.st
    return [*losses, st.grad.clone(), st.w32.clone(), st.w16.clone(), ts.m.clone(), ts.v.clone(), ts.ema_st.w32.clone()]


def det_steps(mt, R, ncls, dec, B, mask, n=3, golden=None, seed=0, budget=0, grad_accum=1, **kw):
    """n deterministic-mode steps of a fresh TrainStep; returns step_state()."""
    from maskdit_b200 import ops
    from maskdit_b200.train_step import TrainStep
    torch.use_deterministic_algorithms(True)
    net = oracle_net(mt, R, ncls, dec)
    ts = TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, loss_fn=GoldenLoss(golden) if golden else None, **kw)
    gen = torch.Generator().manual_seed(seed)
    if golden:
        x, lab = golden["images"].cuda(), (golden["labels"].cuda() if "labels" in golden else None)
    else:
        x = (torch.randn(B, 4, R, R, generator=gen) * 0.5).cuda()
        lab = torch.eye(ncls)[torch.randint(0, ncls, (B,), generator=gen)].cuda() if ncls else None
    torch.manual_seed(seed)
    ops.check(ops.lib().mdt_set_sm_budget(budget), "mdt_set_sm_budget", 0)
    losses = [ts.step(x, lab, mask, 0.1, grad_accum=grad_accum).clone() for _ in range(n)]
    ops.check(ops.lib().mdt_set_sm_budget(0), "mdt_set_sm_budget", 0)
    assert ops.lib().mdt_get_deterministic() == 1
    out = step_state(ts, losses)
    del ts, net
    torch.cuda.empty_cache()
    return out


def assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (i, (x.double() - y.double()).abs().max().item())


# ---- steps on VAE moments with live gradients ------------------------------------------------------------------------------
MODELS = {"S/2": ("DiT-S/2", 32, 1000, 4), "XL/2": ("DiT-XL/2", 32, 1000, 8)}   # model type, R, classes, batch


def live_net(model):
    """The training network from torch's init (seed 1), built on the device; the zero-initialised tensors get values
    (a CUDA generator, seed 2), so every gradient is live."""
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


def batches(model, k):
    """k batches of VAE moments and one-hot labels; batch i is drawn with its own seed."""
    _, R, ncls, B = MODELS[model]
    out = []
    for i in range(k):
        g = torch.Generator().manual_seed(100 + i)
        mom = torch.cat([torch.randn(B, 4, R, R, generator=g), torch.randn(B, 4, R, R, generator=g) - 2], 1)
        lab = torch.nn.functional.one_hot(torch.randint(0, ncls, (B,), generator=g), ncls).float()
        out.append((mom.cuda(), lab.cuda(), 1000 + i))
    return out


def poison(batch):
    mom, lab, seed = batch
    mom = mom.clone()
    mom[0, 0, 3, 5] = NAN   # one NaN in the moments' mean
    return mom, lab, seed


def step_batch(ts, batch, ga=1):
    mom, lab, seed = batch
    torch.manual_seed(seed)   # the step's draws (sigma, noise, latent eps, mask noise, label dropout) belong to the batch
    return ts.step(mom, lab, 0.5, 0.1, grad_accum=ga, moments=True, class_dropout_prob=0.1)


def opt_state(ts):
    n = ts.st.n_train
    return {"w32": ts.st.w32[:n].clone(), "w16": ts.st.w16[:n].clone(), "m": ts.m.clone(), "v": ts.v.clone(),
            "ema": ts.ema_st.w32[:n].clone()}


def assert_skipped(before, after, ema_decay):
    """A skipped step: weights, shadow and moments unchanged, the EMA moved towards the weights."""
    for k in ("w32", "w16", "m", "v"):
        assert torch.equal(before[k], after[k]), k
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
        bound = ulp32(want) + ulp32(d * e0) + ulp32((1 - d) * w0)
        assert (err <= bound).all(), (lo, (err / bound).max().item())


# train.py on synthetic latents: DiT-S/2 at 16 x 16, four steps, a checkpoint after the fourth
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
