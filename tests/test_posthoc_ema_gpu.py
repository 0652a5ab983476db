"""GPU: power-function EMA profiles for post-hoc EMA.

1. `mdt_power_ema` against a float64 recurrence with the same fp32 coefficients: k = 1..4, sizes that are not a
   multiple of 4, slices at every 4-byte offset (shared and mixed 16-byte phases), exact copy at t = 1, bitwise repeats.
2. `TrainStep(phema_sigma_rels=(0.05, 0.10))` on DiT-S/2: every profile is the float64 power EMA of the recorded w32
   sequence, eager, with grad_accum = 2, across a step skipped for a non-finite gradient, from CUDA graphs and with
   recomputation.
3. Off by default: no launch and no bit differs; with profiles on, the weights and the EMA are unchanged.
4. Resume: a run interrupted after a state_dict() round trip continues its profiles bit for bit.
5. World > 1 (rank 0 of two identical ranks): every element is updated exactly once per step, after its optimizer
   pass and on that pass's stream.
6. train.py writes snapshots, posthoc_ema.py reconstructs sigma_rel 0.08 and generate.py samples from it.
"""
import copy
import ctypes
import gc
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from maskdit_b200 import phema  # noqa: E402

bf16 = torch.bfloat16
SIGMAS = (0.05, 0.10)


@pytest.fixture(scope="module")
def ops():
    from maskdit_b200 import ops as o
    return o


@pytest.fixture
def det():
    """Deterministic mode on for the test; the torch flag and the SM budget are restored afterwards."""
    from maskdit_b200 import _lib
    flag = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(flag)
    _lib.sync_deterministic()
    assert _lib.lib().mdt_set_sm_budget(0) == 0


def _f32(x):
    return float(np.float32(x))


def _ulp32(x64):
    a = x64.abs().float()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def _replay(ws, gammas, t0=1):
    """float64 power EMA of the w sequence with the fp32-rounded coefficients the kernel receives."""
    es = [torch.zeros_like(ws[0], dtype=torch.float64) for _ in gammas]
    for t, w in enumerate(ws, start=t0):
        w = w.double()
        for j, g in enumerate(gammas):
            es[j] += _f32(phema.one_minus_beta(g, t)) * (w - es[j])
    return es


def _assert_close(got, want, ws, what):
    """Each step rounds w - e, the product and the sum: at most ~2 ulp of max|w| per step (e is a convex combination
    of the w's, so it never exceeds them; an earlier error only shrinks by the factor 1 - c)."""
    mx = torch.stack([w.double().abs() for w in ws]).amax(0)
    bound = 2 * len(ws) * _ulp32(mx) + 1e-30
    err = (got.double() - want).abs()
    assert (err <= bound).all(), (what, (err / bound).max().item())
    return (err / _ulp32(mx).clamp_min(1e-30)).max().item()


# ---- 1. the kernel ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_kernel_vs_float64(ops, k):
    gammas = [phema.sigma_rel_to_gamma(s) for s in (0.05, 0.10, 0.2, 0.03)[:k]]
    worst = 0.0
    for n in (1, 3, 5, 1021, 262_147):
        for w_off, e_off in ((0, 0), (1, 1), (2, 2), (3, 3), (0, 1), (3, 2)):   # elements past a 16-byte boundary
            g = torch.Generator(device="cuda").manual_seed(n + 10 * w_off + e_off)
            wbuf = torch.empty(n + 8, device="cuda")
            ebufs = [torch.full((n + 8,), 7.0, device="cuda") for _ in range(k)]   # t = 1 overwrites whatever is there
            w, es = wbuf[w_off:w_off + n], [b[e_off:e_off + n] for b in ebufs]
            ws = []
            for t in range(1, 7):
                w.copy_(torch.randn(n, device="cuda", generator=g) * (1 + t))
                ws.append(w.clone())
                ops.power_ema(w, es, [phema.one_minus_beta(gm, t) for gm in gammas])
                if t == 1:
                    for e in es:
                        assert torch.equal(e, w), (n, w_off, e_off)      # exact copy
            for b in ebufs:   # nothing outside the slice is touched
                assert (b[:e_off] == 7.0).all() and (b[e_off + n:] == 7.0).all()
            want = _replay(ws, gammas)
            for j in range(k):
                worst = max(worst, _assert_close(es[j], want[j], ws, (k, n, w_off, e_off, j)))
            # bitwise repeatable, whatever the alignment
            es2 = [torch.zeros(n, device="cuda") for _ in range(k)]
            for t, wt in enumerate(ws, start=1):
                ops.power_ema(wt, es2, [phema.one_minus_beta(gm, t) for gm in gammas])
            for a, b in zip(es, es2):   # float4 and scalar paths compute the same bits
                assert torch.equal(a, b), (k, n, w_off, e_off)
    print(f"power_ema k={k}: worst error {worst:.2f} ulp of max|w|")


def test_kernel_refuses_cpu_and_mismatched_buffers(ops):
    from maskdit_b200._lib import MdtError
    w = torch.zeros(16, device="cuda")
    with pytest.raises(MdtError):
        ops.power_ema(w.cpu(), [w.cpu()], [0.5])
    with pytest.raises(MdtError):
        ops.power_ema(w, [torch.zeros(15, device="cuda")], [0.5])
    with pytest.raises(MdtError):
        ops.power_ema(w, [w.clone()], [0.5, 0.5])
    with pytest.raises(MdtError):
        ops.power_ema(w, [w.clone() for _ in range(5)], [0.5] * 5)
    with pytest.raises(MdtError):
        ops.power_ema(w, [w.clone()], [1.5])


# ---- 2. TrainStep -----------------------------------------------------------------------------------------------------------
R, NCLS, B = 32, 1000, 4


def _net():
    from maskdit_b200.maskdit import Precond_models
    torch.manual_seed(1)
    with torch.device("cuda"):
        net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=NCLS, model_type="DiT-S/2",
                                    use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False)
        gz = torch.Generator(device="cuda").manual_seed(2)
        with torch.no_grad():   # the zero-initialised tensors get values: every gradient is live
            for p in net.parameters():
                if p.requires_grad and float(p.abs().sum()) == 0.0:
                    p.copy_(torch.randn(p.shape, generator=gz, device="cuda") * 0.02)
    return net.train()


def _batches(k):
    out = []
    for i in range(k):
        g = torch.Generator().manual_seed(100 + i)
        mom = torch.cat([torch.randn(B, 4, R, R, generator=g), torch.randn(B, 4, R, R, generator=g) - 2], 1)
        lab = torch.nn.functional.one_hot(torch.randint(0, NCLS, (B,), generator=g), NCLS).float()
        out.append((mom.cuda(), lab.cuda(), 1000 + i))
    return out


def _poison(batch):
    mom, lab, seed = batch
    mom = mom.clone()
    mom[0, 0, 3, 5] = float("nan")
    return mom, lab, seed


def _step(ts, batch, ga=1):
    mom, lab, seed = batch
    torch.manual_seed(seed)
    return ts.step(mom, lab, 0.5, 0.1, grad_accum=ga, moments=True, class_dropout_prob=0.1)


def _trainstep(**kw):
    from maskdit_b200.train_step import TrainStep
    net = _net()
    return TrainStep(net, copy.deepcopy(net).eval(), lr=1e-3, weight_decay=0.01, global_batch=B, **kw)


MODES = {
    "eager": dict(),
    "grad_accum2": dict(grad_accum=2),
    "skip_nonfinite": dict(skip_nonfinite=True, poison=2),
    "graph": dict(graph=True),
    "recompute": dict(recompute_blocks=3),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_trainstep_profiles_are_the_power_ema_of_the_weights(mode):
    kw = dict(MODES[mode])
    ga, poison = kw.pop("grad_accum", 1), kw.pop("poison", None)
    ts = _trainstep(phema_sigma_rels=SIGMAS, **kw)
    n = ts.st.n_train
    assert len(ts.phema_emas) == 2 and all(e.numel() == n for e in ts.phema_emas)
    ws = []
    data = _batches(6)
    for i, b in enumerate(data):
        if i == poison:
            b = _poison(b)
            before = ts.st.w32[:n].clone()
        _step(ts, b, ga)
        ws.append(ts.st.w32[:n].clone())
        if i == 0:
            for e in ts.phema_emas:
                assert torch.equal(e, ws[0])       # t = 1: a copy of the weights after the first update
        if i == poison:
            assert torch.equal(ws[-1], before) and int(ts.skipped_steps) == 1
    torch.cuda.synchronize()
    assert ts.phema_origin == 0 and ts.phema_steps == 6
    if mode == "recompute":
        assert ts.recompute_blocks == 3
    want = _replay(ws, ts.phema_gammas)
    worst = max(_assert_close(e, w, ws, (mode, j)) for j, (e, w) in enumerate(zip(ts.phema_emas, want)))
    # the two widths differ, and both differ from the reference-fixed EMA
    assert not torch.equal(ts.phema_emas[0], ts.phema_emas[1])
    print(f"{mode}: worst profile error {worst:.2f} ulp of max|w|")


# ---- 3. off by default -------------------------------------------------------------------------------------------------------
def test_off_by_default_and_invisible_to_training(det, ops):
    runs = {}
    for name, kw in (("default", {}), ("empty", dict(phema_sigma_rels=())), ("on", dict(phema_sigma_rels=SIGMAS))):
        ts = _trainstep(**kw)
        n = ts.st.n_train
        assert bool(ts.phema_emas) == (name == "on")
        n0 = ops.L.LAUNCHES
        for b in _batches(3):
            _step(ts, b)
        torch.cuda.synchronize()
        runs[name] = (ops.L.LAUNCHES - n0, ts.st.w32[:n].clone(), ts.ema_st.w32[:n].clone(), ts.m.clone())
        del ts
        gc.collect()
        torch.cuda.empty_cache()
    d, e, o = runs["default"], runs["empty"], runs["on"]
    assert d[0] == e[0] and all(torch.equal(a, b) for a, b in zip(d[1:], e[1:]))
    assert o[0] == d[0] + 3                                    # one power-EMA launch per optimizer pass
    assert all(torch.equal(a, b) for a, b in zip(d[1:], o[1:]))   # weights, EMA and moments unchanged


# ---- 4. resume ---------------------------------------------------------------------------------------------------------------
def test_resume_continues_the_profiles_bit_for_bit(det):
    data = _batches(5)
    ts = _trainstep(phema_sigma_rels=SIGMAS)
    for b in data:
        _step(ts, b)
    torch.cuda.synchronize()
    a = [e.clone() for e in ts.phema_emas]
    a_snap = ts.phema_snapshot()
    del ts
    gc.collect()
    ts = _trainstep(phema_sigma_rels=SIGMAS)
    for b in data[:2]:
        _step(ts, b)
    buf = io.BytesIO()
    torch.save({"model": ts.net.state_dict(), "ema": ts.ema.state_dict(), "opt": ts.state_dict()}, buf)
    del ts
    gc.collect()
    torch.cuda.empty_cache()
    buf.seek(0)
    ck = torch.load(buf, weights_only=False)
    assert ck["opt"]["phema"]["steps"] == 2 and ck["opt"]["phema"]["origin"] == 0
    from maskdit_b200.train_step import TrainStep
    net = _net()
    net.load_state_dict(ck["model"])
    ema = copy.deepcopy(net).eval()
    ema.load_state_dict(ck["ema"])
    ts2 = TrainStep(net, ema, lr=1e-3, weight_decay=0.01, global_batch=B, phema_sigma_rels=SIGMAS)
    ts2.load_state_dict(ck["opt"])
    for b in data[2:]:
        _step(ts2, b)
    torch.cuda.synchronize()
    for x, y in zip(a, ts2.phema_emas):
        assert torch.equal(x, y)
    b_snap = ts2.phema_snapshot()
    assert (b_snap["step"], b_snap["origin"]) == (a_snap["step"], a_snap["origin"]) == (5, 0)
    for pa, pb in zip(a_snap["profiles"], b_snap["profiles"]):
        assert pa["gamma"] == pb["gamma"] and list(pa["ema"]) == list(net.state_dict())
        for k in pa["ema"]:
            assert torch.equal(pa["ema"][k], pb["ema"][k]), k
    # frozen tensors are the model's, trainable ones the profile's
    assert torch.equal(b_snap["profiles"][0]["ema"]["model.pos_embed"], net.model.pos_embed.detach().cpu())
    # a checkpoint without profiles (a reference one): new profiles counted from the resume step
    opt = dict(ck["opt"])
    del opt["phema"]
    net3 = _net()
    ts3 = TrainStep(net3, copy.deepcopy(net3).eval(), lr=1e-3, global_batch=B, phema_sigma_rels=SIGMAS)
    ts3.load_state_dict(opt)
    ts3.lr_step_offset = 7 - ts3.step_count       # as train.py sets it for a checkpoint of run step 7
    _step(ts3, data[0])
    assert ts3.phema_origin == 7 and ts3.phema_steps == 1
    assert all(torch.equal(e, ts3.st.w32[:ts3.st.n_train]) for e in ts3.phema_emas)


# ---- 5. world > 1 ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def comm(ops):
    """A one-rank communicator."""
    L = ops.lib()
    uid = ctypes.create_string_buffer(128)
    assert L.mdt_nccl_unique_id(uid) == 0
    c = ctypes.c_void_p()
    assert L.mdt_nccl_comm_create(bytes(uid.raw), 0, 1, 0, ctypes.byref(c)) == 0 and c.value
    yield c
    assert L.mdt_nccl_comm_destroy(c) == 0


class TwoIdenticalRanks:
    """Stand-in for `GradComm` on rank 0 of two ranks that hold the same gradient: the real one-rank
    `mdt_allreduce_grads`, then the buffer doubled (the exact sum of the two ranks)."""

    def __init__(self, comm):
        self.comm = comm

    def all_reduce(self, t):
        from maskdit_b200 import ops
        assert ops.lib().mdt_allreduce_grads(self.comm, t.data_ptr(), t.numel(), int(t.dtype == bf16),
                                             ops.stream_ptr()) == 0
        t.mul_(2)

    def close(self):
        pass


WORLD2 = {
    "bf16-chunked": dict(grad_dtype="bf16", ar_chunks=4),
    "bf16-flat": dict(grad_dtype="bf16", ar_chunks=1),
    "fp32-chunked": dict(grad_dtype="fp32", ar_chunks=4),
    "bf16-chunked-skip": dict(grad_dtype="bf16", ar_chunks=4, skip_nonfinite=True),
}


@pytest.mark.parametrize("mode", list(WORLD2))
def test_world2_every_element_once_after_its_pass(ops, comm, monkeypatch, mode):
    from maskdit_b200.train_step import ar_chunk_bounds
    for k in ("MDT_GRAD_AR", "MDT_COLLECTIVE", "MDT_AR_CHUNKS", "MDT_TRAIN_GRAPH"):
        monkeypatch.delenv(k, raising=False)
    kw = dict(WORLD2[mode])
    chunks = kw.pop("ar_chunks")
    ts = _trainstep(phema_sigma_rels=SIGMAS, **kw)
    ts.world = 2
    ts.comm = TwoIdenticalRanks(comm)
    if ts.grad_dtype == "bf16":
        ts.g16 = torch.empty(ts.st.n_train, dtype=bf16, device="cuda")
    ts.ar_chunks = chunks
    n = ts.st.n_train
    log = []

    def recorder(name, fn):
        def call(*a, **k):
            lo = (a[0].data_ptr() - ts.st.w32.data_ptr()) // 4
            log.append((name, lo, lo + a[0].numel(), torch.cuda.current_stream().cuda_stream))
            return fn(*a, **k)
        return call

    for name in ("adamw_ema", "adamw_ema_guarded", "power_ema"):
        monkeypatch.setattr(ops, name, recorder(name, getattr(ops, name)))
    ws = []
    for step, b in enumerate(_batches(3)):
        log.clear()
        _step(ts, b)
        ws.append(ts.st.w32[:n].clone())
        what = f"{mode} step {step}"
        pe = [(lo, hi, s) for name, lo, hi, s in log if name == "power_ema"]
        spans = sorted((lo, hi) for lo, hi, _ in pe)
        assert spans[0][0] == 0 and spans[-1][1] == n and all(a[1] == b_[0] for a, b_ in zip(spans, spans[1:])), what
        assert spans == ar_chunk_bounds(n, chunks), what
        # each update directly follows the optimizer pass over the same range, on its stream
        for i, (name, lo, hi, s) in enumerate(log):
            if name == "power_ema":
                assert i > 0 and log[i - 1][0].startswith("adamw") and log[i - 1][1:] == (lo, hi, s), (what, i)
    torch.cuda.synchronize()
    ts.close()
    want = _replay(ws, ts.phema_gammas)
    for j, (e, w) in enumerate(zip(ts.phema_emas, want)):
        _assert_close(e, w, ws, (mode, j))


# ---- 6. train.py -> posthoc_ema.py -> generate.py --------------------------------------------------------------------------
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
        max_num_steps: 6}
log: {log_every: 2, ckpt_every: 4, tag: t}
"""


def _run(cmd, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, *cmd], cwd=cwd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def test_train_posthoc_generate(tmp_path):
    cfg = tmp_path / "cfg.yaml"
    cfg.write_text(YAML)
    res = tmp_path / "res"
    out = _run([os.path.join(ROOT, "train.py"), "--config", str(cfg), "--synthetic", "--max_steps", "6",
                "--phema_sigma_rel", "0.05,0.10", "--phema_every", "2", "--results_dir", str(res)], str(tmp_path))
    snaps = sorted(os.listdir(res / "phema"))
    assert snaps == ["phema-0000002.pt", "phema-0000004.pt", "phema-0000006.pt"], snaps
    for s in snaps:
        assert str(res / "phema" / s) in out, out
    s4 = torch.load(res / "phema" / "phema-0000004.pt", weights_only=True)
    assert s4["step"] == 4 and s4["origin"] == 0 and [p["sigma_rel"] for p in s4["profiles"]] == [0.05, 0.10]
    ck = torch.load(res / "checkpoints" / "0000004.pt", map_location="cpu", weights_only=False)
    ph = ck["opt"]["phema"]
    assert ph["steps"] == 4 and ph["origin"] == 0
    assert set(s4["profiles"][0]["ema"]) == set(ck["ema"])
    post = tmp_path / "ema-0.08.pt"
    out = _run([os.path.join(ROOT, "posthoc_ema.py"), "--snapshots", str(res / "phema"), "--sigma_rel", "0.08",
                "--out", str(post)], str(tmp_path))
    assert "relative L2 residual" in out
    p = torch.load(post, weights_only=True)
    assert p["posthoc"]["step"] == 6 and len(p["posthoc"]["coefficients"]) == 6
    assert set(p["ema"]) == set(ck["ema"]) and all(torch.isfinite(v).all() for v in p["ema"].values())
    _run([os.path.join(ROOT, "generate.py"), "--config", str(cfg), "--ckpt_path", str(post), "--seeds", "0-1",
          "--num_steps", "4", "--results_dir", str(tmp_path / "samples")], str(tmp_path))
    z = np.load(tmp_path / "samples" / "000001.npy")
    assert z.shape == (4, 16, 16) and np.isfinite(z).all()
