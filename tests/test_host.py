"""CPU tests of the host-side logic: ABI surface, module/state-dict contract, flat layout, DP helpers (gloo)."""
import ctypes
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_library_exports_every_declared_symbol():
    """The C-ABI library loads without a GPU and exports every function include/maskdit_b200.h declares."""
    from maskdit_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "maskdit_b200.h")).read()
    declared = set(re.findall(r"\b(mdt_[a-z0-9_]+)\s*\(", hdr))
    declared.discard("mdt_gemm_args")
    L = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(L, name), name
    assert declared == set(_lib.exported_symbols()), declared ^ set(_lib.exported_symbols())
    assert _lib.lib().mdt_abi_version() == 2
    assert _lib.lib().mdt_status_string(-1).decode().startswith("invalid argument")


def test_product_path_refuses_cpu_tensors():
    from maskdit_b200 import ops
    from maskdit_b200._lib import MdtError
    from maskdit_b200.maskdit import Precond_models
    with pytest.raises(MdtError):
        ops.mask_indices(torch.rand(2, 16), 8)
    net = Precond_models["edm"](8, 4, num_classes=10, model_type="DiT-S/2", use_decoder=True, mae_loss_coef=0.1)
    with pytest.raises(MdtError):
        net(torch.randn(2, 4, 8, 8), torch.ones(2), None)


def test_product_never_imports_oracle():
    for root, _, files in os.walk(os.path.join(ROOT, "maskdit_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(root, f)).read()
                assert "oracle" not in src.replace("# oracle", ""), f


@pytest.mark.parametrize("mt,R,ncls", [("DiT-S/2", 8, 10), ("DiT-XL/2", 32, 1000)])
def test_state_dict_contract_matches_reference_keys(mt, R, ncls):
    """Key names and shapes of EDMPrecond.state_dict() == the reference's (oracle.param_shapes is pinned to the
    reference module by make_golden.py's strict load)."""
    from maskdit_b200.maskdit import DiT_models, Precond_models
    from oracle import maskdit_oracle as O
    if mt == "DiT-XL/2":
        with torch.device("meta"):
            net = Precond_models["edm"](R, 4, num_classes=ncls, model_type=mt, use_decoder=True, mae_loss_coef=0.1)
    else:
        net = Precond_models["edm"](R, 4, num_classes=ncls, model_type=mt, use_decoder=True, mae_loss_coef=0.1)
    want = O.param_shapes(O.Cfg(model_type=mt, img_resolution=R, num_classes=ncls))
    got = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert got == {k: tuple(v) for k, v in want.items()}
    if mt == "DiT-XL/2":
        assert len(got) == 378 and sum(int(torch.tensor(s).prod()) for s in got.values()) == 730_541_200
    frozen = [k for k, p in net.named_parameters() if not p.requires_grad]
    assert sorted(frozen) == ["model.decoder_pos_embed", "model.pos_embed"]
    assert len(DiT_models) == 15 and net.model.patch_size == 2 and net.model.extras == 0


def test_init_matches_reference_scheme():
    from maskdit_b200.maskdit import Precond_models, sincos_2d
    from oracle import maskdit_oracle as O
    net = Precond_models["edm"](8, 4, num_classes=10, model_type="DiT-S/2", use_decoder=True, mae_loss_coef=0.1)
    sd = net.state_dict()
    zero = [k for k, v in sd.items() if v.abs().sum() == 0]
    for k in sd:
        should = k.endswith(".bias") or "adaLN_modulation" in k or k.startswith(("model.final_layer.linear",
                                                                               "model.decoder_layer.linear"))
        assert (k in zero) == should, k
    assert torch.allclose(sd["model.pos_embed"][0], O.sincos_pos_embed(384, 4))
    assert torch.allclose(sincos_2d(512, 16), O.sincos_pos_embed(512, 16))
    w = sd["model.blocks.0.attn.qkv.weight"]
    bound = (6 / (w.shape[0] + w.shape[1])) ** 0.5
    assert w.abs().max() <= bound + 1e-6 and w.abs().max() > 0.9 * bound
    assert abs(sd["model.y_embedder.embedding_table.weight"].std().item() - 0.02) < 2e-3


def test_flat_layout_plan():
    from maskdit_b200.flat import ALIGN, FlatStore
    from oracle import maskdit_oracle as O
    cfg = O.Cfg(model_type="DiT-XL/2", img_resolution=32, num_classes=1000)
    shapes = O.param_shapes(cfg)
    st = FlatStore()
    st.plan(shapes)
    o, rows, hid = st.ada_w_range
    assert o == 0 and hid == 1152 and rows == 28 * 6912 + 2304 + 8 * 3072 + 1024
    spans = sorted((v[0], v[0] + v[1]) for v in st.offsets.values())
    for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
        assert a1 <= b0 and b0 % ALIGN == 0
    assert st.offsets["model.pos_embed"][0] >= st.n_train  # frozen tensors sit after the trainable region
    n_train = sum(v[1] for k, v in st.offsets.items() if not k.endswith("pos_embed"))
    assert n_train == 730_115_216  # SURVEY §2.2: trainable parameter count
    # per-block gradient ranges (overlapped all-reduce/optimizer): contiguous, disjoint, inside the trainable region
    ranges = [st.prefix_range(f"model.blocks.{i}.") for i in range(28)] + \
             [st.prefix_range(f"model.decoder_blocks.{i}.") for i in range(8)]
    for (a0, a1), (b0, b1) in zip(sorted(ranges), sorted(ranges)[1:]):
        assert a0 < a1 <= b0 < b1 <= st.n_train
    lo, hi = ranges[0]
    assert hi - lo == 3 * 1152 * 1152 + 3456 + 1152 * 1152 + 1152 + 2 * 4608 * 1152 + 4608 + 1152


def test_dp_helpers_and_schedule():
    from maskdit_b200.train_step import lr_at, shard_batch
    assert [shard_batch(1024, 8, r) for r in (0, 7)] == [(0, 128), (896, 1024)]
    with pytest.raises(ValueError):
        shard_batch(10, 4, 0)
    assert lr_at(0, 1e-4, 1024, 10) == 0.0 and lr_at(5, 1e-4, 1024, 10) == pytest.approx(5.12e-5)
    assert lr_at(100, 1e-4, 1024, 10) == 1e-4
    from maskdit_b200.train_step import ar_chunk_bounds
    for n, k in [(730115216, 8), (5000, 8), (1 << 20, 3), (7, 1)]:
        b = ar_chunk_bounds(n, k)
        assert b[0][0] == 0 and b[-1][1] == n and all(x[1] == y[0] for x, y in zip(b, b[1:]))
        assert all(lo % 1024 == 0 for lo, _ in b) and len(b) <= max(k, 1)


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from maskdit_b200.train_step import shard_batch
    # the step's single collective: SUM all-reduce of one flat buffer, 1/world folded in afterwards
    torch.manual_seed(0)
    full = torch.randn(8, 1000)                       # per-sample "gradients" of a global batch of 8
    lo, hi = shard_batch(8, world, rank)
    flat = full[lo:hi].sum(0)
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    ok = torch.allclose(flat / world, full.sum(0) / world, atol=1e-5)
    # chunked, asynchronous form used by TrainStep when world > 1 (optimizer pass of chunk k overlaps chunk k+1)
    from maskdit_b200.train_step import ar_chunk_bounds
    big = torch.randn(3, 10000)[rank % 3].clone()
    ref = big.clone()
    dist.all_reduce(ref, op=dist.ReduceOp.SUM)
    works = [(lo, hi, dist.all_reduce(big[lo:hi], op=dist.ReduceOp.SUM, async_op=True))
             for lo, hi in ar_chunk_bounds(big.numel(), 4)]
    for lo, hi, w in works:
        w.wait()
    q.put((rank, ok and len(works) == 4 and torch.equal(big, ref)))
    dist.barrier()
    dist.destroy_process_group()


def test_gloo_world2_flat_allreduce_equals_single_process():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 1000
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(60)
    assert all(ok for _, ok in res) and sorted(r for r, _ in res) == [0, 1]


YAML = """
data: {dataset: imagenet256-latent, category: lmdb, resolution: 32, num_channels: 4, root: ../data, feat_path: None}
model:
  precond: edm
  model_type: DiT-XL/2
  in_size: 32
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
train: {tf32: False, amp: True, batchsize: 128, grad_accum: 1, epochs: 2800, lr: 0.0001, lr_rampup_kimg: 0,
        xflip: False, max_num_steps: 2000000}
log: {log_every: 500, ckpt_every: 50_000, tag: pretrain}
"""


def test_config_schema_and_mask_schedule():
    """The reference YAML schema (configs/train/imagenet256-latent.yaml) parses with PyYAML; schedules follow
    get_mask_ratio_fn (train_utils/helper.py:9-27) incl. the `cos4` alias of the finetune config."""
    import math
    from maskdit_b200.config import load_config, mask_ratio_schedule, parse_float_none, parse_int_list
    cfg = load_config(YAML)
    assert cfg.model.model_type == "DiT-XL/2" and cfg.train.batchsize == 128 and cfg.data.feat_path is None
    assert cfg.log.ckpt_every == 50000 and cfg.model.get("self_cond") is None
    assert mask_ratio_schedule("constant", 0.5)(0.3) == 0.5
    for name in ("cosine4", "cos4"):
        f = mask_ratio_schedule(name, 0.5, 0.1)
        assert f(0.25) == pytest.approx(0.4 * math.cos(math.pi * 0.125) ** 4 + 0.1)
    assert mask_ratio_schedule("linear", 0.5, 0.1)(0.5) == pytest.approx(0.3)
    assert mask_ratio_schedule("exp", 0.5, 0.0)(1.0) == pytest.approx(0.5 * math.exp(-7))
    with pytest.raises(ValueError):
        mask_ratio_schedule("bogus")
    assert parse_int_list("1,2,5-8") == [1, 2, 5, 6, 7, 8] and parse_float_none("None") is None


@pytest.mark.parametrize("mt,R,ncls", [("DiT-S/2", 8, 10), ("DiT-B/4", 16, 7), ("DiT-XL/2", 32, 1000), ("DiT-XL/2", 64, 1000)])
def test_c_driver_layout_equals_flat_store(mt, R, ncls):
    """The packed parameter blob `mdt_model_param_info` enumerates (csrc/driver.cu) is exactly the layout FlatStore
    builds for the nn.Module — names = the reference's state-dict keys — and the workspace planner is monotone."""
    import ctypes
    from maskdit_b200 import _lib
    from maskdit_b200.flat import FlatStore
    from oracle import maskdit_oracle as O
    from maskdit_b200.maskdit import Precond_models
    cfg = O.Cfg(model_type=mt, img_resolution=R, num_classes=ncls)
    with torch.device("meta"):   # registration order of the module (= the reference's, see make_golden.py's strict load)
        net = Precond_models["edm"](R, 4, num_classes=ncls, model_type=mt, use_decoder=True, mae_loss_coef=0.1)
    shapes = {k: tuple(p.shape) for k, p in net.named_parameters()}
    assert shapes == {k: tuple(v) for k, v in O.param_shapes(cfg).items()}
    st = FlatStore()
    st.plan(shapes)
    L = _lib.lib()
    mc = _lib.ModelCfg(R, 4, cfg.patch, ncls, cfg.hidden, cfg.depth, cfg.heads, 4 * cfg.hidden, 512, 8, 16, 2048, 1, 0.5)
    h = ctypes.c_void_p()
    assert L.mdt_model_create(ctypes.byref(mc), ctypes.byref(h)) == 0
    n = L.mdt_model_num_tensors(h)
    assert n == len(shapes)
    name, off, num = ctypes.create_string_buffer(160), ctypes.c_longlong(), ctypes.c_longlong()
    prev = -1
    for i in range(n):
        assert L.mdt_model_param_info(h, i, name, 160, ctypes.byref(off), ctypes.byref(num)) == 0
        k = name.value.decode()
        assert st.offsets[k][:2] == (off.value, num.value), k
        assert off.value > prev and off.value % 64 == 0
        prev = off.value
    assert L.mdt_model_param_info(h, n, name, 160, None, None) != 0
    assert (L.mdt_model_param_count(h, 1), L.mdt_model_param_count(h, 0)) == (st.n_train, st.n_total)
    if mt == "DiT-XL/2":
        assert L.mdt_model_param_count(h, 1) >= 730_115_216
    T = cfg.num_patches // 2
    tr, ev = L.mdt_workspace_bytes(h, 8, T, 1), L.mdt_workspace_bytes(h, 8, 0, 0)
    assert tr > ev > 0 and L.mdt_workspace_bytes(h, 16, T, 1) > tr and L.mdt_workspace_bytes(h, 0, T, 1) < 0
    bad = _lib.ModelCfg(R, 4, cfg.patch, ncls, cfg.hidden + 1, cfg.depth, cfg.heads, 4 * cfg.hidden, 512, 8, 16, 2048, 1, 0.5)
    h2 = ctypes.c_void_p()
    assert L.mdt_model_create(ctypes.byref(bad), ctypes.byref(h2)) != 0     # hidden not divisible by heads
    L.mdt_model_destroy(h)


def test_gemm_dispatch_plan_for_the_xl2_step():
    """`mdt_gemm_plan` (no device needed): the host-side decisions of the GEMM launches of one XL/2 training step at
    B = 256 (M_e = 32768 kept-token rows, M_d = 65536 decoder rows, SURVEY 8) on an H100 (132 SMs) - tile width, grid,
    the paired half-tile order for N = 1152 / 3456 and the k-slice counts of the wgrad GEMMs."""
    from maskdit_b200 import _lib
    P = _lib.gemm_plan
    Me, Md, D, H4, Dd, H4d = 32768, 65536, 1152, 4608, 512, 2048
    # forward / dgrad: 128 x 256 tiles, one persistent CTA per SM
    for (M, N, K, kw) in ((Me, 3 * D, D, {}), (Me, D, D, {"epi": _lib.EPI_GATE_RESID}), (Me, H4, D, {"epi": _lib.EPI_GELU}),
                          (Me, D, H4, {"epi": _lib.EPI_GATE_RESID}), (Me, D, H4, {"b_mn": True}),
                          (Me, H4, D, {"b_mn": True, "epi": _lib.EPI_DGELU}), (Md, 3 * Dd, Dd, {}), (Md, Dd, H4d, {})):
        p = P(M, N, K, **kw)
        assert (p["block_n"], p["cg"], p["splits"], p["grid"]) == (256, 1, 1, 132), (M, N, K, p)
        narrow = N % 256 != 0 and N % 256 <= 128
        assert p["narrow_last"] == int(narrow) and p["pair_halves"] == int(narrow)
        mt, nt = M // 128, -(-N // 256)
        units = mt * nt if not narrow else (mt // 2) * (2 * (nt - 1) + 1)
        assert (p["num_m_tiles"], p["num_n_tiles"], p["num_kb"], p["units"]) == (mt, nt, K // 64, units)
    # wgrad (accumulating epilogue): LPT inside the k-slices, slice count from the wave-time model
    for (M, N, want) in ((D, H4, 4), (H4, D, 5), (3 * D, D, 9), (D, D, 11)):
        p = P(M, N, Me, a_mn=True, b_mn=True, epi=_lib.EPI_ATOMIC)
        assert (p["block_n"], p["cg"], p["pair_halves"], p["splits"]) == (256, 1, 0, want), (M, N, p)
        assert p["units"] == p["num_m_tiles"] * p["num_n_tiles"] * want and p["grid"] == min(132, p["units"])
    for (M, N, want) in ((Dd, H4d, 4), (H4d, Dd, 4), (3 * Dd, Dd, 11)):
        assert P(M, N, Md, a_mn=True, b_mn=True, epi=_lib.EPI_ATOMIC)["splits"] == want, (M, N)
    # skinny problems: narrow tiles, never more CTAs than units
    p = P(2, 1152, 256)
    assert (p["cg"], p["block_n"], p["grid"]) == (1, 256, 5)
    p = P(1024, 16, 512)
    assert (p["cg"], p["block_n"], p["units"], p["grid"]) == (1, 128, 8, 8)
    p = P(256, 160, 64)
    assert (p["cg"], p["block_n"]) == (1, 192)
    # argument errors surface as a status, not a crash
    with pytest.raises(_lib.MdtError):
        P(0, 16, 16)
    with pytest.raises(_lib.MdtError):
        P(128, 128, 100)      # lda = 100: TMA needs 16-byte row strides
