"""GPU: the held-out denoising loss on the CUDA path (maskdit_b200/validate.py).

1. Against the unmodified reference's golden (tests/golden/val_s2.npz) at the loss tolerance of the CUDA-path loss
   tests (5e-3 relative), for several batchings.
2. Under torch.use_deterministic_algorithms(True) the per-item losses are bit-identical for different batch sizes (one
   with a remainder batch) and for one process against two rank slices scored separately and combined.
3. In the default mode the same comparison holds bit for bit as well: only backward GEMMs accumulate with k-slices
   whose count follows the row count, and the eval forward has none of them (DESIGN §5; measured difference 0).
4. train.py --synthetic --val_every 2 prints the Val Loss line; its training losses and weights are bit-identical to a
   run without validation (deterministic mode); val_loss.py on the saved checkpoint gives train.py's numbers;
   val_loss.py --snapshots scores the post-hoc EMA widths of the run.
"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from maskdit_b200 import validate as V  # noqa: E402
from oracle import maskdit_oracle as O  # noqa: E402
from support import det  # noqa: E402,F401

GOLD = os.path.join(ROOT, "tests", "golden", "val_s2.npz")
LOSS_TOL = 5e-3


def _net(model_type, R, ncls, seed=1):
    from maskdit_b200.maskdit import Precond_models
    cfg = O.Cfg(model_type=model_type, img_resolution=R, num_classes=ncls)
    net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=ncls, model_type=model_type,
                                use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False)
    net.load_state_dict(O.make_state_dict(cfg, seed), strict=True)
    return net.cuda().eval()


# ---- 1. golden -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch", [1, 7, 40])
def test_cuda_path_matches_reference_golden(batch):
    g = np.load(GOLD)
    N, K = g["per_item"].shape
    held = V.HeldOut(torch.from_numpy(g["moments"]), torch.from_numpy(g["labels"]))
    res = V.validate(_net("DiT-S/2", 8, 10), held, levels=K, seed=int(g["seed"]), batch=batch)
    want = torch.from_numpy(g["per_item"])
    rel = ((res["per_item"] - want).abs() / want.abs()).max().item()
    assert rel <= LOSS_TOL, rel
    np.testing.assert_allclose(res["per_level"], g["per_item"].astype(np.float64).mean(0), rtol=LOSS_TOL)
    print(f"batch {batch}: worst per-item relative error against the reference {rel:.2e}")


def test_refuses_training_mode_and_cpu():
    net = _net("DiT-S/2", 8, 10)
    with pytest.raises(ValueError, match="eval"):
        V.CudaScorer(net.train())
    with pytest.raises(ValueError, match="CUDA"):
        V.CudaScorer(_net("DiT-S/2", 8, 10).cpu())


# ---- 2./3. batching and rank slices ----------------------------------------------------------------------------------
N_ITEMS, K_LEVELS = 13, 3


def _variants():
    """Per-item losses of DiT-S/2 at 32x32 (256 tokens, 1000 classes) for several batchings and a two-rank split."""
    net = _net("DiT-S/2", 32, 1000)
    held = V.HeldOut.synthetic(N_ITEMS, 32, 4, 1000, seed=5)
    scorer = V.CudaScorer(net)
    out = {}
    for batch in (N_ITEMS * K_LEVELS, 8, 16, 1):          # 39 rows: 8 and 16 leave a remainder of 7
        out[f"batch{batch}"] = V.score_items(scorer, held, 0, N_ITEMS, K_LEVELS, seed=2, batch=batch)
    parts = [V.score_items(scorer, held, *V.rank_slice(N_ITEMS, r, 2), K_LEVELS, seed=2, batch=8) for r in range(2)]
    out["ranks2"] = torch.cat(parts)
    return out


def test_deterministic_mode_is_bit_identical_across_batching_and_ranks(det):
    out = _variants()
    ref = out.pop(f"batch{N_ITEMS * K_LEVELS}")
    assert torch.isfinite(ref).all()
    for name, v in out.items():
        assert torch.equal(v, ref), (name, ((v - ref).abs() / ref.abs()).max().item())
    again = _variants()[f"batch{N_ITEMS * K_LEVELS}"]
    assert torch.equal(again, ref)


def test_default_mode_is_bit_identical_too():
    from maskdit_b200 import _lib
    assert not torch.are_deterministic_algorithms_enabled()
    _lib.sync_deterministic()
    out = _variants()
    ref = out.pop(f"batch{N_ITEMS * K_LEVELS}")
    worst = 0.0
    for name, v in out.items():
        rel = ((v - ref).abs() / ref.abs()).max().item()
        worst = max(worst, rel)
        assert torch.equal(v, ref), (name, rel)
    print(f"default mode: worst per-item relative difference across batchings / rank split {worst:.3e}")


# ---- 4. train.py / val_loss.py ---------------------------------------------------------------------------------------
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

# runs a script as __main__ under torch.use_deterministic_algorithms(True)
DET = ("import runpy, sys, torch; torch.use_deterministic_algorithms(True); sys.argv = sys.argv[1:]; "
       "runpy.run_path(sys.argv[0], run_name='__main__')")


def _run(args, cwd, deterministic=True):
    env = dict(os.environ, PYTHONPATH=ROOT)
    cmd = [sys.executable, "-c", DET, *args] if deterministic else [sys.executable, *args]
    r = subprocess.run(cmd, cwd=cwd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def _train(tmp_path, name, extra):
    res = tmp_path / name
    out = _run([os.path.join(ROOT, "train.py"), "--config", str(tmp_path / "cfg.yaml"), "--synthetic", "--max_steps",
                "4", "--results_dir", str(res), "--phema_sigma_rel", "0.05,0.10", "--phema_every", "2", *extra],
               str(tmp_path))
    return res, out


def test_train_and_val_loss_end_to_end(tmp_path):
    (tmp_path / "cfg.yaml").write_text(YAML)
    res_on, out_on = _train(tmp_path, "on", ["--val_every", "2", "--val_count", "6", "--val_levels", "4"])
    res_off, out_off = _train(tmp_path, "off", [])
    vals = re.findall(r"\(step=(\d+)\) Val Loss: ([-\d.]+) \[([-\d. ]+)\] \(6 items, EMA\)", out_on)
    assert [int(s) for s, _, _ in vals] == [2, 4], out_on
    assert all(len(lv.split()) == 4 for _, _, lv in vals)
    assert "Val Loss" not in out_off
    # validation changes nothing in training: the same loss lines and bit-identical weights, EMA and optimizer state
    train_lines = lambda out: [re.sub(r"Train Steps/Sec: [\d.]+", "", ln) for ln in out.splitlines()  # noqa: E731
                               if "Train Loss" in ln]
    assert train_lines(out_on) == train_lines(out_off) and len(train_lines(out_on)) == 2
    a = torch.load(res_on / "checkpoints" / "0000004.pt", map_location="cpu", weights_only=False)
    b = torch.load(res_off / "checkpoints" / "0000004.pt", map_location="cpu", weights_only=False)
    for key in ("model", "ema"):
        assert all(torch.equal(a[key][k], b[key][k]) for k in a[key]), key
    for i, st in a["opt"]["state"].items():
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(st[k], b["opt"]["state"][i][k]), (i, k)
    # val_loss.py on the checkpoint gives the number train.py printed at that step (other batch size too)
    for batch in ("8", "5"):
        js = tmp_path / f"ckpt{batch}.json"
        out = _run([os.path.join(ROOT, "val_loss.py"), "--config", str(tmp_path / "cfg.yaml"), "--synthetic",
                    "--ckpt", str(res_on / "checkpoints" / "0000004.pt"), "--count", "6", "--levels", "4",
                    "--batch", batch, "--json", str(js)], str(tmp_path))
        row = json.loads(js.read_text())["rows"][0]
        assert f"{row['mean']:.5f}" == vals[1][1], (row, vals[1], out)
        assert " ".join(f"{v:.5f}" for v in row["per_level"]) == vals[1][2]
        assert "best: 0000004.pt" in out
    # post-hoc EMA widths of the run, rebuilt and scored
    js = tmp_path / "phema.json"
    out = _run([os.path.join(ROOT, "val_loss.py"), "--config", str(tmp_path / "cfg.yaml"), "--synthetic",
                "--snapshots", str(res_on / "phema"), "--sigma_rel", "0.05", "0.08", "0.10", "--count", "6",
                "--levels", "4", "--json", str(js)], str(tmp_path), deterministic=False)
    j = json.loads(js.read_text())
    assert [r["name"] for r in j["rows"]] == ["sigma_rel=0.05@4", "sigma_rel=0.08@4", "sigma_rel=0.1@4"], j
    assert j["best"] in [r["name"] for r in j["rows"]] and f"best: {j['best']}" in out
    assert all(np.isfinite(r["mean"]) for r in j["rows"]) and j["count"] == 6 and j["levels"] == 4
