"""Sharded optimizer state (`TrainStep(shard_optimizer=True)`) against the replicated step: MaskDiT-XL/2 at batch 256,
mask 0.5, two post-hoc EMA profiles (sigma_rel 0.05, 0.10), bf16 exchange in 4 chunks.

One GPU (default): the step runs as simulated rank 0 of 2, 4 and 8 ranks.  The collectives are the library's one-rank
NCCL calls, i.e. local copies, so the numbers are device work without the wire.  Replicated and sharded steps
alternate in one process; each round times `--steps` steps with CUDA events, and the median over `--rounds` rounds is
reported, with the optimizer pass alone (AdamW + EMA + profiles over this rank's elements) and the peak allocated
memory.  Under torchrun on N GPUs the real exchange runs and only the step time is reported.
The card's name and power limit are read in the same run."""
import argparse
import copy
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from maskdit_b200 import ops  # noqa: E402
from maskdit_b200.maskdit import Precond_models  # noqa: E402
from maskdit_b200.train_step import _GATHER_DTYPES, TrainStep  # noqa: E402


class LocalRanks:
    """Rank 0 of `world` ranks on a one-rank communicator: every collective is the real one-rank call only."""

    def __init__(self, world):
        L = ops.lib()
        uid = ctypes.create_string_buffer(128)
        ops.check(L.mdt_nccl_unique_id(uid), "mdt_nccl_unique_id", 0)
        self._c = ctypes.c_void_p()
        ops.check(L.mdt_nccl_comm_create(bytes(uid.raw), 0, 1, 0, ctypes.byref(self._c)), "mdt_nccl_comm_create", 0)
        self.rank, self.world = 0, world

    def all_reduce(self, t):
        ops.check(ops.lib().mdt_allreduce_grads(self._c, t.data_ptr(), t.numel(), int(t.dtype == torch.bfloat16),
                                                ops.stream_ptr()), "mdt_allreduce_grads", 0)

    def reduce_scatter(self, t, count):
        ops.check(ops.lib().mdt_reduce_scatter_grads(self._c, t.data_ptr(), count, int(t.dtype == torch.bfloat16),
                                                     ops.stream_ptr()), "mdt_reduce_scatter_grads", 0)

    def all_gather(self, t, count):
        ops.check(ops.lib().mdt_allgather(self._c, t.data_ptr(), count, _GATHER_DTYPES[t.dtype], ops.stream_ptr()),
                  "mdt_allgather", 0)

    def close(self):
        ops.lib().mdt_nccl_comm_destroy(self._c)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"unknown ({e})"
    return q


def build(shard, world, pg=None):
    torch.manual_seed(0)
    with torch.device("cuda"):
        net = Precond_models["edm"](img_resolution=32, img_channels=4, num_classes=1000, model_type="DiT-XL/2",
                                    use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False).train()
    kw = dict(lr=1e-4, phema_sigma_rels=(0.05, 0.10))
    if pg is not None:
        return TrainStep(net, copy.deepcopy(net).eval(), collective="mdt", shard_optimizer=shard, **kw)
    ts = TrainStep(net, copy.deepcopy(net).eval(), **kw)
    ts.world, ts.rank, ts.comm, ts.shard_optimizer = world, 0, LocalRanks(world), shard
    if shard:
        ts._shard_setup()
    else:
        ts.g16 = torch.empty(ts.st.n_train, dtype=torch.bfloat16, device="cuda")
    return ts


def data(B):
    g = torch.Generator().manual_seed(5)
    mom = torch.cat([torch.randn(B, 4, 32, 32, generator=g), torch.randn(B, 4, 32, 32, generator=g) - 2], 1).cuda()
    lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float().cuda()
    return mom, lab


def timed(fn, k):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(k):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k


def optimizer_pass(ts):
    if ts.sharded:
        for k in range(len(ts._sh.bounds)):
            ts._step_piece(k)
    else:
        ts._step_range(0, ts.st.n_train)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="2,4,8")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    world_env = int(os.environ.get("WORLD_SIZE", 1))
    pg = None
    if world_env > 1:
        import torch.distributed as dist
        local = int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        pg = dist.group.WORLD
    B = args.batch // world_env if pg is not None else args.batch
    mom, lab = data(B)
    out = {"card": card(), "model": "MaskDiT-XL/2", "batch_per_gpu": B, "mask_ratio": 0.5, "profiles": 2}
    worlds = [world_env] if pg is not None else [int(w) for w in args.worlds.split(",")]
    for W in worlds:
        res = {}
        for shard in (False, True):   # built one at a time: both at once do not fit
            ts = build(shard, W, pg)

            def step():
                ts.step(mom, lab, 0.5, 0.1, moments=True, class_dropout_prob=0.1)
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            steps = [timed(step, args.steps) for _ in range(args.rounds)]
            opt = [timed(lambda: optimizer_pass(ts), args.steps) for _ in range(args.rounds)]
            res["sharded" if shard else "replicated"] = {
                "step_ms": round(statistics.median(steps), 2), "step_ms_rounds": [round(s, 2) for s in steps],
                "optimizer_pass_ms": round(statistics.median(opt), 2),
                "peak_alloc_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2),
                "recompute_blocks": ts.recompute_blocks}
            ts.close()
            del ts, step
            torch.cuda.empty_cache()
        out[f"world_{W}" + ("" if pg is not None else "_simulated")] = res
    if pg is None or int(os.environ.get("RANK", 0)) == 0:
        print(json.dumps(out), flush=True)
    if pg is not None:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
