"""torchrun --nproc-per-node N tools/shard_equivalence.py — the sharded optimizer on real GPUs: N ranks with
`TrainStep(shard_optimizer=True)` and N ranks replicated, both with the library's NCCL communicator and the bf16
exchange, give bitwise-equal weights, shadow and EMA after 3 steps under the deterministic mode; a checkpoint written
by the sharded run loads into a replicated run, which then steps on bit for bit with the replicated run.
Prints SHARD_EQUIV_OK on rank 0."""
import copy
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from maskdit_b200.maskdit import Precond_models  # noqa: E402
from maskdit_b200.train_step import TrainStep  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    torch.use_deterministic_algorithms(True)
    R, ncls, B = 32, 1000, 4
    torch.manual_seed(1)
    base = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=ncls, model_type="DiT-S/2",
                                 use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False)
    with torch.no_grad():
        gz = torch.Generator().manual_seed(2)
        for p in base.parameters():
            if p.requires_grad and float(p.abs().sum()) == 0.0:
                p.copy_(torch.randn(p.shape, generator=gz) * 0.02)
    data = []
    for i in range(4):   # a different batch on every rank
        g = torch.Generator().manual_seed(100 * rank + i)
        mom = torch.cat([torch.randn(B, 4, R, R, generator=g), torch.randn(B, 4, R, R, generator=g) - 2], 1).to(dev)
        lab = torch.nn.functional.one_hot(torch.randint(0, ncls, (B,), generator=g), ncls).float().to(dev)
        data.append((mom, lab, 1000 * rank + i))

    def make(shard, net=None, ema=None):
        net = net or copy.deepcopy(base).to(dev).train()
        ema = ema or copy.deepcopy(net).eval()
        return TrainStep(net, ema, lr=1e-3, ema_decay=0.99, phema_sigma_rels=(0.05, 0.10), collective="mdt",
                         grad_dtype="bf16", shard_optimizer=shard)

    def step(ts, b):
        torch.manual_seed(b[2])
        ts.step(b[0], b[1], 0.5, 0.1, moments=True, class_dropout_prob=0.1)

    rep, sh = make(False), make(True)
    assert sh.sharded and sh.m.numel() < rep.m.numel()
    for b in data[:3]:
        step(rep, b)
        step(sh, b)
    sh.materialize()
    torch.cuda.synchronize()
    same = [torch.equal(a, b) for a, b in ((sh.st.w32, rep.st.w32), (sh.st.w16, rep.st.w16),
                                           (sh.ema_st.w32, rep.ema_st.w32))]
    opt = sh.state_dict()
    snap_sh, snap_rep = sh.phema_snapshot(), rep.phema_snapshot()
    same.append(all(torch.equal(x["ema"][k], y["ema"][k].cpu()) for x, y in zip(snap_sh["profiles"],
                                                                                   snap_rep["profiles"])
                    for k in x["ema"]))
    # the sharded run's checkpoint into a replicated run, one more step on both replicated runs
    net = copy.deepcopy(base).to(dev).train()
    net.load_state_dict(sh.net.state_dict())
    ema = copy.deepcopy(net).eval()
    ema.load_state_dict(sh.ema.state_dict())
    resumed = make(False, net, ema)
    resumed.load_state_dict(opt)
    step(rep, data[3])
    step(resumed, data[3])
    torch.cuda.synchronize()
    same += [torch.equal(resumed.st.w32, rep.st.w32), torch.equal(resumed.m, rep.m),
             torch.equal(resumed.phema_emas[0], rep.phema_emas[0])]
    ok = torch.tensor([float(all(same))], device=dev)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(f"sharded vs replicated on {world} GPUs: {same}  [{sh.describe_collective()}]", flush=True)
    for t in (rep, sh, resumed):
        t.close()
    dist.barrier()
    if rank == 0 and ok.item() == 1.0:
        print("SHARD_EQUIV_OK", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
