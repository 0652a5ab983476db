"""torchrun --nproc-per-node N tools/dp_equivalence.py — data-parallel equivalence on real GPUs (SURVEY 8e):
the gradient of a global batch split over N ranks and summed by the step's collective equals (x N) the gradient one
GPU computes on the whole batch, for every exchange mode of TrainStep (the chunked exchange pipelined with the
optimizer): our own NCCL communicator in fp32, torch.distributed, and the bf16 buffer (bf16 tolerance).
Prints DP_EQUIV_OK on rank 0."""
import copy
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from maskdit_b200 import ops  # noqa: E402
from maskdit_b200.loss import EDMLoss  # noqa: E402
from maskdit_b200.maskdit import Precond_models  # noqa: E402
from maskdit_b200.train_step import TrainStep, shard_batch  # noqa: E402


class Draws(EDMLoss):
    """Fixed random draws, sliced to this call's rows."""

    def __init__(self, rnd, noise, mnoise, lo, hi):
        super().__init__()
        self.t, self.k, self.m = (rnd[lo:hi].contiguous(), noise[lo:hi].contiguous()), 0, mnoise[lo:hi].contiguous()

    def _randn(self, shape, device):
        t = self.t[self.k % 2]
        self.k += 1
        return t

    def _rand(self, shape, device):
        return self.m


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    R, ncls, Bper = 32, 1000, 4
    Bg = Bper * world
    g = torch.Generator().manual_seed(0)
    images = (torch.randn(Bg, 4, R, R, generator=g) * 0.5).to(dev)
    labels = torch.nn.functional.one_hot(torch.randint(0, ncls, (Bg,), generator=g), ncls).float().to(dev)
    rnd, noise = torch.randn(Bg, 1, 1, 1, generator=g).to(dev), torch.randn(Bg, 4, R, R, generator=g).to(dev)
    mnoise = torch.rand(Bg, 256, generator=g).to(dev)
    torch.manual_seed(1)
    base = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=ncls, model_type="DiT-B/2",
                                 use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False)
    with torch.no_grad():
        gz = torch.Generator().manual_seed(2)
        for p in base.parameters():
            if p.requires_grad and float(p.abs().sum()) == 0.0:
                p.copy_(torch.randn(p.shape, generator=gz) * 0.02)
    lo, hi = shard_batch(Bg, world, rank)

    # single-GPU gradient of the whole global batch (every rank computes it locally: same weights, same draws)
    ref_net = copy.deepcopy(base).to(dev).train()
    ts_ref = TrainStep(ref_net, None, lr=1e-3, loss_fn=Draws(rnd, noise, mnoise, 0, Bg), process_group=None,
                       grad_dtype="fp32")
    ts_ref.world, ts_ref.comm, ts_ref.g16 = 1, None, None      # a 1-GPU step inside the N-rank job
    ts_ref._grad_scale = 1.0
    ts_ref.step(images, labels, 0.5, 0.1)
    g_ref = ts_ref.st.grad.clone()

    def run(**kw):
        net = copy.deepcopy(base).to(dev).train()
        ts = TrainStep(net, None, lr=1e-3, loss_fn=Draws(rnd, noise, mnoise, lo, hi), global_batch=Bg, **kw)
        n = ts.st.n_train
        w0 = ts.st.w32[:n].clone()
        ts.step(images[lo:hi].contiguous(), labels[lo:hi].contiguous(), 0.5, 0.1)
        torch.cuda.synchronize()
        gbuf = ts.g16 if ts.g16 is not None else ts.st.grad
        # the optimizer pass must be exactly one AdamW pass over the exchanged sum: replay it on the pre-step state
        m, v, w16 = torch.zeros_like(ts.m), torch.zeros_like(ts.v), torch.empty(n, dtype=torch.bfloat16, device=dev)
        ops.adamw_ema(w0, gbuf, m, v, None, w16, n, ts._lr_now, ts.step_count, ts.betas[0], ts.betas[1], ts.eps,
                      ts.wd, ts.ema_decay, 1.0 / world)
        torch.cuda.synchronize()
        replay = all(torch.equal(a, b) for a, b in ((ts.st.w32[:n], w0), (ts.m, m), (ts.v, v), (ts.st.w16[:n], w16)))
        return gbuf.float() / world, replay, ts

    def rel(a, b):
        return ((a.double() - b.double()).norm() / b.double().norm()).item()

    results = {}
    for name, kw, tol in (("mdt fp32 chunked", dict(collective="mdt", grad_dtype="fp32"), 5e-5),
                          ("torch fp32 chunked", dict(collective="torch", grad_dtype="fp32"), 5e-5),
                          ("mdt bf16 chunked", dict(collective="mdt", grad_dtype="bf16"), 6e-3)):
        gm, replay, ts = run(**kw)
        r = rel(gm, g_ref)
        results[name] = (r, replay)
        if rank == 0:
            print(f"{name:22s} gradient rel-L2 vs 1-GPU whole batch: {r:.3e}   optimizer pass == AdamW replay on the "
                  f"exchanged sum: {replay}   [{ts.describe_collective()}]", flush=True)
        assert r <= tol, (name, r)
        assert replay, name
        ts.close()
    dist.barrier()
    if rank == 0:
        print("DP_EQUIV_OK", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
