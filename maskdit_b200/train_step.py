"""Data-parallel training step on the H100 engine (reference: train.py:200-230 inner step, :178 DDP, :141 optimizer,
train_utils/helper.py:47-58 EMA).

One process per GPU.  A step is:
    zero flat grad  ->  fused EDM loss forward/backward (C++ step driver)  ->  sum-all-reduce of the flat gradient
    buffer over NVLink (`GradComm`: our own NCCL communicator behind the C ABI; the 1/world factor is folded into the
    optimizer kernel)  ->  fused AdamW + EMA + bf16-shadow kernel over the flat buffers.
`overlap=False`: literally one all-reduce after the backward and one optimizer launch.  `overlap=True`: a block's
gradient range is exchanged on a side stream as soon as its backward is enqueued (the role DDP's bucketed hooks play in
the reference), through a communicator confined to a few CTAs while the persistent GEMM grids leave those SMs free
(`mdt_set_sm_budget`), then one optimizer pass.  No other collective is issued in the step (SURVEY.md §8e); the loss is
returned as a device tensor (no per-step `.item()` host sync as at train.py:227).
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

from . import ops
from .loss import EDMLoss
from .maskdit import EDMPrecond


class DataParallelB200:
    """What the reference's loss expects from the DDP wrapper: `.module`, `.training`, callable (loss.py:41,47,52).
    Gradient synchronisation is NOT hooked into autograd; `TrainStep` all-reduces the flat gradient buffer once."""

    def __init__(self, module: EDMPrecond):
        self.module = module

    @property
    def training(self):
        return self.module.training

    def train(self, mode=True):
        self.module.train(mode)
        return self

    def eval(self):
        return self.train(False)

    def parameters(self):
        return self.module.parameters()

    def __call__(self, *a, **k):
        return self.module(*a, **k)


def shard_batch(global_batch: int, world_size: int, rank: int):
    """Even batch split by rank (train.py:72-75: global = per-GPU batch x world)."""
    if global_batch % world_size:
        raise ValueError(f"global batch {global_batch} not divisible by world size {world_size}")
    per = global_batch // world_size
    return rank * per, (rank + 1) * per


def lr_at(step: int, base_lr: float, global_batch: int, rampup_kimg: float):
    """train.py:223, evaluated BEFORE `train_steps` is incremented (train.py:232): the very first update of a run
    uses lr = 0 (also with lr_rampup_kimg = 0: min(0 / 1e-8, 1) = 0), every later one base_lr * min(ramp, 1)."""
    return base_lr * min(step * global_batch / max(rampup_kimg * 1000, 1e-8), 1)


def ar_chunk_bounds(n, k):
    """[lo, hi) element ranges of the k all-reduce chunks of a flat buffer of n elements (4 KiB aligned starts)."""
    if k <= 1 or n < k * 1024:
        return [(0, n)]
    step = -(-(-(-n // k)) // 1024) * 1024
    return [(lo, min(n, lo + step)) for lo in range(0, n, step)]


class GradComm:
    """The step's gradient exchange behind the C ABI (`mdt_nccl_*`, `mdt_allreduce_grads`, csrc/driver.cu): an NCCL
    communicator of our own, created from a unique id that rank 0 draws and `torch.distributed` merely ships to the
    other ranks (any backend; it is the bootstrap side channel, nothing else).  `max_ctas` > 0 confines the
    communicator's kernels to that many CTAs so that they run NEXT TO the backward instead of after it."""

    def __init__(self, pg=None, max_ctas=0):
        import ctypes
        self.rank, self.world = dist.get_rank(pg), dist.get_world_size(pg)
        L = ops.lib()
        buf = ctypes.create_string_buffer(128)
        if self.rank == 0:
            ops.check(L.mdt_nccl_unique_id(buf), "mdt_nccl_unique_id", 0)
        box = [bytes(buf.raw)]
        dist.broadcast_object_list(box, src=dist.get_global_rank(pg, 0) if pg is not None else 0, group=pg)
        self._comm = ctypes.c_void_p()
        ops.check(L.mdt_nccl_comm_create(box[0], self.rank, self.world, int(max_ctas), ctypes.byref(self._comm)),
                  "mdt_nccl_comm_create", 0)
        self.max_ctas = max_ctas

    def all_reduce(self, t):
        """In-place SUM over the ranks of a contiguous fp32 / bf16 device tensor, on the current stream."""
        assert t.is_cuda and t.is_contiguous() and t.dtype in (torch.float32, torch.bfloat16)
        ops.check(ops.lib().mdt_allreduce_grads(self._comm, t.data_ptr(), t.numel(), int(t.dtype == torch.bfloat16),
                                                ops.stream_ptr()), "mdt_allreduce_grads", 0)

    def close(self):
        if self._comm:
            ops.lib().mdt_nccl_comm_destroy(self._comm)
            self._comm = None


class TrainStep:
    def __init__(self, net: EDMPrecond, ema: EDMPrecond | None = None, lr=1e-4, betas=(0.9, 0.999), eps=1e-8,
                 weight_decay=0.0, ema_decay=0.9999, loss_fn: EDMLoss | None = None, process_group=None,
                 lr_rampup_kimg=0.0, global_batch=None, device=None, overlap=False, graph=None,
                 reference_lr_schedule=False, collective=None, grad_dtype=None, comm_ctas=None):
        """Multi-GPU options (world > 1; SURVEY 8e: the step's ONLY collective is the sum of the flat gradient buffer):
          collective  'mdt' (default with an NCCL process group): our own communicator behind the C ABI (`GradComm`);
                      'torch': `torch.distributed.all_reduce` on the process group (gloo tests, A/B).
          grad_dtype  'bf16' (default, SURVEY 8e): the fp32 gradient buffer is cast to a bf16 exchange buffer, 1.46 GB cross
                      the links instead of 2.92 GB and the optimizer kernel reads the bf16 sums; local
                      accumulation, moments and master weights stay fp32.  2-rank vs 1-GPU gradient rel-L2 2.3e-3.
                      'fp32': the 2.92 GB buffer is reduced as is (DDP's arithmetic; rel-L2 1e-5, order noise).
          overlap     the exchange of a block's gradients starts as soon as its backward is enqueued, on a side stream,
                      through a communicator confined to `comm_ctas` CTAs while the persistent GEMM / attention grids
                      are sized for (SMs - comm_ctas) (`mdt_set_sm_budget`).  Off by default, kept for A/B.
        Environment overrides: MDT_COLLECTIVE, MDT_GRAD_AR, MDT_OVERLAP, MDT_COMM_CTAS."""
        self.net, self.ema = net, ema
        self.lr, self.betas, self.eps, self.wd, self.ema_decay = lr, betas, eps, weight_decay, ema_decay
        self.loss_fn = loss_fn or EDMLoss()
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self.rampup, self.global_batch = lr_rampup_kimg, global_batch
        # lr: the reference recomputes it every step from the run's step counter (train.py:223); lr_step_offset lets a
        # resumed run continue that counter when it differs from the optimizer's own step count.
        self.reference_lr_schedule = reference_lr_schedule
        self.lr_step_offset = 0
        self._grad_scale = 1.0 / self.world
        self.step_count = 0
        dev = device or next(net.parameters()).device
        self.st = net.prepare(dev)
        self.st.ensure_grad()
        n = self.st.n_train
        self.m = torch.zeros(n, dtype=torch.float32, device=dev)
        self.v = torch.zeros(n, dtype=torch.float32, device=dev)
        self.ema_st = None
        if ema is not None:
            self.ema_st = ema.prepare(dev)
            assert self.ema_st.n_train == n and self.ema_st.offsets == self.st.offsets
        for k, p in net.named_parameters():  # .grad views into the flat buffer (optimizer-compatible)
            if p.requires_grad:
                p.grad = self.st.gview(k)
        # Overlap: gradient ranges are exchanged on a side stream as soon as a block's backward is enqueued.
        env = os.environ
        self.overlap = bool(int(env["MDT_OVERLAP"])) if "MDT_OVERLAP" in env else bool(overlap)
        self.collective = env.get("MDT_COLLECTIVE") or collective or \
            ("mdt" if self.world > 1 and dist.get_backend(process_group) == "nccl" else "torch")
        self.grad_dtype = env.get("MDT_GRAD_AR") or grad_dtype or "bf16"
        assert self.collective in ("mdt", "torch") and self.grad_dtype in ("fp32", "bf16")
        self.comm_ctas = int(env.get("MDT_COMM_CTAS", comm_ctas if comm_ctas is not None else 8))
        self.comm = None
        self.comm_bg = None
        self.g16 = None
        if self.world > 1:
            if self.collective == "mdt":
                self.comm = GradComm(process_group)               # full-width communicator (NVLS, all channels)
                # a second communicator confined to a few CTAs carries the per-block chunks DURING the backward; the
                # gradients that only become final at its very end (adaLN projections = 35 % of the volume, embeddings)
                # go through the full-width one afterwards
                self.comm_bg = GradComm(process_group, max_ctas=max(1, self.comm_ctas // 2)) if self.overlap else None
            if self.grad_dtype == "bf16":
                self.g16 = torch.empty(n, dtype=torch.bfloat16, device=dev)
        self._sms = torch.cuda.get_device_properties(dev).multi_processor_count
        self.graph = (os.environ.get("MDT_TRAIN_GRAPH", "0") == "1") if graph is None else bool(graph)
        self._graphs = {}
        # gradient all-reduce in this many chunks on a side stream, the fused AdamW/EMA pass of chunk k running while
        # chunk k+1 is on the wire.
        self.ar_chunks = int(os.environ.get("MDT_AR_CHUNKS", "4"))
        self.side = torch.cuda.Stream(device=dev, priority=-1) if self.overlap else None
        self._done = []          # [lo, hi) ranges already handled in the current step
        self._lr_now = lr
        net._grad_ready_hook = self._on_grads_ready if (self.overlap and self.world > 1) else None

    # -- optimizer state for checkpoints (reference: train.py:259-270 stores optimizer.state_dict() under 'opt') ------
    def state_dict(self):
        """AdamW state laid out like `torch.optim.AdamW(net.parameters()).state_dict()` / apex FusedAdam's
        (train.py:141,262): `state` is keyed by the parameter's POSITION in `net.parameters()` — frozen tensors
        (pos_embed = 0, decoder_pos_embed = 1) keep their index but own no state, so the first key is 2 — with
        `exp_avg` / `exp_avg_sq` and a per-parameter `step` (torch layout); the step count is also stored in the
        param_group (apex layout).  Tensors are copies on the current device."""
        state, n_all = {}, 0
        for i, (k, p) in enumerate(self.net.named_parameters()):
            n_all = i + 1
            if not p.requires_grad:
                continue
            lo, _, shape = self.st.offsets[k]
            n = p.numel()
            state[i] = {"step": torch.tensor(float(self.step_count)), "exp_avg": self.m[lo:lo + n].view(shape).clone(),
                        "exp_avg_sq": self.v[lo:lo + n].view(shape).clone()}
        return {"state": state,
                "param_groups": [{"lr": self.lr, "betas": self.betas, "eps": self.eps, "weight_decay": self.wd,
                                  "step": self.step_count, "params": list(range(n_all))}]}

    def load_state_dict(self, sd):
        """Accepts (a) this class's own layout, (b) `torch.optim.AdamW(model.parameters()).state_dict()`, (c) apex
        FusedAdam's (same indexing, `step` only in the param_group) and (d) round-1 checkpoints of this repo (compact
        indices over the trainable parameters + `param_names`)."""
        state = {int(k): v for k, v in sd["state"].items()}
        group = sd["param_groups"][0]
        named = list(self.net.named_parameters())
        trainable = [(i, k) for i, (k, p) in enumerate(named) if p.requires_grad]
        if "param_names" in sd:                                    # (d) legacy compact layout
            index_of = {k: j for j, k in enumerate(sd["param_names"])}
            lookup = [(index_of[k], k) for _, k in trainable if k in index_of]
        elif all(i in state for i, _ in trainable):                 # (a) (b) (c): position in net.parameters()
            lookup = trainable
        elif len(state) == len(trainable) and set(state) == set(range(len(trainable))):
            lookup = [(j, k) for j, (_, k) in enumerate(trainable)]  # optimizer built over the trainable params only
        else:
            raise ValueError(f"optimizer state holds {len(state)} entries (keys {sorted(state)[:3]}..), the model has "
                             f"{len(trainable)} trainable of {len(named)} parameters")
        if len(lookup) != len(trainable):
            raise ValueError(f"optimizer state covers {len(lookup)} of {len(trainable)} trainable parameters")
        step = group.get("step", None)
        for j, k in lookup:
            e = state[j]
            lo, _, shape = self.st.offsets[k]
            if tuple(e["exp_avg"].shape) != tuple(shape):
                raise ValueError(f"optimizer state of {k}: shape {tuple(e['exp_avg'].shape)} != {tuple(shape)}")
            n = e["exp_avg"].numel()
            self.m[lo:lo + n].copy_(e["exp_avg"].reshape(-1))
            self.v[lo:lo + n].copy_(e["exp_avg_sq"].reshape(-1))
            if "step" in e:
                step = e["step"]
        if step is None:
            raise ValueError("optimizer state carries no step count (neither per parameter nor in the param_group)")
        self.step_count = int(float(step))
        self.lr, self.betas, self.eps, self.wd = group["lr"], tuple(group["betas"]), group["eps"], \
            group["weight_decay"]

    def close(self):
        """Release the communicator (a TrainStep owns one when world > 1 and collective == 'mdt')."""
        for c in (self.comm, self.comm_bg):
            if c is not None:
                c.close()
        self.comm = self.comm_bg = None
        self.net._grad_ready_hook = None

    # -- gradient exchange + optimizer ------------------------------------------------------------------------------------
    def describe_collective(self):
        if self.world == 1:
            return "none (1 GPU)"
        how = "own NCCL communicator behind the C ABI (mdt_allreduce_grads)" if self.comm else "torch.distributed"
        when = (f"per block during the backward on a side stream ({self.comm_ctas} comm CTAs, persistent grids sized "
                f"for {self._sms - self.comm_ctas} SMs)") if self.overlap else (
            f"after the backward in {self.ar_chunks} chunks on a side stream, pipelined with the optimizer pass"
            if self.ar_chunks > 1 else "one flat call after the backward")
        return f"{self.grad_dtype} sum-all-reduce of the flat gradient buffer, {how}, {when}"

    def _exchange(self, lo, hi, background=False):
        """Sum gradient elements [lo, hi) over the ranks on the current stream (in `grad`, or in the bf16 buffer)."""
        if hi <= lo or self.world == 1:
            return
        st = self.st
        buf = st.grad[lo:hi]
        if self.g16 is not None:
            buf = ops.cast_bf16(buf, out=self.g16[lo:hi])
        if self.comm is not None:
            (self.comm_bg if (background and self.comm_bg is not None) else self.comm).all_reduce(buf)
        else:
            dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.pg)

    def _step_range(self, lo, hi, max_blocks=0):
        st, n = self.st, hi - lo
        if n <= 0:
            return
        g = self.g16[lo:hi] if (self.g16 is not None and self.world > 1) else st.grad[lo:hi]
        ops.adamw_ema(st.w32[lo:hi], g, self.m[lo:hi], self.v[lo:hi],
                      self.ema_st.w32[lo:hi] if self.ema_st is not None else None, st.w16[lo:hi], n, self._lr_now,
                      self.step_count, self.betas[0], self.betas[1], self.eps, self.wd, self.ema_decay,
                      self._grad_scale, max_blocks)

    def _on_grads_ready(self, lo, hi):
        """Called (on the host, from inside mdt_backward) when the kernels finalising gradient elements [lo, hi) of one
        block are enqueued: start their exchange behind them on the side stream."""
        if not self._done:   # first block of this backward: from here on the persistent grids leave SMs to the side stream
            ops.check(ops.lib().mdt_set_sm_budget(self._sms - self.comm_ctas), "mdt_set_sm_budget", 0)
        main = torch.cuda.current_stream()
        self.side.wait_stream(main)
        with torch.cuda.stream(self.side):
            self._exchange(lo, hi, background=True)
        self._done.append((lo, hi))

    def _fwd_bwd_graphed(self, images, labels, mask_ratio, mae_loss_coef, loss_call, moments=False):
        """Gradient zeroing + loss forward + engine backward (~770 launches, 70 ms of host time) replayed from a CUDA
        graph captured once per (shapes, mask_ratio, mae_loss_coef); the all-reduce and the optimizer pass stay eager
        (their scalars change every step).  Opt-in (`TrainStep(graph=True)` / MDT_TRAIN_GRAPH=1): checked by
        tests/test_model_gpu_extra.py::test_train_step_cuda_graph_matches_eager."""
        # keyed on the kept-token count (what shapes the launches), not on the float ratio: a schedule such as cos4
        # (configs/finetune/imagenet256-latent-cos.yaml) revisits few distinct T; at most 2 graphs are kept.
        L = self.net.model.num_patches
        key = (tuple(images.shape), tuple(labels.shape), int(L * (1 - mask_ratio)) if mask_ratio > 0 else -1,
               float(mae_loss_coef), bool(moments))
        ent = self._graphs.get(key)
        if ent is None:
            while len(self._graphs) >= 2:
                self._graphs.pop(next(iter(self._graphs)))
            gx, gy = images.clone(), labels.clone()

            def body():
                self.st.grad.zero_()
                loss = loss_call(self.net, gx, gy, mask_ratio, mae_loss_coef)
                loss.mean().backward()
                return loss.detach()

            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):   # warm-up outside the capture (lazy kernel attributes, allocator pools)
                body()
            cur.wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            n0 = ops.L.LAUNCHES
            with torch.cuda.graph(graph):
                out = body()
            ent = (graph, gx, gy, out, ops.L.LAUNCHES - n0)
            self._graphs[key] = ent
        graph, gx, gy, out, n_launch = ent
        gx.copy_(images), gy.copy_(labels)
        graph.replay()
        ops.L.LAUNCHES += n_launch
        return out.clone()

    def step(self, images, labels, mask_ratio=0.5, mae_loss_coef=0.1, grad_accum=1, moments=False,
             class_dropout_prob=0.0):
        """One optimisation step on this rank's shard.  Returns the per-sample loss [B] (device tensor).
        `grad_accum` > 1: the shard is cut into that many equal micro-batches whose mean-loss gradients are averaged
        (train.py:211-227 under accelerate's `gradient_accumulation_steps`): the wgrad kernels accumulate into the
        flat buffer anyway, so the rounds simply run back to back and 1/rounds is folded into the optimizer kernel.
        `moments=True`: `images` are VAE moments [B,2C,R,R] straight from the dataset; the latent sampling, the label
        dropout (`class_dropout_prob`) and the noise injection run as the fused step-front kernel (EDMLoss.from_moments)."""
        st = self.st
        if moments:
            base_loss = self.loss_fn
            pre = {}
            if grad_accum > 1:   # the reference draws these once for the whole per-GPU batch (train.py:206-209)
                Bt, C2, R, _ = images.shape
                pre["eps"] = base_loss._randn((Bt, C2 // 2, R, R), images.device)
                if class_dropout_prob > 0:
                    pre["drop_u"] = base_loss._rand((Bt, 1), images.device).reshape(Bt)
            rounds = [0]

            def loss_call(net, x, lab, mask_ratio, mae_loss_coef):
                n, r = x.shape[0], rounds[0]
                rounds[0] += 1
                sl = {k: v[r * n:(r + 1) * n].contiguous() for k, v in pre.items()}
                return base_loss.from_moments(net, x, lab, mask_ratio=mask_ratio, mae_loss_coef=mae_loss_coef,
                                              class_dropout_prob=class_dropout_prob, **sl)
        else:
            def loss_call(net, x, lab, mask_ratio, mae_loss_coef):
                return self.loss_fn(net, x, lab, mask_ratio=mask_ratio, mae_loss_coef=mae_loss_coef)
        gb = self.global_batch or images.shape[0] * self.world
        self._lr_now = lr_at(self.step_count + self.lr_step_offset, self.lr, gb, self.rampup) \
            if self.reference_lr_schedule else self.lr
        self.step_count += 1
        self._done = []
        self._grad_scale = 1.0 / (self.world * grad_accum)
        if grad_accum > 1:
            if images.shape[0] % grad_accum:
                raise ValueError(f"batch {images.shape[0]} is not divisible by grad_accum {grad_accum}")
            if self.overlap:
                raise ValueError("overlap=True steps block ranges during the backward: incompatible with grad_accum > 1")
            mb = images.shape[0] // grad_accum
            st.grad.zero_()
            losses = []
            for r in range(grad_accum):
                lr_ = loss_call(self.net, images[r * mb:(r + 1) * mb], labels[r * mb:(r + 1) * mb], mask_ratio,
                                mae_loss_coef)
                lr_.mean().backward()
                losses.append(lr_.detach())
            loss = torch.cat(losses)
        elif self.graph and not self.overlap and ops.L.GEMM_PROFILE is None:
            loss = self._fwd_bwd_graphed(images, labels, mask_ratio, mae_loss_coef, loss_call, moments)
        else:
            st.grad.zero_()
            loss = loss_call(self.net, images, labels, mask_ratio, mae_loss_coef)
            loss.mean().backward()   # engine backward; with overlap=True block ranges are already being reduced/stepped
        main = torch.cuda.current_stream()
        if self.overlap and self._done:
            ops.check(ops.lib().mdt_set_sm_budget(0), "mdt_set_sm_budget", 0)
            self.side.wait_stream(main)
            with torch.cuda.stream(self.side):
                cur = 0
                for lo, hi in sorted(self._done) + [(st.n_train, st.n_train)]:   # the complement of the block ranges
                    self._exchange(cur, lo)
                    cur = max(cur, hi)
            main.wait_stream(self.side)
            self._step_range(0, st.n_train)          # ONE optimizer pass over the whole (reduced) buffer
        elif self.world == 1:
            self._step_range(0, st.n_train)
        elif self.ar_chunks > 1:
            # pipeline the exposed all-reduce against the optimizer pass: chunk k is stepped while k+1 is on the wire
            if self.side is None:
                self.side = torch.cuda.Stream(device=st.grad.device)
            bounds = ar_chunk_bounds(st.n_train, self.ar_chunks)
            self.side.wait_stream(main)
            evs = []
            with torch.cuda.stream(self.side):
                for lo, hi in bounds:
                    self._exchange(lo, hi)
                    ev = torch.cuda.Event()
                    ev.record(self.side)
                    evs.append(ev)
            for (lo, hi), ev in zip(bounds, evs):
                main.wait_event(ev)
                self._step_range(lo, hi)
        else:
            self._exchange(0, st.n_train)            # one flat all-reduce ...
            self._step_range(0, st.n_train)          # ... + one optimizer pass
        st.mark_shadow_fresh(self.net._params())   # the kernel refreshed the bf16 shadow itself
        if self.ema_st is not None:
            self.ema_st._versions = None           # EMA weights changed behind PyTorch's back: shadow is stale
        return loss.detach()
