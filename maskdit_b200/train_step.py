"""Data-parallel training step on the H100 engine (reference: train.py:200-230 inner step, :178 DDP, :141 optimizer,
train_utils/helper.py:47-58 EMA).

One process per GPU.  A step is:
    zero flat grad  ->  fused EDM loss forward/backward (C++ step driver)  ->  sum-all-reduce of the flat gradient
    buffer over NVLink (`GradComm`: our own NCCL communicator behind the C ABI; the 1/world factor is folded into the
    optimizer kernel)  ->  fused AdamW + EMA + bf16-shadow kernel over the flat buffers.
At world > 1 the all-reduce runs after the backward in `ar_chunks` chunks on a side stream, the optimizer pass of chunk
k running on the main stream while chunk k+1 is on the wire.  No other collective is issued in the step (SURVEY.md
§8e); the loss is returned as a device tensor (no per-step `.item()` host sync as at train.py:227).
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

from . import ops, phema
from .loss import ECTLoss, EDMLoss
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


def check_max_grad_norm(c):
    """The clipping bound `TrainStep(max_grad_norm=)` accepts: None (off), or a float > 0, inf included (measure only)."""
    if c is None:
        return None
    c = float(c)
    if not c > 0:   # also NaN
        raise ValueError(f"max_grad_norm must be > 0 (inf: report the norm without clipping), got {c}")
    return c


def ar_chunk_bounds(n, k):
    """[lo, hi) element ranges of the k all-reduce chunks of a flat buffer of n elements (4 KiB aligned starts)."""
    if k <= 1 or n < k * 1024:
        return [(0, n)]
    step = -(-(-(-n // k)) // 1024) * 1024
    return [(lo, min(n, lo + step)) for lo in range(0, n, step)]


class GradComm:
    """The step's gradient exchange behind the C ABI (`mdt_nccl_*`, `mdt_allreduce_grads`, csrc/driver.cu): an NCCL
    communicator of our own, created from a unique id that rank 0 draws and `torch.distributed` merely ships to the
    other ranks (any backend; it is the bootstrap side channel, nothing else)."""

    def __init__(self, pg=None):
        import ctypes
        self.rank, self.world = dist.get_rank(pg), dist.get_world_size(pg)
        L = ops.lib()
        buf = ctypes.create_string_buffer(128)
        if self.rank == 0:
            ops.check(L.mdt_nccl_unique_id(buf), "mdt_nccl_unique_id", 0)
        box = [bytes(buf.raw)]
        dist.broadcast_object_list(box, src=dist.get_global_rank(pg, 0) if pg is not None else 0, group=pg)
        self._comm = ctypes.c_void_p()
        ops.check(L.mdt_nccl_comm_create(box[0], self.rank, self.world, 0, ctypes.byref(self._comm)),
                  "mdt_nccl_comm_create", 0)

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
    phema_emas = ()   # no post-hoc EMA profiles unless the constructor is given widths
    edm_loss = None   # the last step's reference per-sample loss (see `step`)
    # consistency tuning (loss_fn an ECTLoss): the stage's device word q^-(s+1) that the step front reads (allocated by
    # the first tuned step), the run step of the first tuned step, and the last step's stage
    _ect_qs = None
    ect_origin = None
    ect_stage = None

    def __init__(self, net: EDMPrecond, ema: EDMPrecond | None = None, lr=1e-4, betas=(0.9, 0.999), eps=1e-8,
                 weight_decay=0.0, ema_decay=0.9999, loss_fn: EDMLoss | None = None, process_group=None,
                 lr_rampup_kimg=0.0, global_batch=None, device=None, overlap=False, graph=None,
                 reference_lr_schedule=False, collective=None, grad_dtype=None, skip_nonfinite=False,
                 recompute_blocks=None, phema_sigma_rels=(), max_grad_norm=None):
        """max_grad_norm: gradient-norm clipping, torch.nn.utils.clip_grad_norm_'s formula on the device.  None
        (default): off, nothing is allocated or launched.  A float c > 0: every step measures
        norm = grad_scale * ||g||_2 over the trainable region, g being the gradient the optimizer reads (the fp32 flat
        gradient at world 1, the summed exchange buffer at world > 1, bf16 sums under grad_dtype='bf16') and
        grad_scale = 1/(world * grad_accum), i.e. the norm of the averaged gradient that clip_grad_norm_ returns after
        a DDP backward.  The sum of squares runs in fp64 in an order that depends only on the size (bit-reproducible in
        both modes, whatever the SM budget), and the norm is rounded to fp32 once.  The update then uses
        coef * grad_scale * g with coef = min(1, c / (norm + 1e-6)) in fp32; c = inf only measures (coef = 1, and the
        update is the unclipped one bit for bit).  `grad_norm` holds the last step's norm before clipping on the
        device.  Every rank holds the same summed bits, so every rank computes the same norm without a collective.
        Cost: at world 1 one extra read of the gradient, none under skip_nonfinite (the norm pass replaces the check
        pass).  At world > 1 each chunk's sum of squares runs on the exchange stream after that chunk's all-reduce; with
        a finite c every optimizer pass then waits for the last chunk, since clipping needs the global norm, which
        serialises the optimizer behind the whole exchange (c = inf keeps the pipelined order).  With skip_nonfinite a
        non-finite element still skips the step, and with a finite c so does a non-finite norm (a sum that overflows
        although every rank's values were finite).  Without the guard a non-finite norm gives the coefficient the
        formula gives (NaN or 0), as clip_grad_norm_(error_if_nonfinite=False) does, and that poisons or freezes the
        weights; skip_nonfinite is how to avoid it.
        phema_sigma_rels: relative widths of power-function EMA profiles to keep for post-hoc EMA (`phema.py`,
        posthoc_ema.py), e.g. (0.05, 0.10); at most 4.  Each is one fp32 buffer over the trainable region (2.92 GB for XL/2),
        allocated here and advanced after every optimizer pass over a range, on that pass's stream, by `mdt_power_ema`
        with 1 - beta(t) from the host's count t of the profiles' steps: exactly one update per optimizer step (also
        under grad_accum, and toward the unchanged weights when skip_nonfinite skips the step).  The profiles count
        from `phema_origin`, the run step before their first update (`step_count + lr_step_offset` then).  Empty
        (default): nothing is allocated and nothing launches.
        recompute_blocks: how many blocks (in forward order, encoder first) keep only their output and have their
        forward re-run in the backward (activation recomputation, `mdt_model_set_recompute`).  None: automatic, i.e.
        none unless the training workspace of a micro-batch does not fit into device memory, then the fewest that
        make it fit; an int in [0, depth + dec_depth] forces that count.  The count in use is `self.recompute_blocks`.
        The gradients do not depend on it beyond the default mode's summation-order noise (bit for bit under
        `torch.use_deterministic_algorithms(True)`).
        skip_nonfinite:skip every optimizer step whose gradient holds an inf or NaN, as the reference's fp16
        GradScaler does (train.py:39-48): the weights, the bf16 shadow, the moments and Adam's step count stay as they
        are, the EMA still moves toward the unchanged weights (train.py:230), and the lr schedule's counter
        (`step_count`) advances as for any attempted step.  At world 1 the flat gradient is checked; at world > 1
        each rank checks its local values before the exchange (with bf16 exchange the bf16 values, checked while they
        are cast) and one flag word is summed over the ranks, so a non-finite value on any rank skips the step
        everywhere (with `MDT_AR_CHUNKS=1` and fp32 exchange this replaces an earlier check of the summed buffer, which
        could also flag finite values whose sum overflows).  The decision is a device flag (no host
        synchronisation); Adam's step count lives on the device
        (`applied_steps()`), the number of skipped steps in `skipped_steps`.  Off by default: the step is then
        exactly the unguarded one.
        Multi-GPU options (world > 1; SURVEY 8e: the step's ONLY collective is the sum of the flat gradient buffer):
          collective  'mdt' (default with an NCCL process group): our own communicator behind the C ABI (`GradComm`);
                      'torch': `torch.distributed.all_reduce` on the process group (gloo tests, A/B).
          grad_dtype  'bf16' (default, SURVEY 8e): the fp32 gradient buffer is cast to a bf16 exchange buffer, 1.46 GB cross
                      the links instead of 2.92 GB and the optimizer kernel reads the bf16 sums; local
                      accumulation, moments and master weights stay fp32.  2-rank vs 1-GPU gradient rel-L2 2.3e-3.
                      'fp32': the 2.92 GB buffer is reduced as is (DDP's arithmetic; rel-L2 1e-5, order noise).
          The exchange runs after the backward in `ar_chunks` chunks (MDT_AR_CHUNKS, default 4) on a side stream, the
          optimizer pass of chunk k on the main stream while chunk k+1 is on the wire.
          overlap     only False is accepted: the exchange overlapped with the backward was removed (a C caller can
                      still overlap through `mdt_backward`'s `on_ready` callback).  `self.overlap` stays readable
                      and is always False, so code that inspects a TrainStep's configuration keeps working.
        Environment overrides: MDT_COLLECTIVE, MDT_GRAD_AR, MDT_AR_CHUNKS."""
        if overlap:
            raise ValueError("overlap=True: the gradient exchange overlapped with the backward was removed; the "
                             "exchange runs after the backward, chunked and pipelined with the optimizer")
        self.overlap = False
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
        self._engine = net._engine
        if recompute_blocks is not None and not 0 <= int(recompute_blocks) <= self._engine.num_blocks:
            raise ValueError(f"recompute_blocks {recompute_blocks} outside [0, {self._engine.num_blocks}]")
        self._engine.recompute = None if recompute_blocks is None else int(recompute_blocks)
        if recompute_blocks is not None:
            self._engine.recompute_blocks = int(recompute_blocks)
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
        env = os.environ
        self.collective = env.get("MDT_COLLECTIVE") or collective or \
            ("mdt" if self.world > 1 and dist.get_backend(process_group) == "nccl" else "torch")
        self.grad_dtype = env.get("MDT_GRAD_AR") or grad_dtype or "bf16"
        assert self.collective in ("mdt", "torch") and self.grad_dtype in ("fp32", "bf16")
        self.comm = None
        self.g16 = None
        if self.world > 1:
            if self.collective == "mdt":
                self.comm = GradComm(process_group)
            if self.grad_dtype == "bf16":
                self.g16 = torch.empty(n, dtype=torch.bfloat16, device=dev)
        self.graph = (os.environ.get("MDT_TRAIN_GRAPH", "0") == "1") if graph is None else bool(graph)
        self._graphs = {}
        # gradient all-reduce in this many chunks on a side stream, the fused AdamW/EMA pass of chunk k running while
        # chunk k+1 is on the wire.
        self.ar_chunks = int(os.environ.get("MDT_AR_CHUNKS", "4"))
        self.side = None         # the exchange's stream, created by the first step at world > 1
        self._lr_now = lr
        # non-finite guard: flag (fp32, 0 = finite; a SUM over the ranks is their OR), counts {applied, skipped}
        self.skip_nonfinite = bool(skip_nonfinite)
        self._flag = torch.zeros(1, dtype=torch.float32, device=dev) if self.skip_nonfinite else None
        self._counts = torch.zeros(2, dtype=torch.int64, device=dev) if self.skip_nonfinite else None
        # gradient-norm clipping: fp64 sum-of-squares slots (one per exchange chunk), the norm pass's scratch, norm, coef
        self.max_grad_norm = check_max_grad_norm(max_grad_norm)
        if self.max_grad_norm is not None:
            self._gn_slots = torch.zeros(max(len(ar_chunk_bounds(n, self.ar_chunks)), 1), dtype=torch.float64,
                                         device=dev)
            self._gn_scratch = ops.grad_sumsq_scratch(n, dev)
            self._gn = torch.zeros(2, dtype=torch.float32, device=dev)   # {norm, coef}
        # power-function EMA profiles: allocated now, so the recomputation picker sees their memory as used
        self.phema_sigma_rels = tuple(float(s) for s in phema_sigma_rels)
        if len(self.phema_sigma_rels) > 4:   # mdt_power_ema advances up to 4 profiles from one read of the weights
            raise ValueError(f"{len(self.phema_sigma_rels)} post-hoc EMA profiles: at most 4")
        self.phema_gammas = tuple(phema.sigma_rel_to_gamma(s) for s in self.phema_sigma_rels)
        self.phema_emas = [torch.zeros(n, dtype=torch.float32, device=dev) for _ in self.phema_sigma_rels]
        self.phema_origin = None   # run step before the profiles' first update (None: set by the next step)
        self.phema_steps = 0       # updates since the origin (the profiles' t after the last step)
        self._phema_c = None

    @property
    def recompute_blocks(self) -> int:
        """Blocks recomputed by the last training forward (before the first step: the forced count, or 0)."""
        return self._engine.recompute_blocks

    @property
    def skipped_steps(self):
        """Device tensor (int64, 0-dim): optimizer steps skipped for non-finite gradients since this object was built
        (None without `skip_nonfinite`).  Reading its value synchronises; the step itself never does."""
        return self._counts[1] if self._counts is not None else None

    @property
    def grad_norm(self):
        """Device tensor (fp32, 0-dim): the last step's gradient norm before clipping, grad_scale * ||g||_2 (None without
        `max_grad_norm`).  Reading its value synchronises; the step itself never does."""
        return self._gn[0] if self.max_grad_norm is not None else None

    def _tunes(self):
        return isinstance(getattr(self, "loss_fn", None), ECTLoss)

    def applied_steps(self) -> int:
        """Adam's step count: the steps whose update was applied (a host read of the device counter under
        `skip_nonfinite`, i.e. one synchronisation; `step_count` otherwise)."""
        return int(self._counts[0]) if self._counts is not None else self.step_count

    # -- optimizer state for checkpoints (reference: train.py:259-270 stores optimizer.state_dict() under 'opt') ------
    def state_dict(self):
        """AdamW state laid out like `torch.optim.AdamW(net.parameters()).state_dict()` / apex FusedAdam's
        (train.py:141,262): `state` is keyed by the parameter's POSITION in `net.parameters()` — frozen tensors
        (pos_embed = 0, decoder_pos_embed = 1) keep their index but own no state, so the first key is 2 (1 for the
        decoder-less DiT, whose only frozen tensor is pos_embed) — with
        `exp_avg` / `exp_avg_sq` and a per-parameter `step` (torch layout); the step count is also stored in the
        param_group (apex layout).  Tensors are copies on the current device.  The step count is Adam's
        (`applied_steps()`): under `skip_nonfinite` it leaves out the skipped steps.
        With power-function EMA profiles, `phema` holds their widths, exponents, origin, step count and flat buffers
        (host copies: the device keeps no second copy of them).  Under consistency tuning, `ect` holds the tuning
        origin, so a resumed run continues the stage."""
        state, n_all = {}, 0
        adam_step = self.applied_steps()
        for i, (k, p) in enumerate(self.net.named_parameters()):
            n_all = i + 1
            if not p.requires_grad:
                continue
            lo, _, shape = self.st.offsets[k]
            n = p.numel()
            state[i] = {"step": torch.tensor(float(adam_step)), "exp_avg": self.m[lo:lo + n].view(shape).clone(),
                        "exp_avg_sq": self.v[lo:lo + n].view(shape).clone()}
        sd = {"state": state,
              "param_groups": [{"lr": self.lr, "betas": self.betas, "eps": self.eps, "weight_decay": self.wd,
                                "step": adam_step, "params": list(range(n_all))}]}
        if self._tunes():
            sd["ect"] = {"origin": self.ect_origin, "stage_steps": self.loss_fn.stage_steps}
        if self.phema_emas:
            sd["phema"] = {"sigma_rels": list(self.phema_sigma_rels), "gammas": list(self.phema_gammas),
                           "origin": self.phema_origin, "steps": self.phema_steps,
                           "emas": [e.to("cpu", copy=True) for e in self.phema_emas]}
        return sd

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
        if self._counts is not None:   # Adam continues from the stored count; the skip tally is this object's own
            self._counts[0].fill_(self.step_count)
        self.lr, self.betas, self.eps, self.wd = group["lr"], tuple(group["betas"]), group["eps"], \
            group["weight_decay"]
        if self.phema_emas:
            self._load_phema(sd.get("phema"))
        if self._tunes():   # a state without it (an EDM run's) starts tuning at the next step
            self.ect_origin = (sd.get("ect") or {}).get("origin")

    def _load_phema(self, ph):
        """Continue the stored profiles, or (a state without them, e.g. a reference checkpoint) start new ones whose
        origin is the run step of the next update."""
        if ph is None:
            for e in self.phema_emas:
                e.zero_()
            self.phema_origin, self.phema_steps = None, 0
            return
        if [round(s, 9) for s in ph["sigma_rels"]] != [round(s, 9) for s in self.phema_sigma_rels]:
            raise ValueError(f"the state holds post-hoc EMA profiles of sigma_rel {list(ph['sigma_rels'])}, this "
                             f"TrainStep keeps {list(self.phema_sigma_rels)}")
        for e, src in zip(self.phema_emas, ph["emas"]):
            if src.numel() != e.numel():
                raise ValueError(f"post-hoc EMA profile of {src.numel()} elements, the model trains {e.numel()}")
            e.copy_(src.reshape(-1))
        self.phema_origin, self.phema_steps = int(ph["origin"]), int(ph["steps"])

    # -- power-function EMA profiles (post-hoc EMA) ----------------------------------------------------------------
    def phema_state_dicts(self):
        """The profiles as model state dicts with the module's keys (host copies; frozen tensors from the weights)."""
        out = []
        for e in self.phema_emas:
            flat = e.to("cpu", copy=True)   # one host storage per profile; the trainable tensors are views into it
            sd = {}
            for k, v in self.net.state_dict().items():
                o, cnt, shape = self.st.offsets.get(k, (None, None, None))
                if o is not None and o + cnt <= self.st.n_train:
                    sd[k] = flat[o:o + cnt].view(shape)
                else:
                    sd[k] = v.detach().to("cpu", copy=True)
            out.append(sd)
        return out

    def phema_snapshot(self):
        """What post-hoc EMA reconstruction reads: {step, origin, profiles: [{sigma_rel, gamma, ema}]}, where step is
        the run step of the last update and each ema a state dict."""
        if self.phema_origin is None:
            raise ValueError("the post-hoc EMA profiles have not been updated yet")
        return {"step": self.phema_origin + self.phema_steps, "origin": self.phema_origin,
                "profiles": [{"sigma_rel": s, "gamma": g, "ema": sd} for s, g, sd in
                             zip(self.phema_sigma_rels, self.phema_gammas, self.phema_state_dicts())]}

    def close(self):
        """Release the communicator (a TrainStep owns one when world > 1 and collective == 'mdt')."""
        if self.comm is not None:
            self.comm.close()
        self.comm = None

    # -- gradient exchange + optimizer ------------------------------------------------------------------------------------
    def describe_collective(self):
        if self.world == 1:
            return "none (1 GPU)"
        how = "own NCCL communicator behind the C ABI (mdt_allreduce_grads)" if self.comm else "torch.distributed"
        when = f"after the backward in {self.ar_chunks} chunks on a side stream, pipelined with the optimizer pass" \
            if self.ar_chunks > 1 else "one flat call after the backward"
        return f"{self.grad_dtype} sum-all-reduce of the flat gradient buffer, {how}, {when}"

    def _cast(self, lo, hi):
        """fp32 gradient [lo, hi) -> the bf16 exchange buffer; under the guard the cast also checks what it stores."""
        if self._flag is not None:
            return ops.cast_bf16_check(self.st.grad[lo:hi], self._flag, out=self.g16[lo:hi])
        return ops.cast_bf16(self.st.grad[lo:hi], out=self.g16[lo:hi])

    def _all_reduce(self, buf):
        if self.comm is not None:
            self.comm.all_reduce(buf)
        else:
            dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.pg)

    def _exchange(self, lo, hi, cast=True):
        """Sum gradient elements [lo, hi) over the ranks on the current stream (in `grad`, or in the bf16 buffer;
        cast=False: the bf16 buffer already holds this range's cast)."""
        buf = self.st.grad[lo:hi]
        if self.g16 is not None:
            buf = self._cast(lo, hi) if cast else self.g16[lo:hi]
        self._all_reduce(buf)

    def _clips(self):
        return self.max_grad_norm is not None and self.max_grad_norm != float("inf")

    def _grad_norm_coef(self, k):
        """norm and coef from the first k sum-of-squares slots; with a finite bound a non-finite norm sets the guard's
        flag."""
        ops.grad_clip_coef(self._gn_slots[:k], self._grad_scale, self.max_grad_norm, self._gn[:1], self._gn[1:],
                           flag=self._flag if self._clips() else None)

    def _step_range(self, lo, hi):
        st, n = self.st, hi - lo
        if n <= 0:
            return
        g = self.g16[lo:hi] if (self.g16 is not None and self.world > 1) else st.grad[lo:hi]
        ema = self.ema_st.w32[lo:hi] if self.ema_st is not None else None
        # a finite clipping bound: the optimizer reads the coefficient (c = inf keeps the plain kernels)
        coef = self._gn[1:] if self._clips() else None
        if self._flag is not None:   # Adam's step number comes from the device counter, the skip from the flag
            ops.adamw_ema_guarded(st.w32[lo:hi], g, self.m[lo:hi], self.v[lo:hi], ema, st.w16[lo:hi], n, self._lr_now,
                                  self._flag, self._counts, self.betas[0], self.betas[1], self.eps, self.wd,
                                  self.ema_decay, self._grad_scale, coef=coef)
        else:
            ops.adamw_ema(st.w32[lo:hi], g, self.m[lo:hi], self.v[lo:hi], ema, st.w16[lo:hi], n, self._lr_now,
                          self.step_count, self.betas[0], self.betas[1], self.eps, self.wd, self.ema_decay,
                          self._grad_scale, coef=coef)
        if self.phema_emas:   # the profiles follow the range's new (or, skipped, unchanged) weights on the same stream
            ops.power_ema(st.w32[lo:hi], [e[lo:hi] for e in self.phema_emas], self._phema_c)

    def _fwd_bwd_graphed(self, images, labels, mask_ratio, mae_loss_coef, loss_call, moments=False):
        """Gradient zeroing + loss forward + engine backward (~770 launches, 70 ms of host time) replayed from a CUDA
        graph captured once per (shapes, mask_ratio, mae_loss_coef); the all-reduce and the optimizer pass stay eager
        (their scalars change every step).  Opt-in (`TrainStep(graph=True)` / MDT_TRAIN_GRAPH=1): checked by
        tests/test_model_gpu_extra.py::test_train_step_cuda_graph_matches_eager."""
        # keyed on the kept-token count (what shapes the launches), not on the float ratio: a schedule such as cos4
        # (configs/finetune/imagenet256-latent-cos.yaml) revisits few distinct T; at most 2 graphs are kept.
        L = self.net.model.num_patches
        # the deterministic mode is part of the key: a captured graph replays the reductions it was captured with
        key = (tuple(images.shape), tuple(labels.shape), int(L * (1 - mask_ratio)) if mask_ratio > 0 else -1,
               float(mae_loss_coef), bool(moments), ops.L.sync_deterministic())
        ent = self._graphs.get(key)
        if ent is None:
            while len(self._graphs) >= 2:
                self._graphs.pop(next(iter(self._graphs)))
            gx, gy = images.clone(), labels.clone()

            def body():
                self.st.grad.zero_()
                loss = loss_call(self.net, gx, gy, mask_ratio, mae_loss_coef)
                loss.mean().backward()
                return loss.detach(), self._last_edm_loss()

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
        graph, gx, gy, (out, out_edm), n_launch = ent
        gx.copy_(images), gy.copy_(labels)
        graph.replay()
        ops.L.LAUNCHES += n_launch
        loss = out.clone()
        return loss, (out_edm.clone() if out_edm is not None else loss)

    def _last_edm_loss(self):
        """The reference loss of the last loss call when the network learns its loss weighting, else None."""
        return self.loss_fn.last_edm_loss.detach() if self.net.logvar_channels else None

    def step(self, images, labels, mask_ratio=0.5, mae_loss_coef=0.1, grad_accum=1, moments=False,
             class_dropout_prob=0.0):
        """One optimisation step on this rank's shard.  Returns the per-sample loss [B] (device tensor): the objective
        the gradient follows, which for a network with a learned loss weighting (`EDMPrecond(logvar_channels=C)`) is
        exp(-u) E + u + mae_coef M.  `edm_loss` then holds the reference's per-sample loss E + mae_coef M [B] of the
        step (concatenated over the grad_accum rounds), comparable with runs without the weighting; without one it is
        the returned tensor.  w, the weighting's one trainable tensor, lives in the flat buffers like every other
        weight, so AdamW, the EMA, the post-hoc EMA profiles, clipping, the non-finite guard and the exchange cover it.
        `grad_accum` > 1: the shard is cut into that many equal micro-batches whose mean-loss gradients are averaged
        (train.py:211-227 under accelerate's `gradient_accumulation_steps`): the wgrad kernels accumulate into the
        flat buffer anyway, so the rounds simply run back to back and 1/rounds is folded into the optimizer kernel.
        `moments=True`: `images` are VAE moments [B,2C,R,R] straight from the dataset; the latent sampling, the label
        dropout (`class_dropout_prob`) and the noise injection run as the fused step-front kernel (EDMLoss.from_moments).
        With an `ECTLoss` the step runs at tuning stage s = floor((run step - ect_origin) / stage_steps), the run step
        being `step_count + lr_step_offset` before the call and `ect_origin` the run step of the first tuned step.
        Under `torch.use_deterministic_algorithms(True)` the library's deterministic mode is on for the step
        (`mdt_set_deterministic`): the gradients, and so the weights, moments and EMA, repeat bit for bit."""
        st = self.st
        ops.L.sync_deterministic()
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
        if self.phema_emas:
            if self.phema_origin is None:
                self.phema_origin = self.step_count - 1 + self.lr_step_offset
            self.phema_steps += 1
            self._phema_c = [phema.one_minus_beta(g, self.phema_steps) for g in self.phema_gammas]
        if self._tunes():   # the stage word changes on the device, so a replayed graph reads it too
            if self._ect_qs is None:
                self._ect_qs = torch.zeros(1, dtype=torch.float32, device=st.w32.device)
            self.loss_fn.stage_scale = self._ect_qs
            run = self.step_count - 1 + self.lr_step_offset
            if self.ect_origin is None:
                self.ect_origin = run
            self.ect_stage = self.loss_fn.stage_at(run, self.ect_origin)
            self._ect_qs.fill_(self.loss_fn.scale_of(self.ect_stage))
        guard = self._flag is not None
        if guard:
            self._flag.zero_()
        self._grad_scale = 1.0 / (self.world * grad_accum)
        if grad_accum > 1:
            if images.shape[0] % grad_accum:
                raise ValueError(f"batch {images.shape[0]} is not divisible by grad_accum {grad_accum}")
            mb = images.shape[0] // grad_accum
            st.grad.zero_()
            losses, edm = [], []
            for r in range(grad_accum):
                lr_ = loss_call(self.net, images[r * mb:(r + 1) * mb], labels[r * mb:(r + 1) * mb], mask_ratio,
                                mae_loss_coef)
                lr_.mean().backward()
                losses.append(lr_.detach())
                edm.append(self._last_edm_loss())
            loss = torch.cat(losses)
            edm_loss = torch.cat(edm) if self.net.logvar_channels else loss
        elif self.graph and ops.L.GEMM_PROFILE is None:
            loss, edm_loss = self._fwd_bwd_graphed(images, labels, mask_ratio, mae_loss_coef, loss_call, moments)
        else:
            st.grad.zero_()
            loss = loss_call(self.net, images, labels, mask_ratio, mae_loss_coef)
            loss.mean().backward()   # engine backward
            edm_loss = self._last_edm_loss()
        loss = loss.detach()
        self.edm_loss = loss if edm_loss is None else edm_loss
        main = torch.cuda.current_stream()
        n = st.n_train
        # Under the guard the flag must be final before the first optimizer pass.  At world > 1 every rank checks its
        # local values (bf16 exchange: while casting them) and one flag word is summed over the ranks.
        measure = self.max_grad_norm is not None
        if self.world == 1:
            if measure:   # one read of the gradient: the norm, and under the guard the non-finite check
                ops.grad_sumsq(st.grad[:n], self._gn_slots[:1], self._gn_scratch, flag=self._flag)
                self._grad_norm_coef(1)
            elif guard:
                ops.nonfinite_check(st.grad[:n], self._flag)
            self._step_range(0, n)
        else:
            # pipeline the exposed all-reduce against the optimizer pass: chunk k is stepped while k+1 is on the wire
            if self.side is None:
                self.side = torch.cuda.Stream(device=st.grad.device)
            bounds = ar_chunk_bounds(n, self.ar_chunks)
            if measure and self._gn_slots.numel() < len(bounds):
                self._gn_slots = torch.zeros(len(bounds), dtype=torch.float64, device=st.grad.device)
            self.side.wait_stream(main)
            evs = []
            with torch.cuda.stream(self.side):
                if guard:   # chunk 0's optimizer pass needs the decision: check every local chunk first
                    if self.g16 is not None:
                        for lo, hi in bounds:
                            self._cast(lo, hi)
                    else:
                        ops.nonfinite_check(st.grad[:n], self._flag)
                    self._all_reduce(self._flag)
                for k, (lo, hi) in enumerate(bounds):
                    self._exchange(lo, hi, cast=not guard)
                    ev = torch.cuda.Event()
                    ev.record(self.side)
                    evs.append(ev)
                    if measure:   # the chunk's summed values, while the optimizer steps it
                        g = self.g16[lo:hi] if self.g16 is not None else st.grad[lo:hi]
                        ops.grad_sumsq(g, self._gn_slots[k:k + 1], self._gn_scratch)
                if measure:
                    self._grad_norm_coef(len(bounds))
            if self._clips():   # clipping needs the global norm: every chunk's pass waits for the coefficient
                main.wait_stream(self.side)
                evs = [None] * len(bounds)
            for (lo, hi), ev in zip(bounds, evs):
                if ev is not None:
                    main.wait_event(ev)
                self._step_range(lo, hi)
            if measure:   # the norm passes read buffers the next step writes on this stream
                main.wait_stream(self.side)
        if guard:
            ops.optim_guard_advance(self._flag, self._counts)
        st.mark_shadow_fresh(self.net._params())   # the kernel refreshed the bf16 shadow itself
        if self.ema_st is not None:
            self.ema_st._versions = None           # EMA weights changed behind PyTorch's back: shadow is stale
        return loss
