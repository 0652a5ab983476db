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
from .loss import ECTLoss, EDMLoss, MGLoss
from .maskdit import EDMPrecond

_GATHER_DTYPES = {torch.float32: 0, torch.bfloat16: 1, torch.float64: 2}   # MDT_DTYPE_F32 / _BF16 / _F64


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


SHARD_ALIGN = 64   # elements: 256 B of fp32, the optimizer kernels' float4 and alignment rules


def shard_piece(count, world):
    """Elements per rank of an exchange chunk of `count` elements under `TrainStep(shard_optimizer=True)`: count / world
    rounded up to a multiple of SHARD_ALIGN."""
    return -(-(-(-count // world)) // SHARD_ALIGN) * SHARD_ALIGN


def owned_ranges(n, world, chunks):
    """Per rank, the [lo, hi) element ranges of a flat buffer of n elements whose optimizer state the rank owns under
    `TrainStep(shard_optimizer=True)`: one range per exchange chunk (`ar_chunk_bounds(n, chunks)`), rank r owning piece r
    of the chunk's split into `world` pieces of `shard_piece(chunk, world)` elements.  So each chunk's reduce-scatter
    and all-gather are one call with equal counts.  The pieces of the last ranks may run past the chunk's end: the
    exchange buffer pads them, and their ranges here are clamped to the chunk (shorter, or empty with lo == hi)."""
    for name, v in (("n", n), ("world", world), ("chunks", chunks)):
        if isinstance(v, bool) or not isinstance(v, int) or v < 1:
            raise ValueError(f"owned_ranges: {name} must be an int >= 1, got {v!r}")
    out = [[] for _ in range(world)]
    for lo, hi in ar_chunk_bounds(n, chunks):
        p = shard_piece(hi - lo, world)
        for r in range(world):
            a = min(hi, lo + r * p)
            out[r].append((a, min(hi, a + p)))
    return out


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

    def reduce_scatter(self, t, count):
        """In-place SUM of t (world * count elements) whose share `count` elements at rank * count is this rank's."""
        assert t.is_cuda and t.is_contiguous() and t.dtype in (torch.float32, torch.bfloat16)
        assert t.numel() == count * self.world
        ops.check(ops.lib().mdt_reduce_scatter_grads(self._comm, t.data_ptr(), count, int(t.dtype == torch.bfloat16),
                                                     ops.stream_ptr()), "mdt_reduce_scatter_grads", 0)

    def all_gather(self, t, count):
        """In place: every rank's `count` elements at rank * count of t (world * count elements) to every rank."""
        assert t.is_cuda and t.is_contiguous() and t.dtype in _GATHER_DTYPES and t.numel() == count * self.world
        ops.check(ops.lib().mdt_allgather(self._comm, t.data_ptr(), count, _GATHER_DTYPES[t.dtype], ops.stream_ptr()),
                  "mdt_allgather", 0)

    def close(self):
        if self._comm:
            ops.lib().mdt_nccl_comm_destroy(self._comm)
            self._comm = None


class TrainStep:
    phema_emas = ()   # no post-hoc EMA profiles unless the constructor is given widths
    _sh = None        # the sharded layout (shard_optimizer at world > 1)
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
                 recompute_blocks=None, phema_sigma_rels=(), max_grad_norm=None, shard_optimizer=False):
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
          shard_optimizer  False (default): every rank keeps the whole optimizer state.  True (ZeRO stage 1, needs
                      collective 'mdt'): the all-reduce is split into its two halves.  Each exchange chunk is
                      reduce-scattered, each rank runs AdamW, the EMA and the post-hoc EMA profiles on its own piece of
                      every chunk (`owned_ranges`), then the bf16 shadow is all-gathered, and once per step the ranges
                      the step reads from the fp32 masters (`CEngine.fp32_read_ranges`).  m, v and the profiles are
                      allocated at 1/world of the trainable region; the weights, the shadow, the gradient and the EMA
                      keep their full buffers.  The update is elementwise, so the weights are the replicated step's bit
                      for bit (the clipping norm may differ by fp64 reassociation).  A rank's fp32 masters outside its
                      pieces and that set are stale between steps: `materialize()` gathers them and the EMA, and
                      `state_dict()` / `phema_snapshot()` become collectives that return the replicated layout.
                      At world 1 the flag changes nothing.
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
        self.shard_optimizer = bool(shard_optimizer)
        sharded = self.shard_optimizer and self.world > 1
        if sharded and self.collective != "mdt":
            raise ValueError("shard_optimizer=True needs collective='mdt' (the library's own NCCL communicator): the "
                             "torch.distributed exchange has no reduce-scatter / all-gather path")
        self.rank = dist.get_rank(process_group) if self.world > 1 else 0
        self.comm = None
        self.g16 = None
        if self.world > 1:
            if self.collective == "mdt":
                self.comm = GradComm(process_group)
            if self.grad_dtype == "bf16" and not sharded:
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
        self._sh = None   # the sharded layout (`_shard_setup`), None when every rank keeps the whole state
        if sharded:
            self._shard_setup()
        else:
            self.m = torch.zeros(n, dtype=torch.float32, device=dev)
            self.v = torch.zeros(n, dtype=torch.float32, device=dev)
            self.phema_emas = [torch.zeros(n, dtype=torch.float32, device=dev) for _ in self.phema_sigma_rels]
        self.phema_origin = None   # run step before the profiles' first update (None: set by the next step)
        self.phema_steps = 0       # updates since the origin (the profiles' t after the last step)
        self._phema_c = None

    # -- sharded optimizer state (shard_optimizer=True) ---------------------------------------------------------------
    def _shard_setup(self):
        """Lay out and allocate the sharded state for (world, rank, ar_chunks): per chunk k of `ar_chunk_bounds`, the
        piece p_k = `shard_piece`, this rank's owned range, the chunk's place in the padded exchange buffer (world * p_k
        elements) and in the local state (p_k elements: m, v and the profiles); then the fp32-read set's pack tables."""
        n, W, r, dev = self.st.n_train, self.world, self.rank, self.st.w32.device
        bounds = ar_chunk_bounds(n, self.ar_chunks)
        owned = owned_ranges(n, W, self.ar_chunks)
        pieces = [shard_piece(hi - lo, W) for lo, hi in bounds]
        xoff, loff = [0], [0]
        for p in pieces:
            xoff.append(xoff[-1] + W * p)
            loff.append(loff[-1] + p)
        self._sh = sh = type("ShardLayout", (), {})()
        sh.bounds, sh.pieces, sh.owned, sh.own, sh.xoff, sh.loff = bounds, pieces, owned, owned[r], xoff, loff
        self.m = self.v = None
        self.phema_emas = []
        self.m = torch.zeros(loff[-1], dtype=torch.float32, device=dev)
        self.v = torch.zeros(loff[-1], dtype=torch.float32, device=dev)
        self.phema_emas = [torch.zeros(loff[-1], dtype=torch.float32, device=dev) for _ in self.phema_sigma_rels]
        # the exchange buffer: chunk k at xoff[k], its padding (world * p_k - chunk elements) zero and never read
        self.g16 = None
        self.xbuf = torch.zeros(xoff[-1], dtype=torch.bfloat16 if self.grad_dtype == "bf16" else torch.float32,
                                device=dev)
        if self.max_grad_norm is not None:   # one fp64 sum of squares per (chunk, rank)
            self._gn_slots = torch.zeros(len(bounds) * W, dtype=torch.float64, device=dev)
        # fp32-read set: each rank packs its owned part of the set into its slot of `_rset`, one all-gather, and every
        # rank unpacks the other ranks' slots into w32
        read = self._engine.fp32_read_ranges()
        segs, sizes = [], []
        for rr in range(W):
            mine, o = [], 0
            for a, b in owned[rr]:
                for lo, hi in read:
                    lo, hi = max(a, lo), min(b, hi)
                    if lo < hi:
                        mine.append((lo, o, hi - lo))
                        o += hi - lo
            segs.append(mine)
            sizes.append(o)
        P = max(SHARD_ALIGN, -(-max(sizes) // SHARD_ALIGN) * SHARD_ALIGN)
        sh.read, sh.read_segs, sh.rset_piece = read, segs, P
        self._rset = torch.zeros(W * P, dtype=torch.float32, device=dev)
        pack = [(g, r * P + o, c) for g, o, c in segs[r]]
        unpack = [(rr * P + o, g, c) for rr in range(W) if rr != r for g, o, c in segs[rr]]
        sh.pack = torch.tensor(pack, dtype=torch.int64).reshape(-1, 3).to(dev)
        sh.unpack = torch.tensor(unpack, dtype=torch.int64).reshape(-1, 3).to(dev)

    def _xchunk(self, k):
        sh = self._sh
        return self.xbuf[sh.xoff[k]:sh.xoff[k + 1]]

    def _fill_x(self, k):
        """Chunk k of the local fp32 gradient into its exchange slot (bf16: cast, under the guard with the check)."""
        lo, hi = self._sh.bounds[k]
        x = self._xchunk(k)
        if x.dtype == torch.bfloat16:
            if self._flag is not None:
                ops.cast_bf16_check(self.st.grad[lo:hi], self._flag, out=x[:hi - lo])
            else:
                ops.cast_bf16(self.st.grad[lo:hi], out=x[:hi - lo])
        else:
            x[:hi - lo].copy_(self.st.grad[lo:hi])
            if x.numel() > hi - lo:   # the slot doubled as the shadow's staging last step
                x[hi - lo:].zero_()
        return x

    def _own_grad(self, k):
        """This rank's summed gradient of chunk k (its owned range's elements) in the exchange buffer."""
        sh = self._sh
        a, b = sh.own[k]
        o = sh.xoff[k] + self.rank * sh.pieces[k]
        return self.xbuf[o:o + b - a]

    def _step_piece(self, k):
        sh = self._sh
        a, b = sh.own[k]
        if b > a:
            self._step_range(a, b, self._own_grad(k), sh.loff[k])

    def _gather_w16(self, k):
        """All-gather chunk k of the bf16 shadow: in place, or (a padded chunk, whose last pieces would run past it)
        staged through the chunk's exchange slot, which the optimizer has read by now."""
        sh, st, W, r = self._sh, self.st, self.world, self.rank
        lo, hi = sh.bounds[k]
        p = sh.pieces[k]
        if W * p == hi - lo:
            self.comm.all_gather(st.w16[lo:hi], p)
            return
        a, b = sh.own[k]
        stage = self._xchunk(k).view(torch.bfloat16)[:W * p]
        stage[r * p:r * p + b - a].copy_(st.w16[a:b])
        self.comm.all_gather(stage, p)
        st.w16[lo:hi].copy_(stage[:hi - lo])

    def _gather_chunk(self, k, piece, out):
        """out (chunk k's hi - lo elements, host or device) = chunk k assembled from every rank's `piece` (its owned
        range's values): one all-gather through a chunk-sized device temporary."""
        sh = self._sh
        lo, hi = sh.bounds[k]
        p = sh.pieces[k]
        tmp = torch.zeros(self.world * p, dtype=piece.dtype, device=self.st.w32.device)
        tmp[self.rank * p:self.rank * p + piece.numel()].copy_(piece)
        self.comm.all_gather(tmp, p)
        out.copy_(tmp[:hi - lo])

    def _full(self, local):
        """A host fp32 tensor of the trainable region holding the replicated layout of the local state `local`
        (a collective under sharding; a host copy otherwise)."""
        if self._sh is None:
            return local.to("cpu", copy=True)
        sh = self._sh
        out = torch.empty(self.st.n_train, dtype=torch.float32)
        for k, ((lo, hi), (a, b)) in enumerate(zip(sh.bounds, sh.own)):
            self._gather_chunk(k, local[sh.loff[k]:sh.loff[k] + b - a], out[lo:hi])
        return out

    def _keep(self, local, lo, src):
        """Store the replicated-layout values src, which start at element lo, into the local state: all of them, or
        under sharding the part inside this rank's pieces."""
        if self._sh is None:
            local[lo:lo + src.numel()].copy_(src)
            return
        sh = self._sh
        for k, (a, b) in enumerate(sh.own):
            x, y = max(a, lo), min(b, lo + src.numel())
            if x < y:
                o = sh.loff[k] + x - a
                local[o:o + y - x].copy_(src[x - lo:y - lo])

    def materialize(self, ema=True, params=True):
        """Under sharding, a collective that every rank calls: all-gather the fp32 masters of the EMA network
        (`ema`) and of the trained network (`params`) into their full buffers, so that host reads (state dicts,
        validation, sampling) see current values.  The bf16 shadow is current already and is not recast.  Does nothing
        without sharding."""
        if self._sh is None:
            return
        sh = self._sh
        flats = ([self.st.w32] if params else []) + ([self.ema_st.w32] if ema and self.ema_st is not None else [])
        with torch.no_grad():
            for w in flats:
                for k, ((lo, hi), (a, b)) in enumerate(zip(sh.bounds, sh.own)):
                    self._gather_chunk(k, w[a:b], w[lo:hi])
        if params:   # the writes went through views of the parameters' storage: the shadow already holds these values
            self.st.mark_shadow_fresh(self.net._params())
        if ema and self.ema_st is not None:
            self.ema_st._versions = None

    @property
    def sharded(self) -> bool:
        """Whether the optimizer state is sharded across the ranks (`shard_optimizer` at world > 1)."""
        return self._sh is not None

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
        origin, so a resumed run continues the stage.
        Under `shard_optimizer` this is a collective that every rank calls.  It returns the replicated layout and
        values, gathered chunk by chunk into host tensors (no full-size device temporary)."""
        state, n_all = {}, 0
        adam_step = self.applied_steps()
        m, v = (self.m, self.v) if self._sh is None else (self._full(self.m), self._full(self.v))
        for i, (k, p) in enumerate(self.net.named_parameters()):
            n_all = i + 1
            if not p.requires_grad:
                continue
            lo, _, shape = self.st.offsets[k]
            n = p.numel()
            state[i] = {"step": torch.tensor(float(adam_step)), "exp_avg": m[lo:lo + n].view(shape).clone(),
                        "exp_avg_sq": v[lo:lo + n].view(shape).clone()}
        sd = {"state": state,
              "param_groups": [{"lr": self.lr, "betas": self.betas, "eps": self.eps, "weight_decay": self.wd,
                                "step": adam_step, "params": list(range(n_all))}]}
        if self._tunes():
            sd["ect"] = {"origin": self.ect_origin, "stage_steps": self.loss_fn.stage_steps}
        if self.phema_emas:
            sd["phema"] = {"sigma_rels": list(self.phema_sigma_rels), "gammas": list(self.phema_gammas),
                           "origin": self.phema_origin, "steps": self.phema_steps,
                           "emas": [self._full(e) for e in self.phema_emas]}
        return sd

    def load_state_dict(self, sd):
        """Accepts (a) this class's own layout, (b) `torch.optim.AdamW(model.parameters()).state_dict()`, (c) apex
        FusedAdam's (same indexing, `step` only in the param_group) and (d) round-1 checkpoints of this repo (compact
        indices over the trainable parameters + `param_names`).  Under `shard_optimizer` a rank keeps the part of
        the (full-layout) state inside its pieces, so states move between world sizes and between sharded and
        replicated runs."""
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
            self._keep(self.m, lo, e["exp_avg"].reshape(-1).to(self.m.device))
            self._keep(self.v, lo, e["exp_avg_sq"].reshape(-1).to(self.v.device))
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
            if src.numel() != self.st.n_train:
                raise ValueError(f"post-hoc EMA profile of {src.numel()} elements, the model trains "
                                 f"{self.st.n_train}")
            self._keep(e, 0, src.reshape(-1).to(e.device))
        self.phema_origin, self.phema_steps = int(ph["origin"]), int(ph["steps"])

    # -- power-function EMA profiles (post-hoc EMA) ----------------------------------------------------------------
    def phema_state_dicts(self):
        """The profiles as model state dicts with the module's keys (host copies; frozen tensors from the weights).  A
        collective under sharding."""
        out = []
        for e in self.phema_emas:
            flat = self._full(e)   # one host storage per profile; the trainable tensors are views into it
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
        the run step of the last update and each ema a state dict.  A collective under sharding, with the replicated
        run's layout and values."""
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
        if self._sh is not None:
            return (f"sharded optimizer state (rank {self.rank} of {self.world}): {self.grad_dtype} reduce-scatter of "
                    f"the flat gradient buffer in {len(self._sh.bounds)} chunks on a side stream, the optimizer on "
                    f"this rank's piece of each chunk, then an all-gather of the bf16 shadow and one of the fp32-read "
                    f"set, own NCCL communicator behind the C ABI (mdt_reduce_scatter_grads, mdt_allgather)")
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

    def _step_range(self, lo, hi, g=None, s=None):
        """The optimizer pass over weights [lo, hi): gradient `g` (default: the range of the summed buffer), moments
        and profiles from element `s` of the local state (default lo: the whole state is local)."""
        st, n = self.st, hi - lo
        if n <= 0:
            return
        if g is None:
            g = self.g16[lo:hi] if (self.g16 is not None and self.world > 1) else st.grad[lo:hi]
        s = lo if s is None else s
        m, v = self.m[s:s + n], self.v[s:s + n]
        ema = self.ema_st.w32[lo:hi] if self.ema_st is not None else None
        # a finite clipping bound: the optimizer reads the coefficient (c = inf keeps the plain kernels)
        coef = self._gn[1:] if self._clips() else None
        if self._flag is not None:   # Adam's step number comes from the device counter, the skip from the flag
            ops.adamw_ema_guarded(st.w32[lo:hi], g, m, v, ema, st.w16[lo:hi], n, self._lr_now,
                                  self._flag, self._counts, self.betas[0], self.betas[1], self.eps, self.wd,
                                  self.ema_decay, self._grad_scale, coef=coef)
        else:
            ops.adamw_ema(st.w32[lo:hi], g, m, v, ema, st.w16[lo:hi], n, self._lr_now,
                          self.step_count, self.betas[0], self.betas[1], self.eps, self.wd, self.ema_decay,
                          self._grad_scale, coef=coef)
        if self.phema_emas:   # the profiles follow the range's new (or, skipped, unchanged) weights on the same stream
            ops.power_ema(st.w32[lo:hi], [e[s:s + n] for e in self.phema_emas], self._phema_c)

    def _sharded_exchange_step(self, guard, measure):
        """Reduce-scatter -> optimizer on the owned pieces -> all-gather, chunk by chunk.  Every collective runs on the
        exchange stream in the same order on every rank; the optimizer pass of chunk k runs on the main stream while
        chunk k+1 is on the wire, and the shadow of chunk k is gathered while chunk k+1 is stepped."""
        st, sh, W, r = self.st, self._sh, self.world, self.rank
        main = torch.cuda.current_stream()
        if self.side is None:
            self.side = torch.cuda.Stream(device=st.grad.device)
        self.side.wait_stream(main)
        evs = []
        with torch.cuda.stream(self.side):
            cast_first = guard and self.xbuf.dtype == torch.bfloat16
            if guard:   # chunk 0's optimizer pass needs the decision: check every local chunk first
                if cast_first:
                    for k in range(len(sh.bounds)):
                        self._fill_x(k)
                else:
                    ops.nonfinite_check(st.grad[:st.n_train], self._flag)
                self._all_reduce(self._flag)
            for k in range(len(sh.bounds)):
                x = self._xchunk(k) if cast_first else self._fill_x(k)
                self.comm.reduce_scatter(x, sh.pieces[k])
                ev = torch.cuda.Event()
                ev.record(self.side)
                evs.append(ev)
                if measure:   # this rank's sum of squares of the chunk, then every rank's, in (chunk, rank) order
                    slot = self._gn_slots[k * W + r:k * W + r + 1]
                    g = self._own_grad(k)
                    if g.numel():
                        ops.grad_sumsq(g, slot, self._gn_scratch)
                    else:
                        slot.zero_()
                    self.comm.all_gather(self._gn_slots[k * W:(k + 1) * W], 1)
            if measure:
                self._grad_norm_coef(len(sh.bounds) * W)
        if self._clips():   # clipping needs the global norm: every chunk's pass waits for the coefficient
            main.wait_stream(self.side)
            evs = [None] * len(sh.bounds)
        stepped = []
        for k, ev in enumerate(evs):
            if ev is not None:
                main.wait_event(ev)
            self._step_piece(k)
            done = torch.cuda.Event()
            done.record(main)
            stepped.append(done)
        with torch.cuda.stream(self.side):
            for k, done in enumerate(stepped):
                self.side.wait_event(done)
                self._gather_w16(k)
            # the masters the step reads in fp32, from every rank's pieces
            ops.copy_segments_f32(st.w32, self._rset, sh.pack)
            self.comm.all_gather(self._rset, sh.rset_piece)
            ops.copy_segments_f32(self._rset, st.w32, sh.unpack)
        main.wait_stream(self.side)

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

    def _splits_loss(self):
        """Whether the objective the gradient follows differs from the plain loss: a learned loss weighting, or model
        guidance."""
        return bool(self.net.logvar_channels) or isinstance(self.loss_fn, MGLoss)

    def _last_edm_loss(self):
        """The plain loss of the last loss call when the objective differs from it (`_splits_loss`), else None."""
        return self.loss_fn.last_edm_loss.detach() if self._splits_loss() else None

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
        With an `MGLoss` (model guidance) the returned tensor is the MG objective and `edm_loss` the plain EDM or flow
        loss against the unguided target.
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
            edm_loss = torch.cat(edm) if self._splits_loss() else loss
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
        elif self._sh is not None:
            self._sharded_exchange_step(guard, measure)
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
