#!/usr/bin/env python
"""Benchmark of the MaskDiT hot path on H100 (one JSON line on rank 0).

  python bench.py --gpus N --steps K --warmup W                 # GPU arm: MaskDiT-XL/2 ImageNet-256 train step
  python bench.py --impl reference --gpus N --steps K --warmup W  # reference arm: the CPU oracle port of the same workload
  python bench.py --workload sampler                            # EDM sampler, 18 steps, CFG 1.5, batch 64

A "step" = EDMLoss forward + hand-written backward + (N>1: one NCCL all-reduce of the flat fp32 gradient) +
fused AdamW + EMA, on synthetic latents of BASELINE.json's shape with random-init XL/2 weights (the reference's
zero-initialised tensors are randomised, SURVEY.md §3.3 — otherwise the net is the identity).
`value`  : samples/s, inputs resident in HBM.      `e2e.value`: same, inputs copied from pinned host memory
every step and the loss read back to the host every step.
`--dump-outputs DIR`: after the timed steps, what the last timed step computed is written as DIR/<name>.npy, so that
two builds can be compared output for output on identical inputs: for training the per-sample loss and a fixed, seeded
sample of the trained and EMA weights it left behind (float32); for `--workload sampler` the sampled latents (float64).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FLOP_PER_SAMPLE = {256: 392.72e9, 512: 1680.98e9}   # SURVEY.md §8(d): 3 x forward matmul FLOPs, no recompute
SAMPLER_FLOP_PER_IMAGE = 17.608e12                   # 251.55 GF x 2 (CFG) x 35 evals


def peaks():
    try:
        p = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return dict(burst=p["bf16_tflops"], sustained=p["bf16_tflops_sustained"], hbm=p["hbm_gbs"], src="measured")
    except Exception:
        # H100 SXM data sheet (dense bf16, HBM3 at 700 W): a reference point, not a measured rate
        return dict(burst=989.0, sustained=989.0, hbm=3350.0, src="H100 SXM data sheet")


class ClockSampler:
    """nvidia-smi sampling DURING the timed region (profiling guide's clocks line)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx, self.proc, self.path = gpu_index, None, f"/tmp/mdt_clocks_{os.getpid()}.csv"

    def start(self):
        try:
            self.f = open(self.path, "w")
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "200", "-i", str(self.idx)], stdout=self.f,
                                         stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(5)
        except Exception:
            self.proc.kill()
        self.f.close()
        sm, mx, reasons = [], [], set()
        for line in open(self.path):
            c = [x.strip() for x in line.split(",")]
            if len(c) < 8:
                continue
            try:
                sm.append(float(c[1])), mx.append(float(c[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), c[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no samples"]}
        busy = [x for x in sm if x > 0]
        return {"sm_mhz": statistics.median(busy), "sm_max_mhz": max(mx), "reasons": sorted(reasons),
                "samples": len(sm)}


def randomise_zero_init(net, seed=1):
    """SURVEY §8(d): overwrite the adaLN-Zero / zero-init tensors with N(0, 0.02) so every block is active."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k, p in net.named_parameters():
            if p.requires_grad and float(p.abs().sum()) == 0.0:
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)


def make_batches(n, B, R, ncls, seed=0):
    """Synthetic latents ~ N(0, sigma_data^2) and one-hot labels with 10 % dropped rows (train.py:209), pinned."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        x = (torch.randn(B, 4, R, R, generator=g) * 0.5).pin_memory()
        y = torch.nn.functional.one_hot(torch.randint(0, ncls, (B,), generator=g), ncls).float()
        y = (y * (torch.rand(B, 1, generator=g) >= 0.1)).pin_memory()
        out.append((x, y))
    return out


# ---------------------------------------------------------------------------------------------------------------
def pin_to_one_socket():
    """CPU baseline stability (VERDICT r1: the CPU arm moved 13x between runs): bind this process to the physical cores
    of socket 0 (one hardware thread per core) and size torch's pool to match.  Returns (threads, description)."""
    try:
        cores = {}
        for c in sorted(os.sched_getaffinity(0)):
            base = f"/sys/devices/system/cpu/cpu{c}/topology/"
            pkg = int(open(base + "physical_package_id").read())
            core = int(open(base + "core_id").read())
            cores.setdefault(pkg, {}).setdefault(core, c)     # first hardware thread of every physical core
        pkg0 = min(cores)
        cpus = sorted(cores[pkg0].values())
        os.sched_setaffinity(0, cpus)
        torch.set_num_threads(len(cpus))
        return len(cpus), f"pinned to the {len(cpus)} physical cores of socket {pkg0} (of {len(cores)} sockets)"
    except Exception as e:  # no sysfs topology: leave the affinity alone
        return torch.get_num_threads(), f"unpinned ({type(e).__name__})"


def cpu_reference_train(B, steps, warmup, R=32):
    """The reference's algorithm on the host CPU (oracle port, fp32, AdamW(wd=0)): samples/s.  Checker code timed as a
    BASELINE only — never on the product path.  SURVEY 8(d): full train step at B=8, 1 warm-up + 3 timed."""
    from oracle import maskdit_oracle as O
    cfg = O.Cfg(model_type="DiT-XL/2", img_resolution=R, num_classes=1000)
    sd = {k: v.requires_grad_(not k.endswith("pos_embed")) for k, v in O.make_state_dict(cfg, 1).items()}
    m = {k: torch.zeros_like(v) for k, v in sd.items() if v.requires_grad}
    v2 = {k: torch.zeros_like(v) for k, v in sd.items() if v.requires_grad}
    g = torch.Generator().manual_seed(0)
    times = []
    for it in range(warmup + steps):
        x = torch.randn(B, 4, R, R, generator=g) * 0.5
        y = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float()
        t0 = time.perf_counter()
        md = O.mask_from_noise(torch.rand(B, cfg.num_patches, generator=g), 0.5)
        loss, _ = O.edm_loss(sd, cfg, x, y, torch.randn(B, 1, 1, 1, generator=g), torch.randn(x.shape, generator=g),
                             md, 0.1)
        loss.mean().backward()
        with torch.no_grad():
            for k in m:
                O.adamw_ema_step(sd[k], sd[k].grad, m[k], v2[k], None, it + 1)
                sd[k].grad = None
        if it >= warmup:
            times.append(time.perf_counter() - t0)
    return B * len(times) / sum(times), sum(times)


def cpu_reference_eval(R=32):
    """SURVEY 8(d) (i) config 1: XL/2 masked forward at B=2, fp32; (iii) sampler at B=2, CFG 1.5: three network
    evaluations are timed and scaled to the 35 of an 18-step run (the sampler is 35 identical evaluations + axpys)."""
    from oracle import maskdit_oracle as O
    cfg = O.Cfg(model_type="DiT-XL/2", img_resolution=R, num_classes=1000)
    sd = O.make_state_dict(cfg, 1)
    g = torch.Generator().manual_seed(0)
    B = 2
    x = torch.randn(B, 4, R, R, generator=g) * 0.5
    y = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float()
    md = O.mask_from_noise(torch.rand(B, cfg.num_patches, generator=g), 0.5)
    with torch.no_grad():
        O.edm_loss(sd, cfg, x, y, torch.randn(B, 1, 1, 1, generator=g), torch.randn(x.shape, generator=g), md, 0.1)
        t0 = time.perf_counter()
        for _ in range(2):
            O.edm_loss(sd, cfg, x, y, torch.randn(B, 1, 1, 1, generator=g), torch.randn(x.shape, generator=g), md, 0.1)
        fwd = 2 * B / (time.perf_counter() - t0)
        t0 = time.perf_counter()
        for s_ in (80.0, 10.0, 0.5):
            O.edm_precond(sd, cfg, x, torch.tensor(s_, dtype=torch.float64), y, cfg_scale=1.5, training=False)
        per_eval = (time.perf_counter() - t0) / 3
    return fwd, B / (35 * per_eval)


def cpu_baseline_record(steps, warmup, R=32, B=8, extras=False):
    """CPU arm: the oracle port (oracle/maskdit_oracle.py, pinned to the unmodified reference by tests/golden)."""
    threads, how = pin_to_one_socket()
    sps, secs = cpu_reference_train(B, steps, warmup, R=R)
    extra = {}
    if extras:
        fwd, ips = cpu_reference_eval(R)
        extra = {"c1_forward_b2": {"value": fwd, "unit": "samples/s"},
                 "c5_sampler_b2_scaled": {"value": ips, "unit": "img/s",
                                          "how": "3 CFG network evaluations at B=2 timed, scaled to the 35 of an 18-step run"}}
    return sps, secs, {**extra, "value": sps, "unit": "samples/s", "cores": threads, "kind": "port", "same_config": False,
                       "sample": f"{steps} timed steps (+{warmup} warm-up) of batch {B} (SURVEY 8d), EDM loss fwd + bwd + "
                                 f"AdamW, torch CPU fp32, {threads} threads {how}; host has {os.cpu_count()} logical "
                                 f"CPUs; {secs:.1f} s timed; the oracle port, pinned to the unmodified reference by "
                                 "tests/golden"}


def run_reference_arm(args, rank):
    if rank != 0:
        return
    R = 64 if args.workload == "train512" else 32
    B = 8 if R == 32 else 2
    sps, secs, rec = cpu_baseline_record(args.steps, max(1, min(args.warmup, 2)), R=R, B=B)
    line = {"impl": "reference", "metric": "train_samples_per_sec", "value": sps, "unit": "samples/s",
            "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * secs / args.steps,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"MaskDiT-XL/2 ImageNet-{256 if R == 32 else 512} train step ({R}x{R}x4 latents, "
                                   "mask 0.5) on host CPU", "batch_per_step": B, "same_config": False},
            "cpu_baseline": rec,
            "e2e": {"value": sps, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


# ---------------------------------------------------------------------------------------------------------------
def build_xl2(R, dev):
    from maskdit_b200.maskdit import Precond_models
    torch.manual_seed(0)
    net = Precond_models["edm"](img_resolution=R, img_channels=4, num_classes=1000, model_type="DiT-XL/2",
                                use_decoder=True, mae_loss_coef=0.1, pad_cls_token=False)
    randomise_zero_init(net)
    return net.to(dev)


class Env:
    def __init__(self, dev, world, rank):
        self.dev, self.world, self.rank = dev, world, rank

    def sync_all(self):
        if self.world > 1:
            import torch.distributed as dist
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(self, ms):
        if self.world == 1:
            return ms
        import torch.distributed as dist
        t = torch.tensor([ms], device=self.dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def timed(self, fn, K):
        """K calls of fn bracketed by barrier + synchronize on both sides, CUDA events on the launching stream, max
        over ranks (ms)."""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self.sync_all()
        e0.record()
        for i in range(K):
            fn(i)
        e1.record()
        self.sync_all()
        return self.max_over_ranks(e0.elapsed_time(e1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="train256", choices=["train256", "train512", "sampler"])
    ap.add_argument("--batch-per-gpu", type=int, default=None)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the last timed step's outputs as DIR/<name>.npy (training: float32; sampler: float64 latents)")
    ap.add_argument("--no-sub", action="store_true",
                    help="skip the sub-records (BASELINE configs 3-5: 128/GPU, 64x64x4 latents, sampler)")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if args.impl == "reference":
        run_reference_arm(args, rank)
        return
    assert args.warmup >= 3, "timing rules: at least 3 warm-up steps"

    import torch.distributed as dist
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    PK = peaks()
    env = Env(dev, world, rank)

    R = 64 if args.workload == "train512" else 32
    net = build_xl2(R, dev)
    if args.workload == "sampler":
        line = bench_sampler(args, net, env, PK)
    else:
        line = bench_train(args, net, env, R, PK, args.batch_per_gpu or (256 if R == 32 else 64), args.steps,
                           args.warmup, full=True)
        if args.workload == "train256" and not args.no_sub and args.batch_per_gpu is None:
            # BASELINE.json configs 3, 4, 5 next to the headline (config 2), same process, same box, same clocks
            # (a sub-record that fails - symmetrically on every rank, e.g. out of memory - must not cost the headline)
            sub = {}

            def guarded(name, fn):
                try:
                    sub[name] = fn()
                except Exception as e:  # noqa: BLE001
                    sub[name] = {"error": f"{type(e).__name__}: {e}"[:300]}
                    torch.cuda.empty_cache()

            guarded("c3_global1024_at_8gpu",
                    lambda: bench_train(args, net, env, 32, PK, 128, max(5, args.steps // 2), 3, full=False))
            guarded("c5_sampler", lambda: bench_sampler(args, net, env, PK, iters=2, warm=1))
            del net
            torch.cuda.empty_cache()

            def c4():
                net64 = None
                try:
                    net64 = build_xl2(64, dev)
                    # batch 64: the largest the 80 GB of an H100 holds at 512 px (batch 128 needs a 108 GB workspace)
                    return bench_train(args, net64, env, 64, PK, 64, max(4, args.steps // 4), 3, full=False)
                finally:
                    net64 = None
                    torch.cuda.empty_cache()

            guarded("c4_512px", c4)
            line["sub"] = sub
        if world > 1 and not args.no_sub and args.workload == "train256" and args.batch_per_gpu is None:
            # the same step with the fp32 gradient exchange (DDP's arithmetic) next to the default bf16 exchange buffer
            os.environ["MDT_GRAD_AR"] = "fp32"
            try:
                net2 = build_xl2(32, dev)
                line.setdefault("sub", {})["c2_fp32_grad_exchange"] = bench_train(args, net2, env, 32, PK, 256,
                                                                               max(5, args.steps // 2), 3, full=False)
                del net2
            except Exception as e:  # noqa: BLE001
                line.setdefault("sub", {})["c2_fp32_grad_exchange"] = {"error": f"{type(e).__name__}: {e}"[:300]}
            del os.environ["MDT_GRAD_AR"]
            torch.cuda.empty_cache()
        if rank == 0 and world == 1 and not args.no_cpu_baseline:
            _, _, line["cpu_baseline"] = cpu_baseline_record(3, 1, R=R, B=8 if R == 32 else 2, extras=(R == 32))
    if rank == 0:
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def bench_train(args, net, env, R, PK, B, steps, warmup, full):
    """One training-step measurement.  full=True: the headline record (resident + e2e + per-launch GEMM timing +
    clocks); full=False: a compact sub-record (resident inputs only)."""
    import copy

    from maskdit_b200 import _lib
    from maskdit_b200.train_step import TrainStep
    dev, world, rank = env.dev, env.world, env.rank
    net.train()
    ema = copy.deepcopy(net).eval()
    ts = TrainStep(net, ema, lr=1e-4, global_batch=B * world, overlap=os.environ.get("MDT_OVERLAP", "0") == "1")
    pool = make_batches(4, B, R, 1000, seed=rank)
    resident = [(x.to(dev), y.to(dev)) for x, y in pool]
    h2d = pool[0][0].numel() * 4 + pool[0][1].numel() * 4
    loss_host = torch.zeros(1).pin_memory()

    last = {}

    def step_resident(i):
        x, y = resident[i % len(resident)]
        last["loss"] = ts.step(x, y, 0.5, 0.1)
        return last["loss"]

    def step_e2e(i):
        xh, yh = pool[i % len(pool)]
        x, y = xh.to(dev, non_blocking=True), yh.to(dev, non_blocking=True)
        loss = ts.step(x, y, 0.5, 0.1)
        loss_host.copy_(loss.mean().reshape(1), non_blocking=True)   # D2H read of the step's result

    for i in range(warmup):
        step_resident(i)
    clocks = ClockSampler(torch.cuda.current_device())
    if rank == 0 and full:
        clocks.start()
    n0 = _lib.LAUNCHES
    ms = env.timed(step_resident, steps)
    launches = _lib.LAUNCHES - n0
    clk = clocks.stop() if (rank == 0 and full) else None
    if full and rank == 0 and args.dump_outputs:
        dump_outputs(args.dump_outputs, last["loss"], ts)
    ms_step = ms / steps
    sps = B * world * steps / (ms / 1e3)
    flop = FLOP_PER_SAMPLE[256 if R == 32 else 512]
    step_tf = sps / world * flop / 1e12
    workload = (f"MaskDiT-XL/2 ImageNet-{256 if R == 32 else 512} training step ({R}x{R}x4 latents, bf16 GEMM operands / "
                f"fp32 accumulate+residual, mask_ratio 0.5, EDM+MAE loss, AdamW+EMA)")
    if not full:
        rec = {"metric": "train_samples_per_sec", "value": sps, "unit": "samples/s", "n_gpus": world, "steps": steps,
               "warmup": warmup, "ms_per_step": ms_step, "gpu_launches": launches,
               "config": {"workload": workload, "batch_per_gpu": B, "global_batch": B * world,
                          "grad_allreduce": ts.describe_collective()},
               "roofline": {"bound": "tensor", "step_achieved": step_tf, "peak": PK["sustained"], "unit": "TFLOP/s",
                            "step_frac": step_tf / PK["sustained"], "peak_source": f"{PK['src']} sustained bf16"}}
        ts.close()
        del ts, ema, resident
        torch.cuda.empty_cache()
        return rec
    for i in range(2):
        step_e2e(i)
    ms_e2e = env.timed(step_e2e, steps)
    final_loss = float(loss_host.item())

    # dominant kernel (the wgmma GEMM family) timed per launch with CUDA events inside real steps: the library brackets
    # every mdt_gemm_bf16 launch - the C++ step driver's own - with an event pair on the launching stream
    # (mdt_gemm_profile_enable); three steps, per launch the median of the three.
    import ctypes
    L = _lib.lib()
    runs = []
    for i in range(3):
        L.mdt_gemm_profile_enable(1)
        step_resident(i)
        torch.cuda.synchronize()
        L.mdt_gemm_profile_enable(0)
        n = L.mdt_gemm_profile_read(None, None, 0)
        ms_buf, fl_buf = (ctypes.c_float * n)(), (ctypes.c_double * n)()
        assert L.mdt_gemm_profile_read(ms_buf, fl_buf, n) == n
        runs.append(list(zip(list(fl_buf), list(ms_buf))))
    prof = runs[0]
    assert all(len(r) == len(prof) for r in runs)
    gemm_ms = sum(sorted(r[j][1] for r in runs)[1] for j in range(len(prof)))
    gemm_flops = sum(f for f, _ in prof)
    sps_e2e = B * world * steps / (ms_e2e / 1e3)
    achieved = gemm_flops / (gemm_ms * 1e-3) / 1e12 if gemm_ms > 0 else 0.0
    line = {
        "metric": "train_samples_per_sec", "value": sps, "unit": "samples/s", "n_gpus": world, "steps": steps,
        "warmup": warmup, "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": {"workload": workload, "batch_per_gpu": B, "global_batch": B * world, "parallelism": f"dp{world}",
                   "grad_allreduce": ts.describe_collective(),
                   "l2_policy": "per-step working set (activations > 40 GB) far exceeds the 50 MB L2; no flush needed",
                   "final_loss": final_loss},
        "clocks": clk,
        "e2e": {"value": sps_e2e, "unit": "samples/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4},
        "gpu_launches": launches,
        "roofline": {"bound": "tensor", "kernel": "gemm_wgmma_kernel (all GEMM launches of one step)",
                     "achieved": achieved, "peak": PK["sustained"], "unit": "TFLOP/s",
                     "frac": achieved / PK["sustained"], "peak_source": f"{PK['src']} sustained bf16",
                     "traffic": None, "traffic_source": "not measured on this GPU",
                     "launches_per_step": len(prof), "share_of_step": gemm_ms / ms_step,
                     "step_achieved": step_tf, "step_frac": step_tf / PK["sustained"]},
    }
    ts.close()
    del ts, ema, resident
    torch.cuda.empty_cache()
    return line


def dump_outputs(out_dir, loss, ts, n_sample=1 << 20, seed=0):
    """What the timed training step hands back: the per-sample loss, plus the weights and EMA weights it updated
    (a fixed seeded sample of n_sample entries of each flat fp32 store; 8 MB in all at the default)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    np.save(os.path.join(out_dir, "loss.npy"), loss.float().cpu().numpy())
    n = ts.st.n_train
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, n, (min(n_sample, n),), generator=g).to(ts.st.w32.device)
    np.save(os.path.join(out_dir, "weights_sample.npy"), ts.st.w32[:n][idx].float().cpu().numpy())
    if ts.ema_st is not None:
        np.save(os.path.join(out_dir, "ema_weights_sample.npy"), ts.ema_st.w32[:n][idx].float().cpu().numpy())


def bench_sampler(args, net, env, PK, iters=None, warm=None):
    from maskdit_b200 import _lib
    from maskdit_b200.sampler import edm_sampler
    dev, world, rank = env.dev, env.world, env.rank
    B = (args.batch_per_gpu if args.workload == "sampler" else None) or 64
    net.eval()
    g = torch.Generator().manual_seed(rank)
    lat_h = torch.randn(B, 4, 32, 32, generator=g).pin_memory()
    lab_h = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float().pin_memory()
    out_h = torch.zeros(B, 4, 32, 32, dtype=torch.float64).pin_memory()

    def run(i):
        with torch.no_grad():
            z = edm_sampler(net, lat_h.to(dev, non_blocking=True), lab_h.to(dev, non_blocking=True), cfg_scale=1.5,
                            num_steps=18)
            out_h.copy_(z, non_blocking=True)

    W = warm if warm is not None else max(1, args.warmup // 3)
    for i in range(W):
        run(i)
    K = iters if iters is not None else max(1, args.steps // 5)
    clocks = ClockSampler(torch.cuda.current_device())
    if rank == 0:
        clocks.start()
    n0 = _lib.LAUNCHES
    ms = env.timed(run, K)
    if args.dump_outputs and args.workload == "sampler" and rank == 0:  # the sampled latents of the last timed run
        import numpy as np
        os.makedirs(args.dump_outputs, exist_ok=True)
        torch.cuda.synchronize()
        np.save(os.path.join(args.dump_outputs, "latents.npy"), out_h.numpy())
    ips = B * world * K / (ms / 1e3)
    ach = ips / world * SAMPLER_FLOP_PER_IMAGE / 1e12
    return {"metric": "edm_sampler_imgs_per_sec", "value": ips, "unit": "img/s", "n_gpus": world, "steps": K,
            "warmup": W, "ms_per_step": ms / K, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": "EDM sampler 18 steps (35 net evals), CFG 1.5, 32x32x4 latents, MaskDiT-XL/2",
                       "batch_per_gpu": B, "parallelism": f"replicas x{world}"},
            "clocks": clocks.stop() if rank == 0 else None,
            "e2e": {"value": ips, "unit": "img/s", "h2d_bytes_per_step": lat_h.numel() * 4 + lab_h.numel() * 4,
                    "d2h_bytes_per_step": out_h.numel() * 8},
            "gpu_launches": _lib.LAUNCHES - n0,
            "roofline": {"bound": "tensor", "achieved": ach, "peak": PK["sustained"], "unit": "TFLOP/s",
                         "frac": ach / PK["sustained"], "peak_source": f"{PK['src']} sustained bf16",
                         "traffic": None}}


if __name__ == "__main__":
    main()
