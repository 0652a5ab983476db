#!/usr/bin/env python
"""Every distinct GEMM of the MaskDiT-XL/2 ImageNet-256 training step (batch 256, mask ratio 0.5), timed on its own.

    python tools/gemm_step_shapes.py [--iters 10] [--warmup 3] [--dump DIR] [--only NAME,...]

The shapes, operand majors, epilogues and gate groups are those `block_fwd` / `block_bwd` and the step's embedding,
adaLN, decoder-layer and final-layer GEMMs launch (csrc/driver.cu), with the count of launches per step.  Each one
runs through `_lib.gemm` on seeded inputs and is timed with CUDA events over `--iters` launches after `--warmup`.
One JSON line per shape: time, TFLOP/s, epilogue bytes/s, the shape's share of the step's GEMM FLOPs, and the card's
name, power limit and max SM clock, read in the same run.  `--dump DIR` writes each non-accumulating shape's outputs
(out, aux, colsum) as .npy after one launch on fresh buffers, for a bit-for-bit comparison of two builds
(MDT_LIB_PATH selects the library).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from maskdit_b200 import _lib  # noqa: E402
from maskdit_b200._lib import EPI_ATOMIC, EPI_DGELU, EPI_GATE_RESID, EPI_GELU, EPI_STORE  # noqa: E402

B, D, H4, DEPTH, Dd, H4d, DDEPTH, NCLS, PD = 256, 1152, 4608, 28, 512, 2048, 8, 1000, 16
T, L = 128, 256                                      # kept tokens (mask 0.5), decoder tokens
ME, MD = B * T, B * L
NA = DEPTH * 6 * D + 2 * D + DDEPTH * 6 * Dd + 2 * Dd  # adaLN modulation width of all blocks


def step_shapes():
    """(name, count per step, M, N, K, a_mn, b_mn, epi, out fp32, bias, resid, rows_per_group)."""
    s = []
    for tag, M, d, h4, t, n in (("enc", ME, D, H4, T, DEPTH), ("dec", MD, Dd, H4d, L, DDEPTH)):
        s += [
            (f"{tag}.qkv.fwd", n, M, 3 * d, d, 0, 0, EPI_STORE, 0, 1, 0, 1),
            (f"{tag}.proj.fwd", n, M, d, d, 0, 0, EPI_GATE_RESID, 1, 1, 1, t),
            (f"{tag}.fc1.fwd", n, M, h4, d, 0, 0, EPI_GELU, 0, 1, 0, 1),
            (f"{tag}.fc2.fwd", n, M, d, h4, 0, 0, EPI_GATE_RESID, 1, 1, 1, t),
            (f"{tag}.fc2.dgrad", n, M, h4, d, 0, 1, EPI_DGELU, 0, 0, 0, 1),
            (f"{tag}.fc2.wgrad", n, d, h4, M, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
            (f"{tag}.fc1.dgrad", n, M, d, h4, 0, 1, EPI_STORE, 0, 0, 0, 1),
            (f"{tag}.fc1.wgrad", n, h4, d, M, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
            (f"{tag}.proj.dgrad", n, M, d, d, 0, 1, EPI_STORE, 0, 0, 0, 1),
            (f"{tag}.proj.wgrad", n, d, d, M, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
            (f"{tag}.qkv.dgrad", n, M, d, 3 * d, 0, 1, EPI_STORE, 0, 0, 0, 1),
            (f"{tag}.qkv.wgrad", n, 3 * d, d, M, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
        ]
    s += [
        ("t_emb.fc0.fwd", 1, B, D, 256, 0, 0, EPI_STORE, 1, 1, 0, 1),
        ("t_emb.fc2.fwd", 1, B, D, D, 0, 0, EPI_STORE, 1, 1, 0, 1),
        ("y_emb.fwd", 1, B, D, NCLS, 0, 0, EPI_STORE, 1, 0, 1, 1),
        ("adaln.fwd", 1, B, NA, D, 0, 0, EPI_STORE, 1, 1, 0, 1),
        ("declayer.fwd", 1, ME, Dd, D, 0, 0, EPI_STORE, 1, 1, 0, 1),
        ("final.fwd", 1, MD, PD, Dd, 0, 0, EPI_STORE, 1, 1, 0, 1),
        ("final.wgrad", 1, PD, Dd, MD, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
        ("final.dgrad", 1, MD, Dd, PD, 0, 1, EPI_STORE, 0, 0, 0, 1),
        ("declayer.wgrad", 1, Dd, D, ME, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
        ("declayer.dgrad", 1, ME, D, Dd, 0, 1, EPI_STORE, 0, 0, 0, 1),
        ("adaln.wgrad", 1, NA, D, B, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
        ("adaln.dgrad", 1, B, D, NA, 0, 1, EPI_ATOMIC, 1, 0, 0, 1),
        ("y_emb.wgrad", 1, D, NCLS, B, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
        ("t_emb.fc2.wgrad", 1, D, D, B, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
        ("t_emb.fc2.dgrad", 1, B, D, D, 0, 1, EPI_ATOMIC, 1, 0, 0, 1),
        ("t_emb.fc0.wgrad", 1, D, 256, B, 1, 1, EPI_ATOMIC, 1, 0, 0, 1),
    ]
    return s


def epilogue_bytes(M, N, epi, out32, resid, splits):
    """Global bytes the epilogue moves: outputs written, operands it reads (residual, GELU pre-activation); a
    red.add counts its 4-byte payload once per k-slice.  Bias and gate rows are negligible and not counted."""
    per = {EPI_STORE: (4 if out32 else 2) + (4 if resid else 0), EPI_GELU: 4, EPI_GATE_RESID: 10, EPI_DGELU: 4,
           EPI_ATOMIC: 4 * splits}[epi]
    return float(M) * N * per


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clk = (s.strip() for s in r.stdout.strip().split(","))
    except Exception:                                   # nvidia-smi missing: the name still comes from the runtime
        name, power, clk = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "sm_clock_max": clk}


class Problem:
    """Seeded operands and fresh output buffers of one shape (layouts as the step driver passes them)."""

    def __init__(self, shape, seed):
        name, _, M, N, K, a_mn, b_mn, epi, out32, bias, resid, rpg = shape
        g = torch.Generator(device="cuda").manual_seed(seed)
        dev = "cuda"

        def rnd(*shp, scale=1.0, dtype=torch.bfloat16):
            return (torch.randn(*shp, generator=g, device=dev) * scale).to(dtype)

        self.shape = shape
        self.A = rnd(*((K, M) if a_mn else (M, K)), scale=1.0)
        self.B = rnd(*((K, N) if b_mn else (N, K)), scale=K ** -0.5)
        self.bias = rnd(N, scale=0.1, dtype=torch.float32) if bias else None
        self.resid = rnd(M, N, dtype=torch.float32) if resid else None
        ngroups = (M + rpg - 1) // rpg
        self.gate = rnd(ngroups, N, dtype=torch.float32) if epi == EPI_GATE_RESID else None
        self.aux_in = rnd(M, N) if epi == EPI_DGELU else None
        self.fresh()

    def fresh(self):
        _, _, M, N, K, a_mn, b_mn, epi, out32, *_ = self.shape
        self.out = torch.zeros(M, N, device="cuda", dtype=torch.float32 if out32 else torch.bfloat16)
        self.aux = (torch.zeros(M, N, device="cuda", dtype=torch.bfloat16) if epi in (EPI_GELU, EPI_GATE_RESID)
                    else self.aux_in)
        self.colsum = torch.zeros(N, device="cuda") if epi == EPI_DGELU else None

    def launch(self):
        _, _, M, N, K, a_mn, b_mn, epi, out32, _, _, rpg = self.shape
        _lib.gemm(self.A, self.B, M, N, K, a_mn=bool(a_mn), b_mn=bool(b_mn), epi=epi, out=self.out, bias=self.bias,
                  aux=self.aux, ld_aux=N if self.aux is not None else 0, resid=self.resid,
                  ld_resid=N if self.resid is not None else 0, gate=self.gate, ld_gate=N if self.gate is not None else 0,
                  rows_per_group=rpg, colsum=self.colsum)


def as_numpy(t):
    t = t.detach().cpu()
    return (t.view(torch.int16) if t.dtype == torch.bfloat16 else t).numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump", default=None, metavar="DIR", help="write the non-accumulating shapes' outputs here")
    ap.add_argument("--only", default=None, help="comma-separated shape names")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_step_shapes needs a CUDA device")
    info = card()
    shapes = step_shapes()
    total_flop = sum(2.0 * n * M * N * K for _, n, M, N, K, *_ in shapes)
    only = set(args.only.split(",")) if args.only else None
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
    for i, shape in enumerate(shapes):
        name, n, M, N, K, a_mn, b_mn, epi, out32, bias, resid, rpg = shape
        if only and name not in only:
            continue
        plan = _lib.gemm_plan(M, N, K, a_mn=bool(a_mn), b_mn=bool(b_mn), epi=epi)
        pr = Problem(shape, seed=1000 + i)
        if args.dump and epi != EPI_ATOMIC:
            pr.launch()
            torch.cuda.synchronize()
            np.save(os.path.join(args.dump, f"{name}.out.npy"), as_numpy(pr.out))
            if epi in (EPI_GELU, EPI_GATE_RESID):
                np.save(os.path.join(args.dump, f"{name}.aux.npy"), as_numpy(pr.aux))
            if epi == EPI_DGELU:
                np.save(os.path.join(args.dump, f"{name}.colsum.npy"), as_numpy(pr.colsum))
        for _ in range(args.warmup):
            pr.launch()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            pr.launch()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        flop = 2.0 * M * N * K
        ebytes = epilogue_bytes(M, N, epi, out32, resid, plan["splits"])
        epi_name = {EPI_STORE: "store", EPI_GELU: "gelu", EPI_GATE_RESID: "gate_resid", EPI_DGELU: "dgelu",
                    EPI_ATOMIC: "atomic"}[epi]
        rec = {"metric": "gemm_step_shape", "name": name, "per_step": n, "M": M, "N": N, "K": K,
               "a_major": "mn" if a_mn else "k", "b_major": "mn" if b_mn else "k", "epilogue": epi_name,
               "out": "f32" if out32 else "bf16", "rows_per_group": rpg, "block_n": plan["block_n"],
               "splits": plan["splits"], "ms": round(ms, 4), "tflops": round(flop / ms / 1e9, 1),
               "epilogue_gb_per_s": round(ebytes / ms / 1e6, 1), "step_ms": round(n * ms, 3),
               "flop_share": round(n * flop / total_flop, 4), **info}
        print(json.dumps(rec), flush=True)
        del pr
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
