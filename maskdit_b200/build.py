"""Build the in-tree CUDA library (`maskdit_b200/libmaskdit_b200.so`) for sm_90a (H100) with nvcc.

nvcc cross-compiles without a GPU, so this runs in the CPU container; the .so then travels to the GPU box with
the repo snapshot.  Objects are rebuilt only when a source or header is newer than the object.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libmaskdit_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hs.append(os.path.join(HERE, "..", "include", "maskdit_b200.h"))
    return max(os.path.getmtime(h) for h in hs)


def build(verbose: bool = False, force: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    hm = _headers_mtime()
    jobs = []
    objs = []
    for s in _sources():
        src = os.path.join(CSRC, s)
        obj = os.path.join(BUILD, s[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hm):
            jobs.append((src, obj))

    def run(job):
        src, obj = job
        cmd = [NVCC, *FLAGS, *os.environ.get("MDT_NVCC_EXTRA", "").split(), "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for src, r in ex.map(run, jobs):
                if verbose or r.returncode:
                    sys.stderr.write(r.stdout + r.stderr)
                if r.returncode:
                    raise RuntimeError(f"nvcc failed on {src}")
    if jobs or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [NVCC, "-shared", "-o", LIB, *objs, "-Xcompiler", "-fPIC"]  # static cudart (nvcc default)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
