"""Host-side test of the persistent GEMM's work-unit order: the header the kernel includes
(`maskdit_b200/csrc/unit_sched.h`) is compiled with g++ and walked for every CTA group.

Checks: every (k-slice, m, n) tile is produced exactly once, and identically by every CTA of a group when a tile is
shared (cg = 2, kept as a property of the scheduler; the shipped kernel runs cg = 1); for the N = 1152 GEMMs of the
XL/2 encoder (4.5 column tiles of 256) the paired order has the same makespan as LPT while an m-panel's column tiles
stay within adjacent waves (L2 locality of the A panel), both in the shipped H100 geometry (256 row tiles of 128 on
132 CTAs) and in a 2-CTA one (128 row tiles of 256 on 74 CTA pairs).
"""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("needs g++ and the CUDA headers (gemm.h includes cuda_runtime.h)")
    exe = str(tmp_path_factory.mktemp("usc") / "unit_sched_check")
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "maskdit_b200", "csrc"),
                    "-I", "/usr/local/cuda/include", os.path.join(ROOT, "tests", "host", "unit_sched_check.cpp"),
                    "-o", exe], check=True)

    def run(mt, nt, kb, splits, narrow, pair, grid, cg):
        r = subprocess.run([exe] + [str(v) for v in (mt, nt, kb, splits, narrow, pair, grid, cg)],
                           capture_output=True, text=True)
        f = r.stdout.split()
        assert r.returncode == 0 and f[0] == "covered" and f[1] == "1", (r.returncode, r.stdout, r.stderr)
        return {"units": int(f[3]), "makespan": float(f[5]), "min": float(f[7]), "gap": int(f[9])}
    return run


def test_encoder_n1152_orders_h100(checker):
    # the shipped launch: M = 32768 (256 row tiles of 128), N = 1152 (4 full + 1 half column tile), K = 4608, 132 CTAs
    lpt = checker(256, 5, 72, 1, 1, 0, 132, 1)
    paired = checker(256, 5, 72, 1, 1, 1, 132, 1)
    assert lpt["makespan"] == paired["makespan"]                 # 1152 units of work on 132 CTAs
    assert paired["makespan"] <= 2 * (256 * 4.5 / 132 + 1) + 1e-9  # within one full tile of the ideal share
    assert lpt["gap"] >= 7 and paired["gap"] <= 1               # LPT revisits every A panel at the very end


def test_encoder_n1152_orders(checker):
    # M = 32768 (128 row tiles of 256), N = 1152 (4 full + 1 half column tile), K = 4608, 74 CTA pairs
    lpt = checker(128, 5, 72, 1, 1, 0, 148, 2)
    paired = checker(128, 5, 72, 1, 1, 1, 148, 2)
    assert lpt["makespan"] == paired["makespan"] == 16.0        # 8 full tile-times (7.78 of work)
    assert lpt["gap"] >= 7 and paired["gap"] <= 1               # LPT revisits every A panel at the very end
    plain = checker(128, 5, 72, 1, 0, 0, 148, 2)                # (narrow_last off: every tile counted full width)
    assert plain["units"] == 640


@pytest.mark.parametrize("mt,nt", [(1, 5), (2, 5), (3, 2), (7, 3), (129, 5), (64, 2), (255, 9)])
@pytest.mark.parametrize("grid,cg", [(148, 2), (148, 1), (4, 2), (6, 1), (132, 1)])
def test_paired_order_covers_every_tile(checker, mt, nt, grid, cg):
    r = checker(mt, nt, 18, 1, 1, 1, grid, cg)
    groups = grid // cg
    # a panel pair's 2 (nt - 1) + 1 units are consecutive: they span that many units' worth of waves, no more
    assert r["units"] == mt * nt and r["gap"] <= (2 * nt - 1 + groups - 1) // groups + 1
    # balance: no group carries more than one full tile over the ideal share
    ideal = (2 * mt * (nt - 1) + mt) / groups
    assert r["makespan"] <= ideal + 2.0 + 1e-9


@pytest.mark.parametrize("splits", [1, 2, 3, 6, 16])
@pytest.mark.parametrize("narrow,pair", [(0, 0), (1, 0), (1, 1)])
def test_k_slices_tile_the_k_range(checker, splits, narrow, pair):
    r = checker(5, 5, 512, splits, narrow, pair, 148, 2)
    assert r["units"] == 25 * splits
