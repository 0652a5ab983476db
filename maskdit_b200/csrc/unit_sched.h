// Work-unit order of the persistent GEMM (gemm_wgmma.cu).  Plain C++ so that the host-side test
// (tests/test_unit_sched.py) compiles the very same code with g++ and checks coverage and balance.
#pragma once
#include "gemm.h"

#if defined(__CUDACC__)
#define MDT_HD __host__ __device__ __forceinline__
#else
#define MDT_HD inline
#endif

namespace mdt {

// Units (tiles x k-slices) the launch is cut into for a given GemmParams (host side: grid size, slice heuristic).
MDT_HD long long gemm_units_per_slice(const GemmParams& p) {
  const long long tiles = static_cast<long long>(p.num_m_tiles) * p.num_n_tiles;
  if (!(p.narrow_last && p.pair_halves)) return tiles;
  const int n_full = p.num_n_tiles - 1;
  return static_cast<long long>(p.num_m_tiles / 2) * (2 * n_full + 1) + ((p.num_m_tiles & 1) ? n_full + 1 : 0);
}

struct UnitSched {
  // Iterates the work units of this CTA group; identical sequence in every warp role (and in both CTAs of a pair).
  // Units are (k-slice, tile) pairs in SLICE-major order, dealt round-robin to the groups: at any moment the resident
  // groups work on the same k-slice of different tiles, so A/B panels are shared through L2 exactly as in a plain
  // tiled GEMM (a tile-major stream-K order made the wgrad GEMMs DRAM-bound: every unit streamed private panels).
  // splits == 1 is the ordinary persistent tile loop.
  // Tile order inside a slice: when the last column tile is a half-width one (N = 1152 = 4.5 x 256: every N = 1152
  // GEMM of the encoder, 58 % of the GEMM flops) the full-width tiles are dealt first and the half-cost tiles last,
  // continuing the same round robin - longest-processing-time-first.  With the plain (m, n) order a CTA pair's 8-9
  // tiles contained 1-2 half tiles at random and the makespan was 8.5 tile-times for 7.78 of work (ncu launch list r01:
  // fc2 263 us vs 240 us for the same-flop fc1 dgrad); now it is 8.0.
  // Paired order (p.pair_halves, used for the non-accumulating epilogues): LPT leaves ALL half-width tiles for the end
  // of the launch, when the A panels they need (the whole activation matrix: 226-302 MB for the K = 3456 / 4608
  // GEMMs) have long left the L2 (the fc2 forward then reads its A panels from DRAM more than once), and
  // the tail (74 pairs, each streaming a private 256-row A panel for half a tile-time of MMAs) is DRAM-bound.  Here
  // the tiles stay in m-major order and the two half tiles of an m-panel PAIR form one unit (walked back to back by the
  // same CTA group): every unit costs one full tile-time again (makespan 8.0 for N = 1152, as with LPT) and a panel's
  // 4.5 column tiles run in the same wave, so A is read from DRAM once.
  int num_kb, num_tiles, num_n_tiles, num_m_tiles, splits, grid, n_full, full_count;
  int pair, grp_units, num_groups, units_per_slice;
  bool pending;
  int unit, num_units;
  int cur_tile, cur_m, cur_n, kb0, kb1;
  MDT_HD void init(const GemmParams& p, int cg, int grid_dim, int block_idx) {
    num_kb = p.num_kb;
    num_n_tiles = p.num_n_tiles;
    num_m_tiles = p.num_m_tiles;
    num_tiles = p.num_m_tiles * p.num_n_tiles;
    splits = p.streamk;  // number of k-slices (>= 1)
    n_full = p.narrow_last ? p.num_n_tiles - 1 : p.num_n_tiles;
    full_count = p.num_m_tiles * n_full;
    pair = p.narrow_last && p.pair_halves;
    grp_units = 2 * n_full + 1;
    num_groups = p.num_m_tiles >> 1;
    units_per_slice = pair ? num_groups * grp_units + ((p.num_m_tiles & 1) ? n_full + 1 : 0) : num_tiles;
    num_units = units_per_slice * splits;
    pending = false;
    grid = grid_dim / cg;
    unit = block_idx / cg;
  }
  MDT_HD bool next() {
    if (pending) {  // second half tile of a paired unit: next m-panel, same (last) column tile, same k range
      pending = false;
      ++cur_m;
      return true;
    }
    if (unit >= num_units) return false;
    const int slice = unit / units_per_slice;
    cur_tile = unit - slice * units_per_slice;
    if (pair) {
      const int g = cur_tile / grp_units, r = cur_tile - g * grp_units;
      if (g < num_groups) {
        if (r < 2 * n_full) {
          const int dm = r >= n_full ? 1 : 0;
          cur_m = 2 * g + dm, cur_n = r - dm * n_full;
        } else {
          cur_m = 2 * g, cur_n = n_full, pending = true;
        }
      } else {  // odd panel left over: its full tiles, then its single half tile
        cur_m = num_m_tiles - 1, cur_n = r;
      }
    } else if (cur_tile < full_count) {
      cur_m = cur_tile / n_full, cur_n = cur_tile - cur_m * n_full;
    } else {
      cur_m = cur_tile - full_count, cur_n = n_full;
    }
    kb0 = static_cast<int>(static_cast<long long>(num_kb) * slice / splits);
    kb1 = static_cast<int>(static_cast<long long>(num_kb) * (slice + 1) / splits);
    unit += grid;
    return true;
  }
  MDT_HD int m_tile() const { return cur_m; }
  MDT_HD int n_tile() const { return cur_n; }
};

}  // namespace mdt
