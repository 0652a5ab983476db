// Internal declarations shared by gemm_wgmma.cu and api.cu.
#pragma once
#include <cuda_runtime.h>

#include "../../include/maskdit_b200.h"

namespace mdt {

enum { EPI_STORE = MDT_EPI_STORE, EPI_GELU = MDT_EPI_GELU, EPI_GATE_RESID = MDT_EPI_GATE_RESID,
       EPI_DGELU = MDT_EPI_DGELU, EPI_ATOMIC = MDT_EPI_ATOMIC };
enum { ACT_NONE = MDT_ACT_NONE, ACT_SILU = MDT_ACT_SILU };

struct GemmParams {
  int M, N, K;
  int epi, act;
  int num_m_tiles, num_n_tiles, num_kb;
  int streamk;
  int narrow_last;  // 1: the last column tile runs at half width (<= BLOCK_N/2 columns remain) - see UnitSched
  int pair_halves;  // 1: m-major tile order, the half tiles of two adjacent m-panels form one unit - see UnitSched
  void* out;
  int ldo, out_fp32;
  const float* bias;
  void* aux;
  int ld_aux;
  const float* resid;
  int ld_resid;
  const float* gate;
  int ld_gate, rows_per_group;
  float* colsum;
};

int gemm_launch(const mdt_gemm_args& a, cudaStream_t stream);

// Host-side decisions of one launch (tile width, CTAs per tile, k-slices, unit order, grid) - what mdt_gemm_plan reports.
struct GemmPlan {
  int block_n, cg, splits, pair_halves, narrow_last, num_m_tiles, num_n_tiles, num_kb;
  long long units;
  int grid;
};
int gemm_plan(const mdt_gemm_args& a, GemmPlan* out);

// Tensor map of one head's columns in a token-major bf16 matrix [rows, heads * dh]: the 3-D tensor {dh, heads, rows};
// a box {64, 1, 64} lands in smem as 64 rows x 128 B, SWIZZLE_128B, columns >= dh zero-filled.  `m` is a CUtensorMap
// (opaque here to keep cuda.h out of this header).
int make_head_tile_tmap(void* m, const void* ptr, unsigned long long dh, unsigned long long heads,
                        unsigned long long rows);

}  // namespace mdt
