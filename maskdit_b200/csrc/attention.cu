// Multi-head softmax attention core of timm Attention (reference ctor site models/maskdit.py:178), forward and
// backward, for the short sequences of MaskDiT (T = 128..1024 tokens, head_dim 72 in the encoder, 32 in the decoder).
//
//   qkv [B, T, 3, H, dh] bf16  ->  out [B, T, H*dh] bf16,  lse [B, H, T] fp32 (natural-log-sum-exp of scaled scores)
//
// The production shapes (T a multiple of 64, head_dim 32 / 64 / 72) run on the wgmma + TMA kernels of
// attention_wgmma.cu.  This file holds the dispatch and the general kernels for every other shape (odd token counts of
// class-unconditional or differently masked inputs): flash-style tiles on the warp-level tensor-core path (mma.sync
// m16n8k16 bf16, ldmatrix), fp32 online softmax.
// head_dim is zero-padded to DP (multiple of 16) in shared memory; rows are padded by 8 elements so that ldmatrix
// is bank-conflict free.
//
// Backward = two kernels with no atomics: dQ (block = 64 queries, loops over keys; also emits delta = rowsum(dO*O))
// and dK/dV (block = 64 keys, loops over queries, transposed formulation S^T = K Q^T).
#include <stdlib.h>

#include "common.cuh"
#include "../../include/maskdit_b200.h"

namespace mdt {

constexpr int kTile = 64;  // rows per block (4 warps x 16) and keys per inner chunk

MDT_DEVINL void ldsm_x4(uint32_t* r, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
MDT_DEVINL void ldsm_x4_t(uint32_t* r, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
MDT_DEVINL void mma16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int DP>
struct Tile {
  static constexpr int LD = DP + 8;  // smem row stride (elements)
  // Load `rows` rows x dh columns (bf16) from global (row stride gstride elements) into smem, zero-padding
  // columns dh..DP and rows >= valid.
  static MDT_DEVINL void load(__nv_bfloat16* s, const __nv_bfloat16* g, long long gstride, int valid, int dh) {
    constexpr int CH = DP / 8;  // 16-byte chunks per row
    for (int e = threadIdx.x; e < kTile * CH; e += blockDim.x) {
      const int r = e / CH, c = (e % CH) * 8;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (r < valid && c < dh) v = *reinterpret_cast<const uint4*>(g + r * gstride + c);
      *reinterpret_cast<uint4*>(s + r * LD + c) = v;
    }
  }
  // A fragment (16 rows x 16 k) at (row0, k0): lanes address row (lane%8)+((lane/8)%2)*8, col (lane/16)*8
  static MDT_DEVINL void lda(uint32_t* r, const __nv_bfloat16* s, int row0, int k0, int lane) {
    ldsm_x4(r, smem_u32(s + (row0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + k0 + (lane >> 4) * 8));
  }
  // B fragments for two adjacent n-tiles from an [n][k] row-major tile (n = rows): r[0],r[1] -> n-tile n0, r[2],r[3] -> n0+8
  static MDT_DEVINL void ldb_nk(uint32_t* r, const __nv_bfloat16* s, int n0, int k0, int lane) {
    ldsm_x4(r, smem_u32(s + (n0 + (lane & 7) + (lane >> 4) * 8) * LD + k0 + ((lane >> 3) & 1) * 8));
  }
  // B fragments for two adjacent n-tiles from a [k][n] row-major tile (k = rows), via transposing ldmatrix
  static MDT_DEVINL void ldb_kn(uint32_t* r, const __nv_bfloat16* s, int k0, int n0, int lane) {
    ldsm_x4_t(r, smem_u32(s + (k0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + n0 + (lane >> 4) * 8));
  }
};

MDT_DEVINL float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
MDT_DEVINL float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// S[16 x 64] = A(16 x DP, smem rows row0..) * Bt(64 x DP smem)^T
template <int DP>
MDT_DEVINL void gemm_rows_nk(float (*acc)[4], const __nv_bfloat16* sA, int row0, const __nv_bfloat16* sB, int lane) {
#pragma unroll
  for (int ks = 0; ks < DP / 16; ++ks) {
    uint32_t a[4];
    Tile<DP>::lda(a, sA, row0, ks * 16, lane);
#pragma unroll
    for (int np = 0; np < kTile / 16; ++np) {
      uint32_t b[4];
      Tile<DP>::ldb_nk(b, sB, np * 16, ks * 16, lane);
      mma16816(acc[2 * np], a, b[0], b[1]);
      mma16816(acc[2 * np + 1], a, b[2], b[3]);
    }
  }
}
// O[16 x DP] += P(16 x 64, fragments pa[4 k-slices][4]) * B(64 x DP smem, [k][n] layout)
template <int DP>
MDT_DEVINL void gemm_p_kn(float (*acc)[4], const uint32_t (*pa)[4], const __nv_bfloat16* sB, int lane) {
#pragma unroll
  for (int kk = 0; kk < kTile / 16; ++kk) {
#pragma unroll
    for (int np = 0; np < DP / 16; ++np) {
      uint32_t b[4];
      Tile<DP>::ldb_kn(b, sB, kk * 16, np * 16, lane);
      mma16816(acc[2 * np], pa[kk], b[0], b[1]);
      mma16816(acc[2 * np + 1], pa[kk], b[2], b[3]);
    }
  }
}
// C-fragment layout (16 x 64 fp32) -> A fragments (bf16) for the next matmul
MDT_DEVINL void pack_p(uint32_t (*pa)[4], const float (*s)[4]) {
#pragma unroll
  for (int kk = 0; kk < kTile / 16; ++kk) {
    pa[kk][0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
    pa[kk][1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
    pa[kk][2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
    pa[kk][3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
  }
}
// store a 16 x DP accumulator (C layout) as bf16 rows; cols >= dh and rows >= valid are dropped
template <int DP>
MDT_DEVINL void store_rows(__nv_bfloat16* g, long long gstride, const float (*acc)[4], int row0, int valid, int dh,
                           int lane, float mul0, float mul1) {
  const int r0 = row0 + (lane >> 2), r1 = r0 + 8, cq = (lane & 3) * 2;
#pragma unroll
  for (int nt = 0; nt < DP / 8; ++nt) {
    const int c = nt * 8 + cq;
    if (c < dh) {
      if (r0 < valid) *reinterpret_cast<uint32_t*>(g + r0 * gstride + c) = pack_bf16(acc[nt][0] * mul0, acc[nt][1] * mul0);
      if (r1 < valid) *reinterpret_cast<uint32_t*>(g + r1 * gstride + c) = pack_bf16(acc[nt][2] * mul1, acc[nt][3] * mul1);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------
template <int DP>
__global__ void __launch_bounds__(128)
attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
                int T, int H, int dh, float scale) {
  using TL = Tile<DP>;
  __shared__ __align__(16) __nv_bfloat16 sQ[kTile * TL::LD];
  __shared__ __align__(16) __nv_bfloat16 sK[kTile * TL::LD];
  __shared__ __align__(16) __nv_bfloat16 sV[kTile * TL::LD];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y / H, h = blockIdx.y % H;
  const int q0 = blockIdx.x * kTile;
  const long long rs = 3LL * H * dh;
  const __nv_bfloat16* base = qkv + static_cast<long long>(b) * T * rs;
  const float sl = scale * 1.4426950408889634f;

  TL::load(sQ, base + q0 * rs + h * dh, rs, T - q0, dh);
  float o[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  for (int k0 = 0; k0 < T; k0 += kTile) {
    __syncthreads();
    TL::load(sK, base + k0 * rs + (H + h) * dh, rs, T - k0, dh);
    TL::load(sV, base + k0 * rs + (2 * H + h) * dh, rs, T - k0, dh);
    __syncthreads();
    float s[kTile / 8][4];
#pragma unroll
    for (int i = 0; i < kTile / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    gemm_rows_nk<DP>(s, sQ, warp * 16, sK, lane);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < kTile / 8; ++nt) {
      const int c = k0 + nt * 8 + (lane & 3) * 2;
      if (c >= T) s[nt][0] = s[nt][2] = -INFINITY;
      if (c + 1 >= T) s[nt][1] = s[nt][3] = -INFINITY;
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    const float mn0 = fmaxf(m0, quad_max(mx0)), mn1 = fmaxf(m1, quad_max(mx1));
    const float a0 = fast_exp2((m0 - mn0) * sl), a1 = fast_exp2((m1 - mn1) * sl);
    m0 = mn0, m1 = mn1;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < kTile / 8; ++nt) {
      s[nt][0] = fast_exp2(s[nt][0] * sl - m0 * sl), s[nt][1] = fast_exp2(s[nt][1] * sl - m0 * sl);
      s[nt][2] = fast_exp2(s[nt][2] * sl - m1 * sl), s[nt][3] = fast_exp2(s[nt][3] * sl - m1 * sl);
      rs0 += s[nt][0] + s[nt][1], rs1 += s[nt][2] + s[nt][3];
    }
    l0 = l0 * a0 + rs0, l1 = l1 * a1 + rs1;
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) o[i][0] *= a0, o[i][1] *= a0, o[i][2] *= a1, o[i][3] *= a1;
    uint32_t pa[kTile / 16][4];
    pack_p(pa, s);
    gemm_p_kn<DP>(o, pa, sV, lane);
  }
  l0 = quad_sum(l0), l1 = quad_sum(l1);
  const int HD = H * dh;
  store_rows<DP>(out + (static_cast<long long>(b) * T + q0) * HD + h * dh, HD, o, warp * 16, T - q0, dh, lane,
                 1.f / l0, 1.f / l1);
  if ((lane & 3) == 0 && lse) {
    const int r0 = q0 + warp * 16 + (lane >> 2);
    float* L = lse + (static_cast<long long>(b) * H + h) * T;
    if (r0 < T) L[r0] = m0 * scale + logf(l0);
    if (r0 + 8 < T) L[r0 + 8] = m1 * scale + logf(l1);
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward: dQ (+ delta)
// ------------------------------------------------------------------------------------------------------------
template <int DP>
__global__ void __launch_bounds__(128)
attn_bwd_dq_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ out,
                   const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse,
                   __nv_bfloat16* __restrict__ dqkv, float* __restrict__ delta, int T, int H, int dh, float scale) {
  using TL = Tile<DP>;
  __shared__ __align__(16) __nv_bfloat16 sQ[kTile * TL::LD];
  __shared__ __align__(16) __nv_bfloat16 sdO[kTile * TL::LD];
  __shared__ __align__(16) __nv_bfloat16 sK[kTile * TL::LD];
  __shared__ __align__(16) __nv_bfloat16 sV[kTile * TL::LD];
  __shared__ float sDelta[kTile];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y / H, h = blockIdx.y % H;
  const int q0 = blockIdx.x * kTile;
  const long long rs = 3LL * H * dh;
  const int HD = H * dh;
  const __nv_bfloat16* base = qkv + static_cast<long long>(b) * T * rs;
  const float sl = scale * 1.4426950408889634f;

  TL::load(sQ, base + q0 * rs + h * dh, rs, T - q0, dh);
  TL::load(sdO, dout + (static_cast<long long>(b) * T + q0) * HD + h * dh, HD, T - q0, dh);
  TL::load(sK, out + (static_cast<long long>(b) * T + q0) * HD + h * dh, HD, T - q0, dh);  // O, temporarily
  __syncthreads();
  {
    const int r = threadIdx.x >> 1, half = threadIdx.x & 1;
    float acc = 0.f;
    for (int c = half * (DP / 2); c < (half + 1) * (DP / 2); ++c)
      acc += __bfloat162float(sdO[r * TL::LD + c]) * __bfloat162float(sK[r * TL::LD + c]);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (half == 0) {
      sDelta[r] = acc;
      if (q0 + r < T) delta[(static_cast<long long>(b) * H + h) * T + q0 + r] = acc;
    }
  }
  __syncthreads();
  const int r0 = warp * 16 + (lane >> 2);
  const float* L = lse + (static_cast<long long>(b) * H + h) * T;
  const float ls0 = (q0 + r0 < T) ? L[q0 + r0] * 1.4426950408889634f : 0.f;
  const float ls1 = (q0 + r0 + 8 < T) ? L[q0 + r0 + 8] * 1.4426950408889634f : 0.f;
  const float dl0 = sDelta[r0], dl1 = sDelta[r0 + 8];

  float dq[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;

  for (int k0 = 0; k0 < T; k0 += kTile) {
    __syncthreads();
    TL::load(sK, base + k0 * rs + (H + h) * dh, rs, T - k0, dh);
    TL::load(sV, base + k0 * rs + (2 * H + h) * dh, rs, T - k0, dh);
    __syncthreads();
    float s[kTile / 8][4], dp[kTile / 8][4];
#pragma unroll
    for (int i = 0; i < kTile / 8; ++i) {
      s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    }
    gemm_rows_nk<DP>(s, sQ, warp * 16, sK, lane);
    gemm_rows_nk<DP>(dp, sdO, warp * 16, sV, lane);
#pragma unroll
    for (int nt = 0; nt < kTile / 8; ++nt) {
      const int c = k0 + nt * 8 + (lane & 3) * 2;
      const float p0 = (c < T) ? fast_exp2(s[nt][0] * sl - ls0) : 0.f;
      const float p1 = (c + 1 < T) ? fast_exp2(s[nt][1] * sl - ls0) : 0.f;
      const float p2 = (c < T) ? fast_exp2(s[nt][2] * sl - ls1) : 0.f;
      const float p3 = (c + 1 < T) ? fast_exp2(s[nt][3] * sl - ls1) : 0.f;
      s[nt][0] = p0 * (dp[nt][0] - dl0) * scale, s[nt][1] = p1 * (dp[nt][1] - dl0) * scale;
      s[nt][2] = p2 * (dp[nt][2] - dl1) * scale, s[nt][3] = p3 * (dp[nt][3] - dl1) * scale;
    }
    uint32_t pa[kTile / 16][4];
    pack_p(pa, s);
    gemm_p_kn<DP>(dq, pa, sK, lane);
  }
  store_rows<DP>(dqkv + (static_cast<long long>(b) * T + q0) * rs + h * dh, rs, dq, warp * 16, T - q0, dh, lane, 1.f,
                 1.f);
}

// ------------------------------------------------------------------------------------------------------------
// backward: dK, dV  (rows = keys)
// ------------------------------------------------------------------------------------------------------------
template <int DP>
__global__ void __launch_bounds__(128)
attn_bwd_dkv_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ dout,
                    const float* __restrict__ lse, const float* __restrict__ delta,
                    __nv_bfloat16* __restrict__ dqkv, int T, int H, int dh, float scale) {
  using TL = Tile<DP>;
  __shared__ __align__(16) __nv_bfloat16 sK[kTile * TL::LD];
  __shared__ __align__(16) __nv_bfloat16 sV[kTile * TL::LD];
  __shared__ __align__(16) __nv_bfloat16 sQ[kTile * TL::LD];
  __shared__ __align__(16) __nv_bfloat16 sdO[kTile * TL::LD];
  __shared__ float sLse[kTile], sDelta[kTile];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y / H, h = blockIdx.y % H;
  const int k0 = blockIdx.x * kTile;
  const long long rs = 3LL * H * dh;
  const int HD = H * dh;
  const __nv_bfloat16* base = qkv + static_cast<long long>(b) * T * rs;
  const float sl = scale * 1.4426950408889634f;
  const float* L = lse + (static_cast<long long>(b) * H + h) * T;
  const float* Dl = delta + (static_cast<long long>(b) * H + h) * T;

  TL::load(sK, base + k0 * rs + (H + h) * dh, rs, T - k0, dh);
  TL::load(sV, base + k0 * rs + (2 * H + h) * dh, rs, T - k0, dh);
  float dk[DP / 8][4], dv[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) {
    dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
    dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  }
  for (int q0 = 0; q0 < T; q0 += kTile) {
    __syncthreads();
    TL::load(sQ, base + q0 * rs + h * dh, rs, T - q0, dh);
    TL::load(sdO, dout + (static_cast<long long>(b) * T + q0) * HD + h * dh, HD, T - q0, dh);
    if (threadIdx.x < kTile) {
      const int q = q0 + threadIdx.x;
      sLse[threadIdx.x] = (q < T) ? L[q] * 1.4426950408889634f : 0.f;
      sDelta[threadIdx.x] = (q < T) ? Dl[q] : 0.f;
    }
    __syncthreads();
    float st[kTile / 8][4], dpt[kTile / 8][4];
#pragma unroll
    for (int i = 0; i < kTile / 8; ++i) {
      st[i][0] = st[i][1] = st[i][2] = st[i][3] = 0.f;
      dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f;
    }
    gemm_rows_nk<DP>(st, sK, warp * 16, sQ, lane);    // S^T[key, query]
    gemm_rows_nk<DP>(dpt, sV, warp * 16, sdO, lane);  // dP^T[key, query]
    float ds[kTile / 8][4];
#pragma unroll
    for (int nt = 0; nt < kTile / 8; ++nt) {
      const int cl = nt * 8 + (lane & 3) * 2, c = q0 + cl;
      const float e0 = sLse[cl], e1 = sLse[cl + 1], d0 = sDelta[cl], d1 = sDelta[cl + 1];
      const float p0 = (c < T) ? fast_exp2(st[nt][0] * sl - e0) : 0.f;
      const float p1 = (c + 1 < T) ? fast_exp2(st[nt][1] * sl - e1) : 0.f;
      const float p2 = (c < T) ? fast_exp2(st[nt][2] * sl - e0) : 0.f;
      const float p3 = (c + 1 < T) ? fast_exp2(st[nt][3] * sl - e1) : 0.f;
      st[nt][0] = p0, st[nt][1] = p1, st[nt][2] = p2, st[nt][3] = p3;
      ds[nt][0] = p0 * (dpt[nt][0] - d0) * scale, ds[nt][1] = p1 * (dpt[nt][1] - d1) * scale;
      ds[nt][2] = p2 * (dpt[nt][2] - d0) * scale, ds[nt][3] = p3 * (dpt[nt][3] - d1) * scale;
    }
    uint32_t pa[kTile / 16][4];
    pack_p(pa, st);
    gemm_p_kn<DP>(dv, pa, sdO, lane);  // dV += P^T dO
    pack_p(pa, ds);
    gemm_p_kn<DP>(dk, pa, sQ, lane);   // dK += dS^T Q
  }
  store_rows<DP>(dqkv + (static_cast<long long>(b) * T + k0) * rs + (H + h) * dh, rs, dk, warp * 16, T - k0, dh, lane,
                 1.f, 1.f);
  store_rows<DP>(dqkv + (static_cast<long long>(b) * T + k0) * rs + (2 * H + h) * dh, rs, dv, warp * 16, T - k0, dh,
                 lane, 1.f, 1.f);
}

}  // namespace mdt

namespace mdt {
// attention_wgmma.cu: T a multiple of 64, head_dim 32 / 64 / 72; MDT_ERR_UNSUPPORTED otherwise -> the kernels above
int attention_wg_fwd(const void* qkv, void* out, float* lse, int B, int T, int H, int dh, float scale, cudaStream_t st);
int attention_wg_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta, void* dqkv,
                     int B, int T, int H, int dh, float scale, cudaStream_t st);
}  // namespace mdt

using namespace mdt;

static int dp_of(int dh) {
  if (dh % 8) return 0;
  if (dh <= 32) return 32;
  if (dh <= 64) return 64;
  if (dh <= 80) return 80;
  return 0;
}

#define MDT_DP_DISPATCH(DPV, ...)                               \
  switch (DPV) {                                                \
    case 32: { constexpr int kDP = 32; __VA_ARGS__; } break;    \
    case 64: { constexpr int kDP = 64; __VA_ARGS__; } break;    \
    case 80: { constexpr int kDP = 80; __VA_ARGS__; } break;    \
    default: return MDT_ERR_UNSUPPORTED;                        \
  }

// Which implementation served the last call (tests assert the production kernels ran instead of trusting the
// fallthrough): 0 = mma.sync (this file: sequence lengths that are not a multiple of 64, other head_dims), 1 = wgmma +
// TMA (attention_wgmma.cu).
static int g_attn_last_impl[2] = {-1, -1};
constexpr int kAttnLogCap = 1024;
static int g_attn_log[kAttnLogCap][4];  // (which, T, head_dim, impl) of every call since the last reset
static int g_attn_log_n = 0;
static void attn_log(int which, int T, int dh, int impl) {
  g_attn_last_impl[which] = impl;
  if (g_attn_log_n < kAttnLogCap) {
    int* e = g_attn_log[g_attn_log_n++];
    e[0] = which, e[1] = T, e[2] = dh, e[3] = impl;
  }
}

extern "C" {

int mdt_attention_last_impl(int which) { return (which == 0 || which == 1) ? g_attn_last_impl[which] : -1; }

int mdt_attention_impl_log(int* out4, int cap) {
  if (!out4) {  // reset
    g_attn_log_n = 0;
    return 0;
  }
  const int n = g_attn_log_n < cap ? g_attn_log_n : cap;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 4; ++j) out4[4 * i + j] = g_attn_log[i][j];
  return n;
}

int mdt_attention_fwd(const void* qkv, void* out, float* lse, int B, int T, int H, int dh, void* stream) {
  if (!qkv || !out || B <= 0 || T <= 0 || H <= 0) return MDT_ERR_ARG;
  const int dp = dp_of(dh);
  if (!dp) return MDT_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(qkv) & 15) || (reinterpret_cast<uintptr_t>(out) & 15)) return MDT_ERR_ARG;
  dim3 grid((T + kTile - 1) / kTile, B * H);
  const float scale = 1.f / sqrtf(static_cast<float>(dh));
  {
    const int rc = attention_wg_fwd(qkv, out, lse, B, T, H, dh, scale, static_cast<cudaStream_t>(stream));
    if (rc != MDT_ERR_UNSUPPORTED) {
      if (rc == MDT_OK) attn_log(0, T, dh, 1);
      return rc;
    }
  }
  attn_log(0, T, dh, 0);
  MDT_DP_DISPATCH(dp, attn_fwd_kernel<kDP><<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(
                          static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(out), lse, T, H, dh,
                          scale));
  return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA;
}

// `lse` doubles as scratch: delta is written to lse + B*H*T (caller allocates 2*B*H*T floats).
int mdt_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, int B, int T,
                      int H, int dh, void* stream) {
  if (!qkv || !out || !dout || !lse || !dqkv || B <= 0 || T <= 0 || H <= 0) return MDT_ERR_ARG;
  const int dp = dp_of(dh);
  if (!dp) return MDT_ERR_UNSUPPORTED;
  dim3 grid((T + kTile - 1) / kTile, B * H);
  const float scale = 1.f / sqrtf(static_cast<float>(dh));
  float* delta = const_cast<float*>(lse) + static_cast<size_t>(B) * H * T;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  {
    const int rc = attention_wg_bwd(qkv, out, dout, lse, delta, dqkv, B, T, H, dh, scale, st);
    if (rc != MDT_ERR_UNSUPPORTED) {
      if (rc == MDT_OK) attn_log(1, T, dh, 1);
      return rc;
    }
  }
  attn_log(1, T, dh, 0);
  MDT_DP_DISPATCH(dp, {
    attn_bwd_dq_kernel<kDP><<<grid, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(qkv),
                                                  static_cast<const __nv_bfloat16*>(out),
                                                  static_cast<const __nv_bfloat16*>(dout), lse,
                                                  static_cast<__nv_bfloat16*>(dqkv), delta, T, H, dh, scale);
    attn_bwd_dkv_kernel<kDP><<<grid, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(qkv),
                                                   static_cast<const __nv_bfloat16*>(dout), lse, delta,
                                                   static_cast<__nv_bfloat16*>(dqkv), T, H, dh, scale);
  });
  return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA;
}

}  // extern "C"
