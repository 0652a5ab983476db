// Multi-head softmax attention on the Hopper tensor cores (wgmma), forward and backward, for the sequence lengths of
// MaskDiT (T a multiple of 64: 128 / 256 / 512 / 1024 tokens) and head_dim 32 / 64 / 72.
//
//   qkv [B, T, 3, H, dh] bf16  ->  out [B, T, H*dh] bf16,  lse [B, H, T] fp32 (natural-log-sum-exp of scaled scores)
//
// One warpgroup (128 threads) per CTA owns a block of 64 rows (queries, or keys in the dK/dV kernel) of one (b, h).
// The other side streams through a two-slot smem ring in blocks of 64 rows: one thread issues the TMA loads of block
// i + 2 as soon as block i is consumed, completion is signalled on the slot's mbarrier.  Every tile is one 3-D TMA box
// per 64 columns of the head ({64 columns, 1 head, 64 rows}, SWIZZLE_128B); head_dim 72 takes two boxes, the columns
// beyond dh are zero-filled by TMA, so the products over head_dim need no masking.
//   S  = A B^T      wgmma m64n64k16, both operands K-major from smem (the contraction is over head_dim)
//   O += P V        wgmma m64n{dh}k16, P from registers (the S accumulator repacked to bf16 A fragments), V read
//                   MN-major from the same [rows][head_dim] tiles (the contraction is over the 64 streamed rows)
// fp32 online softmax in registers.  Backward = two kernels with no atomics: dQ (64 queries, loops over keys; also
// emits delta = rowsum(dO * O)) and dK / dV (64 keys, loops over queries, transposed formulation S^T = K Q^T).
#include "common.cuh"
#include "gemm.h"
#include "wgmma.cuh"

#include <type_traits>

namespace mdt {

constexpr int kAB = 64;                 // rows per block on either side
constexpr uint32_t kBox = 64 * 128;     // bytes of one [64 rows][64 columns] bf16 SW128 tile
constexpr float kLog2e = 1.4426950408889634f;

MDT_DEVINL void tma_load_3d(const CUtensorMap* m, uint64_t* bar, uint32_t smem_dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// inline spin: a call (the bounded wait's slow path) inside the loops would make ptxas serialise the wgmma pipeline
MDT_DEVINL void spin_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// S[64 x 64] = A[64 x DH] B[64 x DH]^T, both stored as SW128 tiles of 64 columns; ceil(DH / 16) k-steps (the
// zero-filled columns beyond them are not multiplied)
template <int DH>
MDT_DEVINL void mma_abt(float* s, uint32_t sa, uint32_t sb) {
  constexpr int kSteps = (DH + 15) / 16;
  wgmma_fence();
#pragma unroll
  for (int t = 0; t < kSteps; ++t) {
    const uint32_t off = (t / 4) * kBox + (t % 4) * 32;
    Wgmma<64, 0, 0>::mma(s, make_smem_desc_sw128(sa + off, 16, 1024), make_smem_desc_sw128(sb + off, 16, 1024),
                         t > 0 ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
}
// O[64 x N] += P[64 x 64] (bf16 A fragments in registers) * V[64 x N] (the 64-row tile, N = head_dim, MN-major)
template <int N>
MDT_DEVINL void mma_pv(float* o, const uint32_t (*pa)[4], uint32_t sv) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) WgmmaRS<N, 1>::mma(o, pa[kk], make_smem_desc_sw128(sv + kk * (16 * 128), kBox, 1024), 1u);
  wgmma_commit();
  wgmma_wait<0>();
}
// m64n64 accumulator -> the four k16 A fragments of the next product
MDT_DEVINL void pack_a(uint32_t (*pa)[4], const float* s) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    pa[kk][0] = pack_bf16(s[8 * kk + 0], s[8 * kk + 1]);
    pa[kk][1] = pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
    pa[kk][2] = pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
    pa[kk][3] = pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
  }
}
MDT_DEVINL float quad_max4(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
MDT_DEVINL float quad_sum4(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// store a 64 x N accumulator (this thread: rows r, r + 8, columns 8g + 2q, +1) as bf16 to rows of stride ld
template <int N>
MDT_DEVINL void store_acc(__nv_bfloat16* g, long long ld, const float* o, float mul0, float mul1) {
  const int lane = threadIdx.x & 31, r = 16 * (threadIdx.x >> 5) + (lane >> 2), c = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<uint32_t*>(g + r * ld + 8 * j + c) = pack_bf16(o[4 * j] * mul0, o[4 * j + 1] * mul0);
    *reinterpret_cast<uint32_t*>(g + (r + 8) * ld + 8 * j + c) = pack_bf16(o[4 * j + 2] * mul1, o[4 * j + 3] * mul1);
  }
}

// Shared memory of every kernel: two resident tiles (R0, R1; R1 unused by the forward) and a two-slot ring of two
// streamed tiles (S0, S1), each KCH * 8 KB, then the barriers.
template <int KCH>
struct AttnSmem {
  static constexpr uint32_t kTile = KCH * kBox;
  static constexpr uint32_t kBytes = 6 * kTile + 512 /*barriers, delta*/ + 1024 /*align slack*/;
};

// Loads the two streamed tiles of block `blk` (rows tok0 + 64 blk) of heads (c1a, c1b) into ring slot `slot`.
template <int KCH>
MDT_DEVINL void load_pair(const CUtensorMap* ma, int c1a, const CUtensorMap* mb, int c1b, int tok, uint64_t* bar,
                          uint32_t sa, uint32_t sb) {
  mbar_arrive_expect_tx(bar, 2 * AttnSmem<KCH>::kTile);
#pragma unroll
  for (int c = 0; c < KCH; ++c) {
    tma_load_3d(ma, bar, sa + c * kBox, 64 * c, c1a, tok);
    tma_load_3d(mb, bar, sb + c * kBox, 64 * c, c1b, tok);
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------
template <int KCH, int N>
__global__ void __launch_bounds__(128)
attn_wg_fwd_kernel(const __grid_constant__ CUtensorMap tqkv, __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
                   int T, int H, float scale) {
  using SM = AttnSmem<KCH>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023) & ~1023u;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + (base - smem_u32(smem_raw)) + 6 * SM::kTile);
  const uint32_t sQ = base, sK = base + 2 * SM::kTile, sV = base + 4 * SM::kTile;  // ring: slot s at + s * kTile
  const int tid = threadIdx.x, lane = tid & 31;
  const int b = blockIdx.y / H, h = blockIdx.y % H, q0 = blockIdx.x * kAB, tok = b * T, nkb = T / kAB;
  const float sl = scale * kLog2e;
  if (tid == 0) {
    tma_prefetch_desc(&tqkv);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bars[2], SM::kTile);
    for (int c = 0; c < KCH; ++c) tma_load_3d(&tqkv, &bars[2], sQ + c * kBox, 64 * c, h, tok + q0);
    for (int i = 0; i < 2 && i < nkb; ++i)
      load_pair<KCH>(&tqkv, H + h, &tqkv, 2 * H + h, tok + i * kAB, &bars[i], sK + i * SM::kTile, sV + i * SM::kTile);
  }
  float o[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  spin_wait(&bars[2], 0);
  for (int i = 0; i < nkb; ++i) {
    const int s = i & 1;
    spin_wait(&bars[s], (i >> 1) & 1);
    float sc[32];
    mma_abt<N>(sc, sQ, sK + s * SM::kTile);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      mx0 = fmaxf(mx0, fmaxf(sc[4 * g], sc[4 * g + 1]));
      mx1 = fmaxf(mx1, fmaxf(sc[4 * g + 2], sc[4 * g + 3]));
    }
    const float mn0 = fmaxf(m0, quad_max4(mx0)), mn1 = fmaxf(m1, quad_max4(mx1));
    const float a0 = fast_exp2((m0 - mn0) * sl), a1 = fast_exp2((m1 - mn1) * sl);
    m0 = mn0, m1 = mn1;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      sc[4 * g] = fast_exp2(sc[4 * g] * sl - m0 * sl), sc[4 * g + 1] = fast_exp2(sc[4 * g + 1] * sl - m0 * sl);
      sc[4 * g + 2] = fast_exp2(sc[4 * g + 2] * sl - m1 * sl), sc[4 * g + 3] = fast_exp2(sc[4 * g + 3] * sl - m1 * sl);
      rs0 += sc[4 * g] + sc[4 * g + 1], rs1 += sc[4 * g + 2] + sc[4 * g + 3];
    }
    l0 = l0 * a0 + rs0, l1 = l1 * a1 + rs1;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) o[4 * j] *= a0, o[4 * j + 1] *= a0, o[4 * j + 2] *= a1, o[4 * j + 3] *= a1;
    uint32_t pa[4][4];
    pack_a(pa, sc);
    mma_pv<N>(o, pa, sV + s * SM::kTile);
    __syncthreads();  // every warp is done with slot s
    if (tid == 0 && i + 2 < nkb)
      load_pair<KCH>(&tqkv, H + h, &tqkv, 2 * H + h, tok + (i + 2) * kAB, &bars[s], sK + s * SM::kTile,
                     sV + s * SM::kTile);
  }
  l0 = quad_sum4(l0), l1 = quad_sum4(l1);
  const int HD = H * N;
  store_acc<N>(out + static_cast<long long>(tok + q0) * HD + h * N, HD, o, 1.f / l0, 1.f / l1);
  if ((lane & 3) == 0 && lse) {
    const int r = q0 + 16 * (tid >> 5) + (lane >> 2);
    float* L = lse + (static_cast<long long>(b) * H + h) * T;
    L[r] = m0 * scale + logf(l0);
    L[r + 8] = m1 * scale + logf(l1);
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward: dQ (+ delta)
// ------------------------------------------------------------------------------------------------------------
template <int KCH, int N>
__global__ void __launch_bounds__(128)
attn_wg_bwd_dq_kernel(const __grid_constant__ CUtensorMap tqkv, const __grid_constant__ CUtensorMap tdo,
                      const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                      const float* __restrict__ lse, __nv_bfloat16* __restrict__ dqkv, float* __restrict__ delta, int T,
                      int H, float scale) {
  using SM = AttnSmem<KCH>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023) & ~1023u;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + (base - smem_u32(smem_raw)) + 6 * SM::kTile);
  float* sDelta = reinterpret_cast<float*>(bars + 4);
  const uint32_t sQ = base, sdO = base + SM::kTile, sK = base + 2 * SM::kTile, sV = base + 4 * SM::kTile;
  const int tid = threadIdx.x, lane = tid & 31;
  const int b = blockIdx.y / H, h = blockIdx.y % H, q0 = blockIdx.x * kAB, tok = b * T, nkb = T / kAB;
  const int HD = H * N;
  const float sl = scale * kLog2e;
  if (tid == 0) {
    tma_prefetch_desc(&tqkv);
    tma_prefetch_desc(&tdo);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bars[2], 2 * SM::kTile);
    for (int c = 0; c < KCH; ++c) {
      tma_load_3d(&tqkv, &bars[2], sQ + c * kBox, 64 * c, h, tok + q0);
      tma_load_3d(&tdo, &bars[2], sdO + c * kBox, 64 * c, h, tok + q0);
    }
    for (int i = 0; i < 2 && i < nkb; ++i)
      load_pair<KCH>(&tqkv, H + h, &tqkv, 2 * H + h, tok + i * kAB, &bars[i], sK + i * SM::kTile, sV + i * SM::kTile);
  }
  {  // delta = rowsum(dO * O): two threads per row, 8 columns per load
    const int r = tid >> 1, half = tid & 1;
    const long long off = static_cast<long long>(tok + q0 + r) * HD + h * N;
    float acc = 0.f;
    for (int c = 8 * half; c < N; c += 16) {
      const uint4 u = *reinterpret_cast<const uint4*>(out + off + c), v = *reinterpret_cast<const uint4*>(dout + off + c);
      acc += bf16_lo(u.x) * bf16_lo(v.x) + bf16_hi(u.x) * bf16_hi(v.x) + bf16_lo(u.y) * bf16_lo(v.y) +
             bf16_hi(u.y) * bf16_hi(v.y) + bf16_lo(u.z) * bf16_lo(v.z) + bf16_hi(u.z) * bf16_hi(v.z) +
             bf16_lo(u.w) * bf16_lo(v.w) + bf16_hi(u.w) * bf16_hi(v.w);
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (half == 0) {
      sDelta[r] = acc;
      delta[(static_cast<long long>(b) * H + h) * T + q0 + r] = acc;
    }
  }
  __syncthreads();
  const int r0 = 16 * (tid >> 5) + (lane >> 2);
  const float* L = lse + (static_cast<long long>(b) * H + h) * T + q0;
  const float ls0 = L[r0] * kLog2e, ls1 = L[r0 + 8] * kLog2e, dl0 = sDelta[r0], dl1 = sDelta[r0 + 8];
  float dq[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) dq[i] = 0.f;
  spin_wait(&bars[2], 0);
  for (int i = 0; i < nkb; ++i) {
    const int s = i & 1;
    spin_wait(&bars[s], (i >> 1) & 1);
    float sc[32], dp[32];
    mma_abt<N>(sc, sQ, sK + s * SM::kTile);
    mma_abt<N>(dp, sdO, sV + s * SM::kTile);
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      sc[4 * g] = fast_exp2(sc[4 * g] * sl - ls0) * (dp[4 * g] - dl0) * scale;
      sc[4 * g + 1] = fast_exp2(sc[4 * g + 1] * sl - ls0) * (dp[4 * g + 1] - dl0) * scale;
      sc[4 * g + 2] = fast_exp2(sc[4 * g + 2] * sl - ls1) * (dp[4 * g + 2] - dl1) * scale;
      sc[4 * g + 3] = fast_exp2(sc[4 * g + 3] * sl - ls1) * (dp[4 * g + 3] - dl1) * scale;
    }
    uint32_t pa[4][4];
    pack_a(pa, sc);
    mma_pv<N>(dq, pa, sK + s * SM::kTile);  // dQ += dS K
    __syncthreads();
    if (tid == 0 && i + 2 < nkb)
      load_pair<KCH>(&tqkv, H + h, &tqkv, 2 * H + h, tok + (i + 2) * kAB, &bars[s], sK + s * SM::kTile,
                     sV + s * SM::kTile);
  }
  store_acc<N>(dqkv + static_cast<long long>(tok + q0) * 3 * HD + h * N, 3 * HD, dq, 1.f, 1.f);
}

// ------------------------------------------------------------------------------------------------------------
// backward: dK, dV  (rows = keys)
// ------------------------------------------------------------------------------------------------------------
template <int KCH, int N>
__global__ void __launch_bounds__(128)
attn_wg_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tqkv, const __grid_constant__ CUtensorMap tdo,
                       const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv,
                       int T, int H, float scale) {
  using SM = AttnSmem<KCH>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023) & ~1023u;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + (base - smem_u32(smem_raw)) + 6 * SM::kTile);
  const uint32_t sK = base, sV = base + SM::kTile, sQ = base + 2 * SM::kTile, sdO = base + 4 * SM::kTile;
  const int tid = threadIdx.x, lane = tid & 31;
  const int b = blockIdx.y / H, h = blockIdx.y % H, k0 = blockIdx.x * kAB, tok = b * T, nqb = T / kAB;
  const int HD = H * N;
  const float sl = scale * kLog2e;
  if (tid == 0) {
    tma_prefetch_desc(&tqkv);
    tma_prefetch_desc(&tdo);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    load_pair<KCH>(&tqkv, H + h, &tqkv, 2 * H + h, tok + k0, &bars[2], sK, sV);
    for (int i = 0; i < 2 && i < nqb; ++i)
      load_pair<KCH>(&tqkv, h, &tdo, h, tok + i * kAB, &bars[i], sQ + i * SM::kTile, sdO + i * SM::kTile);
  }
  const float* L = lse + (static_cast<long long>(b) * H + h) * T;
  const float* Dl = delta + (static_cast<long long>(b) * H + h) * T;
  const int cq = (lane & 3) * 2;
  float dk[N / 2], dv[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) dk[i] = dv[i] = 0.f;
  spin_wait(&bars[2], 0);
  for (int i = 0; i < nqb; ++i) {
    const int s = i & 1;
    spin_wait(&bars[s], (i >> 1) & 1);
    float st[32], dpt[32];
    mma_abt<N>(st, sK, sQ + s * SM::kTile);     // S^T[key, query]
    mma_abt<N>(dpt, sV, sdO + s * SM::kTile);   // dP^T[key, query]
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      const int q = i * kAB + 8 * g + cq;
      const float2 e = *reinterpret_cast<const float2*>(L + q), d = *reinterpret_cast<const float2*>(Dl + q);
      const float p0 = fast_exp2(st[4 * g] * sl - e.x * kLog2e), p1 = fast_exp2(st[4 * g + 1] * sl - e.y * kLog2e);
      const float p2 = fast_exp2(st[4 * g + 2] * sl - e.x * kLog2e), p3 = fast_exp2(st[4 * g + 3] * sl - e.y * kLog2e);
      st[4 * g] = p0, st[4 * g + 1] = p1, st[4 * g + 2] = p2, st[4 * g + 3] = p3;
      dpt[4 * g] = p0 * (dpt[4 * g] - d.x) * scale, dpt[4 * g + 1] = p1 * (dpt[4 * g + 1] - d.y) * scale;
      dpt[4 * g + 2] = p2 * (dpt[4 * g + 2] - d.x) * scale, dpt[4 * g + 3] = p3 * (dpt[4 * g + 3] - d.y) * scale;
    }
    uint32_t pa[4][4];
    pack_a(pa, st);
    mma_pv<N>(dv, pa, sdO + s * SM::kTile);  // dV += P^T dO
    pack_a(pa, dpt);
    mma_pv<N>(dk, pa, sQ + s * SM::kTile);   // dK += dS^T Q
    __syncthreads();
    if (tid == 0 && i + 2 < nqb)
      load_pair<KCH>(&tqkv, h, &tdo, h, tok + (i + 2) * kAB, &bars[s], sQ + s * SM::kTile, sdO + s * SM::kTile);
  }
  __nv_bfloat16* g = dqkv + static_cast<long long>(tok + k0) * 3 * HD;
  store_acc<N>(g + (H + h) * N, 3 * HD, dk, 1.f, 1.f);
  store_acc<N>(g + (2 * H + h) * N, 3 * HD, dv, 1.f, 1.f);
}

// ------------------------------------------------------------------------------------------------------------
// host side: MDT_ERR_UNSUPPORTED for a shape outside the kernels' range (T % 64 != 0, other head_dims)
// ------------------------------------------------------------------------------------------------------------
template <typename F>
static int run_dh(int dh, F&& f) {
  switch (dh) {
    case 32: return f(std::integral_constant<int, 1>(), std::integral_constant<int, 32>());
    case 64: return f(std::integral_constant<int, 1>(), std::integral_constant<int, 64>());
    case 72: return f(std::integral_constant<int, 2>(), std::integral_constant<int, 72>());
    default: return MDT_ERR_UNSUPPORTED;
  }
}
template <typename K>
static int set_smem(K kern, uint32_t bytes) {
  return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess ? MDT_OK
                                                                                                      : MDT_ERR_CUDA;
}

int attention_wg_fwd(const void* qkv, void* out, float* lse, int B, int T, int H, int dh, float scale, cudaStream_t st) {
  if (T % kAB) return MDT_ERR_UNSUPPORTED;
  return run_dh(dh, [&](auto kch, auto n) {
    constexpr int KCH = decltype(kch)::value, N = decltype(n)::value;
    CUtensorMap tq;
    int rc = make_head_tile_tmap(&tq, qkv, N, 3ull * H, static_cast<unsigned long long>(B) * T);
    if (rc) return rc;
    auto kern = attn_wg_fwd_kernel<KCH, N>;
    static int attr = set_smem(kern, AttnSmem<KCH>::kBytes);
    if (attr) return attr;
    kern<<<dim3(T / kAB, B * H), 128, AttnSmem<KCH>::kBytes, st>>>(tq, static_cast<__nv_bfloat16*>(out), lse, T, H,
                                                                   scale);
    return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA;
  });
}

int attention_wg_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta, void* dqkv,
                     int B, int T, int H, int dh, float scale, cudaStream_t st) {
  if (T % kAB) return MDT_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(dout) & 15)) return MDT_ERR_UNSUPPORTED;
  return run_dh(dh, [&](auto kch, auto n) {
    constexpr int KCH = decltype(kch)::value, N = decltype(n)::value;
    const unsigned long long rows = static_cast<unsigned long long>(B) * T;
    CUtensorMap tq, tdo;
    int rc = make_head_tile_tmap(&tq, qkv, N, 3ull * H, rows);
    if (rc) return rc;
    rc = make_head_tile_tmap(&tdo, dout, N, H, rows);
    if (rc) return rc;
    auto kdq = attn_wg_bwd_dq_kernel<KCH, N>;
    auto kdkv = attn_wg_bwd_dkv_kernel<KCH, N>;
    static int attr = set_smem(kdq, AttnSmem<KCH>::kBytes) | set_smem(kdkv, AttnSmem<KCH>::kBytes);
    if (attr) return MDT_ERR_CUDA;
    const dim3 grid(T / kAB, B * H);
    kdq<<<grid, 128, AttnSmem<KCH>::kBytes, st>>>(tq, tdo, static_cast<const __nv_bfloat16*>(out),
                                                  static_cast<const __nv_bfloat16*>(dout), lse,
                                                  static_cast<__nv_bfloat16*>(dqkv), delta, T, H, scale);
    kdkv<<<grid, 128, AttnSmem<KCH>::kBytes, st>>>(tq, tdo, lse, delta, static_cast<__nv_bfloat16*>(dqkv), T, H,
                                                   scale);
    return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA;
  });
}

}  // namespace mdt
