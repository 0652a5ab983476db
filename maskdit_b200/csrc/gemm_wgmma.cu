// bf16 GEMM on the Hopper tensor cores (wgmma.mma_async, accumulators in registers, operands staged by TMA).
//
//   out[M,N] (+)= sum_k A[m,k] * B[n,k]      fp32 accumulate
//
// One persistent CTA per SM, warp-specialised, 128 x BLOCK_N output tiles:
//   warpgroup 0      TMA producer (one thread)  global -> 128B-swizzled smem ring, mbarrier complete_tx
//   warpgroups 1, 2  consumers                  wgmma 64 x BLOCK_N x 16 on rows 64 * (wg - 1) .. +63 of the tile, then
//                                               the fused epilogue straight from the accumulator registers
// The producer runs ahead into the next unit while the consumers are in their epilogue.  The register file is split
// with setmaxnreg: the producer warpgroup keeps 40 registers per thread, each consumer thread gets 232 (a 64 x 256 fp32
// accumulator is 128 of them).
//
// Operand majors: "K-major" = contraction index contiguous in memory (activations [M,K], nn.Linear weights
// [N,K]); "MN-major" = the M/N index contiguous (used by dgrad: B = W[N,K] read as [K_out, N_contract]; and by
// wgrad: both operands are token-major [tokens, features] with the contraction over tokens).  wgmma reads both from
// shared memory through the transpose bits of the instruction.
//
// Scheduling: persistent tile loop (each CTA takes whole output tiles, strided) for forward/dgrad; for the
// accumulate epilogue (wgrad, long-K small-output GEMMs) the K range is additionally cut into slices so that
// tiles x slices fills the machine, units are walked slice-major and partial tiles are reduced with fp32
// red.global.add.v4 in the epilogue.
//
// Reference ops this replaces: every nn.Linear of models/maskdit.py (timm Attention.qkv/proj, Mlp.fc1/fc2,
// adaLN_modulation, DecoderLayer.linear, TimestepEmbedder.mlp, LabelEmbedder) and their autograd backward.
#include "common.cuh"
#include "deterministic.h"
#include "gemm.h"
#include "unit_sched.h"
#include "wgmma.cuh"

#include <stdlib.h>

#include <mutex>

namespace mdt {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 B = one swizzle-128B row
constexpr int WG_K = 16;
constexpr int kNumConsumerWGs = 2;
constexpr int kNumThreads = 128 * (1 + kNumConsumerWGs);
constexpr int kConsumerRegs = 232, kProducerRegs = 40;  // (40 + 2 * 232) * 128 <= 64 K registers
constexpr int kRowsPerWarp = 16;                         // wgmma m64: warp w of a warpgroup owns rows 16w .. 16w+15
constexpr int kRowGroups = kRowsPerWarp / 4;

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStagingBytes = kNumConsumerWGs * 4 * kRowsPerWarp * 40 * 4;  // per-warp 16x40 fp32 tiles
  static constexpr int kFixed = kStagingBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int kStagesFit = (232448 - kFixed) / kStageBytes;
  static constexpr int kStages = kStagesFit > 8 ? 8 : kStagesFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixed;
  static_assert(kStages >= 3, "pipeline too shallow");
};

// ---- fused epilogue ---------------------------------------------------------------------------------------
// The wgmma accumulator fragment gives each thread 2 adjacent columns of 2 rows per 8-column group.  Storing that
// straight to global would make every warp store touch 16 rows.  Each 16 x 32 chunk of a warp is therefore
// transposed through a per-warp smem staging tile (row stride 40 words: the 8-byte fragment stores of a half warp and
// the LDS.128 of a quarter warp are both conflict free).  In the second phase lane -> (row = lane/8 + 4i, 4 columns =
// lane%8): one warp instruction covers 4 rows x 128 contiguous bytes (fp32) or 64 bytes (bf16), and bias / gate /
// residual / aux are read with the same coalesced vector pattern.
// The per-epilogue loops are separate template instances selected by ONE switch per launch, so a launch only ever
// touches the instructions of its own epilogue.
constexpr int kStgStride = 40;
constexpr int kStgFloats = kRowsPerWarp * kStgStride;

MDT_DEVINL uint2 pack4_bf16(float4 v) { return make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w)); }
MDT_DEVINL float4 unpack4_bf16(uint2 u) { return make_float4(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y)); }
MDT_DEVINL void sts64(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// Global operands of one chunk (this lane's 4 columns x the row groups) are fetched for all row groups BEFORE any
// dependent store is issued: issue is in order, so a load -> store dependency inside the row loop would expose the
// full global latency once per row group.
struct EpiCoord {
  int row_base, nrows, col;  // col = this lane's first column
  bool valid;                // nrows > 0 && col + 4 <= N
};
MDT_DEVINL EpiCoord make_coord(const GemmParams& p, int row_base, int nrows, int col) {
  return EpiCoord{row_base, nrows, col, nrows > 0 && col + 4 <= p.N};
}

template <int EPI>
struct EpiOps {
  float4 bias4, gate4;
  bool gate_uniform;
  float4 res[(EPI == EPI_GATE_RESID || EPI == EPI_STORE) ? kRowGroups : 1];
  uint2 auxv[EPI == EPI_DGELU ? kRowGroups : 1];
};

template <int EPI>
MDT_DEVINL void epi_load(const GemmParams& p, const EpiCoord& c, int lane, EpiOps<EPI>& o) {
  if (!c.valid) return;
  const int rsub = lane >> 3;
  const size_t row0 = static_cast<size_t>(c.row_base + rsub);
  o.bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (EPI != EPI_ATOMIC && p.bias) o.bias4 = ldg128_nc(gaddr(p.bias + c.col));
  if constexpr (EPI == EPI_GATE_RESID) {
    const int b0 = c.row_base / p.rows_per_group, b1 = (c.row_base + c.nrows - 1) / p.rows_per_group;
    o.gate_uniform = b0 == b1;
    o.gate4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (o.gate_uniform) o.gate4 = ldg128_nc(gaddr(p.gate + static_cast<size_t>(b0) * p.ld_gate + c.col));
  }
  if constexpr (EPI == EPI_GATE_RESID || EPI == EPI_STORE) {
    if (EPI == EPI_GATE_RESID || p.resid) {
      const uint64_t a_res = gaddr(p.resid) + (row0 * p.ld_resid + c.col) * 4, s_res = 16ull * p.ld_resid;
#pragma unroll
      for (int i = 0; i < kRowGroups; ++i)
        if (4 * i + rsub < c.nrows) o.res[i] = ldg128(a_res + i * s_res);
    }
  }
  if constexpr (EPI == EPI_DGELU) {
    const uint64_t a_aux = gaddr(p.aux) + (row0 * p.ld_aux + c.col) * 2, s_aux = 8ull * p.ld_aux;
#pragma unroll
    for (int i = 0; i < kRowGroups; ++i)
      if (4 * i + rsub < c.nrows) o.auxv[i] = ldg64_nc(a_aux + i * s_aux);
  }
}

// chunk `c` (valid for this lane): transpose-read, fused arithmetic, coalesced stores
template <int EPI>
MDT_DEVINL void epilogue_chunk(const GemmParams& p, uint32_t stg, const EpiCoord& c, int lane, const EpiOps<EPI>& o,
                               float4& cs_out) {
  const int rsub = lane >> 3, c4 = (lane & 7) * 4;
  const float4 bias4 = o.bias4;
  const size_t row0 = static_cast<size_t>(c.row_base + rsub);
  const int osz = (EPI == EPI_ATOMIC || EPI == EPI_GATE_RESID || (EPI == EPI_STORE && p.out_fp32)) ? 4 : 2;
  const uint64_t a_out = gaddr(p.out) + (row0 * p.ldo + c.col) * osz;
  const uint64_t a_aux = gaddr(p.aux) + (row0 * p.ld_aux + c.col) * 2;
  const uint64_t s_out = 4ull * p.ldo * osz, s_aux = 8ull * p.ld_aux;
  const uint32_t sp = stg + (rsub * kStgStride + c4) * 4;
  float4 cs = make_float4(0.f, 0.f, 0.f, 0.f);  // EPI_DGELU: column sums of this lane's outputs (bias gradient)
#pragma unroll
  for (int i = 0; i < kRowGroups; ++i) {
    if (4 * i + rsub >= c.nrows) break;
    float4 v = lds128(sp + i * (4 * kStgStride * 4));
    const uint64_t ao = a_out + i * s_out;
    if constexpr (EPI == EPI_ATOMIC) {
      red_add_v4(ao, v);
    } else {
      v.x += bias4.x, v.y += bias4.y, v.z += bias4.z, v.w += bias4.w;
      if constexpr (EPI == EPI_STORE) {
        if (p.resid) v.x += o.res[i].x, v.y += o.res[i].y, v.z += o.res[i].z, v.w += o.res[i].w;
        if (p.act == ACT_SILU) v = make_float4(silu(v.x), silu(v.y), silu(v.z), silu(v.w));
        if (p.out_fp32) stg128(ao, v); else stg64(ao, pack4_bf16(v));
      } else if constexpr (EPI == EPI_GELU) {
        // pre-activation is rounded to bf16 first (as a bf16 nn.Linear output would be), GELU on the rounded value
        const uint2 pre = pack4_bf16(v);
        if (p.aux) stg64(a_aux + i * s_aux, pre);
        const float4 h = unpack4_bf16(pre);
        stg64(ao, pack4_bf16(make_float4(gelu_tanh(h.x), gelu_tanh(h.y), gelu_tanh(h.z), gelu_tanh(h.w))));
      } else if constexpr (EPI == EPI_GATE_RESID) {
        if (p.aux) stg64(a_aux + i * s_aux, pack4_bf16(v));
        float4 g = o.gate4;
        if (!o.gate_uniform) {
          const size_t b = (row0 + 4 * i) / p.rows_per_group;
          g = ldg128_nc(gaddr(p.gate + b * p.ld_gate + c.col));
        }
        const float4 r = o.res[i];  // may alias `out` (in-place residual update): each element is read before written
        stg128(ao, make_float4(fmaf(g.x, v.x, r.x), fmaf(g.y, v.y, r.y), fmaf(g.z, v.z, r.z), fmaf(g.w, v.w, r.w)));
      } else if constexpr (EPI == EPI_DGELU) {
        const float4 h = unpack4_bf16(o.auxv[i]);
        const uint2 ov = pack4_bf16(make_float4(v.x * gelu_tanh_grad(h.x), v.y * gelu_tanh_grad(h.y),
                                                v.z * gelu_tanh_grad(h.z), v.w * gelu_tanh_grad(h.w)));
        stg64(ao, ov);
        const float4 r = unpack4_bf16(ov);  // sum what was stored (what a separate column-sum pass would read back)
        cs.x += r.x, cs.y += r.y, cs.z += r.z, cs.w += r.w;
      }
    }
  }
  if constexpr (EPI == EPI_DGELU) cs_out = cs;
}

// ragged right edge (N % 4 != 0 inside this 4-column group): element-wise, same arithmetic, cold path
__device__ __noinline__ void epilogue_ragged(const GemmParams& p, uint32_t stg, int row_base, int nrows, int col,
                                             int lane) {
  const int rsub = lane >> 3, c4 = (lane & 7) * 4;
  for (int i = 0; i < kRowGroups; ++i) {
    const int rr = 4 * i + rsub;
    if (rr >= nrows) break;
    const size_t row = static_cast<size_t>(row_base + rr);
    for (int j = 0; j < 4 && col + j < p.N; ++j) {
      float v = lds32(stg + (rr * kStgStride + c4 + j) * 4);
      const int c = col + j;
      if (p.epi == EPI_ATOMIC) {
        atomicAdd(reinterpret_cast<float*>(p.out) + row * p.ldo + c, v);
        continue;
      }
      if (p.bias) v += p.bias[c];
      __nv_bfloat16* o16 = reinterpret_cast<__nv_bfloat16*>(p.out) + row * p.ldo + c;
      float* o32 = reinterpret_cast<float*>(p.out) + row * p.ldo + c;
      __nv_bfloat16* aux = reinterpret_cast<__nv_bfloat16*>(p.aux) + row * p.ld_aux + c;
      switch (p.epi) {
        case EPI_STORE:
          if (p.resid) v += p.resid[row * p.ld_resid + c];
          if (p.act == ACT_SILU) v = silu(v);
          if (p.out_fp32) *o32 = v; else *o16 = __float2bfloat16_rn(v);
          break;
        case EPI_GELU: {
          const __nv_bfloat16 pre = __float2bfloat16_rn(v);
          if (p.aux) *aux = pre;
          *o16 = __float2bfloat16_rn(gelu_tanh(__bfloat162float(pre)));
        } break;
        case EPI_GATE_RESID:
          if (p.aux) *aux = __float2bfloat16_rn(v);
          *o32 = fmaf(p.gate[(row / p.rows_per_group) * p.ld_gate + c], v, p.resid[row * p.ld_resid + c]);
          break;
        case EPI_DGELU: {
          const __nv_bfloat16 r = __float2bfloat16_rn(v * gelu_tanh_grad(__bfloat162float(*aux)));
          *o16 = r;
          if (p.colsum) atomicAdd(p.colsum + c, __bfloat162float(r));
        } break;
        default: break;
      }
    }
  }
}

// One staged 16 x 32 chunk of a warp -> global.  Kept out of line: the consumer loop around it holds the whole
// accumulator in registers, and inlining the epilogue arithmetic there pushes the accumulator into local memory.
// `p` is the kernel's __grid_constant__ parameter, so the reference points into parameter space: a plain by-value
// kernel parameter would be copied to a stack frame for its address and every field read here would be a local load.
template <int EPI>
__device__ __noinline__ void epilogue_staged(const GemmParams& p, uint32_t stg, int row_base, int nrows, int col0,
                                             int lane) {
  const EpiCoord c = make_coord(p, row_base, nrows, col0 + (lane & 7) * 4);
  EpiOps<EPI> ops;
  epi_load<EPI>(p, c, lane, ops);
  float4 cs = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c.valid) epilogue_chunk<EPI>(p, stg, c, lane, ops, cs);
  else if (c.col < p.N) epilogue_ragged(p, stg, row_base, nrows, c.col, lane);
  if constexpr (EPI == EPI_DGELU) {
    if (p.colsum) {  // launch-uniform: bias gradient = column sums of the stored tile (fused colsum pass)
      __syncwarp();  // lanes l, l^8, l^16, l^24 own the same 4 columns (different row groups)
      cs.x += __shfl_xor_sync(0xffffffffu, cs.x, 8), cs.y += __shfl_xor_sync(0xffffffffu, cs.y, 8);
      cs.z += __shfl_xor_sync(0xffffffffu, cs.z, 8), cs.w += __shfl_xor_sync(0xffffffffu, cs.w, 8);
      cs.x += __shfl_xor_sync(0xffffffffu, cs.x, 16), cs.y += __shfl_xor_sync(0xffffffffu, cs.y, 16);
      cs.z += __shfl_xor_sync(0xffffffffu, cs.z, 16), cs.w += __shfl_xor_sync(0xffffffffu, cs.w, 16);
      if (lane < 8 && c.valid) red_add_v4(gaddr(p.colsum + c.col), cs);
    }
  }
}

// The k-blocks of one unit: wgmma 64 x WN x 16 from the smem ring into `acc`, each slot handed back to the producer as
// soon as the MMAs that read it have retired.
template <int WN, int BLOCK_N, bool A_MN, bool B_MN>
MDT_DEVINL void mainloop(const UnitSched& sched, uint8_t* smem_tiles, uint64_t* full_bar, uint64_t* empty_bar,
                         float* acc, int cwg, int lane, int& stage, uint32_t& phase) {
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int kStages = Cfg::kStages;
  int prev = -1;
  for (int kb = sched.kb0; kb < sched.kb1; ++kb) {
    // inline spin: a call here (the bounded wait's slow path) would make ptxas serialise the wgmma pipeline
    while (!mbar_try_wait(&full_bar[stage], phase)) {
    }
    const uint32_t sa = smem_u32(smem_tiles + stage * Cfg::kStageBytes) + cwg * (64 * 128);
    const uint32_t sb = smem_u32(smem_tiles + stage * Cfg::kStageBytes) + Cfg::kABytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / WG_K; ++k) {
      // K-major: +32 B per WG_K inside the 128B swizzle row; SBO = 8 rows * 128 B.
      // MN-major: +16 k-rows * 128 B per WG_K; LBO = one 64-wide MN atom (64 k-rows * 128 B), SBO = 8 k-rows.
      const uint64_t da = A_MN ? make_smem_desc_sw128(sa + k * (WG_K * 128), 64 * BLOCK_K * 2, 1024)
                               : make_smem_desc_sw128(sa + k * (WG_K * 2), 16, 1024);
      const uint64_t db = B_MN ? make_smem_desc_sw128(sb + k * (WG_K * 128), 64 * BLOCK_K * 2, 1024)
                               : make_smem_desc_sw128(sb + k * (WG_K * 2), 16, 1024);
      const uint32_t scale_d = (kb > sched.kb0 || k > 0) ? 1u : 0u;
      Wgmma<WN, A_MN, B_MN>::mma(acc, da, db, scale_d);
    }
    wgmma_commit();
    // the previous k-block's MMAs have retired: its smem slot goes back to the producer
    wgmma_wait<1>();
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }
    prev = stage;
    if (++stage == kStages) stage = 0, phase ^= 1;
  }
  wgmma_wait<0>();
  __syncwarp();
  if (lane == 0 && prev >= 0) mbar_arrive(&empty_bar[prev]);
}

// The consumer warpgroups' whole persistent loop for ONE epilogue kind: main loop over the unit's k-blocks, then the
// epilogue of the warp's 16 rows x BLOCK_N columns from the accumulator registers.
template <int EPI, int BLOCK_N, bool A_MN, bool B_MN>
MDT_DEVINL void consumer_loop(const GemmParams& p, UnitSched& sched, uint8_t* smem_tiles, uint64_t* full_bar,
                              uint64_t* empty_bar, uint32_t stg, int cwg, int warp, int lane) {
  const int wq = warp & 3;  // warp within the warpgroup
  int stage = 0;
  uint32_t phase = 0;
  float acc[BLOCK_N / 2];
  while (sched.next()) {
    const int nt0 = sched.n_tile() * BLOCK_N;
    // ragged last column tile: when <= 128 columns remain the MMAs run at half width (the columns beyond N are zero-
    // filled by TMA and never touch DRAM)
    const bool narrow = BLOCK_N == 256 && (p.N - nt0) <= BLOCK_N / 2;
    // (the tile width is chosen once per unit: a branch between wgmma shapes inside the k-loop makes ptxas serialise
    // the wgmma pipeline)
    if (BLOCK_N == 256 && narrow)
      mainloop<128, BLOCK_N, A_MN, B_MN>(sched, smem_tiles, full_bar, empty_bar, acc, cwg, lane, stage, phase);
    else
      mainloop<BLOCK_N, BLOCK_N, A_MN, B_MN>(sched, smem_tiles, full_bar, empty_bar, acc, cwg, lane, stage, phase);

    const int row_base = sched.m_tile() * BLOCK_M + cwg * 64 + wq * kRowsPerWarp;
    const int nrows = p.M - row_base > kRowsPerWarp ? kRowsPerWarp : p.M - row_base;
    const int fr = lane >> 2, fc = (lane & 3) * 2;  // accumulator fragment: rows fr / fr + 8, columns fc, fc + 1
#pragma unroll
    for (int ci = 0; ci < BLOCK_N / 32; ++ci) {
      const int col0 = nt0 + ci * 32;
      if (nrows <= 0 || col0 >= p.N) continue;  // warp-uniform
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const float* d = acc + 4 * (4 * ci + g);
        sts64(stg + (fr * kStgStride + 8 * g + fc) * 4, d[0], d[1]);
        sts64(stg + ((fr + 8) * kStgStride + 8 * g + fc) * 4, d[2], d[3]);
      }
      __syncwarp();
      epilogue_staged<EPI>(p, stg, row_base, nrows, col0, lane);
      __syncwarp();
    }
  }
}

template <int BLOCK_N, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ GemmParams p) {
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_tiles = smem;
  float* staging = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes + Cfg::kStagingBytes);
  uint64_t* full_bar = bars;             // [kStages]  TMA -> consumers
  uint64_t* empty_bar = bars + kStages;  // [kStages]  consumers (one arrive per warp) -> TMA

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kNumConsumerWGs * 4);
    }
    fence_barrier_init();
  }
  __syncthreads();

  UnitSched sched;
  sched.init(p, 1, static_cast<int>(gridDim.x), static_cast<int>(blockIdx.x));

  if (wg == 0) {
    // setmaxnreg sits at the top of each role branch and every warp of the warpgroup executes it
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == 0 && lane == 0) {
      // ===================== TMA producer =====================
      int stage = 0;
      uint32_t phase = 0;
      while (sched.next()) {
        const int m0 = sched.m_tile() * BLOCK_M;
        const int n0 = sched.n_tile() * BLOCK_N;
        for (int kb = sched.kb0; kb < sched.kb1; ++kb) {
          while (!mbar_try_wait(&empty_bar[stage], phase ^ 1)) {
          }
          uint8_t* sa = smem_tiles + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          const int k0 = kb * BLOCK_K;
          if constexpr (!A_MN) {
            tma_load_2d(&tmap_a, &full_bar[stage], sa, k0, m0);  // box {64 k, 128 rows}
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_M / 64; ++j)  // boxes {64 mn, 64 k}
              tma_load_2d(&tmap_a, &full_bar[stage], sa + j * (64 * BLOCK_K * 2), m0 + j * 64, k0);
          }
          if constexpr (!B_MN) {
            tma_load_2d(&tmap_b, &full_bar[stage], sb, k0, n0);  // box {64 k, BLOCK_N rows}
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_N / 64; ++j)
              tma_load_2d(&tmap_b, &full_bar[stage], sb + j * (64 * BLOCK_K * 2), n0 + j * 64, k0);
          }
          if (++stage == kStages) stage = 0, phase ^= 1;
        }
      }
    }
  } else {
    // ===================== consumers: MMA + epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int cwg = wg - 1;
    const uint32_t stg = smem_u32(staging) + (warp - 4) * kStgFloats * 4;
#define MDT_CONSUMER(E) \
  consumer_loop<E, BLOCK_N, A_MN, B_MN>(p, sched, smem_tiles, full_bar, empty_bar, stg, cwg, warp, lane)
    switch (p.epi) {
      case EPI_STORE: MDT_CONSUMER(EPI_STORE); break;
      case EPI_GELU: MDT_CONSUMER(EPI_GELU); break;
      case EPI_GATE_RESID: MDT_CONSUMER(EPI_GATE_RESID); break;
      case EPI_DGELU: MDT_CONSUMER(EPI_DGELU); break;
      default: MDT_CONSUMER(EPI_ATOMIC); break;
    }
#undef MDT_CONSUMER
  }
}

// ---------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(f);
  });
  return fn;
}

// 2-D bf16 tensor map: dims {inner, outer}, row stride ld elements, box {box_inner, box_outer}, 128B swizzle.
static int make_tmap(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                     uint32_t box_outer) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return MDT_ERR_DRIVER;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? MDT_OK : MDT_ERR_TMAP;
}

int make_head_tile_tmap(void* m, const void* ptr, unsigned long long dh, unsigned long long heads,
                        unsigned long long rows) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return MDT_ERR_DRIVER;
  if ((dh % 8) || (reinterpret_cast<uintptr_t>(ptr) & 15)) return MDT_ERR_ARG;
  cuuint64_t dims[3] = {dh, heads, rows};
  cuuint64_t strides[2] = {dh * 2, heads * dh * 2};
  cuuint32_t box[3] = {64, 1, 64};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(static_cast<CUtensorMap*>(m), CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? MDT_OK : MDT_ERR_TMAP;
}

extern int g_sm_budget;
static int g_num_sms = 0;
static int num_sms_device() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = kNumSMsDefault;
  }
  return g_num_sms;
}
// SMs the persistent grid is sized for: the device's, or the budget set by mdt_set_sm_budget
static int num_sms() {
  const int n = num_sms_device();
  if (g_sm_budget > 0 && g_sm_budget < n) return g_sm_budget;
  return n;
}

extern int g_gemm_last_config, g_gemm_configs_seen;
static thread_local GemmPlan* g_plan_out = nullptr;  // set by gemm_plan() around a gemm_launch() call
template <int BLOCK_N, bool A_MN, bool B_MN>
static int launch(const mdt_gemm_args& a, cudaStream_t stream) {
  using Cfg = GemmCfg<BLOCK_N>;
  GemmParams p;
  p.M = a.M, p.N = a.N, p.K = a.K;
  p.epi = a.epi, p.act = a.act;
  p.num_m_tiles = (a.M + BLOCK_M - 1) / BLOCK_M;
  p.num_n_tiles = (a.N + BLOCK_N - 1) / BLOCK_N;
  p.num_kb = (a.K + BLOCK_K - 1) / BLOCK_K;
  p.narrow_last = (BLOCK_N == 256 && p.num_n_tiles > 1 && (a.N - (p.num_n_tiles - 1) * BLOCK_N) <= BLOCK_N / 2) ? 1 : 0;
  p.out = a.out, p.ldo = a.ldo, p.out_fp32 = a.out_fp32;
  p.bias = a.bias;
  p.aux = a.aux, p.ld_aux = a.ld_aux;
  p.resid = a.resid, p.ld_resid = a.ld_resid;
  p.gate = a.gate, p.ld_gate = a.ld_gate, p.rows_per_group = a.rows_per_group > 0 ? a.rows_per_group : 1;
  p.colsum = a.epi == EPI_DGELU ? a.colsum : nullptr;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int groups = num_sms();  // CTAs resident at once (1 CTA per SM)
  // k-slices: only for the accumulate epilogue (fp32 red.add).  Units = tiles x slices are dealt round robin to the
  // CTAs, so a launch lasts ceil(units / CTAs) unit-times; a unit costs its k-blocks plus a fixed part (pipeline fill,
  // the tile's reduction epilogue: ~4 k-blocks' worth).  Pick the slice count that minimises
  // waves x (num_kb / slices + 4).  Deterministic mode (mdt_set_deterministic): one slice, so every output element
  // receives exactly one fp32 reduction per launch and its k order is fixed by the shape, whatever the SM count.
  int splits = 1;
  if (a.epi == EPI_ATOMIC && !g_deterministic) {
    double best = 0.0;
    for (int c = 1; c <= 32 && c <= p.num_kb; ++c) {
      const long long u = static_cast<long long>(tiles) * c;
      const double t = static_cast<double>((u + groups - 1) / groups) * (static_cast<double>(p.num_kb) / c + 4.0);
      if (c == 1 || t < best * 0.995) best = t, splits = c;  // ties and near-ties go to fewer slices (fewer reductions)
    }
  }
  p.streamk = splits;
  // half-width last column: paired tile order (locality) for the non-accumulating epilogues, LPT for the accumulating
  p.pair_halves = (p.narrow_last && a.epi != EPI_ATOMIC) ? 1 : 0;
  const long long units = gemm_units_per_slice(p) * splits;
  const int grid = static_cast<int>(units < groups ? units : groups);
  if (g_plan_out) {  // mdt_gemm_plan: report the decisions, launch nothing (no device, no driver needed)
    *g_plan_out = GemmPlan{BLOCK_N, 1, splits, p.pair_halves, p.narrow_last, p.num_m_tiles, p.num_n_tiles, p.num_kb,
                           units, grid};
    return MDT_OK;
  }
  if (grid <= 0) return MDT_OK;
  CUtensorMap ta, tb;
  int rc;
  // A: K-major stored [M, K] ld=lda -> dims {K, M}, box {64, 128}; MN-major stored [K, M] -> dims {M, K}, box {64, 64}
  rc = A_MN ? make_tmap(&ta, a.A, a.M, a.K, a.lda, 64, 64) : make_tmap(&ta, a.A, a.K, a.M, a.lda, 64, BLOCK_M);
  if (rc) return rc;
  rc = B_MN ? make_tmap(&tb, a.B, a.N, a.K, a.ldb, 64, 64) : make_tmap(&tb, a.B, a.K, a.N, a.ldb, 64, BLOCK_N);
  if (rc) return rc;
  auto kern = gemm_wgmma_kernel<BLOCK_N, A_MN, B_MN>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes) != cudaSuccess)
      return MDT_ERR_CUDA;
    attr_set = true;
  }
  kern<<<grid, kNumThreads, Cfg::kSmemBytes, stream>>>(ta, tb, p);
  g_gemm_last_config = BLOCK_N * 10 + 1;
  g_gemm_configs_seen |= 1 << ((BLOCK_N / 64 - 2) * 2);
  return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA;
}

int g_gemm_last_config = 0;   // BLOCK_N * 10 + 1 of the last launch (one CTA per tile)
int g_gemm_configs_seen = 0;  // bit (BLOCK_N/64 - 2) * 2 per instance launched since the last reset

template <bool A_MN, bool B_MN>
static int dispatch_n(const mdt_gemm_args& a, cudaStream_t stream) {
  // Tile width: 256 columns unless the problem is narrower (the epilogue and the per-tile pipeline fill are amortised
  // over the most MMA work per tile).
  int best = 256;
  if (a.N <= 128) best = 128;
  else if (a.N <= 192) best = 192;
  if (a.block_n == 128 || a.block_n == 192 || a.block_n == 256) best = a.block_n;
  switch (best) {
    case 256: return launch<256, A_MN, B_MN>(a, stream);
    case 192: return launch<192, A_MN, B_MN>(a, stream);
    default: return launch<128, A_MN, B_MN>(a, stream);
  }
}

int gemm_launch(const mdt_gemm_args& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return MDT_ERR_ARG;
  if ((a.lda % 8) || (a.ldb % 8)) return MDT_ERR_ARG;                                   // TMA: 16-byte row strides
  if ((reinterpret_cast<uintptr_t>(a.A) & 15) || (reinterpret_cast<uintptr_t>(a.B) & 15)) return MDT_ERR_ARG;
  if (a.epi == EPI_ATOMIC && !a.out_fp32) return MDT_ERR_ARG;
  if (a.epi == EPI_GATE_RESID && (!a.gate || !a.resid)) return MDT_ERR_ARG;
  if (a.epi == EPI_DGELU && !a.aux) return MDT_ERR_ARG;
  if (a.epi < EPI_STORE || a.epi > EPI_ATOMIC) return MDT_ERR_ARG;
  // vectorised epilogue accesses need 32-column chunks to start 16B-aligned
  if (a.ldo % 8) return MDT_ERR_ARG;
  if (a.a_mn && a.b_mn) return dispatch_n<true, true>(a, stream);
  if (!a.a_mn && a.b_mn) return dispatch_n<false, true>(a, stream);
  if (!a.a_mn && !a.b_mn) return dispatch_n<false, false>(a, stream);
  return MDT_ERR_ARG;  // (MN, K) is never needed by this path
}

int gemm_plan(const mdt_gemm_args& a, GemmPlan* out) {
  GemmPlan pl = {};
  g_plan_out = &pl;
  const int rc = gemm_launch(a, nullptr);
  g_plan_out = nullptr;
  if (rc == MDT_OK && out) *out = pl;
  return rc;
}

}  // namespace mdt
