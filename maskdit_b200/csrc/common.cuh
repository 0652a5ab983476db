// Shared device helpers for the maskdit_b200 sm_90a kernels: mbarrier, TMA, wgmma PTX wrappers,
// bf16 packing and warp reductions.  Everything here is inline PTX; no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define MDT_DEVINL __device__ __forceinline__

namespace mdt {

constexpr int kNumSMsDefault = 132;  // H100 SXM

// ----------------------------------------------------------------------------------------------
// Generic helpers
// ----------------------------------------------------------------------------------------------
MDT_DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

MDT_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
MDT_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

MDT_DEVINL uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
MDT_DEVINL float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
MDT_DEVINL float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
MDT_DEVINL float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

MDT_DEVINL float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// GELU(tanh) exactly as torch.nn.GELU(approximate="tanh") (reference models/maskdit.py:181)
// (written as the shortest FMA chains: 6 / 10 instructions incl. MUFU.TANH - the GEMM epilogues that apply them run
// on two warps per scheduler and are bound by their instruction count)
MDT_DEVINL float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k01 = 0.7978845608028654f * 0.044715f;
  const float u = x * fmaf(x * x, k01, k0);
  const float hx = 0.5f * x;
  return fmaf(hx, tanh_fast(u), hx);
}
MDT_DEVINL float gelu_tanh_grad(float x) {
  const float k0 = 0.7978845608028654f, k01 = 0.7978845608028654f * 0.044715f;
  const float x2 = x * x;
  const float t = tanh_fast(x * fmaf(x2, k01, k0));
  const float du = fmaf(x2, 3.f * k01, k0);
  // 0.5 (1 + t) + 0.5 x (1 - t^2) du
  return fmaf((0.5f * x) * du, fmaf(-t, t, 1.f), fmaf(0.5f, t, 0.5f));
}
// 2^x as ONE MUFU.EX2 (ex2.approx.ftz, 2 ulp): exp2f() wraps the same instruction in a denormal-range rescale
// (4 more instructions per element; ncu r01: 43 % of all instructions of the attention forward).  Softmax arguments
// are <= 0 and results below 2^-126 flush to zero, which bf16 P cannot represent anyway.
MDT_DEVINL float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
MDT_DEVINL float silu(float x) { return x / (1.f + __expf(-x)); }
MDT_DEVINL float silu_grad(float x) {
  float s = 1.f / (1.f + __expf(-x));
  return s * (1.f + x * (1.f - s));
}

// explicit shared-state-space vector accesses (pointers carved out of the dynamic smem blob via integer casts
// degrade to generic LD/ST otherwise)
MDT_DEVINL void sts128(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
MDT_DEVINL float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
MDT_DEVINL float lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// explicit global-state-space accesses for pointers that arrive as void* kernel parameters (generic LD/ST/ATOM
// otherwise: the compiler cannot prove the address space)
MDT_DEVINL uint64_t gaddr(const void* p) { return static_cast<uint64_t>(__cvta_generic_to_global(p)); }
MDT_DEVINL void stg128(uint64_t a, float4 v) {
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
MDT_DEVINL void stg64(uint64_t a, uint2 v) {
  asm volatile("st.global.v2.b32 [%0], {%1, %2};" ::"l"(a), "r"(v.x), "r"(v.y) : "memory");
}
// streaming variants (evict-first in L2): epilogue traffic that is touched once must not push the GEMM's A panels out
MDT_DEVINL void stg128_cs(uint64_t a, float4 v) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
MDT_DEVINL void stg64_cs(uint64_t a, uint2 v) {
  asm volatile("st.global.cs.v2.b32 [%0], {%1, %2};" ::"l"(a), "r"(v.x), "r"(v.y) : "memory");
}
MDT_DEVINL float4 ldg128_cs(uint64_t a) {
  float4 v;
  asm volatile("ld.global.cs.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(a) : "memory");
  return v;
}
MDT_DEVINL float4 ldg128(uint64_t a) {
  float4 v;
  asm volatile("ld.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(a) : "memory");
  return v;
}
MDT_DEVINL float4 ldg128_nc(uint64_t a) {
  float4 v;
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(a));
  return v;
}
MDT_DEVINL uint2 ldg64_nc(uint64_t a) {
  uint2 v;
  asm volatile("ld.global.nc.v2.b32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(a));
  return v;
}
MDT_DEVINL void red_add_v4(uint64_t a, float4 v) {  // one 16-byte fp32 reduction (REDG.E.ADD.F32x4)
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
MDT_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
MDT_DEVINL void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
MDT_DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

MDT_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
MDT_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
MDT_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (launch failure) instead of hanging the GPU box.  The slow path is kept out of
// line so that the hot loops stay small in the instruction cache.
static __device__ __noinline__ void mbar_wait_slow(uint64_t* bar, uint32_t parity) {
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {  // ~2 s at 2 GHz
      printf("mdt: mbarrier timeout block %d thread %d\n", blockIdx.x, threadIdx.x);
      __trap();
    }
  }
}
MDT_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  if (mbar_try_wait(bar, parity)) return;
  mbar_wait_slow(bar, parity);
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor)
// ----------------------------------------------------------------------------------------------
MDT_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
MDT_DEVINL void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* smem_dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// L2 cache-policy operands for TMA loads (the fixed encodings CUTLASS uses, cute/arch/copy_sm90_desc.hpp)
constexpr uint64_t kL2EvictNormal = 0x1000000000000000ull, kL2EvictFirst = 0x12F0000000000000ull,
                   kL2EvictLast = 0x14F0000000000000ull;
MDT_DEVINL void tma_load_2d_hint(const CUtensorMap* m, uint64_t* bar, void* smem_dst, int c0, int c1, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], "
      "[%2], %5;" ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "l"(hint)
      : "memory");
}

MDT_DEVINL void tma_load_4d(const CUtensorMap* m, uint64_t* bar, uint32_t smem_dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// smem -> global bulk tensor store (bulk async-group completion)
MDT_DEVINL void tma_store_4d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
MDT_DEVINL void tma_store_2d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
MDT_DEVINL void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
MDT_DEVINL void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }  // smem reusable
MDT_DEVINL void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }            // writes done

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a)
// ----------------------------------------------------------------------------------------------
MDT_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
MDT_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
MDT_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Shared-memory matrix descriptor of sm_90 (cute::GMMA::DescriptorIterator bit layout):
//  [0,14) start address >> 4 | [16,30) leading byte offset >> 4 | [32,46) stride byte offset >> 4 |
//  [49,52) base offset (0: tiles are 1024-byte aligned) | [62,64) layout type (1 = SWIZZLE_128B)
MDT_DEVINL uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3fffu);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3fffu) << 32;
  d |= 1ull << 62;
  return d;
}

}  // namespace mdt
