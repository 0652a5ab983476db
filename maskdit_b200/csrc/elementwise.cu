// HBM-bound side kernels of the MaskDiT path: mask index path, patch embedding, conditioning pointwise ops,
// LayerNorm+modulate (fwd/bwd), gate/residual backward, unmask scatter/gather, column sums.
// All are coalesced, 8/16-byte vectorised streaming kernels with warp-level reductions; none has data reuse that
// would justify smem tiling (guide: elementwise/reduction kernels are fixed by fusion + vector width).
#include "common.cuh"
#include "deterministic.h"
#include "../../include/maskdit_b200.h"

namespace mdt {

static inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }
static inline int launch_status() { return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA; }

// =========================================================================================================
// get_mask (models/maskdit.py:88-113): rank-by-counting, ties by ascending index == stable argsort.
// One block per batch row; noise row staged in smem; each thread ranks its elements against the row.
// =========================================================================================================
__global__ void mask_indices_kernel(const float* __restrict__ noise, int L, int len_keep,
                                    int64_t* __restrict__ ids_keep, int64_t* __restrict__ ids_restore,
                                    float* __restrict__ mask) {
  extern __shared__ float s_noise[];
  const int b = blockIdx.x;
  const float* row = noise + static_cast<size_t>(b) * L;
  for (int i = threadIdx.x; i < L; i += blockDim.x) s_noise[i] = row[i];
  __syncthreads();
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const float v = s_noise[i];
    int rank = 0;
    for (int j = 0; j < L; ++j) {
      const float u = s_noise[j];
      rank += (u < v) || (u == v && j < i);
    }
    ids_restore[static_cast<size_t>(b) * L + i] = rank;
    mask[static_cast<size_t>(b) * L + i] = rank >= len_keep ? 1.f : 0.f;
    if (rank < len_keep) ids_keep[static_cast<size_t>(b) * len_keep + rank] = i;
  }
}

// =========================================================================================================
// PatchEmbed (+c_in, +pos_embed, +kept-token gather).  Block = kPeTok tokens of one sample, threads over D.
// =========================================================================================================
constexpr int kPeTok = 32;   // tokens per block: the weight row of a channel (C*p*p floats) is read once per 32 tokens
constexpr int kPeMaxCpp = 48 * 1024 / (kPeTok * 4);   // 384: the [kPeTok][cpp] patch block within 48 KB of smem
__global__ void patch_embed_kernel(const float* __restrict__ x, const float* __restrict__ sigma, float sigma_data,
                                   const float* __restrict__ W, const float* __restrict__ bias,
                                   const float* __restrict__ pos, const int64_t* __restrict__ ids_keep,
                                   float* __restrict__ out, int C, int R, int p, int D, int T) {
  extern __shared__ float s_patch[];  // [kPeTok][C*p*p]
  __shared__ int s_tok[kPeTok];
  const int cpp = C * p * p, G = R / p;
  const int b = blockIdx.y, i0 = blockIdx.x * kPeTok;
  const float c_in = sigma ? rsqrtf(sigma_data * sigma_data + sigma[b] * sigma[b]) : 1.f;
  for (int e = threadIdx.x; e < kPeTok * cpp; e += blockDim.x) {
    const int ti = e / cpp, j = e % cpp;
    const int i = i0 + ti;
    float v = 0.f;
    if (i < T) {
      const int tok = ids_keep ? static_cast<int>(ids_keep[static_cast<size_t>(b) * T + i]) : i;
      if (j == 0) s_tok[ti] = tok;
      const int c = j / (p * p), ph = (j / p) % p, pw = j % p;
      const int hh = (tok / G) * p + ph, ww = (tok % G) * p + pw;
      v = c_in * x[((static_cast<size_t>(b) * C + c) * R + hh) * R + ww];
    }
    s_patch[e] = v;
  }
  __syncthreads();
  const int nt = min(kPeTok, T - i0);
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const float* w = W + static_cast<size_t>(d) * cpp;
    const float bd = bias[d];
    if (cpp == 16) {  // patch 2 x 4 channels (every shipped config): the weight row lives in registers
      float wr[16];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(w) + q);
        wr[4 * q] = v.x, wr[4 * q + 1] = v.y, wr[4 * q + 2] = v.z, wr[4 * q + 3] = v.w;
      }
      for (int t = 0; t < nt; ++t) {
        float acc = bd;
        const float4* sp = reinterpret_cast<const float4*>(s_patch + t * 16);  // smem broadcast reads
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 v = sp[q];
          acc = fmaf(wr[4 * q], v.x, acc), acc = fmaf(wr[4 * q + 1], v.y, acc);
          acc = fmaf(wr[4 * q + 2], v.z, acc), acc = fmaf(wr[4 * q + 3], v.w, acc);
        }
        out[(static_cast<size_t>(b) * T + i0 + t) * D + d] = acc + pos[static_cast<size_t>(s_tok[t]) * D + d];
      }
    } else {
      for (int t = 0; t < nt; ++t) {
        float acc = bd;
        for (int j = 0; j < cpp; ++j) acc = fmaf(__ldg(w + j), s_patch[t * cpp + j], acc);
        out[(static_cast<size_t>(b) * T + i0 + t) * D + d] = acc + pos[static_cast<size_t>(s_tok[t]) * D + d];
      }
    }
  }
}

// gW[d, j] += sum_tokens g[tok, d] * patch[tok, j]; gb[d] += sum g.  Block = kPebTok tokens of one sample.
// kPebTok = 128 tokens per block (one atomic per (channel, weight) per block) for cpp <= 96 (patch 2 and 4 at 4
// channels); 32 for cpp <= 384 (patch 8: cpp = 256), so the [kPebTok][cpp] patch block stays within 48 KB of smem.
constexpr int kPebMaxCpp = 48 * 1024 / (32 * 4);
// kStore (deterministic mode): the block's sums are stored, not added, into its own row of per-block partials
// (gW -> [blocks, D * cpp], gb -> [blocks, D]); colsum_ordered reduces the rows afterwards.
template <int kPebTok, bool kStore>
__device__ __forceinline__ void patch_embed_bwd_body(const float* __restrict__ x, const float* __restrict__ sigma,
                                                     float sigma_data, const int64_t* __restrict__ ids_keep,
                                                     const float* __restrict__ g, float* __restrict__ gW,
                                                     float* __restrict__ gb, int C, int R, int p, int D, int T) {
  extern __shared__ float s_patch[];  // [kPebTok][cpp]
  const int cpp = C * p * p, G = R / p;
  const int b = blockIdx.y, i0 = blockIdx.x * kPebTok;
  const int nt = min(kPebTok, T - i0);
  const float c_in = sigma ? rsqrtf(sigma_data * sigma_data + sigma[b] * sigma[b]) : 1.f;
  for (int e = threadIdx.x; e < nt * cpp; e += blockDim.x) {
    const int ti = e / cpp, j = e % cpp;
    const int i = i0 + ti;
    const int tok = ids_keep ? static_cast<int>(ids_keep[static_cast<size_t>(b) * T + i]) : i;
    const int c = j / (p * p), ph = (j / p) % p, pw = j % p;
    const int hh = (tok / G) * p + ph, ww = (tok % G) * p + pw;
    s_patch[e] = c_in * x[((static_cast<size_t>(b) * C + c) * R + hh) * R + ww];
  }
  __syncthreads();
  if (kStore) {
    const size_t blk = static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x;
    gW += blk * D * cpp, gb += blk * D;
  }
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float sb = 0.f;
    // cpp is processed in slabs of 16 accumulators to bound registers (cpp = 16 for patch 2, C 4)
    for (int j0 = 0; j0 < cpp; j0 += 16) {
      float acc[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] = 0.f;
      for (int t = 0; t < nt; ++t) {
        const float gv = g[(static_cast<size_t>(b) * T + i0 + t) * D + d];
        if (j0 == 0) sb += gv;
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (j0 + j < cpp) acc[j] = fmaf(gv, s_patch[t * cpp + j0 + j], acc[j]);
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        if (j0 + j >= cpp) continue;
        if (kStore) gW[static_cast<size_t>(d) * cpp + j0 + j] = acc[j];
        else atomicAdd(gW + static_cast<size_t>(d) * cpp + j0 + j, acc[j]);
      }
    }
    if (kStore) gb[d] = sb;
    else atomicAdd(gb + d, sb);
  }
}
template <int kPebTok>
__global__ void patch_embed_bwd_kernel(const float* __restrict__ x, const float* __restrict__ sigma,
                                       float sigma_data, const int64_t* __restrict__ ids_keep,
                                       const float* __restrict__ g, float* __restrict__ gW, float* __restrict__ gb,
                                       int C, int R, int p, int D, int T) {
  patch_embed_bwd_body<kPebTok, false>(x, sigma, sigma_data, ids_keep, g, gW, gb, C, R, p, D, T);
}
template <int kPebTok>
__global__ void patch_embed_bwd_partial_kernel(const float* __restrict__ x, const float* __restrict__ sigma,
                                               float sigma_data, const int64_t* __restrict__ ids_keep,
                                               const float* __restrict__ g, float* __restrict__ pW,
                                               float* __restrict__ pb, int C, int R, int p, int D, int T) {
  patch_embed_bwd_body<kPebTok, true>(x, sigma, sigma_data, ids_keep, g, pW, pb, C, R, p, D, T);
}

// =========================================================================================================
// Conditioning pointwise ops
// =========================================================================================================
// kPrecond: MDT_PRECOND_EDM reads sigma and embeds c_noise = ln(sigma) / 4; MDT_PRECOND_FLOW reads the flow time t and
// embeds c_noise = t (SiT).
template <int kPrecond>
__global__ void timestep_freq_kernel(const float* __restrict__ sigma, int B, int dim,
                                     __nv_bfloat16* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (idx >= B * half) return;
  const int b = idx / half, k = idx % half;
  const float t = kPrecond == MDT_PRECOND_FLOW ? sigma[b] : logf(sigma[b]) * 0.25f;  // c_noise, models/maskdit.py:767
  const float f = expf(-logf(10000.f) * static_cast<float>(k) / static_cast<float>(half));
  const float a = t * f;
  out[static_cast<size_t>(b) * dim + k] = __float2bfloat16_rn(cosf(a));
  out[static_cast<size_t>(b) * dim + half + k] = __float2bfloat16_rn(sinf(a));
}

__global__ void silu_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ sum,
                            __nv_bfloat16* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float v = a[i] + (b ? b[i] : 0.f);
    if (sum) sum[i] = v;
    out[i] = __float2bfloat16_rn(silu(v));
  }
}
__global__ void silu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dx32,
                                __nv_bfloat16* __restrict__ dx16, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float v = dy[i] * silu_grad(x[i]);
    if (dx32) dx32[i] = v;
    if (dx16) dx16[i] = __float2bfloat16_rn(v);
  }
}
__global__ void cast_f32_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, long long n) {
  const long long n4 = n >> 2;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const float4* in4 = reinterpret_cast<const float4*>(in);
  uint2* out2 = reinterpret_cast<uint2*>(out);
  for (long long i = t; i < n4; i += stride) {
    float4 v = in4[i];
    out2[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
  }
  for (long long i = (n4 << 2) + t; i < n; i += stride) out[i] = __float2bfloat16_rn(in[i]);
}

// Column sums.  Thread owns 2 adjacent columns; block = 128 threads (256 columns) x a chunk of rows.
constexpr int kCsRows = 256;
__global__ void colsum_bf16_kernel(const __nv_bfloat16* __restrict__ in, int M, int N, int ld,
                                   float* __restrict__ out) {
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (c >= N) return;
  const int r0 = blockIdx.y * kCsRows, r1 = min(M, r0 + kCsRows);
  float s0 = 0.f, s1 = 0.f;
  if (c + 1 < N) {
    for (int r = r0; r < r1; ++r) {
      const uint32_t v = *reinterpret_cast<const uint32_t*>(in + static_cast<size_t>(r) * ld + c);
      s0 += bf16_lo(v), s1 += bf16_hi(v);
    }
    atomicAdd(out + c, s0);
    atomicAdd(out + c + 1, s1);
  } else {
    for (int r = r0; r < r1; ++r) s0 += __bfloat162float(in[static_cast<size_t>(r) * ld + c]);
    atomicAdd(out + c, s0);
  }
}
__global__ void colsum_f32_kernel(const float* __restrict__ in, int M, int N, int ld, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  const int r0 = blockIdx.y * kCsRows, r1 = min(M, r0 + kCsRows);
  float s = 0.f;
  for (int r = r0; r < r1; ++r) s += in[static_cast<size_t>(r) * ld + c];
  atomicAdd(out + c, s);
}

// Column sums in a fixed order (deterministic mode).  Block = one strip of kCoCols columns and ALL rows: row lane w
// sums rows w, w + kCoLanes, ... in ascending order, then one thread per column adds the lanes' sums in lane order and
// adds the total to out[c] (the address's only write in the launch).  The order depends on M alone.
constexpr int kCoCols = 32, kCoLanes = 32, kCoUnroll = 8;
MDT_DEVINL float load_f32(const float* p) { return __ldg(p); }
MDT_DEVINL float load_f32(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T>
__global__ void __launch_bounds__(kCoCols * kCoLanes)
colsum_ordered_kernel(const T* __restrict__ in, int M, int N, long long ld, float* __restrict__ out) {
  __shared__ float s_part[kCoLanes][kCoCols + 1];
  const int tx = threadIdx.x % kCoCols, lane = threadIdx.x / kCoCols;
  const int c = blockIdx.x * kCoCols + tx;
  float s = 0.f;
  if (c < N) {
    const T* col = in + c;
    int r = lane;
    // kCoUnroll independent loads in flight, added in row order
    for (; r + (kCoUnroll - 1) * kCoLanes < M; r += kCoUnroll * kCoLanes) {
      float v[kCoUnroll];
#pragma unroll
      for (int u = 0; u < kCoUnroll; ++u) v[u] = load_f32(col + static_cast<long long>(r + u * kCoLanes) * ld);
#pragma unroll
      for (int u = 0; u < kCoUnroll; ++u) s += v[u];
    }
    for (; r < M; r += kCoLanes) s += load_f32(col + static_cast<long long>(r) * ld);
  }
  s_part[lane][tx] = s;
  __syncthreads();
  if (lane == 0 && c < N) {
    float t = s_part[0][tx];
    for (int w = 1; w < kCoLanes; ++w) t += s_part[w][tx];
    out[c] += t;
  }
}

// =========================================================================================================
// Deterministic mode (mdt_set_deterministic): the process-wide setting and the ordered reduction every variant ends in
// =========================================================================================================
int g_deterministic = 0;

int colsum_ordered(const void* in, int in_bf16, int M, int N, long long ld, float* out, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return MDT_OK;
  const int grid = (N + kCoCols - 1) / kCoCols;
  if (in_bf16)
    colsum_ordered_kernel<<<grid, kCoCols * kCoLanes, 0, stream>>>(static_cast<const __nv_bfloat16*>(in), M, N, ld, out);
  else
    colsum_ordered_kernel<<<grid, kCoCols * kCoLanes, 0, stream>>>(static_cast<const float*>(in), M, N, ld, out);
  return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA;
}

// =========================================================================================================
// LayerNorm (no affine) + modulate.  One warp per row; the row lives in registers (NV float4 per lane).
// =========================================================================================================
template <int NV>
__global__ void __launch_bounds__(256)
ln_modulate_kernel(const float* __restrict__ x, const float* __restrict__ shift, const float* __restrict__ scale,
                   int ld_mod, int rows_per_group, __nv_bfloat16* __restrict__ out, float* __restrict__ mean_out,
                   float* __restrict__ rstd_out, int M, float eps) {
  constexpr int D = NV * 128;
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    v[k] = xr[lane + 32 * k];
    s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
  }
  const float mean = warp_sum(s) * (1.f / D);
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const float a = v[k].x - mean, b = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  const size_t mo = static_cast<size_t>(row / rows_per_group) * ld_mod;
  const float4* sh = reinterpret_cast<const float4*>(shift + mo);
  const float4* sc = reinterpret_cast<const float4*>(scale + mo);
  uint2* o = reinterpret_cast<uint2*>(out + static_cast<size_t>(row) * D);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const float4 a = sh[lane + 32 * k], c = sc[lane + 32 * k];
    const float y0 = fmaf((v[k].x - mean) * rstd, 1.f + c.x, a.x);
    const float y1 = fmaf((v[k].y - mean) * rstd, 1.f + c.y, a.y);
    const float y2 = fmaf((v[k].z - mean) * rstd, 1.f + c.z, a.z);
    const float y3 = fmaf((v[k].w - mean) * rstd, 1.f + c.w, a.w);
    o[lane + 32 * k] = make_uint2(pack_bf16(y0, y1), pack_bf16(y2, y3));
  }
}

// Backward.  Block = 4 warps = kLnbRows = gcd(rows_per_group, 32) consecutive rows of ONE sample;
// each warp walks kLnbRows/4 rows keeping the dshift/dscale partial sums of its columns in registers, the block
// combines them through smem and issues one set of atomics.
constexpr int kLnbRowsMax = 32;
static inline int gcd_int(int a, int b) { while (b) { int t = a % b; a = b; b = t; } return a; }
template <int NV>
__global__ void __launch_bounds__(128)
ln_modulate_bwd_kernel(const __nv_bfloat16* __restrict__ dxmod, const float* __restrict__ x,
                       const float* __restrict__ mean, const float* __restrict__ rstd,
                       const float* __restrict__ scale, int ld_mod, int rows_per_group, float* __restrict__ g,
                       int accumulate, float* __restrict__ dshift, float* __restrict__ dscale, int ld_dmod, int M,
                       int kLnbRows) {
  constexpr int D = NV * 128;
  __shared__ float s_red[2 * D];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row0 = blockIdx.x * kLnbRows;
  const int b = row0 / rows_per_group;
  for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) s_red[i] = 0.f;
  __syncthreads();
  float4 sc1[NV];  // 1 + scale
  {
    const float4* sc = reinterpret_cast<const float4*>(scale + static_cast<size_t>(b) * ld_mod);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      float4 c = sc[lane + 32 * k];
      sc1[k] = make_float4(1.f + c.x, 1.f + c.y, 1.f + c.z, 1.f + c.w);
    }
  }
  float4 a_sh[NV], a_sc[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) a_sh[k] = make_float4(0, 0, 0, 0), a_sc[k] = make_float4(0, 0, 0, 0);

  for (int r = warp; r < kLnbRows; r += 4) {
    const int row = row0 + r;
    if (row >= M) break;
    const float mu = mean[row], rs = rstd[row];
    const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
    const uint2* dr = reinterpret_cast<const uint2*>(dxmod + static_cast<size_t>(row) * D);
    float4 xh[NV], dy[NV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const float4 xv = xr[lane + 32 * k];
      const uint2 dv = dr[lane + 32 * k];
      const float4 d = make_float4(bf16_lo(dv.x), bf16_hi(dv.x), bf16_lo(dv.y), bf16_hi(dv.y));
      xh[k] = make_float4((xv.x - mu) * rs, (xv.y - mu) * rs, (xv.z - mu) * rs, (xv.w - mu) * rs);
      a_sh[k].x += d.x, a_sh[k].y += d.y, a_sh[k].z += d.z, a_sh[k].w += d.w;
      a_sc[k].x = fmaf(d.x, xh[k].x, a_sc[k].x), a_sc[k].y = fmaf(d.y, xh[k].y, a_sc[k].y);
      a_sc[k].z = fmaf(d.z, xh[k].z, a_sc[k].z), a_sc[k].w = fmaf(d.w, xh[k].w, a_sc[k].w);
      dy[k] = make_float4(d.x * sc1[k].x, d.y * sc1[k].y, d.z * sc1[k].z, d.w * sc1[k].w);
      s1 += (dy[k].x + dy[k].y) + (dy[k].z + dy[k].w);
      s2 += (dy[k].x * xh[k].x + dy[k].y * xh[k].y) + (dy[k].z * xh[k].z + dy[k].w * xh[k].w);
    }
    s1 = warp_sum(s1) * (1.f / D);
    s2 = warp_sum(s2) * (1.f / D);
    float4* gr = reinterpret_cast<float4*>(g + static_cast<size_t>(row) * D);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      float4 o;
      o.x = rs * (dy[k].x - s1 - xh[k].x * s2);
      o.y = rs * (dy[k].y - s1 - xh[k].y * s2);
      o.z = rs * (dy[k].z - s1 - xh[k].z * s2);
      o.w = rs * (dy[k].w - s1 - xh[k].w * s2);
      if (accumulate) {
        const float4 p = gr[lane + 32 * k];
        o.x += p.x, o.y += p.y, o.z += p.z, o.w += p.w;
      }
      gr[lane + 32 * k] = o;
    }
  }
  // block reduction of the modulation gradients
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = (lane + 32 * k) * 4;
    atomicAdd(&s_red[c + 0], a_sh[k].x), atomicAdd(&s_red[c + 1], a_sh[k].y);
    atomicAdd(&s_red[c + 2], a_sh[k].z), atomicAdd(&s_red[c + 3], a_sh[k].w);
    atomicAdd(&s_red[D + c + 0], a_sc[k].x), atomicAdd(&s_red[D + c + 1], a_sc[k].y);
    atomicAdd(&s_red[D + c + 2], a_sc[k].z), atomicAdd(&s_red[D + c + 3], a_sc[k].w);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    atomicAdd(dshift + static_cast<size_t>(b) * ld_dmod + i, s_red[i]);
    atomicAdd(dscale + static_cast<size_t>(b) * ld_dmod + i, s_red[D + i]);
  }
}

// =========================================================================================================
// gate backward: dy = g * gate (bf16), dgate[b,:] += sum_t g*y, dbias[:] += sum dy.
// Thread owns 4 adjacent columns; block = D/4 threads x kGbRows rows of one sample.
// =========================================================================================================
constexpr int kGbRowsMax = 32;
__global__ void gate_bwd_kernel(const float* __restrict__ g, const __nv_bfloat16* __restrict__ y,
                                const float* __restrict__ gate, int ld_gate, int rows_per_group,
                                __nv_bfloat16* __restrict__ dy, float* __restrict__ dgate, int ld_dgate,
                                float* __restrict__ dbias, int M, int D, int kGbRows) {
  const int c = threadIdx.x * 4;
  if (c >= D) return;
  const int row0 = blockIdx.x * kGbRows;
  const int b = row0 / rows_per_group;
  const float4 gt = *reinterpret_cast<const float4*>(gate + static_cast<size_t>(b) * ld_gate + c);
  float4 ag = make_float4(0, 0, 0, 0), ab = make_float4(0, 0, 0, 0);
  const int r1 = min(M, row0 + kGbRows);
  // 8 rows per trip, all loads issued before the first dependent store (in-order issue: a load->store dependency per
  // row would expose the HBM latency every iteration; v1 of this kernel reached only 53 % of the HBM roofline)
  for (int r = row0; r < r1; r += 8) {
    float4 gv[8];
    uint2 yv[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (r + u < r1) {
        gv[u] = __ldcs(reinterpret_cast<const float4*>(g + static_cast<size_t>(r + u) * D + c));
        yv[u] = __ldcs(reinterpret_cast<const uint2*>(y + static_cast<size_t>(r + u) * D + c));
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (r + u < r1) {
        const float4 d = make_float4(gv[u].x * gt.x, gv[u].y * gt.y, gv[u].z * gt.z, gv[u].w * gt.w);
        *reinterpret_cast<uint2*>(dy + static_cast<size_t>(r + u) * D + c) =
            make_uint2(pack_bf16(d.x, d.y), pack_bf16(d.z, d.w));
        ag.x = fmaf(gv[u].x, bf16_lo(yv[u].x), ag.x), ag.y = fmaf(gv[u].y, bf16_hi(yv[u].x), ag.y);
        ag.z = fmaf(gv[u].z, bf16_lo(yv[u].y), ag.z), ag.w = fmaf(gv[u].w, bf16_hi(yv[u].y), ag.w);
        ab.x += d.x, ab.y += d.y, ab.z += d.z, ab.w += d.w;
      }
    }
  }
  float* dg = dgate + static_cast<size_t>(b) * ld_dgate + c;
  atomicAdd(dg + 0, ag.x), atomicAdd(dg + 1, ag.y), atomicAdd(dg + 2, ag.z), atomicAdd(dg + 3, ag.w);
  if (dbias) {
    atomicAdd(dbias + c + 0, ab.x), atomicAdd(dbias + c + 1, ab.y);
    atomicAdd(dbias + c + 2, ab.z), atomicAdd(dbias + c + 3, ab.w);
  }
}

// =========================================================================================================
// LN-modulate backward FUSED with the gate backward that consumes its result.  In the block backward every LN
// backward (which finishes the residual-stream gradient g) is followed by the gate backward of the next branch, which
// re-reads all of g: fusing the two removes that 4 B/element read and a launch (22 -> 18 B/element for the pair).
// Column-owner layout (thread = 4 adjacent columns, block = D/4 threads x rows_per_block rows of one sample): the
// per-column reductions (dshift, dscale, dgate, dbias) stay in 16 registers; the two per-row LN statistics are
// block-reduced for 4 rows at a time (warp shuffles + one __syncthreads per batch, smem double-buffered by parity).
// =========================================================================================================
constexpr int kLgBatch = 4;
constexpr int kLgMaxThreads = 320;  // D <= 1280
// kBiasRows (deterministic mode, one block per sample): the block's bias-gradient sum is stored into row b of dbias
// ([samples, D] scratch) instead of being added to dbias[:]; colsum_ordered reduces the rows afterwards.
template <bool GATE, bool kBiasRows>
__device__ __forceinline__ void ln_bwd_gate_body(
    const __nv_bfloat16* __restrict__ dxmod, const float* __restrict__ x, const float* __restrict__ mean,
    const float* __restrict__ rstd, const float* __restrict__ scale, int ld_mod, int rows_per_group,
    float* __restrict__ g, int accumulate, float* __restrict__ dshift, float* __restrict__ dscale, int ld_dmod,
    const __nv_bfloat16* __restrict__ y, const float* __restrict__ gate, int ld_gate, __nv_bfloat16* __restrict__ dy,
    float* __restrict__ dgate, int ld_dgate, float* __restrict__ dbias, int M, int D, int rows_per_block) {
  __shared__ float4 s_part[2][kLgMaxThreads / 32][2];  // [parity][warp][{s1 x4}, {s2 x4}]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int c = tid * 4;
  const int row0 = blockIdx.x * rows_per_block;
  const int r_end = min(M, row0 + rows_per_block);
  const int b = row0 / rows_per_group;
  const float inv_d = 1.f / D;
  float4 sc1 = ldg128_nc(gaddr(scale + static_cast<size_t>(b) * ld_mod + c));
  sc1.x += 1.f, sc1.y += 1.f, sc1.z += 1.f, sc1.w += 1.f;
  float4 gt = make_float4(0, 0, 0, 0);
  if (GATE) gt = ldg128_nc(gaddr(gate + static_cast<size_t>(b) * ld_gate + c));
  float4 a_sh = make_float4(0, 0, 0, 0), a_sc = a_sh, ag = a_sh, ab = a_sh;
  int parity = 0;
  for (int r = row0; r < r_end; r += kLgBatch, parity ^= 1) {
    uint2 dv[kLgBatch], yv[kLgBatch];
    float4 xv[kLgBatch], gv[kLgBatch];
    float mu[kLgBatch], rs[kLgBatch];
#pragma unroll
    for (int j = 0; j < kLgBatch; ++j) {
      const bool ok = r + j < r_end;
      const size_t e = static_cast<size_t>(r + j) * D + c;
      dv[j] = ok ? ldg64_nc(gaddr(dxmod + e)) : make_uint2(0, 0);
      xv[j] = ok ? ldg128_nc(gaddr(x + e)) : make_float4(0, 0, 0, 0);
      gv[j] = (ok && accumulate) ? ldg128(gaddr(g + e)) : make_float4(0, 0, 0, 0);
      if (GATE) yv[j] = ok ? ldg64_nc(gaddr(y + e)) : make_uint2(0, 0);
      mu[j] = ok ? mean[r + j] : 0.f;
      rs[j] = ok ? rstd[r + j] : 0.f;
    }
    float s1[kLgBatch], s2[kLgBatch];
#pragma unroll
    for (int j = 0; j < kLgBatch; ++j) {
      const float4 d = make_float4(bf16_lo(dv[j].x), bf16_hi(dv[j].x), bf16_lo(dv[j].y), bf16_hi(dv[j].y));
      const float4 xh = make_float4((xv[j].x - mu[j]) * rs[j], (xv[j].y - mu[j]) * rs[j], (xv[j].z - mu[j]) * rs[j],
                                    (xv[j].w - mu[j]) * rs[j]);
      xv[j] = xh;
      a_sh.x += d.x, a_sh.y += d.y, a_sh.z += d.z, a_sh.w += d.w;
      a_sc.x = fmaf(d.x, xh.x, a_sc.x), a_sc.y = fmaf(d.y, xh.y, a_sc.y);
      a_sc.z = fmaf(d.z, xh.z, a_sc.z), a_sc.w = fmaf(d.w, xh.w, a_sc.w);
      const float4 t = make_float4(d.x * sc1.x, d.y * sc1.y, d.z * sc1.z, d.w * sc1.w);
      s1[j] = (t.x + t.y) + (t.z + t.w);
      s2[j] = (t.x * xh.x + t.y * xh.y) + (t.z * xh.z + t.w * xh.w);
    }
#pragma unroll
    for (int j = 0; j < kLgBatch; ++j) s1[j] = warp_sum(s1[j]), s2[j] = warp_sum(s2[j]);
    if (lane == 0) {
      s_part[parity][warp][0] = make_float4(s1[0], s1[1], s1[2], s1[3]);
      s_part[parity][warp][1] = make_float4(s2[0], s2[1], s2[2], s2[3]);
    }
    __syncthreads();
    float4 t1 = make_float4(0, 0, 0, 0), t2 = t1;
    for (int w = 0; w < nwarps; ++w) {
      const float4 p1 = s_part[parity][w][0], p2 = s_part[parity][w][1];
      t1.x += p1.x, t1.y += p1.y, t1.z += p1.z, t1.w += p1.w;
      t2.x += p2.x, t2.y += p2.y, t2.z += p2.z, t2.w += p2.w;
    }
    s1[0] = t1.x, s1[1] = t1.y, s1[2] = t1.z, s1[3] = t1.w;
    s2[0] = t2.x, s2[1] = t2.y, s2[2] = t2.z, s2[3] = t2.w;
#pragma unroll
    for (int j = 0; j < kLgBatch; ++j) {
      if (r + j >= r_end) break;
      const size_t e = static_cast<size_t>(r + j) * D + c;
      const float m1 = s1[j] * inv_d, m2 = s2[j] * inv_d;
      const float4 d = make_float4(bf16_lo(dv[j].x), bf16_hi(dv[j].x), bf16_lo(dv[j].y), bf16_hi(dv[j].y));
      const float4 xh = xv[j];
      float4 o;
      o.x = fmaf(rs[j], d.x * sc1.x - m1 - xh.x * m2, gv[j].x);
      o.y = fmaf(rs[j], d.y * sc1.y - m1 - xh.y * m2, gv[j].y);
      o.z = fmaf(rs[j], d.z * sc1.z - m1 - xh.z * m2, gv[j].z);
      o.w = fmaf(rs[j], d.w * sc1.w - m1 - xh.w * m2, gv[j].w);
      stg128(gaddr(g + e), o);
      if (GATE) {
        const float4 q = make_float4(o.x * gt.x, o.y * gt.y, o.z * gt.z, o.w * gt.w);
        stg64(gaddr(dy + e), make_uint2(pack_bf16(q.x, q.y), pack_bf16(q.z, q.w)));
        ag.x = fmaf(o.x, bf16_lo(yv[j].x), ag.x), ag.y = fmaf(o.y, bf16_hi(yv[j].x), ag.y);
        ag.z = fmaf(o.z, bf16_lo(yv[j].y), ag.z), ag.w = fmaf(o.w, bf16_hi(yv[j].y), ag.w);
        ab.x += q.x, ab.y += q.y, ab.z += q.z, ab.w += q.w;
      }
    }
  }
  red_add_v4(gaddr(dshift + static_cast<size_t>(b) * ld_dmod + c), a_sh);
  red_add_v4(gaddr(dscale + static_cast<size_t>(b) * ld_dmod + c), a_sc);
  if (GATE) {
    red_add_v4(gaddr(dgate + static_cast<size_t>(b) * ld_dgate + c), ag);
    if (kBiasRows) stg128(gaddr(dbias + static_cast<size_t>(b) * D + c), ab);
    else if (dbias) red_add_v4(gaddr(dbias + c), ab);
  }
}
template <bool GATE>
__global__ void __launch_bounds__(kLgMaxThreads, 2)
ln_bwd_gate_kernel(const __nv_bfloat16* __restrict__ dxmod, const float* __restrict__ x,
                   const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ scale,
                   int ld_mod, int rows_per_group, float* __restrict__ g, int accumulate, float* __restrict__ dshift,
                   float* __restrict__ dscale, int ld_dmod, const __nv_bfloat16* __restrict__ y,
                   const float* __restrict__ gate, int ld_gate, __nv_bfloat16* __restrict__ dy,
                   float* __restrict__ dgate, int ld_dgate, float* __restrict__ dbias, int M, int D,
                   int rows_per_block) {
  ln_bwd_gate_body<GATE, false>(dxmod, x, mean, rstd, scale, ld_mod, rows_per_group, g, accumulate, dshift, dscale,
                                ld_dmod, y, gate, ld_gate, dy, dgate, ld_dgate, dbias, M, D, rows_per_block);
}
__global__ void __launch_bounds__(kLgMaxThreads, 2)
ln_bwd_gate_bias_rows_kernel(const __nv_bfloat16* __restrict__ dxmod, const float* __restrict__ x,
                             const float* __restrict__ mean, const float* __restrict__ rstd,
                             const float* __restrict__ scale, int ld_mod, int rows_per_group, float* __restrict__ g,
                             int accumulate, float* __restrict__ dshift, float* __restrict__ dscale, int ld_dmod,
                             const __nv_bfloat16* __restrict__ y, const float* __restrict__ gate, int ld_gate,
                             __nv_bfloat16* __restrict__ dy, float* __restrict__ dgate, int ld_dgate,
                             float* __restrict__ dbias_rows, int M, int D, int rows_per_block) {
  ln_bwd_gate_body<true, true>(dxmod, x, mean, rstd, scale, ld_mod, rows_per_group, g, accumulate, dshift, dscale,
                               ld_dmod, y, gate, ld_gate, dy, dgate, ld_dgate, dbias_rows, M, D, rows_per_block);
}

// =========================================================================================================
// unmask_tokens (+ decoder_pos_embed) and its backward.  Thread owns 4 columns; block = D/4 threads x 16 positions.
// =========================================================================================================
constexpr int kUmPos = 64;  // positions per block (backward: one 16-byte mask-token reduction per thread and block)
template <bool kPos>  // false: no position term (the decoder-less DiT's zero-filled output scatter)
__global__ void unmask_kernel(const float* __restrict__ u, const float* __restrict__ mask_token,
                              const float* __restrict__ pos, const int64_t* __restrict__ ids_restore,
                              float* __restrict__ out, int T, int L, int D) {
  const int c = threadIdx.x * 4;
  if (c >= D) return;
  const int b = blockIdx.y, l0 = blockIdx.x * kUmPos, l1 = min(L, l0 + kUmPos);
  const float4 mt = mask_token ? *reinterpret_cast<const float4*>(mask_token + c) : make_float4(0, 0, 0, 0);
  // 4 positions per iteration: the index loads, then the 8 independent 16-byte row loads, are issued back to back
  for (int l = l0; l < l1; l += 4) {
    int r[4];
    float4 v[4], pe[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      r[j] = (l + j < l1) ? (ids_restore ? static_cast<int>(ids_restore[static_cast<size_t>(b) * L + l + j]) : l + j) : -1;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (r[j] < 0) continue;
      v[j] = (r[j] < T) ? *reinterpret_cast<const float4*>(u + (static_cast<size_t>(b) * T + r[j]) * D + c) : mt;
      pe[j] = kPos ? *reinterpret_cast<const float4*>(pos + static_cast<size_t>(l + j) * D + c) : make_float4(0, 0, 0, 0);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (r[j] < 0) continue;
      *reinterpret_cast<float4*>(out + (static_cast<size_t>(b) * L + l + j) * D + c) =
          make_float4(v[j].x + pe[j].x, v[j].y + pe[j].y, v[j].z + pe[j].z, v[j].w + pe[j].w);
    }
  }
}
// kStore (deterministic mode): the block's mask-token sum is stored into its own row of dmask_token ([blocks, D]
// scratch, block = blockIdx.y * gridDim.x + blockIdx.x); colsum_ordered reduces the rows afterwards.
template <bool kStore>
__device__ __forceinline__ void unmask_bwd_body(const float* __restrict__ g, const int64_t* __restrict__ ids_restore,
                                                __nv_bfloat16* __restrict__ du, float* __restrict__ dmask_token, int T,
                                                int L, int D) {
  const int c = threadIdx.x * 4;
  if (c >= D) return;
  const int b = blockIdx.y, l0 = blockIdx.x * kUmPos, l1 = min(L, l0 + kUmPos);
  float4 acc = make_float4(0, 0, 0, 0);
  for (int l = l0; l < l1; l += 4) {
    int r[4];
    float4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      r[j] = (l + j < l1) ? (ids_restore ? static_cast<int>(ids_restore[static_cast<size_t>(b) * L + l + j]) : l + j) : -1;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (r[j] >= 0) v[j] = *reinterpret_cast<const float4*>(g + (static_cast<size_t>(b) * L + l + j) * D + c);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (r[j] < 0) continue;
      if (r[j] < T) {
        *reinterpret_cast<uint2*>(du + (static_cast<size_t>(b) * T + r[j]) * D + c) =
            make_uint2(pack_bf16(v[j].x, v[j].y), pack_bf16(v[j].z, v[j].w));
      } else {
        acc.x += v[j].x, acc.y += v[j].y, acc.z += v[j].z, acc.w += v[j].w;
      }
    }
  }
  if (kStore) {
    const size_t blk = static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x;
    *reinterpret_cast<float4*>(dmask_token + blk * D + c) = acc;
  } else if (dmask_token) {  // one 16-byte reduction per thread and block (64 positions): [B * L / 64] per address
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dmask_token + c), "f"(acc.x), "f"(acc.y),
                 "f"(acc.z), "f"(acc.w)
                 : "memory");
  }
}
__global__ void unmask_bwd_kernel(const float* __restrict__ g, const int64_t* __restrict__ ids_restore,
                                  __nv_bfloat16* __restrict__ du, float* __restrict__ dmask_token, int T, int L,
                                  int D) {
  unmask_bwd_body<false>(g, ids_restore, du, dmask_token, T, L, D);
}
__global__ void unmask_bwd_rows_kernel(const float* __restrict__ g, const int64_t* __restrict__ ids_restore,
                                       __nv_bfloat16* __restrict__ du, float* __restrict__ dmask_rows, int T, int L,
                                       int D) {
  unmask_bwd_body<true>(g, ids_restore, du, dmask_rows, T, L, D);
}


// Row gather of a bf16 matrix: out[b*T + i, :] = in[b*L + idx[b*T + i], :].  Thread moves 4 elements (8 bytes).
__global__ void gather_rows_bf16_kernel(const uint2* __restrict__ in, const int64_t* __restrict__ idx,
                                        uint2* __restrict__ out, int T, int L, int D4, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / D4;
    const int c = static_cast<int>(i - row * D4);
    const long long b = row / T;
    out[i] = in[(b * L + idx[row]) * D4 + c];
  }
}

long long det_scratch_floats(int B, int T, int L, int D, int Dd, int cpp, int has_mask_token) {
  const long long tok = 128 * cpp * sizeof(float) <= 48 * 1024 ? 128 : 32;
  const long long pe = static_cast<long long>(B) * ((T + tok - 1) / tok) * D * (cpp + 1);
  const long long um = has_mask_token ? static_cast<long long>(B) * ((L + kUmPos - 1) / kUmPos) * Dd : 0;
  const long long ln = static_cast<long long>(B) * (D > Dd ? D : Dd);
  return pe > um ? (pe > ln ? pe : ln) : (um > ln ? um : ln);
}

int patch_embed_bwd_s(const float* x, const float* sigma, float sigma_data, const int64_t* ids_keep, const float* g,
                      float* gW, float* gb, int B, int C, int R, int p, int D, int T, float* scratch,
                      cudaStream_t stream) {
  if (!x || !g || !gW || !gb || B <= 0 || T <= 0 || R % p) return MDT_ERR_ARG;
  const int cpp = C * p * p;
  if (cpp > kPebMaxCpp) return MDT_ERR_UNSUPPORTED;
  const int tok = 128 * cpp * sizeof(float) <= 48 * 1024 ? 128 : 32;
  const dim3 grid((T + tok - 1) / tok, B);
  const size_t smem = tok * cpp * sizeof(float);
  if (!g_deterministic) {
    if (tok == 128)
      patch_embed_bwd_kernel<128><<<grid, 384, smem, stream>>>(x, sigma, sigma_data, ids_keep, g, gW, gb, C, R, p, D, T);
    else
      patch_embed_bwd_kernel<32><<<grid, 384, smem, stream>>>(x, sigma, sigma_data, ids_keep, g, gW, gb, C, R, p, D, T);
    return launch_status();
  }
  if (!scratch) return MDT_ERR_UNSUPPORTED;
  const long long blocks = static_cast<long long>(grid.x) * grid.y;
  float* pW = scratch;
  float* pb = scratch + blocks * D * cpp;
  if (tok == 128)
    patch_embed_bwd_partial_kernel<128><<<grid, 384, smem, stream>>>(x, sigma, sigma_data, ids_keep, g, pW, pb, C, R,
                                                                     p, D, T);
  else
    patch_embed_bwd_partial_kernel<32><<<grid, 384, smem, stream>>>(x, sigma, sigma_data, ids_keep, g, pW, pb, C, R,
                                                                    p, D, T);
  int rc = launch_status();
  if (rc == MDT_OK) rc = colsum_ordered(pW, 0, static_cast<int>(blocks), D * cpp, D * cpp, gW, stream);
  if (rc == MDT_OK) rc = colsum_ordered(pb, 0, static_cast<int>(blocks), D, D, gb, stream);
  return rc;
}

int ln_modulate_bwd_gate_s(const void* dxmod_bf16, const float* x, const float* mean, const float* rstd,
                           const float* scale, int ld_mod, int rows_per_group, float* g, int accumulate, float* dshift,
                           float* dscale, int ld_dmod, const void* y_bf16, const float* gate, int ld_gate,
                           void* dy_bf16, float* dgate, int ld_dgate, float* dbias, int M, int D, float* scratch,
                           cudaStream_t stream) {
  if (!dxmod_bf16 || !x || !mean || !rstd || !scale || !g || !dshift || !dscale || M <= 0) return MDT_ERR_ARG;
  if (rows_per_group <= 0 || M % rows_per_group || (ld_mod & 3) || (ld_dmod & 3)) return MDT_ERR_ARG;
  if (y_bf16 && (!gate || !dy_bf16 || !dgate || (ld_gate & 3) || (ld_dgate & 3))) return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(dshift) | reinterpret_cast<uintptr_t>(dscale) |
       reinterpret_cast<uintptr_t>(gate) | reinterpret_cast<uintptr_t>(dgate) | reinterpret_cast<uintptr_t>(dbias)) & 15)
    return MDT_ERR_ARG;
  if (D % 128 || D / 4 > kLgMaxThreads) return MDT_ERR_UNSUPPORTED;  // D <= 1280, as the LN kernels
  // deterministic: one block per sample (rows_per_group rows), so the per-sample sums have one writer each; the bias
  // gradient, a sum over samples, goes through per-sample rows in `scratch`
  const bool bias_rows = g_deterministic && y_bf16 && dbias;
  if (bias_rows && (!scratch || (reinterpret_cast<uintptr_t>(scratch) & 15))) return MDT_ERR_UNSUPPORTED;
  const int rpb = g_deterministic ? rows_per_group : gcd_int(rows_per_group, 32);
  const int grid = M / rpb;
  const __nv_bfloat16* dx = static_cast<const __nv_bfloat16*>(dxmod_bf16);
  const __nv_bfloat16* y = static_cast<const __nv_bfloat16*>(y_bf16);
  __nv_bfloat16* dy = static_cast<__nv_bfloat16*>(dy_bf16);
  if (bias_rows) {
    ln_bwd_gate_bias_rows_kernel<<<grid, D / 4, 0, stream>>>(dx, x, mean, rstd, scale, ld_mod, rows_per_group, g,
                                                             accumulate, dshift, dscale, ld_dmod, y, gate, ld_gate, dy,
                                                             dgate, ld_dgate, scratch, M, D, rpb);
    const int rc = launch_status();
    return rc == MDT_OK ? colsum_ordered(scratch, 0, grid, D, D, dbias, stream) : rc;
  }
  if (y_bf16)
    ln_bwd_gate_kernel<true><<<grid, D / 4, 0, stream>>>(dx, x, mean, rstd, scale, ld_mod, rows_per_group, g,
                                                         accumulate, dshift, dscale, ld_dmod, y, gate, ld_gate, dy,
                                                         dgate, ld_dgate, dbias, M, D, rpb);
  else
    ln_bwd_gate_kernel<false><<<grid, D / 4, 0, stream>>>(dx, x, mean, rstd, scale, ld_mod, rows_per_group, g,
                                                          accumulate, dshift, dscale, ld_dmod, nullptr, nullptr, 0,
                                                          nullptr, nullptr, 0, nullptr, M, D, rpb);
  return launch_status();
}

int unmask_tokens_bwd_s(const float* g, const int64_t* ids_restore, void* du_bf16, float* dmask_token, int B, int T,
                        int L, int D, float* scratch, cudaStream_t stream) {
  if (!g || !du_bf16 || B <= 0 || T <= 0 || L <= 0 || D % 4 || D > 4096) return MDT_ERR_ARG;
  if (!ids_restore && T != L) return MDT_ERR_ARG;
  const dim3 grid((L + kUmPos - 1) / kUmPos, B);
  const int threads = ((D / 4 + 31) / 32) * 32;
  __nv_bfloat16* du = static_cast<__nv_bfloat16*>(du_bf16);
  if (!g_deterministic || !dmask_token) {
    unmask_bwd_kernel<<<grid, threads, 0, stream>>>(g, ids_restore, du, dmask_token, T, L, D);
    return launch_status();
  }
  if (!scratch || (reinterpret_cast<uintptr_t>(scratch) & 15)) return MDT_ERR_UNSUPPORTED;
  unmask_bwd_rows_kernel<<<grid, threads, 0, stream>>>(g, ids_restore, du, scratch, T, L, D);
  const int rc = launch_status();
  return rc == MDT_OK ? colsum_ordered(scratch, 0, static_cast<int>(grid.x * grid.y), D, D, dmask_token, stream) : rc;
}

}  // namespace mdt

using namespace mdt;

extern "C" {

int mdt_mask_indices(const float* noise, int B, int L, int len_keep, int64_t* ids_keep, int64_t* ids_restore,
                     float* mask, void* stream) {
  if (!noise || !ids_keep || !ids_restore || !mask || B <= 0 || L <= 0 || len_keep < 0 || len_keep > L)
    return MDT_ERR_ARG;
  if (L * sizeof(float) > 200 * 1024) return MDT_ERR_UNSUPPORTED;
  const int threads = L >= 1024 ? 1024 : ((L + 31) / 32) * 32;
  const size_t smem = L * sizeof(float);
  if (smem > 48 * 1024)
    cudaFuncSetAttribute(mask_indices_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  mask_indices_kernel<<<B, threads, smem, S(stream)>>>(noise, L, len_keep, ids_keep, ids_restore, mask);
  return launch_status();
}

int mdt_patch_embed(const float* x, const float* sigma, float sigma_data, const float* W, const float* bias,
                    const float* pos, const int64_t* ids_keep, float* out, int B, int C, int R, int p, int D, int T,
                    void* stream) {
  if (!x || !W || !bias || !pos || !out || B <= 0 || T <= 0 || R % p) return MDT_ERR_ARG;
  const int cpp = C * p * p;
  if (cpp > kPeMaxCpp) return MDT_ERR_UNSUPPORTED;
  dim3 grid((T + kPeTok - 1) / kPeTok, B);
  patch_embed_kernel<<<grid, 384, kPeTok * cpp * sizeof(float), S(stream)>>>(x, sigma, sigma_data, W, bias, pos,
                                                                             ids_keep, out, C, R, p, D, T);
  return launch_status();
}

int mdt_patch_embed_bwd(const float* x, const float* sigma, float sigma_data, const int64_t* ids_keep,
                        const float* g, float* gW, float* gb, int B, int C, int R, int p, int D, int T, void* stream) {
  return patch_embed_bwd_s(x, sigma, sigma_data, ids_keep, g, gW, gb, B, C, R, p, D, T, nullptr, S(stream));
}

int mdt_timestep_freq(const float* sigma, int B, int dim, void* out_bf16, void* stream) {
  if (!sigma || !out_bf16 || B <= 0 || dim <= 0 || dim % 2) return MDT_ERR_ARG;
  const int n = B * dim / 2;
  timestep_freq_kernel<MDT_PRECOND_EDM><<<(n + 255) / 256, 256, 0, S(stream)>>>(sigma, B, dim,
                                                                                 static_cast<__nv_bfloat16*>(out_bf16));
  return launch_status();
}

int mdt_flow_timestep_freq(const float* t, int B, int dim, void* out_bf16, void* stream) {
  if (!t || !out_bf16 || B <= 0 || dim <= 0 || dim % 2) return MDT_ERR_ARG;
  const int n = B * dim / 2;
  timestep_freq_kernel<MDT_PRECOND_FLOW><<<(n + 255) / 256, 256, 0, S(stream)>>>(t, B, dim,
                                                                                  static_cast<__nv_bfloat16*>(out_bf16));
  return launch_status();
}

static int ew_grid(long long n, int per_thread = 1) {
  long long blocks = (n / per_thread + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > kNumSMsDefault * 16) blocks = kNumSMsDefault * 16;
  return static_cast<int>(blocks);
}

int mdt_silu(const float* a, const float* b, float* sum_f32, void* out_bf16, long long n, void* stream) {
  if (!a || !out_bf16 || n <= 0) return MDT_ERR_ARG;
  silu_kernel<<<ew_grid(n), 256, 0, S(stream)>>>(a, b, sum_f32, static_cast<__nv_bfloat16*>(out_bf16), n);
  return launch_status();
}
int mdt_silu_bwd(const float* dy, const float* x, float* dx_f32, void* dx_bf16, long long n, void* stream) {
  if (!dy || !x || n <= 0) return MDT_ERR_ARG;
  silu_bwd_kernel<<<ew_grid(n), 256, 0, S(stream)>>>(dy, x, dx_f32, static_cast<__nv_bfloat16*>(dx_bf16), n);
  return launch_status();
}
int mdt_cast_f32_bf16(const float* in, void* out_bf16, long long n, void* stream) {
  if (!in || !out_bf16 || n <= 0) return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(in) & 15) || (reinterpret_cast<uintptr_t>(out_bf16) & 7)) return MDT_ERR_ARG;
  cast_f32_bf16_kernel<<<ew_grid(n, 4), 256, 0, S(stream)>>>(in, static_cast<__nv_bfloat16*>(out_bf16), n);
  return launch_status();
}
int mdt_colsum_bf16(const void* in_bf16, int M, int N, int ld, float* out, void* stream) {
  if (!in_bf16 || !out || M <= 0 || N <= 0 || (ld & 1)) return MDT_ERR_ARG;
  if (g_deterministic) return colsum_ordered(in_bf16, 1, M, N, ld, out, S(stream));
  dim3 grid((N + 255) / 256, (M + kCsRows - 1) / kCsRows);
  colsum_bf16_kernel<<<grid, 128, 0, S(stream)>>>(static_cast<const __nv_bfloat16*>(in_bf16), M, N, ld, out);
  return launch_status();
}
int mdt_colsum_f32(const float* in, int M, int N, int ld, float* out, void* stream) {
  if (!in || !out || M <= 0 || N <= 0) return MDT_ERR_ARG;
  if (g_deterministic) return colsum_ordered(in, 0, M, N, ld, out, S(stream));
  dim3 grid((N + 127) / 128, (M + kCsRows - 1) / kCsRows);
  colsum_f32_kernel<<<grid, 128, 0, S(stream)>>>(in, M, N, ld, out);
  return launch_status();
}

#define MDT_LN_DISPATCH(NV, ...)                 \
  switch (NV) {                                  \
    case 3: { constexpr int kNV = 3; __VA_ARGS__; } break;   \
    case 4: { constexpr int kNV = 4; __VA_ARGS__; } break;   \
    case 6: { constexpr int kNV = 6; __VA_ARGS__; } break;   \
    case 8: { constexpr int kNV = 8; __VA_ARGS__; } break;   \
    case 9: { constexpr int kNV = 9; __VA_ARGS__; } break;   \
    case 10: { constexpr int kNV = 10; __VA_ARGS__; } break; \
    default: return MDT_ERR_UNSUPPORTED;         \
  }

int mdt_ln_modulate(const float* x, const float* shift, const float* scale, int ld_mod, int rows_per_group,
                    void* out_bf16, float* mean, float* rstd, int M, int D, float eps, void* stream) {
  if (!x || !shift || !scale || !out_bf16 || M <= 0 || D % 128 || rows_per_group <= 0 || (ld_mod & 3))
    return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(shift) & 15) || (reinterpret_cast<uintptr_t>(scale) & 15)) return MDT_ERR_ARG;
  const int grid = (M + 7) / 8;
  MDT_LN_DISPATCH(D / 128, ln_modulate_kernel<kNV><<<grid, 256, 0, S(stream)>>>(
                               x, shift, scale, ld_mod, rows_per_group, static_cast<__nv_bfloat16*>(out_bf16), mean,
                               rstd, M, eps));
  return launch_status();
}

int mdt_ln_modulate_bwd(const void* dxmod_bf16, const float* x, const float* mean, const float* rstd,
                        const float* scale, int ld_mod, int rows_per_group, float* g, int accumulate, float* dshift,
                        float* dscale, int ld_dmod, int M, int D, void* stream) {
  if (!dxmod_bf16 || !x || !mean || !rstd || !scale || !g || !dshift || !dscale || M <= 0 || D % 128)
    return MDT_ERR_ARG;
  if (rows_per_group <= 0 || M % rows_per_group || (ld_mod & 3)) return MDT_ERR_ARG;
  if (reinterpret_cast<uintptr_t>(scale) & 15) return MDT_ERR_ARG;
  if (g_deterministic) {  // the fused kernel with one block per sample: each dshift / dscale address has one writer
    if (D / 4 > kLgMaxThreads || (ld_dmod & 3) ||
        ((reinterpret_cast<uintptr_t>(dshift) | reinterpret_cast<uintptr_t>(dscale)) & 15))
      return MDT_ERR_UNSUPPORTED;
    return ln_modulate_bwd_gate_s(dxmod_bf16, x, mean, rstd, scale, ld_mod, rows_per_group, g, accumulate, dshift,
                                  dscale, ld_dmod, nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr, M, D, nullptr,
                                  S(stream));
  }
  const int rpb = gcd_int(rows_per_group, kLnbRowsMax);
  const int grid = M / rpb;
  MDT_LN_DISPATCH(D / 128, ln_modulate_bwd_kernel<kNV><<<grid, 128, 0, S(stream)>>>(
                               static_cast<const __nv_bfloat16*>(dxmod_bf16), x, mean, rstd, scale, ld_mod,
                               rows_per_group, g, accumulate, dshift, dscale, ld_dmod, M, rpb));
  return launch_status();
}

int mdt_gate_bwd(const float* g, const void* y_bf16, const float* gate, int ld_gate, int rows_per_group,
                 void* dy_bf16, float* dgate, int ld_dgate, float* dbias, int M, int D, void* stream) {
  if (!g || !y_bf16 || !gate || !dy_bf16 || !dgate || M <= 0 || D % 4 || D > 4096) return MDT_ERR_ARG;
  if (rows_per_group <= 0 || M % rows_per_group || (ld_gate & 3)) return MDT_ERR_ARG;
  if (reinterpret_cast<uintptr_t>(gate) & 15) return MDT_ERR_ARG;
  const int threads = ((D / 4 + 31) / 32) * 32;
  // deterministic: one block per sample (one writer per dgate address); the bias gradient sums over samples and this
  // entry point has no scratch for per-sample rows
  if (g_deterministic && dbias) return MDT_ERR_UNSUPPORTED;
  const int rpb = g_deterministic ? rows_per_group : gcd_int(rows_per_group, kGbRowsMax);
  gate_bwd_kernel<<<M / rpb, threads, 0, S(stream)>>>(g, static_cast<const __nv_bfloat16*>(y_bf16), gate, ld_gate,
                                                      rows_per_group, static_cast<__nv_bfloat16*>(dy_bf16), dgate,
                                                      ld_dgate, dbias, M, D, rpb);
  return launch_status();
}

// LN-modulate backward + the gate backward of the branch that consumes the finished residual gradient (y == NULL:
// plain LN backward).  Same arithmetic as mdt_ln_modulate_bwd followed by mdt_gate_bwd.
int mdt_ln_modulate_bwd_gate(const void* dxmod_bf16, const float* x, const float* mean, const float* rstd,
                             const float* scale, int ld_mod, int rows_per_group, float* g, int accumulate,
                             float* dshift, float* dscale, int ld_dmod, const void* y_bf16, const float* gate,
                             int ld_gate, void* dy_bf16, float* dgate, int ld_dgate, float* dbias, int M, int D,
                             void* stream) {
  return ln_modulate_bwd_gate_s(dxmod_bf16, x, mean, rstd, scale, ld_mod, rows_per_group, g, accumulate, dshift, dscale,
                                ld_dmod, y_bf16, gate, ld_gate, dy_bf16, dgate, ld_dgate, dbias, M, D, nullptr,
                                S(stream));
}

int mdt_unmask_tokens(const float* u, const float* mask_token, const float* pos, const int64_t* ids_restore,
                      float* out, int B, int T, int L, int D, void* stream) {
  if (!u || !out || B <= 0 || T <= 0 || L <= 0 || D % 4 || D > 4096) return MDT_ERR_ARG;
  if (!ids_restore && T != L) return MDT_ERR_ARG;
  dim3 grid((L + kUmPos - 1) / kUmPos, B);
  const int threads = ((D / 4 + 31) / 32) * 32;
  if (pos)
    unmask_kernel<true><<<grid, threads, 0, S(stream)>>>(u, mask_token, pos, ids_restore, out, T, L, D);
  else
    unmask_kernel<false><<<grid, threads, 0, S(stream)>>>(u, mask_token, nullptr, ids_restore, out, T, L, D);
  return launch_status();
}

int mdt_unmask_tokens_bwd(const float* g, const int64_t* ids_keep, const int64_t* ids_restore, void* du_bf16,
                          float* dmask_token, int B, int T, int L, int D, void* stream) {
  (void)ids_keep;
  return unmask_tokens_bwd_s(g, ids_restore, du_bf16, dmask_token, B, T, L, D, nullptr, S(stream));
}

int mdt_gather_rows_bf16(const void* in_bf16, const int64_t* idx, void* out_bf16, int B, int T, int L, int D,
                         void* stream) {
  if (!in_bf16 || !idx || !out_bf16 || B <= 0 || T <= 0 || T > L || D <= 0 || D % 4) return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(in_bf16) | reinterpret_cast<uintptr_t>(out_bf16)) & 7) return MDT_ERR_ARG;
  const long long n = static_cast<long long>(B) * T * (D / 4);
  gather_rows_bf16_kernel<<<ew_grid(n), 256, 0, S(stream)>>>(static_cast<const uint2*>(in_bf16), idx,
                                                              static_cast<uint2*>(out_bf16), T, L, D / 4, n);
  return launch_status();
}

}  // extern "C"
