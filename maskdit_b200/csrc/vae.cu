// Sampler tail: the SD-VAE DECODE path the reference runs on every batch of sampled latents (sample.py:275
// `images = vae.decode(z)`; autoencoder.py:306-453: post_quant_conv, conv_in, ResnetBlocks with GroupNorm(32)+swish,
// one single-head AttnBlock, nearest-2x Upsample + conv, norm_out + conv_out), and the ENCODE path that turns a dataset
// into training latents (extract_latent.py:66 `model(img, fn='encode_moments')`; autoencoder.py:212-303: conv_in,
// ResnetBlocks, stride-2 Downsample convolutions, the AttnBlock, norm_out + conv_out, then quant_conv).
//
// Layout: activations are pixel-major ("NHWC") fp32 row matrices [B*H*W, C], so every convolution is a GEMM on the
// wgmma kernel of gemm_wgmma.cu: a 3x3 convolution reads an im2col operand A[(b,y,x), (ky,kx,c)] (bf16) that ONE
// kernel builds with the GroupNorm affine, the swish and the nearest-2x upsample of the source fused in (the normalised
// tensor is never materialised), weights are pre-flattened to [C_out, (ky,kx,c)]; bias and the residual add ride in the
// GEMM epilogue.  The kernels here are the HBM-bound glue: statistics, im2col, row softmax, layout conversion.
#include <math.h>

#include "common.cuh"
#include "../../include/maskdit_b200.h"

namespace mdt {

static inline cudaStream_t VS(void* s) { return static_cast<cudaStream_t>(s); }
static inline int vae_status() { return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA; }

// z [B,Cz,h,w] f32 (NCHW, the sampler's latent) -> out [B*h*w, Cz] f32 = post_quant_conv(z / scale_factor)
// (FrozenAutoencoderKL.decode, autoencoder.py:449-451; a 1x1 convolution over <= 8 channels)
__global__ void vae_post_quant_kernel(const float* __restrict__ z, const float* __restrict__ W,
                                      const float* __restrict__ bias, float inv_sf, float* __restrict__ out, int B,
                                      int C, int P) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;  // (b, pixel)
  if (i >= static_cast<long long>(B) * P) return;
  const int b = static_cast<int>(i / P), p = static_cast<int>(i % P);
  float v[8];
  for (int c = 0; c < C; ++c) v[c] = inv_sf * z[(static_cast<long long>(b) * C + c) * P + p];
  for (int o = 0; o < C; ++o) {
    float acc = bias[o];
    for (int c = 0; c < C; ++c) acc = fmaf(W[o * C + c], v[c], acc);
    out[i * C + o] = acc;
  }
}

// GroupNorm(32) statistics of x [B, P, C] f32, DETERMINISTIC (no atomics: with bf16 GEMM operands downstream, 1e-7
// order noise in a mean flips bf16 roundings and shows up as 4e-3 run-to-run differences in the decoded image, measured):
//   pass 1: block (b, chunk of kGnPix pixels) -> partial[b][chunk][g] = (sum, sum of squares) of x - K fp32,
//           fixed-order tree
//   pass 2: sums[b][g] = fixed-order fp64 sum of the partials, with the shift K folded back in fp64.
// K is the group's first value (pixel 0, its first channel).  Summing x - K instead of x keeps the fp32 partials at the
// scale of the group's spread, so a group whose mean is large against its spread does not lose its variance to
// cancellation (the one-pass q/n - m^2 that mdt_vae_im2col forms then cancels in fp64), and an exactly constant group
// sums to exactly zero deviation.
// Thread = 4 channels of one pixel lane; block = C/4 x (256 / (C/4)) threads: always 8 threads per group.
constexpr int kGnPix = 256;
__global__ void __launch_bounds__(256)
vae_gn_partial_kernel(const float* __restrict__ x, float* __restrict__ partial, int P, int C) {
  __shared__ float s_part[256][2];
  const int tx = threadIdx.x, ty = threadIdx.y, b = blockIdx.y;
  const int p0 = blockIdx.x * kGnPix;
  const int tpg = (C / 32) / 4;                       // threads per group along x (1, 2 or 4)
  const int g = tx / tpg, member = ty * tpg + (tx - g * tpg);
  const float k = x[static_cast<long long>(b) * P * C + g * (C / 32)];
  float s = 0.f, ss = 0.f;
  for (int p = p0 + ty; p < min(P, p0 + kGnPix); p += blockDim.y) {
    float4 v = *reinterpret_cast<const float4*>(x + (static_cast<long long>(b) * P + p) * C + 4 * tx);
    v.x -= k, v.y -= k, v.z -= k, v.w -= k;
    s += (v.x + v.y) + (v.z + v.w);
    ss += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  // slot = (group, member): the 8 threads of a group occupy 8 consecutive slots
  s_part[g * 8 + member][0] = s;
  s_part[g * 8 + member][1] = ss;
  __syncthreads();
  const int tid = ty * blockDim.x + tx;
  if (tid < 64) {
    const int gg = tid >> 1, w = tid & 1;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) acc += s_part[gg * 8 + k][w];
    partial[((static_cast<long long>(b) * gridDim.x + blockIdx.x) * 32 + gg) * 2 + w] = acc;
  }
}
__global__ void vae_gn_finish_kernel(const float* __restrict__ x, const float* __restrict__ partial,
                                     double* __restrict__ sums, int nchunk, int P, int C) {
  const int b = blockIdx.x, g = threadIdx.x;  // 32 threads: one group each
  double s = 0.0, q = 0.0;
  for (int k = 0; k < nchunk; ++k) {
    const float2 v = *reinterpret_cast<const float2*>(partial + (static_cast<long long>(b) * nchunk + k) * 64 + 2 * g);
    s += static_cast<double>(v.x);
    q += static_cast<double>(v.y);
  }
  const double K = x[static_cast<long long>(b) * P * C + g * (C / 32)];
  const double n = static_cast<double>(P) * (C / 32);
  sums[(static_cast<long long>(b) * 32 + g) * 2] = fma(n, K, s);                 // sum x   = nK + S
  sums[(static_cast<long long>(b) * 32 + g) * 2 + 1] = fma(K, fma(n, K, 2.0 * s), q);  // sum x^2 = K(nK + 2S) + Q
}

// im2col with the producer fused in:
//   A[(b, y, x), (ky, kx, c)] = f(src[b, (s*y+ky-pad)/up, (s*x+kx-pad)/up, c])  (0 outside the s*H x s*W input)
//   f = identity | GroupNorm affine (sums / gamma / beta given) | GroupNorm affine then swish (silu != 0)
//   ks = 3 or 1; pad = low-side zero padding (ks/2 for the "same" convolutions; 0 for Downsample, whose padding
//   (0,1,0,1) only adds a high-side border, autoencoder.py:56-75); up = 1 or 2 (nearest upsample of the source,
//   Upsample.forward autoencoder.py:49-53); stride s = 1 or 2 (not together with up = 2)
//   src [B, s*H/up, s*W/up, C] f32  ->  A [B*H*W, Kp] bf16,  Kp >= ks*ks*C (extra columns zero)
// Thread = 4 channels; blockDim = (C/4, 256/(C/4)) (C = 4: 1 x 256); each y-lane walks output pixels.
__global__ void __launch_bounds__(256)
vae_im2col_kernel(const float* __restrict__ src, const double* __restrict__ sums, const float* __restrict__ gamma,
                  const float* __restrict__ beta, int silu_on, int ks, int up, int stride, int pad,
                  __nv_bfloat16* __restrict__ A, int B, int H, int W, int C, int Kp, float eps) {
  const int tx = threadIdx.x, c = 4 * tx;
  const int Hi = stride * H, Wi = stride * W;  // input extent (after the upsample)
  const int Hs = Hi / up, Ws = Wi / up;
  const long long npix = static_cast<long long>(B) * H * W;
  const int taps = ks * ks;
  float4 ga = make_float4(1.f, 1.f, 1.f, 1.f), be = make_float4(0.f, 0.f, 0.f, 0.f);
  if (sums) {
    ga = *reinterpret_cast<const float4*>(gamma + c);
    be = *reinterpret_cast<const float4*>(beta + c);
  }
  const int cg = C / 32 > 0 ? C / 32 : 1;
  const double cnt = static_cast<double>(Hs) * Ws * cg;
  // GroupNorm of this thread's group in the current image, recomputed only when the image changes.
  // mean = mean_hi + mean_lo: x - mean_hi is exact for x near a large mean, so normalising a group whose mean is
  // large against its spread keeps the fp32 accuracy of x - mean.  The one-pass variance may round below zero
  // (a constant group): it is clamped before eps.
  float mean_hi = 0.f, mean_lo = 0.f, rstd = 1.f;
  int stats_b = -1;
  for (long long pix = blockIdx.x * static_cast<long long>(blockDim.y) + threadIdx.y; pix < npix;
       pix += static_cast<long long>(gridDim.x) * blockDim.y) {
    const int b = static_cast<int>(pix / (static_cast<long long>(H) * W));
    const int yx = static_cast<int>(pix - static_cast<long long>(b) * H * W);
    const int y = yx / W, x = yx - y * W;
    if (sums && b != stats_b) {
      const int g = c / cg;
      const double s = sums[(static_cast<long long>(b) * 32 + g) * 2], q = sums[(static_cast<long long>(b) * 32 + g) * 2 + 1];
      const double m = s / cnt;
      mean_hi = static_cast<float>(m);
      mean_lo = static_cast<float>(m - static_cast<double>(mean_hi));
      rstd = rsqrtf(fmaxf(static_cast<float>(q / cnt - m * m), 0.f) + eps);
      stats_b = b;
    }
    __nv_bfloat16* arow = A + pix * Kp;
    for (int t = 0; t < taps; ++t) {
      const int ky = t / ks, kx = t - ky * ks;
      const int sy = stride * y + ky - pad, sx = stride * x + kx - pad;
      uint2 o = make_uint2(0u, 0u);
      if (sy >= 0 && sy < Hi && sx >= 0 && sx < Wi) {
        const float4 v = *reinterpret_cast<const float4*>(
            src + ((static_cast<long long>(b) * Hs + sy / up) * Ws + sx / up) * C + c);
        float4 r = v;
        if (sums) {
          r.x = fmaf(((v.x - mean_hi) - mean_lo) * rstd, ga.x, be.x);
          r.y = fmaf(((v.y - mean_hi) - mean_lo) * rstd, ga.y, be.y);
          r.z = fmaf(((v.z - mean_hi) - mean_lo) * rstd, ga.z, be.z);
          r.w = fmaf(((v.w - mean_hi) - mean_lo) * rstd, ga.w, be.w);
        }
        if (silu_on) r = make_float4(silu(r.x), silu(r.y), silu(r.z), silu(r.w));
        o = make_uint2(pack_bf16(r.x, r.y), pack_bf16(r.z, r.w));
      }
      *reinterpret_cast<uint2*>(arow + t * C + c) = o;
    }
    if (tx == 0)
      for (int k = taps * C; k < Kp; ++k) arow[k] = __float2bfloat16_rn(0.f);
  }
}

// P[r, :] = softmax(scale * S[r, :]) as bf16; one warp per row (AttnBlock, autoencoder.py:186-187)
__global__ void __launch_bounds__(256)
vae_softmax_rows_kernel(const float* __restrict__ S, float scale, __nv_bfloat16* __restrict__ P, int rows, int cols) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* s = S + static_cast<long long>(row) * cols;
  float mx = -INFINITY;
  for (int j = lane; j < cols; j += 32) mx = fmaxf(mx, s[j]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < cols; j += 32) sum += __expf(scale * (s[j] - mx));
  const float inv = 1.f / warp_sum(sum);
  __nv_bfloat16* p = P + static_cast<long long>(row) * cols;
  for (int j = lane; j < cols; j += 32) p[j] = __float2bfloat16_rn(__expf(scale * (s[j] - mx)) * inv);
}

// x [B, P, ldx] f32 (first C columns valid) -> out [B, C, P] f32 (the [B,3,H,W] image the reference's decode returns)
__global__ void vae_rows_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int P, int C,
                                        int ldx) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(B) * C * P) return;
  const int p = static_cast<int>(i % P), c = static_cast<int>((i / P) % C), b = static_cast<int>(i / (static_cast<long long>(P) * C));
  out[i] = x[(static_cast<long long>(b) * P + p) * ldx + c];
}

// ---- encode half (FrozenAutoencoderKL.encode_moments / encode, autoencoder.py:212-303,431-446) ----------------------
// img [B,3,H,W] f32 (NCHW, [-1, 1]) -> rows [B*H*W, 4] f32, channel 3 zero (conv_in then runs the C = 4 im2col);
// flip != 0 reads column W-1-x (the `img.flip(dims=[-1])` pass of extract_latent.py:87)
__global__ void vae_image_to_rows_kernel(const float* __restrict__ img, float* __restrict__ rows, int B, int H, int W,
                                         int flip) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;  // (b, y, x)
  const long long P = static_cast<long long>(H) * W;
  if (i >= B * P) return;
  const int b = static_cast<int>(i / P), yx = static_cast<int>(i % P);
  const int y = yx / W, x = yx - y * W;
  const long long s = (static_cast<long long>(b) * 3 * H + y) * W + (flip ? W - 1 - x : x);
  *reinterpret_cast<float4*>(rows + 4 * i) = make_float4(img[s], img[s + P], img[s + 2 * P], 0.f);
}

// x [B*P, ldx] f32 (conv_out rows, first C valid) -> moments [B,C,P] f32 = quant_conv(x) (1x1, C -> C, C <= 8);
// z (if eps given) [B,C/2,P] = sf * (mean + exp(0.5 * clamp(logvar, -30, 20)) * eps): FrozenAutoencoderKL.sample,
// rounded step by step as the reference's separate tensor ops are (autoencoder.py:436-442)
__global__ void vae_quant_moments_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ W,
                                         const float* __restrict__ bias, const float* __restrict__ eps, float sf,
                                         float* __restrict__ moments, float* __restrict__ z, int B, int C, int P) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;  // (b, pixel)
  if (i >= static_cast<long long>(B) * P) return;
  const int b = static_cast<int>(i / P), p = static_cast<int>(i % P);
  float v[8], m[8];
  for (int c = 0; c < C; ++c) v[c] = x[i * ldx + c];
  for (int o = 0; o < C; ++o) {
    float acc = bias[o];
    for (int c = 0; c < C; ++c) acc = fmaf(W[o * C + c], v[c], acc);
    m[o] = acc;
    moments[(static_cast<long long>(b) * C + o) * P + p] = acc;
  }
  if (!eps) return;
  const int h = C / 2;
  for (int o = 0; o < h; ++o) {
    const long long zi = (static_cast<long long>(b) * h + o) * P + p;
    const float std_ = expf(__fmul_rn(0.5f, fminf(fmaxf(m[h + o], -30.f), 20.f)));
    z[zi] = __fmul_rn(sf, __fadd_rn(m[o], __fmul_rn(std_, eps[zi])));
  }
}

}  // namespace mdt

using namespace mdt;

extern "C" {

int mdt_vae_post_quant(const float* z, const float* W, const float* bias, float scale_factor, float* out, int B,
                       int C, int P, void* stream) {
  if (!z || !W || !bias || !out || B <= 0 || C <= 0 || C > 8 || P <= 0 || scale_factor == 0.f) return MDT_ERR_ARG;
  const long long n = static_cast<long long>(B) * P;
  vae_post_quant_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, VS(stream)>>>(z, W, bias, 1.f / scale_factor, out,
                                                                                  B, C, P);
  return vae_status();
}

int mdt_vae_gn_stats(const float* x, double* sums, float* scratch, int B, int P, int C, void* stream) {
  if (!x || !sums || !scratch || B <= 0 || P <= 0 || C % 128 || C > 512) return MDT_ERR_ARG;  // 4..16 channels / group
  if (reinterpret_cast<uintptr_t>(x) & 15) return MDT_ERR_ARG;
  const int nchunk = (P + kGnPix - 1) / kGnPix;
  dim3 block(C / 4, 256 / (C / 4)), grid(nchunk, B);
  vae_gn_partial_kernel<<<grid, block, 0, VS(stream)>>>(x, scratch, P, C);
  vae_gn_finish_kernel<<<B, 32, 0, VS(stream)>>>(x, scratch, sums, nchunk, P, C);
  return vae_status();
}

int mdt_vae_im2col(const float* src, const double* sums, const float* gamma, const float* beta, int silu, int ks,
                   int up, void* A_bf16, int B, int H, int W, int C, int Kp, void* stream) {
  return mdt_vae_im2col_strided(src, sums, gamma, beta, silu, ks, up, 1, ks / 2, A_bf16, B, H, W, C, Kp, stream);
}

int mdt_vae_im2col_strided(const float* src, const double* sums, const float* gamma, const float* beta, int silu,
                           int ks, int up, int stride, int pad, void* A_bf16, int B, int H, int W, int C, int Kp,
                           void* stream) {
  if (!src || !A_bf16 || B <= 0 || H <= 0 || W <= 0 || C % 4 || C > 1024 || (ks != 1 && ks != 3) ||
      (up != 1 && up != 2) || (stride != 1 && stride != 2) || (up == 2 && stride == 2) || pad < 0 || pad >= ks ||
      H % up || W % up || Kp < ks * ks * C || Kp % 8)
    return MDT_ERR_ARG;
  if (sums && (!gamma || !beta || C % 128)) return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(A_bf16)) & 15) return MDT_ERR_ARG;
  const int tx = C / 4, ty = tx >= 256 ? 1 : 256 / tx;
  const long long npix = static_cast<long long>(B) * H * W;
  long long blocks = (npix + ty - 1) / ty;
  if (blocks > kNumSMsDefault * 16) blocks = kNumSMsDefault * 16;
  vae_im2col_kernel<<<static_cast<int>(blocks), dim3(tx, ty), 0, VS(stream)>>>(
      src, sums, gamma, beta, silu, ks, up, stride, pad, static_cast<__nv_bfloat16*>(A_bf16), B, H, W, C, Kp, 1e-6f);
  return vae_status();
}

int mdt_vae_softmax_rows(const float* S, float scale, void* P_bf16, int rows, int cols, void* stream) {
  if (!S || !P_bf16 || rows <= 0 || cols <= 0) return MDT_ERR_ARG;
  vae_softmax_rows_kernel<<<(rows + 7) / 8, 256, 0, VS(stream)>>>(S, scale, static_cast<__nv_bfloat16*>(P_bf16), rows,
                                                                  cols);
  return vae_status();
}

int mdt_vae_rows_to_nchw(const float* x, float* out, int B, int P, int C, int ldx, void* stream) {
  if (!x || !out || B <= 0 || P <= 0 || C <= 0 || ldx < C) return MDT_ERR_ARG;
  const long long n = static_cast<long long>(B) * C * P;
  vae_rows_to_nchw_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, VS(stream)>>>(x, out, B, P, C, ldx);
  return vae_status();
}

int mdt_vae_image_to_rows(const float* img, float* rows, int B, int H, int W, int flip, void* stream) {
  if (!img || !rows || B <= 0 || H <= 0 || W <= 0 || (reinterpret_cast<uintptr_t>(rows) & 15)) return MDT_ERR_ARG;
  const long long n = static_cast<long long>(B) * H * W;
  vae_image_to_rows_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, VS(stream)>>>(img, rows, B, H, W, flip != 0);
  return vae_status();
}

int mdt_vae_quant_moments(const float* x, int ldx, const float* W, const float* bias, const float* eps,
                          float scale_factor, float* moments, float* z, int B, int C, int P, void* stream) {
  if (!x || !W || !bias || !moments || B <= 0 || C <= 0 || C > 8 || C % 2 || ldx < C || P <= 0) return MDT_ERR_ARG;
  if (eps && !z) return MDT_ERR_ARG;
  const long long n = static_cast<long long>(B) * P;
  vae_quant_moments_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, VS(stream)>>>(x, ldx, W, bias, eps,
                                                                                     scale_factor, moments, z, B, C, P);
  return vae_status();
}

}  // extern "C"
