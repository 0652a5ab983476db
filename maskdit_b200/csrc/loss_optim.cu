// EDM preconditioning output, EDM + MAE loss (forward + gradient seed), CFG combine, Heun update, fused AdamW+EMA.
#include <math.h>

#include "common.cuh"
#include "../../include/maskdit_b200.h"

namespace mdt {

static inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }
static inline int launch_status() { return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA; }

constexpr int kMaxPD = 64;  // p*p*C per patch (16 for patch 2 x 4 channels)

struct PatchGeom {
  int C, R, p, G, L, pd;
  // element j of a patch vector is ordered (ph, pw, c) — DiT.unpatchify 'nhwpqc->nchpwq', models/maskdit.py:421-423
  MDT_DEVINL size_t pix(int b, int l, int j) const {
    const int c = j % C, pw = (j / C) % p, ph = j / (C * p);
    const int hh = (l / G) * p + ph, ww = (l % G) * p + pw;
    return ((static_cast<size_t>(b) * C + c) * R + hh) * R + ww;
  }
};

MDT_DEVINL float block_sum(float v, float* s_buf) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) s_buf[warp] = v;
  __syncthreads();
  float t = (threadIdx.x < (blockDim.x >> 5)) ? s_buf[threadIdx.x] : 0.f;
  if (warp == 0) t = warp_sum(t);
  if (threadIdx.x == 0) s_buf[0] = t;
  __syncthreads();
  t = s_buf[0];
  return t;
}

// One block per sample.  Thread per token.
__global__ void __launch_bounds__(256)
edm_loss_kernel(const float* __restrict__ F, const float* __restrict__ xin, const float* __restrict__ y,
                const float* __restrict__ sigma, const float* __restrict__ mask, const float* __restrict__ gl,
                float sd, float mae_coef, float* __restrict__ loss, float* __restrict__ Dx,
                __nv_bfloat16* __restrict__ dF, PatchGeom gm) {
  __shared__ float s_buf[32];
  const int b = blockIdx.x;
  const float sg = sigma[b];
  const float den = sg * sg + sd * sd;
  const float c_skip = sd * sd / den, c_out = sg * sd * rsqrtf(den);
  const float w = den / ((sg * sd) * (sg * sd));
  const float glb = gl ? gl[b] : 0.f;
  float n_mask = 0.f;
  if (mask) {
    float cnt = 0.f;
    for (int l = threadIdx.x; l < gm.L; l += blockDim.x) cnt += mask[static_cast<size_t>(b) * gm.L + l];
    n_mask = block_sum(cnt, s_buf);
  }
  const float n_keep = static_cast<float>(gm.L) - n_mask;
  float acc = 0.f;
  for (int l = threadIdx.x; l < gm.L; l += blockDim.x) {
    const float* f = F + (static_cast<size_t>(b) * gm.L + l) * gm.pd;
    float dv[kMaxPD], xv[kMaxPD];
    float se = 0.f, sx = 0.f;
    for (int j = 0; j < gm.pd; ++j) {
      const size_t px = gm.pix(b, l, j);
      const float xi = xin[px];
      const float d = c_skip * xi + c_out * f[j];
      if (Dx) Dx[px] = d;
      const float e = d - y[px];
      dv[j] = d, xv[j] = xi;
      se += e * e, sx += xi;
    }
    const float inv_pd = 1.f / gm.pd;
    if (!mask) {
      acc += w * se;  // mean over all elements of the sample, applied below
      if (dF) {
        const float k = glb * w * 2.f * c_out / (static_cast<float>(gm.L) * gm.pd);
        for (int j = 0; j < gm.pd; ++j)
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(k * (dv[j] - y[gm.pix(b, l, j)]));
      }
    } else {
      const float mk = mask[static_cast<size_t>(b) * gm.L + l];
      float contrib = (1.f - mk) * w * se * inv_pd / n_keep;
      float k_edm = glb * (1.f - mk) / n_keep * w * 2.f * inv_pd * c_out;
      float k_mae = 0.f, mu = 0.f, rstd = 0.f;
      if (mae_coef > 0.f && mk != 0.f) {
        // mae_loss (train_utils/loss.py:87-101): target = per-patch normalised NOISY INPUT, unbiased variance
        mu = sx * inv_pd;
        float var = 0.f;
        for (int j = 0; j < gm.pd; ++j) var += (xv[j] - mu) * (xv[j] - mu);
        var /= static_cast<float>(gm.pd - 1);
        rstd = rsqrtf(var + 1e-6f);
        float sm = 0.f;
        for (int j = 0; j < gm.pd; ++j) {
          const float e = dv[j] - (xv[j] - mu) * rstd;
          sm += e * e;
        }
        contrib += mae_coef * mk * sm * inv_pd / n_mask;
        k_mae = glb * mae_coef * mk / n_mask * 2.f * inv_pd * c_out;
      }
      acc += contrib;
      if (dF) {
        for (int j = 0; j < gm.pd; ++j) {
          float gval = k_edm * (dv[j] - y[gm.pix(b, l, j)]);
          if (k_mae != 0.f) gval += k_mae * (dv[j] - (xv[j] - mu) * rstd);
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(gval);
        }
      }
    }
  }
  const float tot = block_sum(acc, s_buf);
  if (threadIdx.x == 0) loss[b] = mask ? tot : tot / (static_cast<float>(gm.L) * gm.pd);
}

// D = c_skip*x + c_out*unpatchify(F) ; optional CFG combine of two halves of F
__global__ void precond_out_kernel(const float* __restrict__ F, const float* __restrict__ xin,
                                   const float* __restrict__ sigma, float sd, float cfg_scale, int use_cfg, int B,
                                   float* __restrict__ Dx, PatchGeom gm) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * gm.L) return;
  const int b = idx / gm.L, l = idx % gm.L;
  const float sg = sigma[b];
  const float den = sg * sg + sd * sd;
  const float c_skip = sd * sd / den, c_out = sg * sd * rsqrtf(den);
  const float* fc = F + (static_cast<size_t>(b) * gm.L + l) * gm.pd;
  const float* fu = F + (static_cast<size_t>(b + B) * gm.L + l) * gm.pd;
  for (int j = 0; j < gm.pd; ++j) {
    float f = fc[j];
    if (use_cfg) f = fu[j] + cfg_scale * (f - fu[j]);
    const size_t px = gm.pix(b, l, j);
    Dx[px] = c_skip * xin[px] + c_out * f;
  }
}
__global__ void precond_out_bwd_kernel(const float* __restrict__ gD, const float* __restrict__ sigma, float sd, int B,
                                       __nv_bfloat16* __restrict__ dF, PatchGeom gm) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * gm.L) return;
  const int b = idx / gm.L, l = idx % gm.L;
  const float sg = sigma[b];
  const float c_out = sg * sd * rsqrtf(sg * sg + sd * sd);
  for (int j = 0; j < gm.pd; ++j)
    dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(c_out * gD[gm.pix(b, l, j)]);
}

__global__ void heun_kernel(int mode, const double* __restrict__ x_hat, const float* __restrict__ den,
                            double* __restrict__ d_cur, double* __restrict__ x_next, float* __restrict__ x_next_f32,
                            double t_hat, double t_next, long long n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  double xn;
  if (mode == 0) {
    const double d = (x_hat[i] - static_cast<double>(den[i])) / t_hat;
    d_cur[i] = d;
    xn = x_hat[i] + (t_next - t_hat) * d;
  } else {
    const double dp = (x_next[i] - static_cast<double>(den[i])) / t_next;
    xn = x_hat[i] + (t_next - t_hat) * (0.5 * d_cur[i] + 0.5 * dp);
  }
  x_next[i] = xn;
  if (x_next_f32) x_next_f32[i] = static_cast<float>(xn);
}

// Generalised sampler state update (ablation_sampler, sample.py:73-188: every Euler / Heun / churn update is a linear
// combination of the fp64 state, a second fp64 tensor and one fp32 network output with host-computed fp64 scalars):
//   out = a*x + b*y + c*z ;  out_f32 = float(out * f32_scale)   (the next network input x / s(t))
// Also: sample -> 8-bit pixel conversion of the sampler tail (sample.py:287): (v + 1) * 127.5 clamped, NCHW -> NHWC.
__global__ void lincomb_f64_kernel(double a, const double* __restrict__ x, double b, const double* __restrict__ y,
                                   double c, const float* __restrict__ z, double* __restrict__ out,
                                   float* __restrict__ out_f32, double f32_scale, long long n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  double v = a * x[i];
  if (y) v += b * y[i];
  if (z) v += c * static_cast<double>(z[i]);
  if (out) out[i] = v;
  if (out_f32) out_f32[i] = static_cast<float>(v * f32_scale);
}

__global__ void to_uint8_nhwc_kernel(const float* __restrict__ img, unsigned char* __restrict__ out, int B, int C,
                                     int H, int W) {
  const long long n = static_cast<long long>(B) * C * H * W;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;  // output index (b, h, w, c)
  if (i >= n) return;
  const int c = static_cast<int>(i % C);
  const long long p = i / C;
  const int w = static_cast<int>(p % W), h = static_cast<int>((p / W) % H), b = static_cast<int>(p / (static_cast<long long>(W) * H));
  float v = (img[((static_cast<long long>(b) * C + c) * H + h) * W + w] + 1.f) * 127.5f;
  v = fminf(fmaxf(v, 0.f), 255.f);
  out[i] = static_cast<unsigned char>(v);  // truncation, as .to(torch.uint8)
}

// Fused AdamW + EMA + bf16 shadow, float4-vectorised over flat buffers.
template <bool G16>  // G16: the gradient operand is bf16 (the buffer a bf16 all-reduce produced), else fp32
__global__ void __launch_bounds__(256)
adamw_ema_kernel(float* __restrict__ w, const void* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 float* __restrict__ ema, __nv_bfloat16* __restrict__ w16, long long n, float lr, float b1, float b2,
                 float eps, float wd, float inv_bc1, float inv_bc2, float ema_decay, float gscale) {
  const long long n4 = n >> 2;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4; i += stride) {
    float4 wv = reinterpret_cast<float4*>(w)[i];
    float4 gv;
    if constexpr (G16) {
      const uint2 u = reinterpret_cast<const uint2*>(g)[i];
      gv = make_float4(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y));
    } else {
      gv = reinterpret_cast<const float4*>(g)[i];
    }
    float4 mv = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    float* wp = &wv.x;
    float* gp = &gv.x;
    float* mp = &mv.x;
    float* vp = &vv.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float gk = gp[k] * gscale;
      mp[k] = b1 * mp[k] + (1.f - b1) * gk;
      vp[k] = b2 * vp[k] + (1.f - b2) * gk * gk;
      const float upd = (mp[k] * inv_bc1) / (sqrtf(vp[k] * inv_bc2) + eps);
      wp[k] = wp[k] * (1.f - lr * wd) - lr * upd;
    }
    reinterpret_cast<float4*>(w)[i] = wv;
    reinterpret_cast<float4*>(m)[i] = mv;
    reinterpret_cast<float4*>(v)[i] = vv;
    if (ema) {
      float4 ev = reinterpret_cast<float4*>(ema)[i];
      ev.x = ema_decay * ev.x + (1.f - ema_decay) * wv.x, ev.y = ema_decay * ev.y + (1.f - ema_decay) * wv.y;
      ev.z = ema_decay * ev.z + (1.f - ema_decay) * wv.z, ev.w = ema_decay * ev.w + (1.f - ema_decay) * wv.w;
      reinterpret_cast<float4*>(ema)[i] = ev;
    }
    if (w16) reinterpret_cast<uint2*>(w16)[i] = make_uint2(pack_bf16(wv.x, wv.y), pack_bf16(wv.z, wv.w));
  }
}


// Step front (SURVEY 8(f)2): VAE moments -> latent (utils.py:59-65), label dropout (train.py:209), sigma draw and
// noise injection (train_utils/loss.py:35-39) in ONE pass over the batch, given the pre-drawn normals / uniforms
// (drawn by the caller's generator in the reference's order).  Thread = 4 consecutive pixels of one channel plane.
//   y  = sf * (mean + exp(0.5 clamp(logvar, -30, 20)) * eps)        sigma = exp(P_std * rnd + P_mean)
//   yn = y + noise * sigma                                            labels[b, :] *= (drop_u[b] >= drop_prob)
__global__ void __launch_bounds__(256)
step_front_kernel(const float* __restrict__ moments, const float* __restrict__ eps, const float* __restrict__ rnd,
                  const float* __restrict__ noise, const float* __restrict__ drop_u, float drop_prob, float sf,
                  float P_mean, float P_std, float* __restrict__ y, float* __restrict__ yn, float* __restrict__ sigma,
                  float* __restrict__ labels, int B, int C, int plane4, int nc) {
  const long long per = static_cast<long long>(C) * plane4;  // float4 groups per sample
  const long long total = static_cast<long long>(B) * per;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / per);
    const long long r = i - b * per;  // (c, pixel group) inside the sample
    const float sg = expf(rnd[b] * P_std + P_mean);
    const float4* mom = reinterpret_cast<const float4*>(moments) + static_cast<long long>(b) * 2 * per;
    const float4 mu = mom[r], lv = mom[per + r];
    const float4 e = reinterpret_cast<const float4*>(eps)[i], nz = reinterpret_cast<const float4*>(noise)[i];
    float4 o, on;
    o.x = sf * (mu.x + expf(0.5f * fminf(fmaxf(lv.x, -30.f), 20.f)) * e.x);
    o.y = sf * (mu.y + expf(0.5f * fminf(fmaxf(lv.y, -30.f), 20.f)) * e.y);
    o.z = sf * (mu.z + expf(0.5f * fminf(fmaxf(lv.z, -30.f), 20.f)) * e.z);
    o.w = sf * (mu.w + expf(0.5f * fminf(fmaxf(lv.w, -30.f), 20.f)) * e.w);
    on = make_float4(fmaf(nz.x, sg, o.x), fmaf(nz.y, sg, o.y), fmaf(nz.z, sg, o.z), fmaf(nz.w, sg, o.w));
    reinterpret_cast<float4*>(y)[i] = o;
    reinterpret_cast<float4*>(yn)[i] = on;
    if (r == 0) sigma[b] = sg;
  }
  if (labels && drop_u) {
    const long long nl = static_cast<long long>(B) * nc;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nl;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      const int b = static_cast<int>(i / nc);
      if (!(drop_u[b] >= drop_prob)) labels[i] = 0.f;   // y * (rand >= p): dropped rows become the CFG-null label
    }
  }
}

}  // namespace mdt

using namespace mdt;

static int make_geom(PatchGeom* gm, int C, int R, int p) {
  if (C <= 0 || R <= 0 || p <= 0 || R % p) return MDT_ERR_ARG;
  gm->C = C, gm->R = R, gm->p = p, gm->G = R / p, gm->L = gm->G * gm->G, gm->pd = p * p * C;
  return gm->pd <= kMaxPD ? MDT_OK : MDT_ERR_UNSUPPORTED;
}

extern "C" {

int mdt_edm_loss(const float* F, const float* xin, const float* y, const float* sigma, const float* mask,
                 const float* gl, float sigma_data, float mae_coef, float* loss, float* Dx, void* dF_bf16, int B,
                 int C, int R, int p, void* stream) {
  if (!F || !xin || !y || !sigma || !loss || B <= 0) return MDT_ERR_ARG;
  if (dF_bf16 && !gl) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  edm_loss_kernel<<<B, 256, 0, S(stream)>>>(F, xin, y, sigma, mask, gl, sigma_data, mae_coef, loss, Dx,
                                            static_cast<__nv_bfloat16*>(dF_bf16), gm);
  return launch_status();
}

int mdt_edm_precond_out(const float* F, const float* xin, const float* sigma, float sigma_data, float* Dx, int B,
                        int C, int R, int p, void* stream) {
  if (!F || !xin || !sigma || !Dx || B <= 0) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  const int n = B * gm.L;
  precond_out_kernel<<<(n + 127) / 128, 128, 0, S(stream)>>>(F, xin, sigma, sigma_data, 0.f, 0, B, Dx, gm);
  return launch_status();
}

int mdt_cfg_precond_out(const float* F, const float* xin, const float* sigma, float sigma_data, float cfg_scale,
                        float* Dx, int B, int C, int R, int p, void* stream) {
  if (!F || !xin || !sigma || !Dx || B <= 0) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  const int n = B * gm.L;
  precond_out_kernel<<<(n + 127) / 128, 128, 0, S(stream)>>>(F, xin, sigma, sigma_data, cfg_scale, 1, B, Dx, gm);
  return launch_status();
}

int mdt_edm_precond_out_bwd(const float* gD, const float* sigma, float sigma_data, void* dF_bf16, int B, int C, int R,
                            int p, void* stream) {
  if (!gD || !sigma || !dF_bf16 || B <= 0) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  const int n = B * gm.L;
  precond_out_bwd_kernel<<<(n + 127) / 128, 128, 0, S(stream)>>>(gD, sigma, sigma_data, B,
                                                                 static_cast<__nv_bfloat16*>(dF_bf16), gm);
  return launch_status();
}

int mdt_heun_update(int mode, const double* x_hat, const float* denoised, double* d_cur, double* x_next,
                    float* x_next_f32, double t_hat, double t_next, long long n, void* stream) {
  if (!x_hat || !denoised || !d_cur || !x_next || n <= 0 || (mode != 0 && mode != 1)) return MDT_ERR_ARG;
  heun_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, S(stream)>>>(mode, x_hat, denoised, d_cur, x_next,
                                                                        x_next_f32, t_hat, t_next, n);
  return launch_status();
}

int mdt_lincomb_f64(double a, const double* x, double b, const double* y, double c, const float* z, double* out,
                    float* out_f32, double f32_scale, long long n, void* stream) {
  if (!x || (!out && !out_f32) || n <= 0) return MDT_ERR_ARG;
  lincomb_f64_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, S(stream)>>>(a, x, b, y, c, z, out, out_f32,
                                                                               f32_scale, n);
  return launch_status();
}

int mdt_to_uint8_nhwc(const float* img, unsigned char* out, int B, int C, int H, int W, void* stream) {
  if (!img || !out || B <= 0 || C <= 0 || H <= 0 || W <= 0) return MDT_ERR_ARG;
  const long long n = static_cast<long long>(B) * C * H * W;
  to_uint8_nhwc_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, S(stream)>>>(img, out, B, C, H, W);
  return launch_status();
}

static int adamw_launch(bool g16, float* w, const void* g, float* m, float* v, float* ema, void* w_bf16, long long n,
                        float lr, float beta1, float beta2, float eps, float weight_decay, int step, float ema_decay,
                        float grad_scale, int max_blocks, void* stream) {
  if (!w || !g || !m || !v || n <= 0 || step < 1 || (n & 3)) return MDT_ERR_ARG;
  const float inv_bc1 = static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(beta1), step)));
  const float inv_bc2 = static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(beta2), step)));
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > kNumSMsDefault * 8) blocks = kNumSMsDefault * 8;
  if (max_blocks > 0 && blocks > max_blocks) blocks = max_blocks;
  auto kern = g16 ? adamw_ema_kernel<true> : adamw_ema_kernel<false>;
  kern<<<static_cast<int>(blocks), 256, 0, S(stream)>>>(w, g, m, v, ema, static_cast<__nv_bfloat16*>(w_bf16), n, lr,
                                                        beta1, beta2, eps, weight_decay, inv_bc1, inv_bc2, ema_decay,
                                                        grad_scale);
  return launch_status();
}

int mdt_adamw_ema(float* w, const float* g, float* m, float* v, float* ema, void* w_bf16, long long n, float lr,
                  float beta1, float beta2, float eps, float weight_decay, int step, float ema_decay,
                  float grad_scale, int max_blocks, void* stream) {
  return adamw_launch(false, w, g, m, v, ema, w_bf16, n, lr, beta1, beta2, eps, weight_decay, step, ema_decay,
                      grad_scale, max_blocks, stream);
}

int mdt_adamw_ema_g16(float* w, const void* g_bf16, float* m, float* v, float* ema, void* w_bf16, long long n,
                      float lr, float beta1, float beta2, float eps, float weight_decay, int step, float ema_decay,
                      float grad_scale, int max_blocks, void* stream) {
  return adamw_launch(true, w, g_bf16, m, v, ema, w_bf16, n, lr, beta1, beta2, eps, weight_decay, step, ema_decay,
                      grad_scale, max_blocks, stream);
}

int mdt_step_front(const float* moments, const float* eps, const float* rnd_normal, const float* noise_unit,
                   const float* drop_u, float drop_prob, float scale_factor, float P_mean, float P_std, float* y,
                   float* yn, float* sigma, float* labels, int B, int C, int R, int num_classes, void* stream) {
  if (!moments || !eps || !rnd_normal || !noise_unit || !y || !yn || !sigma || B <= 0 || C <= 0 || R <= 0)
    return MDT_ERR_ARG;
  if ((R * R) % 4) return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(moments) | reinterpret_cast<uintptr_t>(eps) | reinterpret_cast<uintptr_t>(noise_unit) |
       reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(yn)) & 15)
    return MDT_ERR_ARG;
  const long long total = static_cast<long long>(B) * C * (R * R / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > kNumSMsDefault * 8) blocks = kNumSMsDefault * 8;
  step_front_kernel<<<static_cast<int>(blocks), 256, 0, S(stream)>>>(moments, eps, rnd_normal, noise_unit, drop_u,
                                                                     drop_prob, scale_factor, P_mean, P_std, y, yn,
                                                                     sigma, labels, B, C, R * R / 4, num_classes);
  return launch_status();
}

}  // extern "C"
