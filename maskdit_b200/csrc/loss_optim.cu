// EDM preconditioning output, EDM + MAE loss (forward + gradient seed), CFG and guide-network combines, Heun update,
// the rectified-flow loss, output and step front, fused AdamW+EMA, power-function EMA profiles (post-hoc EMA).
#include <math.h>

#include "common.cuh"
#include "../../include/maskdit_b200.h"

namespace mdt {

static inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }
static inline int launch_status() { return cudaGetLastError() == cudaSuccess ? MDT_OK : MDT_ERR_CUDA; }

constexpr int kMaxPD = 64;  // p*p*C per patch held in registers by edm_loss (16 for patch 2 x 4 channels)

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

// ---- Learned loss weighting (EDM2 uncertainty weighting, Karras et al. CVPR 2024) --------------------------------------
// u(sigma) = sum_j w_j phi_j(c), c = ln(sigma) / 4, phi_j(c) = sqrt(2) cos(freqs_j c + phases_j), j < C <= 256.
constexpr int kMaxLogvar = 256;
struct LogvarArgs {
  const float *freqs, *phases, *w;   // [C] each: the frozen Fourier features and the [1, C] linear's weight
  int C;
  float *objective, *u, *du;         // [B] each (du only with a gradient seed)
};

// The feature is evaluated in fp64 and rounded once: |freqs_j c| reaches ~30, where an fp32 argument alone is ~2e-6 off.
MDT_DEVINL float logvar_phi(float freq, float phase, float sg) {
  const double c = log(static_cast<double>(sg)) * 0.25;
  return static_cast<float>(1.4142135623730951 * cos(static_cast<double>(freq) * c + static_cast<double>(phase)));
}

// u of one sample: thread j < C forms w_j phi_j, one block sum of 256 threads (every caller launches 256).
MDT_DEVINL float logvar_u(const LogvarArgs& lv, float sg, float* s_buf) {
  const int j = threadIdx.x;
  return block_sum(j < lv.C ? lv.w[j] * logvar_phi(lv.freqs[j], lv.phases[j], sg) : 0.f, s_buf);
}

// One block per sample.  Thread per token.  kReg: the token's D and x live in registers (pd <= kMaxPD); otherwise
// (patch 8: pd = 256) every later pass re-reads F and xin and recomputes D with the same expression.
// kLogvar: also the learned weighting's objective exp(-u) E + u + mae_coef M, where E is the EDM term, summed apart,
// and E + mae_coef M is `loss` (accumulated as without kLogvar): the EDM term's gradient seed is scaled by
// gl[b] exp(-u), the MAE term's by gl[b], and du[b] = gl[b] (1 - exp(-u) E).
template <bool kReg, bool kLogvar>
__global__ void __launch_bounds__(256)
edm_loss_kernel(const float* __restrict__ F, const float* __restrict__ xin, const float* __restrict__ y,
                const float* __restrict__ sigma, const float* __restrict__ mask, const float* __restrict__ gl,
                float sd, float mae_coef, float* __restrict__ loss, float* __restrict__ Dx,
                __nv_bfloat16* __restrict__ dF, PatchGeom gm, LogvarArgs lv) {
  __shared__ float s_buf[32];
  const int b = blockIdx.x;
  const float sg = sigma[b];
  const float den = sg * sg + sd * sd;
  const float c_skip = sd * sd / den, c_out = sg * sd * rsqrtf(den);
  const float w = den / ((sg * sd) * (sg * sd));
  const float glb = gl ? gl[b] : 0.f;
  float u = 0.f, glb_e = glb, acc_e = 0.f;   // glb_e: the EDM term's gradient scale
  if constexpr (kLogvar) {
    u = logvar_u(lv, sg, s_buf);
    glb_e = glb * expf(-u);
  }
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
    float dv[kReg ? kMaxPD : 1], xv[kReg ? kMaxPD : 1];
    auto xat = [&](int j) -> float {
      if constexpr (kReg) return xv[j];
      else return xin[gm.pix(b, l, j)];
    };
    auto dat = [&](int j) -> float {
      if constexpr (kReg) return dv[j];
      else return c_skip * xin[gm.pix(b, l, j)] + c_out * f[j];
    };
    float se = 0.f, sx = 0.f;
    for (int j = 0; j < gm.pd; ++j) {
      const size_t px = gm.pix(b, l, j);
      const float xi = xin[px];
      const float d = c_skip * xi + c_out * f[j];
      if (Dx) Dx[px] = d;
      const float e = d - y[px];
      if constexpr (kReg) dv[j] = d, xv[j] = xi;
      se += e * e, sx += xi;
    }
    const float inv_pd = 1.f / gm.pd;
    if (!mask) {
      acc += w * se;  // mean over all elements of the sample, applied below
      if constexpr (kLogvar) acc_e += w * se;
      if (dF) {
        const float k = glb_e * w * 2.f * c_out / (static_cast<float>(gm.L) * gm.pd);
        for (int j = 0; j < gm.pd; ++j)
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(k * (dat(j) - y[gm.pix(b, l, j)]));
      }
    } else {
      const float mk = mask[static_cast<size_t>(b) * gm.L + l];
      float contrib = (1.f - mk) * w * se * inv_pd / n_keep;
      if constexpr (kLogvar) acc_e += contrib;
      float k_edm = glb_e * (1.f - mk) / n_keep * w * 2.f * inv_pd * c_out;
      float k_mae = 0.f, mu = 0.f, rstd = 0.f;
      if (mae_coef > 0.f && mk != 0.f) {
        // mae_loss (train_utils/loss.py:87-101): target = per-patch normalised NOISY INPUT, unbiased variance
        mu = sx * inv_pd;
        float var = 0.f;
        for (int j = 0; j < gm.pd; ++j) var += (xat(j) - mu) * (xat(j) - mu);
        var /= static_cast<float>(gm.pd - 1);
        rstd = rsqrtf(var + 1e-6f);
        float sm = 0.f;
        for (int j = 0; j < gm.pd; ++j) {
          const float e = dat(j) - (xat(j) - mu) * rstd;
          sm += e * e;
        }
        contrib += mae_coef * mk * sm * inv_pd / n_mask;
        k_mae = glb * mae_coef * mk / n_mask * 2.f * inv_pd * c_out;
      }
      acc += contrib;
      if (dF) {
        for (int j = 0; j < gm.pd; ++j) {
          const float dj = dat(j);
          float gval = k_edm * (dj - y[gm.pix(b, l, j)]);
          if (k_mae != 0.f) gval += k_mae * (dj - (xat(j) - mu) * rstd);
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(gval);
        }
      }
    }
  }
  const float tot = block_sum(acc, s_buf);
  if constexpr (kLogvar) {
    float e = block_sum(acc_e, s_buf);
    if (threadIdx.x == 0) {
      const float lb = mask ? tot : tot / (static_cast<float>(gm.L) * gm.pd);
      if (!mask) e /= static_cast<float>(gm.L) * gm.pd;
      // exp(-u) E + u + M written as (E + M) + expm1(-u) E + u: at u = 0 exactly the reference loss
      lv.objective[b] = lb + expm1f(-u) * e + u;
      lv.u[b] = u;
      if (lv.du) lv.du[b] = glb * (1.f - expf(-u) * e);
    }
  }
  if (threadIdx.x == 0) loss[b] = mask ? tot : tot / (static_cast<float>(gm.L) * gm.pd);
}

// Rectified flow (linear interpolant, velocity prediction; DESIGN §5): x_t = (1 - t) x + t eps, F unpatchified is the
// velocity v^, the target is v = eps - x (formed from eps and x, not from x_t) and x^ = x_t - t v^ is the denoised
// estimate that the MAE term reads.  edm_loss_kernel's structure: one block per sample, thread per token, kReg: the
// token's velocity error and x_t live in registers (pd <= kMaxPD), otherwise later passes re-read F, x_t, eps and x.
template <bool kReg>
__global__ void __launch_bounds__(256)
flow_loss_kernel(const float* __restrict__ F, const float* __restrict__ xt, const float* __restrict__ y,
                 const float* __restrict__ eps, const float* __restrict__ tt, const float* __restrict__ mask,
                 const float* __restrict__ gl, float mae_coef, float* __restrict__ loss, float* __restrict__ Dx,
                 __nv_bfloat16* __restrict__ dF, PatchGeom gm) {
  __shared__ float s_buf[32];
  const int b = blockIdx.x;
  const float tb = tt[b];
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
    float ev[kReg ? kMaxPD : 1], xv[kReg ? kMaxPD : 1];
    auto xat = [&](int j) -> float {
      if constexpr (kReg) return xv[j];
      else return xt[gm.pix(b, l, j)];
    };
    auto eat = [&](int j) -> float {   // v^ - v
      if constexpr (kReg) return ev[j];
      else {
        const size_t px = gm.pix(b, l, j);
        return f[j] - (eps[px] - y[px]);
      }
    };
    auto dat = [&](int j) -> float { return __fmaf_rn(-tb, f[j], xat(j)); };   // x^ = x_t - t v^
    float se = 0.f, sx = 0.f;
    for (int j = 0; j < gm.pd; ++j) {
      const size_t px = gm.pix(b, l, j);
      const float xi = xt[px];
      const float e = f[j] - (eps[px] - y[px]);
      if (Dx) Dx[px] = __fmaf_rn(-tb, f[j], xi);
      if constexpr (kReg) ev[j] = e, xv[j] = xi;
      se += e * e, sx += xi;
    }
    const float inv_pd = 1.f / gm.pd;
    if (!mask) {
      acc += se;  // mean over all elements of the sample, applied below
      if (dF) {
        const float k = glb * 2.f / (static_cast<float>(gm.L) * gm.pd);
        for (int j = 0; j < gm.pd; ++j)
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(k * eat(j));
      }
    } else {
      const float mk = mask[static_cast<size_t>(b) * gm.L + l];
      float contrib = (1.f - mk) * se * inv_pd / n_keep;
      const float k_v = glb * (1.f - mk) / n_keep * 2.f * inv_pd;
      float k_mae = 0.f, mu = 0.f, rstd = 0.f;
      if (mae_coef > 0.f && mk != 0.f) {
        // MaskDiT's MAE term with D replaced by x^: target = per-patch normalised x_t, unbiased variance
        mu = sx * inv_pd;
        float var = 0.f;
        for (int j = 0; j < gm.pd; ++j) var += (xat(j) - mu) * (xat(j) - mu);
        var /= static_cast<float>(gm.pd - 1);
        rstd = rsqrtf(var + 1e-6f);
        float sm = 0.f;
        for (int j = 0; j < gm.pd; ++j) {
          const float e = dat(j) - (xat(j) - mu) * rstd;
          sm += e * e;
        }
        contrib += mae_coef * mk * sm * inv_pd / n_mask;
        k_mae = -tb * glb * mae_coef * mk / n_mask * 2.f * inv_pd;   // d x^ / d v^ = -t
      }
      acc += contrib;
      if (dF) {
        for (int j = 0; j < gm.pd; ++j) {
          float gval = k_v * eat(j);
          if (k_mae != 0.f) gval += k_mae * (dat(j) - (xat(j) - mu) * rstd);
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(gval);
        }
      }
    }
  }
  const float tot = block_sum(acc, s_buf);
  if (threadIdx.x == 0) loss[b] = mask ? tot : tot / (static_cast<float>(gm.L) * gm.pd);
}

// Easy Consistency Tuning (DESIGN §5): the student D_t = c_skip(t) x_t + c_out(t) F_t against the no-gradient target
// D_r = c_skip(r) x_r + c_out(r) F_r (r > 0) or the clean latent y (r = 0, selected, so F_r of such a row never enters).
// Per sample: S = (L / T) sum_kept delta^2, loss = (sqrt(S + c^2) - c) / (t - r) + mae_coef M; the pseudo-Huber term is
// formed as S / (sqrt(S + c^2) + c), which has no cancellation when S << c^2 (a small stage gap).  edm_loss_kernel's
// structure: one block per sample, thread per token, fixed block sums.  S must be complete before any gradient seed,
// so the seed is a second pass over the tokens that re-reads its operands (every patch size, pd 16 / 64 / 256).
__global__ void __launch_bounds__(256)
ect_loss_kernel(const float* __restrict__ Ft, const float* __restrict__ Fr, const float* __restrict__ xt,
                const float* __restrict__ xr, const float* __restrict__ y, const float* __restrict__ tt,
                const float* __restrict__ rr, const float* __restrict__ mask, const float* __restrict__ gl, float sd,
                float c_h, float mae_coef, float* __restrict__ loss, float* __restrict__ Dx,
                __nv_bfloat16* __restrict__ dF, PatchGeom gm) {
  __shared__ float s_buf[32];
  const int b = blockIdx.x;
  const float t = tt[b], r = rr[b];
  const bool has_r = r > 0.f;
  const float den_t = t * t + sd * sd, den_r = r * r + sd * sd;
  const float cs_t = sd * sd / den_t, co_t = t * sd * rsqrtf(den_t);
  // r > 0: delta = c_skip(t) (x_t - x_r) + dcs x_r + c_out(t) (F_t - F_r) + dco F_r, where dcs = c_skip(t) - c_skip(r)
  // and dco = c_out(t) - c_out(r) are formed from t - r (exact in fp32 for r >= t / 2) instead of as differences of
  // nearly equal values: at a small gap and small t, fp32 rounding of c_skip alone is as large as c_skip(t) - c_skip(r).
  const float gap = t - r, tpr = t + r, rt_t = sqrtf(den_t), rt_r = sqrtf(den_r);
  const float dcs = -sd * sd * gap * tpr / (den_t * den_r);
  const float dco = sd * sd * sd * gap * tpr / ((t * rt_r + r * rt_t) * rt_t * rt_r);
  auto d_t = [&](size_t px, float f) -> float { return cs_t * xt[px] + co_t * f; };
  auto delta = [&](size_t px, float ft, float fr) -> float {
    if (!has_r) return d_t(px, ft) - y[px];       // a select: F_r of an r = 0 row is never read
    const float xrv = xr[px];
    return cs_t * (xt[px] - xrv) + dcs * xrv + co_t * (ft - fr) + dco * fr;
  };
  // MaskDiT's MAE statistics of one removed token: the per-patch mean and 1 / std (unbiased) of x_t
  auto mae_stats = [&](int l, float* mu, float* rstd) {
    float sx = 0.f;
    for (int j = 0; j < gm.pd; ++j) sx += xt[gm.pix(b, l, j)];
    *mu = sx / gm.pd;
    float var = 0.f;
    for (int j = 0; j < gm.pd; ++j) {
      const float v = xt[gm.pix(b, l, j)] - *mu;
      var += v * v;
    }
    *rstd = rsqrtf(var / static_cast<float>(gm.pd - 1) + 1e-6f);
  };
  float n_mask = 0.f;
  if (mask) {
    float cnt = 0.f;
    for (int l = threadIdx.x; l < gm.L; l += blockDim.x) cnt += mask[static_cast<size_t>(b) * gm.L + l];
    n_mask = block_sum(cnt, s_buf);
  }
  const float n_keep = static_cast<float>(gm.L) - n_mask;
  const bool mae = mask && mae_coef > 0.f;
  float acc_s = 0.f, acc_m = 0.f;
  for (int l = threadIdx.x; l < gm.L; l += blockDim.x) {
    const size_t row = (static_cast<size_t>(b) * gm.L + l) * gm.pd;
    const float mk = mask ? mask[static_cast<size_t>(b) * gm.L + l] : 0.f;
    float se = 0.f;
    for (int j = 0; j < gm.pd; ++j) {
      const size_t px = gm.pix(b, l, j);
      if (Dx) Dx[px] = d_t(px, Ft[row + j]);
      const float e = delta(px, Ft[row + j], Fr[row + j]);
      se += e * e;
    }
    acc_s += (1.f - mk) * se;
    if (mae && mk != 0.f) {
      float mu, rstd, sm = 0.f;
      mae_stats(l, &mu, &rstd);
      for (int j = 0; j < gm.pd; ++j) {
        const size_t px = gm.pix(b, l, j);
        const float e = d_t(px, Ft[row + j]) - (xt[px] - mu) * rstd;
        sm += e * e;
      }
      acc_m += mk * sm / gm.pd / n_mask;
    }
  }
  const float scale = static_cast<float>(gm.L) / n_keep;          // L / T
  const float S = block_sum(acc_s, s_buf) * scale;
  const float M = mae ? block_sum(acc_m, s_buf) : 0.f;
  const float root = sqrtf(S + c_h * c_h);
  if (threadIdx.x == 0) loss[b] = S / (root + c_h) / gap + mae_coef * M;
  if (!dF) return;
  const float glb = gl[b];
  const float k_s = glb * co_t / (gap * root) * scale;
  for (int l = threadIdx.x; l < gm.L; l += blockDim.x) {
    const size_t row = (static_cast<size_t>(b) * gm.L + l) * gm.pd;
    const float mk = mask ? mask[static_cast<size_t>(b) * gm.L + l] : 0.f;
    const float k_d = k_s * (1.f - mk);
    float k_mae = 0.f, mu = 0.f, rstd = 0.f;
    if (mae && mk != 0.f) {
      mae_stats(l, &mu, &rstd);
      k_mae = glb * mae_coef * mk / n_mask * 2.f / gm.pd * co_t;
    }
    for (int j = 0; j < gm.pd; ++j) {
      const size_t px = gm.pix(b, l, j);
      float gval = 0.f;
      if (k_d != 0.f) gval = k_d * delta(px, Ft[row + j], Fr[row + j]);
      if (k_mae != 0.f) gval += k_mae * (d_t(px, Ft[row + j]) - (xt[px] - mu) * rstd);
      dF[row + j] = __float2bfloat16_rn(gval);
    }
  }
}

// ---- Model guidance (DESIGN §5) -----------------------------------------------------------------------------------------
// F is the student's output (gradient-carrying, conditional) and Fu the no-gradient output of the same weights on the
// same input and kept tokens with the null (all-zero) label row.  Row b is guided with w_b = w when its label row is
// non-zero and lo < level_b <= hi, else w_b = 0.  Its target is the plain target plus w_b c_out (F - Fu) (EDM) or
// w_b (F - Fu) (flow); where w_b = 0 it is the plain target itself, a select that never reads Fu.
struct MgArgs {
  const float* Fu;      // [B, L, pd]
  const float* labels;  // [B, nc]
  int nc;
  float w, lo, hi;
  float* edm_loss;      // [B] optional: the plain loss against the unguided target
};

// w_b of sample b, in every thread of the block.
MDT_DEVINL float mg_weight(const MgArgs& mg, int b, float level) {
  int nz = 0;
  for (int k = threadIdx.x; k < mg.nc; k += blockDim.x) nz |= mg.labels[static_cast<size_t>(b) * mg.nc + k] != 0.f;
  const bool kept = __syncthreads_or(nz) != 0;
  return (kept && level > mg.lo && level <= mg.hi) ? mg.w : 0.f;
}

// edm_loss_kernel<kReg, false> with the guided target.  The plain sums (`edm_loss`) are formed with the same operations
// in the same order, and a row with w_b = 0 takes the plain error, so there `loss` and dF are edm_loss_kernel's bits.
template <bool kReg>
__global__ void __launch_bounds__(256)
mg_loss_kernel(const float* __restrict__ F, const float* __restrict__ xin, const float* __restrict__ y,
               const float* __restrict__ sigma, const float* __restrict__ mask, const float* __restrict__ gl,
               float sd, float mae_coef, float* __restrict__ loss, float* __restrict__ Dx,
               __nv_bfloat16* __restrict__ dF, PatchGeom gm, MgArgs mg) {
  __shared__ float s_buf[32];
  const int b = blockIdx.x;
  const float sg = sigma[b];
  const float den = sg * sg + sd * sd;
  const float c_skip = sd * sd / den, c_out = sg * sd * rsqrtf(den);
  const float w = den / ((sg * sd) * (sg * sd));
  const float glb = gl ? gl[b] : 0.f;
  const float wb = mg_weight(mg, b, sg);
  const bool guided = wb != 0.f;
  float n_mask = 0.f;
  if (mask) {
    float cnt = 0.f;
    for (int l = threadIdx.x; l < gm.L; l += blockDim.x) cnt += mask[static_cast<size_t>(b) * gm.L + l];
    n_mask = block_sum(cnt, s_buf);
  }
  const float n_keep = static_cast<float>(gm.L) - n_mask;
  float acc = 0.f, acc_g = 0.f;   // the plain and the guided sums
  for (int l = threadIdx.x; l < gm.L; l += blockDim.x) {
    const float* f = F + (static_cast<size_t>(b) * gm.L + l) * gm.pd;
    const float* fu = mg.Fu + (static_cast<size_t>(b) * gm.L + l) * gm.pd;
    float dv[kReg ? kMaxPD : 1], xv[kReg ? kMaxPD : 1];
    auto xat = [&](int j) -> float {
      if constexpr (kReg) return xv[j];
      else return xin[gm.pix(b, l, j)];
    };
    auto dat = [&](int j) -> float {
      if constexpr (kReg) return dv[j];
      else return c_skip * xin[gm.pix(b, l, j)] + c_out * f[j];
    };
    auto tat = [&](int j) -> float {   // the target of element j
      const float yv = y[gm.pix(b, l, j)];
      if (!guided) return yv;
      return yv + wb * (c_out * (f[j] - fu[j]));
    };
    float se = 0.f, sx = 0.f, sq = 0.f;
    for (int j = 0; j < gm.pd; ++j) {
      const size_t px = gm.pix(b, l, j);
      const float xi = xin[px];
      const float d = c_skip * xi + c_out * f[j];
      if (Dx) Dx[px] = d;
      const float e = d - y[px];
      if constexpr (kReg) dv[j] = d, xv[j] = xi;
      se += e * e, sx += xi;
      if (guided) {
        const float eg = d - tat(j);
        sq += eg * eg;
      }
    }
    if (!guided) sq = se;
    const float inv_pd = 1.f / gm.pd;
    if (!mask) {
      acc += w * se;  // mean over all elements of the sample, applied below
      acc_g += w * sq;
      if (dF) {
        const float k = glb * w * 2.f * c_out / (static_cast<float>(gm.L) * gm.pd);
        for (int j = 0; j < gm.pd; ++j)
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(k * (dat(j) - tat(j)));
      }
    } else {
      const float mk = mask[static_cast<size_t>(b) * gm.L + l];
      float contrib = (1.f - mk) * w * se * inv_pd / n_keep;
      float contrib_g = guided ? (1.f - mk) * w * sq * inv_pd / n_keep : contrib;
      float k_edm = glb * (1.f - mk) / n_keep * w * 2.f * inv_pd * c_out;
      float k_mae = 0.f, mu = 0.f, rstd = 0.f;
      if (mae_coef > 0.f && mk != 0.f) {
        // MaskDiT's MAE term, unchanged: target = per-patch normalised noisy input, unbiased variance
        mu = sx * inv_pd;
        float var = 0.f;
        for (int j = 0; j < gm.pd; ++j) var += (xat(j) - mu) * (xat(j) - mu);
        var /= static_cast<float>(gm.pd - 1);
        rstd = rsqrtf(var + 1e-6f);
        float sm = 0.f;
        for (int j = 0; j < gm.pd; ++j) {
          const float e = dat(j) - (xat(j) - mu) * rstd;
          sm += e * e;
        }
        const float m = mae_coef * mk * sm * inv_pd / n_mask;
        contrib += m;
        contrib_g += m;
        k_mae = glb * mae_coef * mk / n_mask * 2.f * inv_pd * c_out;
      }
      acc += contrib;
      acc_g += contrib_g;
      if (dF) {
        for (int j = 0; j < gm.pd; ++j) {
          const float dj = dat(j);
          float gval = k_edm * (dj - tat(j));
          if (k_mae != 0.f) gval += k_mae * (dj - (xat(j) - mu) * rstd);
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(gval);
        }
      }
    }
  }
  const float tot = block_sum(acc_g, s_buf);
  if (threadIdx.x == 0) loss[b] = mask ? tot : tot / (static_cast<float>(gm.L) * gm.pd);
  if (mg.edm_loss) {
    const float tp = block_sum(acc, s_buf);
    if (threadIdx.x == 0) mg.edm_loss[b] = mask ? tp : tp / (static_cast<float>(gm.L) * gm.pd);
  }
}

// flow_loss_kernel<kReg> with the guided velocity target v' = (eps - x) + w_b (F - Fu), the interval on t; the same bit
// rules as mg_loss_kernel.
template <bool kReg>
__global__ void __launch_bounds__(256)
flow_mg_loss_kernel(const float* __restrict__ F, const float* __restrict__ xt, const float* __restrict__ y,
                    const float* __restrict__ eps, const float* __restrict__ tt, const float* __restrict__ mask,
                    const float* __restrict__ gl, float mae_coef, float* __restrict__ loss, float* __restrict__ Dx,
                    __nv_bfloat16* __restrict__ dF, PatchGeom gm, MgArgs mg) {
  __shared__ float s_buf[32];
  const int b = blockIdx.x;
  const float tb = tt[b];
  const float glb = gl ? gl[b] : 0.f;
  const float wb = mg_weight(mg, b, tb);
  const bool guided = wb != 0.f;
  float n_mask = 0.f;
  if (mask) {
    float cnt = 0.f;
    for (int l = threadIdx.x; l < gm.L; l += blockDim.x) cnt += mask[static_cast<size_t>(b) * gm.L + l];
    n_mask = block_sum(cnt, s_buf);
  }
  const float n_keep = static_cast<float>(gm.L) - n_mask;
  float acc = 0.f, acc_g = 0.f;
  for (int l = threadIdx.x; l < gm.L; l += blockDim.x) {
    const float* f = F + (static_cast<size_t>(b) * gm.L + l) * gm.pd;
    const float* fu = mg.Fu + (static_cast<size_t>(b) * gm.L + l) * gm.pd;
    float ev[kReg ? kMaxPD : 1], xv[kReg ? kMaxPD : 1];
    auto xat = [&](int j) -> float {
      if constexpr (kReg) return xv[j];
      else return xt[gm.pix(b, l, j)];
    };
    auto eat = [&](int j) -> float {   // v^ - v
      if constexpr (kReg) return ev[j];
      else {
        const size_t px = gm.pix(b, l, j);
        return f[j] - (eps[px] - y[px]);
      }
    };
    auto gat = [&](int j) -> float {   // v^ - v'
      if (!guided) return eat(j);
      const size_t px = gm.pix(b, l, j);
      return f[j] - ((eps[px] - y[px]) + wb * (f[j] - fu[j]));
    };
    auto dat = [&](int j) -> float { return __fmaf_rn(-tb, f[j], xat(j)); };   // x^ = x_t - t v^
    float se = 0.f, sx = 0.f, sq = 0.f;
    for (int j = 0; j < gm.pd; ++j) {
      const size_t px = gm.pix(b, l, j);
      const float xi = xt[px];
      const float e = f[j] - (eps[px] - y[px]);
      if (Dx) Dx[px] = __fmaf_rn(-tb, f[j], xi);
      if constexpr (kReg) ev[j] = e, xv[j] = xi;
      se += e * e, sx += xi;
      if (guided) {
        const float eg = gat(j);
        sq += eg * eg;
      }
    }
    if (!guided) sq = se;
    const float inv_pd = 1.f / gm.pd;
    if (!mask) {
      acc += se;  // mean over all elements of the sample, applied below
      acc_g += sq;
      if (dF) {
        const float k = glb * 2.f / (static_cast<float>(gm.L) * gm.pd);
        for (int j = 0; j < gm.pd; ++j)
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(k * gat(j));
      }
    } else {
      const float mk = mask[static_cast<size_t>(b) * gm.L + l];
      float contrib = (1.f - mk) * se * inv_pd / n_keep;
      float contrib_g = guided ? (1.f - mk) * sq * inv_pd / n_keep : contrib;
      const float k_v = glb * (1.f - mk) / n_keep * 2.f * inv_pd;
      float k_mae = 0.f, mu = 0.f, rstd = 0.f;
      if (mae_coef > 0.f && mk != 0.f) {
        // MaskDiT's MAE term with D replaced by x^, unchanged: target = per-patch normalised x_t, unbiased variance
        mu = sx * inv_pd;
        float var = 0.f;
        for (int j = 0; j < gm.pd; ++j) var += (xat(j) - mu) * (xat(j) - mu);
        var /= static_cast<float>(gm.pd - 1);
        rstd = rsqrtf(var + 1e-6f);
        float sm = 0.f;
        for (int j = 0; j < gm.pd; ++j) {
          const float e = dat(j) - (xat(j) - mu) * rstd;
          sm += e * e;
        }
        const float m = mae_coef * mk * sm * inv_pd / n_mask;
        contrib += m;
        contrib_g += m;
        k_mae = -tb * glb * mae_coef * mk / n_mask * 2.f * inv_pd;   // d x^ / d v^ = -t
      }
      acc += contrib;
      acc_g += contrib_g;
      if (dF) {
        for (int j = 0; j < gm.pd; ++j) {
          float gval = k_v * gat(j);
          if (k_mae != 0.f) gval += k_mae * (dat(j) - (xat(j) - mu) * rstd);
          dF[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j] = __float2bfloat16_rn(gval);
        }
      }
    }
  }
  const float tot = block_sum(acc_g, s_buf);
  if (threadIdx.x == 0) loss[b] = mask ? tot : tot / (static_cast<float>(gm.L) * gm.pd);
  if (mg.edm_loss) {
    const float tp = block_sum(acc, s_buf);
    if (threadIdx.x == 0) mg.edm_loss[b] = mask ? tp : tp / (static_cast<float>(gm.L) * gm.pd);
  }
}

// u(sigma_b) alone, one block of 256 threads per sample: the loss kernel's arithmetic, so the same bits.
__global__ void __launch_bounds__(256) logvar_kernel(const float* __restrict__ sigma, LogvarArgs lv) {
  __shared__ float s_buf[32];
  const float u = logvar_u(lv, sigma[blockIdx.x], s_buf);
  if (threadIdx.x == 0) lv.u[blockIdx.x] = u;
}

// dw_j += sum_i du_i phi_j(c_i): thread j sums the samples in index order in fp64 (no atomics, the same bits on every
// run) and adds the rounded sum once, so gradient-accumulation rounds add up.
__global__ void __launch_bounds__(256) logvar_wgrad_kernel(const float* __restrict__ sigma, const float* __restrict__ du,
                                                           LogvarArgs lv, int B, float* __restrict__ dw) {
  const int j = threadIdx.x;
  if (j >= lv.C) return;
  const float f = lv.freqs[j], ph = lv.phases[j];
  double acc = 0.0;
  for (int i = 0; i < B; ++i) acc += static_cast<double>(du[i]) * static_cast<double>(logvar_phi(f, ph, sigma[i]));
  dw[j] += static_cast<float>(acc);
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
// Guidance by a second network: D = c_skip*x + c_out*(Fg + w (Fm - Fg)), one thread per output pixel.  Fm and Fg are
// each read in their own network's patch geometry (the patch sizes may differ); the combine is the CFG branch above.
MDT_DEVINL float patch_at(const float* __restrict__ F, const PatchGeom& gm, int b, int c, int hh, int ww) {
  const int l = (hh / gm.p) * gm.G + ww / gm.p, j = ((hh % gm.p) * gm.p + ww % gm.p) * gm.C + c;
  return F[(static_cast<size_t>(b) * gm.L + l) * gm.pd + j];
}
__global__ void guided_precond_out_kernel(const float* __restrict__ Fm, PatchGeom gm, const float* __restrict__ Fg,
                                          PatchGeom gg, const float* __restrict__ xin, const float* __restrict__ sigma,
                                          float sd, float w, int B, float* __restrict__ Dx) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const int R = gm.R, C = gm.C;
  if (idx >= static_cast<long long>(B) * C * R * R) return;
  const int ww = static_cast<int>(idx % R), hh = static_cast<int>(idx / R % R);
  const int c = static_cast<int>(idx / (static_cast<long long>(R) * R) % C);
  const int b = static_cast<int>(idx / (static_cast<long long>(C) * R * R));
  const float sg = sigma[b];
  const float den = sg * sg + sd * sd;
  const float c_skip = sd * sd / den, c_out = sg * sd * rsqrtf(den);
  const float fm = patch_at(Fm, gm, b, c, hh, ww), fg = patch_at(Fg, gg, b, c, hh, ww);
  const float f = fg + w * (fm - fg);
  Dx[idx] = c_skip * xin[idx] + c_out * f;
}

// Flow sampler output: out = unpatchify(Fu + s (Fc - Fu)) for CFG (cond rows first, uncond rows second), else
// unpatchify(F).  One thread per output pixel.
__global__ void flow_out_kernel(const float* __restrict__ F, float cfg_scale, int use_cfg, int B,
                                float* __restrict__ out, PatchGeom gm) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const int R = gm.R, C = gm.C;
  if (idx >= static_cast<long long>(B) * C * R * R) return;
  const int ww = static_cast<int>(idx % R), hh = static_cast<int>(idx / R % R);
  const int c = static_cast<int>(idx / (static_cast<long long>(R) * R) % C);
  const int b = static_cast<int>(idx / (static_cast<long long>(C) * R * R));
  float f = patch_at(F, gm, b, c, hh, ww);
  if (use_cfg) {
    const float fu = patch_at(F, gm, b + B, c, hh, ww);
    f = fu + cfg_scale * (f - fu);
  }
  out[idx] = f;
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

// One multistep DPM-Solver++ step (dpm_solver_sampler, DESIGN §5): the data prediction D_i of this evaluation (F itself,
// or x - t F for a flow network's velocity), then x' = a x + b0 D_i + b1 H1 + b2 H2 with host-computed fp64 scalars.
// Every product and sum is rounded on its own, in that order (no contraction), so the result is the op-by-op fp64 value.
__global__ void dpm_update_kernel(const float* __restrict__ F, int velocity, double t, double* __restrict__ x,
                                  double* __restrict__ d_out, const double* __restrict__ h1,
                                  const double* __restrict__ h2, double a, double b0, double b1, double b2,
                                  float* __restrict__ x_f32, long long n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const double xi = x[i];
  const double f = static_cast<double>(F[i]);
  const double d = velocity ? __dsub_rn(xi, __dmul_rn(t, f)) : f;
  d_out[i] = d;
  double v = __dadd_rn(__dmul_rn(a, xi), __dmul_rn(b0, d));
  if (h1) v = __dadd_rn(v, __dmul_rn(b1, h1[i]));
  if (h2) v = __dadd_rn(v, __dmul_rn(b2, h2[i]));
  x[i] = v;
  if (x_f32) x_f32[i] = static_cast<float>(v);
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

// Fused AdamW + EMA + bf16 shadow, float4-vectorised over flat buffers.  One pass of the grid-stride loop; the
// unguarded and the guarded kernel share it, so a guarded step with a clear flag computes the same bits.
template <bool G16>  // G16: the gradient operand is bf16 (the buffer a bf16 all-reduce produced), else fp32
MDT_DEVINL void adamw_ema_pass(float* __restrict__ w, const void* __restrict__ g, float* __restrict__ m,
                               float* __restrict__ v, float* __restrict__ ema, __nv_bfloat16* __restrict__ w16,
                               long long n, float lr, float b1, float b2, float eps, float wd, float inv_bc1,
                               float inv_bc2, float ema_decay, float gscale) {
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

template <bool G16>
__global__ void __launch_bounds__(256)
adamw_ema_kernel(float* __restrict__ w, const void* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 float* __restrict__ ema, __nv_bfloat16* __restrict__ w16, long long n, float lr, float b1, float b2,
                 float eps, float wd, float inv_bc1, float inv_bc2, float ema_decay, float gscale) {
  adamw_ema_pass<G16>(w, g, m, v, ema, w16, n, lr, b1, b2, eps, wd, inv_bc1, inv_bc2, ema_decay, gscale);
}

// ---- Non-finite gradient guard (GradScaler's inf-skip, train.py:39-48,230) --------------------------------------------
MDT_DEVINL bool nonfinite_f32(float x) { return (__float_as_uint(x) & 0x7f800000u) == 0x7f800000u; }
MDT_DEVINL bool nonfinite_bf16x2(uint32_t u) {   // either bf16 half of the word has an all-ones exponent
  return (u & 0x7f800000u) == 0x7f800000u || (u & 0x7f80u) == 0x7f80u;
}
// One warp vote per warp; lanes that saw a non-finite element set the flag (every writer stores the same 1.0f, so the
// unordered stores are an OR).  The flag is fp32 so that a SUM all-reduce of the per-rank flags is their OR.
MDT_DEVINL void flag_or(bool bad, float* flag) {
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) *flag = 1.f;
}

__global__ void __launch_bounds__(256) nonfinite_check_kernel(const float* __restrict__ g, long long n,
                                                              float* __restrict__ flag) {
  const long long n4 = n >> 2;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  bool bad = false;
  for (long long i = t; i < n4; i += stride) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    bad |= nonfinite_f32(v.x) | nonfinite_f32(v.y) | nonfinite_f32(v.z) | nonfinite_f32(v.w);
  }
  for (long long i = (n4 << 2) + t; i < n; i += stride) bad |= nonfinite_f32(g[i]);
  flag_or(bad, flag);
}

// mdt_cast_f32_bf16's arithmetic (same rounding, same output bits) plus the check, on the bf16 values it stores.
__global__ void __launch_bounds__(256) cast_f32_bf16_check_kernel(const float* __restrict__ in,
                                                                  __nv_bfloat16* __restrict__ out, long long n,
                                                                  float* __restrict__ flag) {
  const long long n4 = n >> 2;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const float4* in4 = reinterpret_cast<const float4*>(in);
  uint2* out2 = reinterpret_cast<uint2*>(out);
  bool bad = false;
  for (long long i = t; i < n4; i += stride) {
    float4 v = in4[i];
    const uint2 o = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
    out2[i] = o;
    bad |= nonfinite_bf16x2(o.x) | nonfinite_bf16x2(o.y);
  }
  for (long long i = (n4 << 2) + t; i < n; i += stride) {
    const __nv_bfloat16 b = __float2bfloat16_rn(in[i]);
    out[i] = b;
    bad |= nonfinite_f32(__bfloat162float(b));
  }
  flag_or(bad, flag);
}

// Adam's step number of this step: the applied-step counter + 1, as the bias corrections of adamw_launch compute it.
template <bool G16>
__global__ void __launch_bounds__(256)
adamw_ema_guarded_kernel(float* __restrict__ w, const void* __restrict__ g, float* __restrict__ m,
                         float* __restrict__ v, float* __restrict__ ema, __nv_bfloat16* __restrict__ w16, long long n,
                         float lr, float b1, float b2, float eps, float wd, float ema_decay, float gscale,
                         const float* __restrict__ flag, const long long* __restrict__ counts) {
  if (*flag != 0.f) {   // skipped step: only the EMA moves, toward the unchanged weights
    if (!ema) return;
    const long long n4 = n >> 2;
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4; i += stride) {
      const float4 wv = reinterpret_cast<const float4*>(w)[i];
      float4 ev = reinterpret_cast<float4*>(ema)[i];
      ev.x = ema_decay * ev.x + (1.f - ema_decay) * wv.x, ev.y = ema_decay * ev.y + (1.f - ema_decay) * wv.y;
      ev.z = ema_decay * ev.z + (1.f - ema_decay) * wv.z, ev.w = ema_decay * ev.w + (1.f - ema_decay) * wv.w;
      reinterpret_cast<float4*>(ema)[i] = ev;
    }
    return;
  }
  __shared__ float s_bc[2];
  if (threadIdx.x == 0) {
    const double step = static_cast<double>(counts[0] + 1);
    s_bc[0] = static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(b1), step)));
    s_bc[1] = static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(b2), step)));
  }
  __syncthreads();
  adamw_ema_pass<G16>(w, g, m, v, ema, w16, n, lr, b1, b2, eps, wd, s_bc[0], s_bc[1], ema_decay, gscale);
}

// counts = {applied steps, skipped steps}: one of them advances per optimizer step, after its last guarded pass.
__global__ void optim_guard_advance_kernel(const float* __restrict__ flag, long long* __restrict__ counts) {
  counts[*flag != 0.f ? 1 : 0] += 1;
}

// ---- Gradient-norm clipping (torch.nn.utils.clip_grad_norm_) ------------------------------------------------------------
// The AdamW passes with the clip coefficient read from device memory: the gradient scale becomes grad_scale * *coef
// before the loop, so *coef == 1 computes the plain kernels' bits.
template <bool G16>
__global__ void __launch_bounds__(256)
adamw_ema_coef_kernel(float* __restrict__ w, const void* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                      float* __restrict__ ema, __nv_bfloat16* __restrict__ w16, long long n, float lr, float b1,
                      float b2, float eps, float wd, float inv_bc1, float inv_bc2, float ema_decay, float gscale,
                      const float* __restrict__ coef) {
  adamw_ema_pass<G16>(w, g, m, v, ema, w16, n, lr, b1, b2, eps, wd, inv_bc1, inv_bc2, ema_decay, gscale * *coef);
}

// adamw_ema_guarded_kernel's two branches with the scaled gradient (a skipped step reads neither g nor the scale).
template <bool G16>
__global__ void __launch_bounds__(256)
adamw_ema_guarded_coef_kernel(float* __restrict__ w, const void* __restrict__ g, float* __restrict__ m,
                              float* __restrict__ v, float* __restrict__ ema, __nv_bfloat16* __restrict__ w16,
                              long long n, float lr, float b1, float b2, float eps, float wd, float ema_decay,
                              float gscale, const float* __restrict__ coef, const float* __restrict__ flag,
                              const long long* __restrict__ counts) {
  if (*flag != 0.f) {
    if (!ema) return;
    const long long n4 = n >> 2;
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4; i += stride) {
      const float4 wv = reinterpret_cast<const float4*>(w)[i];
      float4 ev = reinterpret_cast<float4*>(ema)[i];
      ev.x = ema_decay * ev.x + (1.f - ema_decay) * wv.x, ev.y = ema_decay * ev.y + (1.f - ema_decay) * wv.y;
      ev.z = ema_decay * ev.z + (1.f - ema_decay) * wv.z, ev.w = ema_decay * ev.w + (1.f - ema_decay) * wv.w;
      reinterpret_cast<float4*>(ema)[i] = ev;
    }
    return;
  }
  __shared__ float s_bc[3];
  if (threadIdx.x == 0) {
    const double step = static_cast<double>(counts[0] + 1);
    s_bc[0] = static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(b1), step)));
    s_bc[1] = static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(b2), step)));
    s_bc[2] = gscale * *coef;
  }
  __syncthreads();
  adamw_ema_pass<G16>(w, g, m, v, ema, w16, n, lr, b1, b2, eps, wd, s_bc[0], s_bc[1], ema_decay, s_bc[2]);
}

// Fixed-order fp64 block sum (xor-shuffle tree per warp, then warp 0 over the warp sums): the same bits on every run.
MDT_DEVINL double block_sum_f64(double v, double* s_buf) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) s_buf[warp] = v;
  __syncthreads();
  double t = (threadIdx.x < (blockDim.x >> 5)) ? s_buf[threadIdx.x] : 0.0;
  if (warp == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  return t;   // valid in thread 0
}

MDT_DEVINL double sq64(float x) { return static_cast<double>(x) * static_cast<double>(x); }

// Per-block partial sums of squares of g[0, n) in fp64.  The grid and every thread's visiting order are functions of n
// alone.  A fp32 square stays below fp64's maximum, so a thread's sum is non-finite exactly when it met an inf or NaN:
// that is the non-finite check (flag != NULL), with flag_or's convention.
template <bool G16>
__global__ void __launch_bounds__(256) grad_sumsq_kernel(const void* __restrict__ g, long long n,
                                                         double* __restrict__ partials, float* __restrict__ flag) {
  __shared__ double s_buf[8];
  const long long n4 = n >> 2;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  double acc = 0.0;
  for (long long i = t; i < n4; i += stride) {
    float4 x;
    if constexpr (G16) {
      const uint2 u = reinterpret_cast<const uint2*>(g)[i];
      x = make_float4(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y));
    } else {
      x = reinterpret_cast<const float4*>(g)[i];
    }
    acc += (sq64(x.x) + sq64(x.y)) + (sq64(x.z) + sq64(x.w));
  }
  for (long long i = (n4 << 2) + t; i < n; i += stride) {
    if constexpr (G16) acc += sq64(__bfloat162float(reinterpret_cast<const __nv_bfloat16*>(g)[i]));
    else acc += sq64(reinterpret_cast<const float*>(g)[i]);
  }
  if (flag) flag_or(!isfinite(acc), flag);
  const double s = block_sum_f64(acc, s_buf);
  if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

// One block: out = the partials' sum in a fixed order (thread j takes partials j, j + 256, ... in index order).
__global__ void __launch_bounds__(256) grad_sumsq_final_kernel(const double* __restrict__ partials, int nb,
                                                               double* __restrict__ out) {
  __shared__ double s_buf[8];
  double acc = 0.0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) acc += partials[i];
  const double s = block_sum_f64(acc, s_buf);
  if (threadIdx.x == 0) *out = s;
}

// norm = fp32(grad_scale * sqrt(sum of the k slots in index order)); coef as clip_grad_norm_ computes it in fp32:
// clamp(reciprocal(norm + 1e-6) * max_norm, max = 1), NaN staying NaN; max_norm = inf measures only (coef = 1).
__global__ void grad_clip_coef_kernel(const double* __restrict__ sumsq, int k, double grad_scale, float max_norm,
                                      float* __restrict__ norm, float* __restrict__ coef, float* __restrict__ flag) {
  double s = 0.0;
  for (int i = 0; i < k; ++i) s += sumsq[i];
  const float nrm = static_cast<float>(grad_scale * sqrt(s));
  *norm = nrm;
  float c = 1.f;
  if (!isinf(max_norm)) {
    const float q = (1.f / (nrm + 1e-6f)) * max_norm;
    c = q > 1.f ? 1.f : q;
    if (flag && !isfinite(nrm)) *flag = 1.f;
  }
  *coef = c;
}

// ---- Power-function EMA profiles (post-hoc EMA, Karras et al. CVPR 2024 §3) ---------------------------------------------
// K profiles advanced from one read of w:  e += c_j * (w - e).  c_j == 1 (a profile's first step) stores w exactly.
constexpr int kMaxPowerEma = 4;
struct PowerEmaArgs {
  float* e[kMaxPowerEma];
  float c[kMaxPowerEma];
};

MDT_DEVINL float power_ema_one(float w, float e, float c) { return c == 1.f ? w : fmaf(c, w - e, e); }

// [0, head): scalar head up to the 16-byte boundary all buffers share; then n4 float4 groups; then the scalar tail.
template <int K>
__global__ void __launch_bounds__(256) power_ema_kernel(const float* __restrict__ w, PowerEmaArgs a, long long n,
                                                        long long head, long long n4) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const float4* w4 = reinterpret_cast<const float4*>(w + head);
  for (long long i = t; i < n4; i += stride) {
    const float4 wv = w4[i];
#pragma unroll
    for (int j = 0; j < K; ++j) {
      float4* e4 = reinterpret_cast<float4*>(a.e[j] + head);
      float4 ev = e4[i];
      ev.x = power_ema_one(wv.x, ev.x, a.c[j]), ev.y = power_ema_one(wv.y, ev.y, a.c[j]);
      ev.z = power_ema_one(wv.z, ev.z, a.c[j]), ev.w = power_ema_one(wv.w, ev.w, a.c[j]);
      e4[i] = ev;
    }
  }
  const long long body_end = head + (n4 << 2);
  const long long n_scalar = head + (n - body_end);
  for (long long s = t; s < n_scalar; s += stride) {
    const long long i = s < head ? s : body_end + (s - head);
    const float wv = w[i];
#pragma unroll
    for (int j = 0; j < K; ++j) a.e[j][i] = power_ema_one(wv, a.e[j][i], a.c[j]);
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


// Flow step front: mdt_step_front with the flow time and interpolant in place of the sigma draw and noise injection.
//   t = 1 / (1 + exp(-(P_mean + P_std * rnd)))                         x_t = (1 - t) y + t noise
// Each product and sum is rounded separately (no contraction), so the fp32 formula evaluated op by op gives the same bits.
__global__ void __launch_bounds__(256)
flow_step_front_kernel(const float* __restrict__ moments, const float* __restrict__ eps, const float* __restrict__ rnd,
                       const float* __restrict__ noise, const float* __restrict__ drop_u, float drop_prob, float sf,
                       float P_mean, float P_std, float* __restrict__ y, float* __restrict__ xt, float* __restrict__ tt,
                       float* __restrict__ labels, int B, int C, int plane4, int nc) {
  const long long per = static_cast<long long>(C) * plane4;  // float4 groups per sample
  const long long total = static_cast<long long>(B) * per;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / per);
    const long long r = i - b * per;
    const float a = __fadd_rn(__fmul_rn(rnd[b], P_std), P_mean);
    const float t = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-a)));
    const float s = __fsub_rn(1.f, t);
    const float4* mom = reinterpret_cast<const float4*>(moments) + static_cast<long long>(b) * 2 * per;
    const float4 mu = mom[r], lv = mom[per + r];
    const float4 e = reinterpret_cast<const float4*>(eps)[i], nz = reinterpret_cast<const float4*>(noise)[i];
    float4 o, on;
    o.x = sf * (mu.x + expf(0.5f * fminf(fmaxf(lv.x, -30.f), 20.f)) * e.x);
    o.y = sf * (mu.y + expf(0.5f * fminf(fmaxf(lv.y, -30.f), 20.f)) * e.y);
    o.z = sf * (mu.z + expf(0.5f * fminf(fmaxf(lv.z, -30.f), 20.f)) * e.z);
    o.w = sf * (mu.w + expf(0.5f * fminf(fmaxf(lv.w, -30.f), 20.f)) * e.w);
    on.x = __fadd_rn(__fmul_rn(s, o.x), __fmul_rn(t, nz.x));
    on.y = __fadd_rn(__fmul_rn(s, o.y), __fmul_rn(t, nz.y));
    on.z = __fadd_rn(__fmul_rn(s, o.z), __fmul_rn(t, nz.z));
    on.w = __fadd_rn(__fmul_rn(s, o.w), __fmul_rn(t, nz.w));
    reinterpret_cast<float4*>(y)[i] = o;
    reinterpret_cast<float4*>(xt)[i] = on;
    if (r == 0) tt[b] = t;
  }
  if (labels && drop_u) {
    const long long nl = static_cast<long long>(B) * nc;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nl;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      const int b = static_cast<int>(i / nc);
      if (!(drop_u[b] >= drop_prob)) labels[i] = 0.f;
    }
  }
}

// ECT step front: mdt_step_front's latent and label dropout, then the pair of noise levels and both noisy inputs.
//   t = exp(P_std rnd + P_mean)      r = t max(0, 1 - qs (1 + k / (1 + exp(b t))))      (k / (1 + exp(b t)) = k sigmoid(-b t))
//   x_t = y + t noise                x_r = y + r noise                                   sr = r > 0 ? r : t
// qs = q^-(s+1) is read from the device, so a replayed graph follows the stage.  Each product and sum is rounded
// separately (no contraction), so the fp32 formula evaluated op by op gives the same bits.
__global__ void __launch_bounds__(256)
ect_step_front_kernel(const float* __restrict__ moments, const float* __restrict__ eps, const float* __restrict__ rnd,
                      const float* __restrict__ noise, const float* __restrict__ drop_u, float drop_prob, float sf,
                      float P_mean, float P_std, const float* __restrict__ qs, float k, float bc,
                      float* __restrict__ y, float* __restrict__ xt, float* __restrict__ xr, float* __restrict__ sr,
                      float* __restrict__ tt, float* __restrict__ rr, float* __restrict__ labels, int B, int C,
                      int plane4, int nc) {
  const long long per = static_cast<long long>(C) * plane4;  // float4 groups per sample
  const long long total = static_cast<long long>(B) * per;
  const float q = qs[0];
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / per);
    const long long rem = i - b * per;
    const float t = expf(__fadd_rn(__fmul_rn(rnd[b], P_std), P_mean));
    const float sig = __fdiv_rn(1.f, __fadd_rn(1.f, expf(__fmul_rn(bc, t))));
    const float w = __fsub_rn(1.f, __fmul_rn(q, __fadd_rn(1.f, __fmul_rn(k, sig))));
    const float r = __fmul_rn(t, fmaxf(w, 0.f));
    const float4* mom = reinterpret_cast<const float4*>(moments) + static_cast<long long>(b) * 2 * per;
    const float4 mu = mom[rem], lv = mom[per + rem];
    const float4 e = reinterpret_cast<const float4*>(eps)[i], nz = reinterpret_cast<const float4*>(noise)[i];
    float4 o, ot, orr;
    o.x = sf * (mu.x + expf(0.5f * fminf(fmaxf(lv.x, -30.f), 20.f)) * e.x);
    o.y = sf * (mu.y + expf(0.5f * fminf(fmaxf(lv.y, -30.f), 20.f)) * e.y);
    o.z = sf * (mu.z + expf(0.5f * fminf(fmaxf(lv.z, -30.f), 20.f)) * e.z);
    o.w = sf * (mu.w + expf(0.5f * fminf(fmaxf(lv.w, -30.f), 20.f)) * e.w);
    ot.x = __fadd_rn(o.x, __fmul_rn(t, nz.x));
    ot.y = __fadd_rn(o.y, __fmul_rn(t, nz.y));
    ot.z = __fadd_rn(o.z, __fmul_rn(t, nz.z));
    ot.w = __fadd_rn(o.w, __fmul_rn(t, nz.w));
    orr.x = __fadd_rn(o.x, __fmul_rn(r, nz.x));
    orr.y = __fadd_rn(o.y, __fmul_rn(r, nz.y));
    orr.z = __fadd_rn(o.z, __fmul_rn(r, nz.z));
    orr.w = __fadd_rn(o.w, __fmul_rn(r, nz.w));
    reinterpret_cast<float4*>(y)[i] = o;
    reinterpret_cast<float4*>(xt)[i] = ot;
    reinterpret_cast<float4*>(xr)[i] = orr;
    if (rem == 0) tt[b] = t, rr[b] = r, sr[b] = r > 0.f ? r : t;
  }
  if (labels && drop_u) {
    const long long nl = static_cast<long long>(B) * nc;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nl;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      const int b = static_cast<int>(i / nc);
      if (!(drop_u[b] >= drop_prob)) labels[i] = 0.f;
    }
  }
}

}  // namespace mdt

using namespace mdt;

static int make_geom(PatchGeom* gm, int C, int R, int p) {
  if (C <= 0 || R <= 0 || p <= 0 || R % p) return MDT_ERR_ARG;
  gm->C = C, gm->R = R, gm->p = p, gm->G = R / p, gm->L = gm->G * gm->G, gm->pd = p * p * C;
  return MDT_OK;
}

extern "C" {

int mdt_edm_loss(const float* F, const float* xin, const float* y, const float* sigma, const float* mask,
                 const float* gl, float sigma_data, float mae_coef, float* loss, float* Dx, void* dF_bf16, int B,
                 int C, int R, int p, void* stream) {
  if (!F || !xin || !y || !sigma || !loss || B <= 0) return MDT_ERR_ARG;
  if (dF_bf16 && !gl) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  auto kern = gm.pd <= kMaxPD ? edm_loss_kernel<true, false> : edm_loss_kernel<false, false>;
  kern<<<B, 256, 0, S(stream)>>>(F, xin, y, sigma, mask, gl, sigma_data, mae_coef, loss, Dx,
                                 static_cast<__nv_bfloat16*>(dF_bf16), gm, LogvarArgs{});
  return launch_status();
}

static bool logvar_args_ok(const float* freqs, const float* phases, int channels) {
  return freqs && phases && channels >= 1 && channels <= kMaxLogvar;
}

int mdt_edm_loss_logvar(const float* F, const float* xin, const float* y, const float* sigma, const float* mask,
                        const float* gl, float sigma_data, float mae_coef, const float* freqs, const float* phases,
                        const float* w, int channels, float* objective, float* loss, float* u, float* du,
                        void* dF_bf16, int B, int C, int R, int p, void* stream) {
  if (!F || !xin || !y || !sigma || !loss || !objective || !u || !w || B <= 0) return MDT_ERR_ARG;
  if (!logvar_args_ok(freqs, phases, channels) || ((dF_bf16 || du) && !gl)) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  const LogvarArgs lv{freqs, phases, w, channels, objective, u, du};
  auto kern = gm.pd <= kMaxPD ? edm_loss_kernel<true, true> : edm_loss_kernel<false, true>;
  kern<<<B, 256, 0, S(stream)>>>(F, xin, y, sigma, mask, gl, sigma_data, mae_coef, loss, nullptr,
                                 static_cast<__nv_bfloat16*>(dF_bf16), gm, lv);
  return launch_status();
}

int mdt_logvar(const float* sigma, const float* freqs, const float* phases, const float* w, int channels, int B,
               float* u, void* stream) {
  if (!sigma || !w || !u || B <= 0 || !logvar_args_ok(freqs, phases, channels)) return MDT_ERR_ARG;
  logvar_kernel<<<B, 256, 0, S(stream)>>>(sigma, LogvarArgs{freqs, phases, w, channels, nullptr, u, nullptr});
  return launch_status();
}

int mdt_logvar_wgrad(const float* sigma, const float* freqs, const float* phases, const float* du, int channels, int B,
                     float* dw, void* stream) {
  if (!sigma || !du || !dw || B <= 0 || !logvar_args_ok(freqs, phases, channels)) return MDT_ERR_ARG;
  logvar_wgrad_kernel<<<1, 256, 0, S(stream)>>>(sigma, du,
                                                LogvarArgs{freqs, phases, nullptr, channels, nullptr, nullptr, nullptr},
                                                B, dw);
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

int mdt_guided_precond_out(const float* F_main, int p_main, const float* F_guide, int p_guide, const float* xin,
                           const float* sigma, float sigma_data, float w, float* Dx, int B, int C, int R,
                           void* stream) {
  if (!F_main || !F_guide || !xin || !sigma || !Dx || B <= 0 || !isfinite(w)) return MDT_ERR_ARG;
  PatchGeom gm, gg;
  if (int rc = make_geom(&gm, C, R, p_main)) return rc;
  if (int rc = make_geom(&gg, C, R, p_guide)) return rc;
  const long long n = static_cast<long long>(B) * C * R * R;
  guided_precond_out_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, S(stream)>>>(F_main, gm, F_guide, gg, xin,
                                                                                       sigma, sigma_data, w, B, Dx);
  return launch_status();
}

int mdt_flow_loss(const float* F, const float* xt, const float* y, const float* eps, const float* t, const float* mask,
                  const float* gl, float mae_coef, float* loss, float* x_hat, void* dF_bf16, int B, int C, int R, int p,
                  void* stream) {
  if (!F || !xt || !y || !eps || !t || !loss || B <= 0) return MDT_ERR_ARG;
  if (dF_bf16 && !gl) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  auto kern = gm.pd <= kMaxPD ? flow_loss_kernel<true> : flow_loss_kernel<false>;
  kern<<<B, 256, 0, S(stream)>>>(F, xt, y, eps, t, mask, gl, mae_coef, loss, x_hat,
                                 static_cast<__nv_bfloat16*>(dF_bf16), gm);
  return launch_status();
}

int mdt_flow_cfg_out(const float* F, int use_cfg, float cfg_scale, float* out, int B, int C, int R, int p,
                     void* stream) {
  if (!F || !out || B <= 0 || (use_cfg && !isfinite(cfg_scale))) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  const long long n = static_cast<long long>(B) * C * R * R;
  flow_out_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, S(stream)>>>(F, cfg_scale, use_cfg != 0, B, out, gm);
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

int mdt_dpm_update(const float* F, int kind, double t, double* x, double* d_out, const double* h1, const double* h2,
                   double a, double b0, double b1, double b2, float* x_f32, long long n, void* stream) {
  if (!F || !x || !d_out || n <= 0 || (kind != MDT_DPM_DATA && kind != MDT_DPM_VELOCITY) ||
      (h2 && !h1) || !isfinite(a) || !isfinite(b0) || !isfinite(b1) || !isfinite(b2) || !isfinite(t))
    return MDT_ERR_ARG;
  dpm_update_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, S(stream)>>>(
      F, kind == MDT_DPM_VELOCITY, t, x, d_out, h1, h2, a, b0, b1, b2, x_f32, n);
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
                        float grad_scale, int max_blocks, void* stream, const float* coef = nullptr) {
  if (!w || !g || !m || !v || n <= 0 || step < 1 || (n & 3)) return MDT_ERR_ARG;
  // the kernel moves 4 elements per access: float4 for the fp32 buffers, uint2 for the bf16 ones
  const uintptr_t a16 = reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(m) |
                        reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(ema) |
                        (g16 ? 0 : reinterpret_cast<uintptr_t>(g));
  const uintptr_t a8 = reinterpret_cast<uintptr_t>(w_bf16) | (g16 ? reinterpret_cast<uintptr_t>(g) : 0);
  if ((a16 & 15) || (a8 & 7)) return MDT_ERR_ARG;
  const float inv_bc1 = static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(beta1), step)));
  const float inv_bc2 = static_cast<float>(1.0 / (1.0 - pow(static_cast<double>(beta2), step)));
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > kNumSMsDefault * 8) blocks = kNumSMsDefault * 8;
  if (max_blocks > 0 && blocks > max_blocks) blocks = max_blocks;
  if (coef) {
    auto kern = g16 ? adamw_ema_coef_kernel<true> : adamw_ema_coef_kernel<false>;
    kern<<<static_cast<int>(blocks), 256, 0, S(stream)>>>(w, g, m, v, ema, static_cast<__nv_bfloat16*>(w_bf16), n,
                                                          lr, beta1, beta2, eps, weight_decay, inv_bc1, inv_bc2,
                                                          ema_decay, grad_scale, coef);
    return launch_status();
  }
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

static int check_grid(long long n) {   // the grid of mdt_cast_f32_bf16: 4 elements per thread, <= 16 CTAs per SM
  long long blocks = (n / 4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > kNumSMsDefault * 16) blocks = kNumSMsDefault * 16;
  return static_cast<int>(blocks);
}

int mdt_nonfinite_check(const float* g, long long n, float* flag, void* stream) {
  if (!g || !flag || n <= 0 || (reinterpret_cast<uintptr_t>(g) & 15)) return MDT_ERR_ARG;
  nonfinite_check_kernel<<<check_grid(n), 256, 0, S(stream)>>>(g, n, flag);
  return launch_status();
}

int mdt_cast_f32_bf16_check(const float* in, void* out_bf16, long long n, float* flag, void* stream) {
  if (!in || !out_bf16 || !flag || n <= 0) return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(in) & 15) || (reinterpret_cast<uintptr_t>(out_bf16) & 7)) return MDT_ERR_ARG;
  cast_f32_bf16_check_kernel<<<check_grid(n), 256, 0, S(stream)>>>(in, static_cast<__nv_bfloat16*>(out_bf16), n,
                                                                    flag);
  return launch_status();
}

static int adamw_guarded_launch(bool g16, float* w, const void* g, float* m, float* v, float* ema, void* w_bf16,
                                long long n, float lr, float beta1, float beta2, float eps, float weight_decay,
                                float ema_decay, float grad_scale, const float* flag, const long long* counts,
                                int max_blocks, void* stream, const float* coef = nullptr) {
  if (!w || !g || !m || !v || !flag || !counts || n <= 0 || (n & 3)) return MDT_ERR_ARG;
  const uintptr_t a16 = reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(m) |
                        reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(ema) |
                        (g16 ? 0 : reinterpret_cast<uintptr_t>(g));
  const uintptr_t a8 = reinterpret_cast<uintptr_t>(w_bf16) | (g16 ? reinterpret_cast<uintptr_t>(g) : 0) |
                       reinterpret_cast<uintptr_t>(counts);
  if ((a16 & 15) || (a8 & 7) || (reinterpret_cast<uintptr_t>(flag) & 3)) return MDT_ERR_ARG;
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > kNumSMsDefault * 8) blocks = kNumSMsDefault * 8;
  if (max_blocks > 0 && blocks > max_blocks) blocks = max_blocks;
  if (coef) {
    auto kern = g16 ? adamw_ema_guarded_coef_kernel<true> : adamw_ema_guarded_coef_kernel<false>;
    kern<<<static_cast<int>(blocks), 256, 0, S(stream)>>>(w, g, m, v, ema, static_cast<__nv_bfloat16*>(w_bf16), n,
                                                          lr, beta1, beta2, eps, weight_decay, ema_decay, grad_scale,
                                                          coef, flag, counts);
    return launch_status();
  }
  auto kern = g16 ? adamw_ema_guarded_kernel<true> : adamw_ema_guarded_kernel<false>;
  kern<<<static_cast<int>(blocks), 256, 0, S(stream)>>>(w, g, m, v, ema, static_cast<__nv_bfloat16*>(w_bf16), n, lr,
                                                        beta1, beta2, eps, weight_decay, ema_decay, grad_scale, flag,
                                                        counts);
  return launch_status();
}

int mdt_adamw_ema_guarded(float* w, const float* g, float* m, float* v, float* ema, void* w_bf16, long long n,
                          float lr, float beta1, float beta2, float eps, float weight_decay, float ema_decay,
                          float grad_scale, const float* flag, const long long* counts, int max_blocks, void* stream) {
  return adamw_guarded_launch(false, w, g, m, v, ema, w_bf16, n, lr, beta1, beta2, eps, weight_decay, ema_decay,
                              grad_scale, flag, counts, max_blocks, stream);
}

int mdt_adamw_ema_guarded_g16(float* w, const void* g_bf16, float* m, float* v, float* ema, void* w_bf16, long long n,
                              float lr, float beta1, float beta2, float eps, float weight_decay, float ema_decay,
                              float grad_scale, const float* flag, const long long* counts, int max_blocks,
                              void* stream) {
  return adamw_guarded_launch(true, w, g_bf16, m, v, ema, w_bf16, n, lr, beta1, beta2, eps, weight_decay, ema_decay,
                              grad_scale, flag, counts, max_blocks, stream);
}

int mdt_optim_guard_advance(const float* flag, long long* counts, void* stream) {
  if (!flag || !counts || (reinterpret_cast<uintptr_t>(counts) & 7) || (reinterpret_cast<uintptr_t>(flag) & 3))
    return MDT_ERR_ARG;
  optim_guard_advance_kernel<<<1, 1, 0, S(stream)>>>(flag, counts);
  return launch_status();
}

// ---- gradient-norm clipping ---------------------------------------------------------------------------------------------
int mdt_grad_sumsq_scratch(long long n) {
  if (n <= 0) return MDT_ERR_ARG;
  return check_grid(n);
}

int mdt_grad_sumsq(const void* g, long long n, int bf16, double* scratch, double* out, float* flag, void* stream) {
  if (!g || !scratch || !out || n <= 0) return MDT_ERR_ARG;
  const uintptr_t ag = reinterpret_cast<uintptr_t>(g);
  if ((bf16 ? (ag & 7) : (ag & 15)) || ((reinterpret_cast<uintptr_t>(scratch) | reinterpret_cast<uintptr_t>(out)) & 7) ||
      (reinterpret_cast<uintptr_t>(flag) & 3))
    return MDT_ERR_ARG;
  const int blocks = check_grid(n);
  if (bf16) grad_sumsq_kernel<true><<<blocks, 256, 0, S(stream)>>>(g, n, scratch, flag);
  else grad_sumsq_kernel<false><<<blocks, 256, 0, S(stream)>>>(g, n, scratch, flag);
  if (int rc = launch_status()) return rc;
  grad_sumsq_final_kernel<<<1, 256, 0, S(stream)>>>(scratch, blocks, out);
  return launch_status();
}

int mdt_grad_clip_coef(const double* sumsq, int k, double grad_scale, float max_norm, float* norm, float* coef,
                       float* flag, void* stream) {
  if (!sumsq || !norm || !coef || k < 1 || !(grad_scale > 0.0) || !(max_norm > 0.f)) return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(sumsq) & 7) ||
      ((reinterpret_cast<uintptr_t>(norm) | reinterpret_cast<uintptr_t>(coef) | reinterpret_cast<uintptr_t>(flag)) & 3))
    return MDT_ERR_ARG;
  grad_clip_coef_kernel<<<1, 1, 0, S(stream)>>>(sumsq, k, grad_scale, max_norm, norm, coef, flag);
  return launch_status();
}

int mdt_adamw_ema_coef(float* w, const float* g, float* m, float* v, float* ema, void* w_bf16, long long n, float lr,
                       float beta1, float beta2, float eps, float weight_decay, int step, float ema_decay,
                       float grad_scale, const float* coef, int max_blocks, void* stream) {
  if (!coef || (reinterpret_cast<uintptr_t>(coef) & 3)) return MDT_ERR_ARG;
  return adamw_launch(false, w, g, m, v, ema, w_bf16, n, lr, beta1, beta2, eps, weight_decay, step, ema_decay,
                      grad_scale, max_blocks, stream, coef);
}

int mdt_adamw_ema_coef_g16(float* w, const void* g_bf16, float* m, float* v, float* ema, void* w_bf16, long long n,
                           float lr, float beta1, float beta2, float eps, float weight_decay, int step, float ema_decay,
                           float grad_scale, const float* coef, int max_blocks, void* stream) {
  if (!coef || (reinterpret_cast<uintptr_t>(coef) & 3)) return MDT_ERR_ARG;
  return adamw_launch(true, w, g_bf16, m, v, ema, w_bf16, n, lr, beta1, beta2, eps, weight_decay, step, ema_decay,
                      grad_scale, max_blocks, stream, coef);
}

int mdt_adamw_ema_guarded_coef(float* w, const float* g, float* m, float* v, float* ema, void* w_bf16, long long n,
                               float lr, float beta1, float beta2, float eps, float weight_decay, float ema_decay,
                               float grad_scale, const float* coef, const float* flag, const long long* counts,
                               int max_blocks, void* stream) {
  if (!coef || (reinterpret_cast<uintptr_t>(coef) & 3)) return MDT_ERR_ARG;
  return adamw_guarded_launch(false, w, g, m, v, ema, w_bf16, n, lr, beta1, beta2, eps, weight_decay, ema_decay,
                              grad_scale, flag, counts, max_blocks, stream, coef);
}

int mdt_adamw_ema_guarded_coef_g16(float* w, const void* g_bf16, float* m, float* v, float* ema, void* w_bf16,
                                   long long n, float lr, float beta1, float beta2, float eps, float weight_decay,
                                   float ema_decay, float grad_scale, const float* coef, const float* flag,
                                   const long long* counts, int max_blocks, void* stream) {
  if (!coef || (reinterpret_cast<uintptr_t>(coef) & 3)) return MDT_ERR_ARG;
  return adamw_guarded_launch(true, w, g_bf16, m, v, ema, w_bf16, n, lr, beta1, beta2, eps, weight_decay, ema_decay,
                              grad_scale, flag, counts, max_blocks, stream, coef);
}

int mdt_power_ema(const float* w, float* const* ema, const float* one_minus_beta, int k, long long n, void* stream) {
  if (!w || !ema || !one_minus_beta || k < 1 || k > kMaxPowerEma || n <= 0) return MDT_ERR_ARG;
  const uintptr_t phase = reinterpret_cast<uintptr_t>(w) & 15;
  if (phase & 3) return MDT_ERR_ARG;
  PowerEmaArgs a{};
  bool same_phase = true;
  for (int j = 0; j < k; ++j) {
    const float c = one_minus_beta[j];
    if (!ema[j] || (reinterpret_cast<uintptr_t>(ema[j]) & 3) || !(c >= 0.f && c <= 1.f)) return MDT_ERR_ARG;
    same_phase &= (reinterpret_cast<uintptr_t>(ema[j]) & 15) == phase;
    a.e[j] = ema[j], a.c[j] = c;
  }
  // float4 body when every buffer reaches a 16-byte boundary after the same number of elements; else all scalar
  long long head = n, n4 = 0;
  if (same_phase) {
    head = static_cast<long long>((16 - phase) & 15) / 4;
    if (head > n) head = n;
    n4 = (n - head) >> 2;
  }
  const int blocks = check_grid(n);
  switch (k) {
    case 1: power_ema_kernel<1><<<blocks, 256, 0, S(stream)>>>(w, a, n, head, n4); break;
    case 2: power_ema_kernel<2><<<blocks, 256, 0, S(stream)>>>(w, a, n, head, n4); break;
    case 3: power_ema_kernel<3><<<blocks, 256, 0, S(stream)>>>(w, a, n, head, n4); break;
    default: power_ema_kernel<4><<<blocks, 256, 0, S(stream)>>>(w, a, n, head, n4); break;
  }
  return launch_status();
}

// One block row per segment (blockIdx.y), the row's blocks striding over its elements: the sharded optimizer's
// pack / unpack of the fp32-read set (a few hundred segments, a few MB).
__global__ void copy_segments_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                     const long long* __restrict__ seg) {
  const long long so = seg[3 * blockIdx.y], d = seg[3 * blockIdx.y + 1], n = seg[3 * blockIdx.y + 2];
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[d + i] = src[so + i];
}

int mdt_copy_segments_f32(const float* src, float* dst, const long long* seg, int nseg, void* stream) {
  if (nseg < 0 || nseg > 65535) return MDT_ERR_ARG;
  if (nseg == 0) return MDT_OK;
  if (!src || !dst || !seg) return MDT_ERR_ARG;
  copy_segments_kernel<<<dim3(8, nseg), 256, 0, S(stream)>>>(src, dst, seg);
  return launch_status();
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


int mdt_flow_step_front(const float* moments, const float* eps, const float* rnd_normal, const float* noise_unit,
                        const float* drop_u, float drop_prob, float scale_factor, float P_mean, float P_std, float* y,
                        float* xt, float* t, float* labels, int B, int C, int R, int num_classes, void* stream) {
  if (!moments || !eps || !rnd_normal || !noise_unit || !y || !xt || !t || B <= 0 || C <= 0 || R <= 0)
    return MDT_ERR_ARG;
  if ((R * R) % 4) return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(moments) | reinterpret_cast<uintptr_t>(eps) | reinterpret_cast<uintptr_t>(noise_unit) |
       reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(xt)) & 15)
    return MDT_ERR_ARG;
  const long long total = static_cast<long long>(B) * C * (R * R / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > kNumSMsDefault * 8) blocks = kNumSMsDefault * 8;
  flow_step_front_kernel<<<static_cast<int>(blocks), 256, 0, S(stream)>>>(moments, eps, rnd_normal, noise_unit, drop_u,
                                                                          drop_prob, scale_factor, P_mean, P_std, y,
                                                                          xt, t, labels, B, C, R * R / 4, num_classes);
  return launch_status();
}

int mdt_ect_step_front(const float* moments, const float* eps, const float* rnd_normal, const float* noise_unit,
                       const float* drop_u, float drop_prob, float scale_factor, float P_mean, float P_std,
                       const float* qs, float k, float b_coef, float* y, float* xt, float* xr, float* sr, float* t,
                       float* r, float* labels, int B, int C, int R, int num_classes, void* stream) {
  if (!moments || !eps || !rnd_normal || !noise_unit || !qs || !y || !xt || !xr || !sr || !t || !r || B <= 0 ||
      C <= 0 || R <= 0)
    return MDT_ERR_ARG;
  if ((R * R) % 4) return MDT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(moments) | reinterpret_cast<uintptr_t>(eps) | reinterpret_cast<uintptr_t>(noise_unit) |
       reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(xt) | reinterpret_cast<uintptr_t>(xr)) & 15)
    return MDT_ERR_ARG;
  const long long total = static_cast<long long>(B) * C * (R * R / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > kNumSMsDefault * 8) blocks = kNumSMsDefault * 8;
  ect_step_front_kernel<<<static_cast<int>(blocks), 256, 0, S(stream)>>>(
      moments, eps, rnd_normal, noise_unit, drop_u, drop_prob, scale_factor, P_mean, P_std, qs, k, b_coef, y, xt, xr,
      sr, t, r, labels, B, C, R * R / 4, num_classes);
  return launch_status();
}

int mdt_ect_loss(const float* Ft, const float* Fr, const float* xt, const float* xr, const float* y, const float* t,
                 const float* r, const float* mask, const float* gl, float sigma_data, float c, float mae_coef,
                 float* loss, float* D_t, void* dF_bf16, int B, int C, int R, int p, void* stream) {
  if (!Ft || !Fr || !xt || !xr || !y || !t || !r || !loss || B <= 0 || !(c > 0.f)) return MDT_ERR_ARG;
  if (dF_bf16 && !gl) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  ect_loss_kernel<<<B, 256, 0, S(stream)>>>(Ft, Fr, xt, xr, y, t, r, mask, gl, sigma_data, c, mae_coef, loss, D_t,
                                            static_cast<__nv_bfloat16*>(dF_bf16), gm);
  return launch_status();
}

static bool mg_args_ok(const float* Fu, const float* labels, int num_classes, float w, float lo, float hi) {
  return Fu && labels && num_classes >= 1 && w >= 0.f && w < 1.f && lo < hi;
}

int mdt_mg_loss(const float* F, const float* Fu, const float* xin, const float* y, const float* sigma,
                const float* labels, int num_classes, const float* mask, const float* gl, float sigma_data,
                float mae_coef, float w, float lo, float hi, float* loss, float* edm_loss, float* Dx, void* dF_bf16,
                int B, int C, int R, int p, void* stream) {
  if (!F || !xin || !y || !sigma || !loss || B <= 0 || !mg_args_ok(Fu, labels, num_classes, w, lo, hi))
    return MDT_ERR_ARG;
  if (dF_bf16 && !gl) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  auto kern = gm.pd <= kMaxPD ? mg_loss_kernel<true> : mg_loss_kernel<false>;
  kern<<<B, 256, 0, S(stream)>>>(F, xin, y, sigma, mask, gl, sigma_data, mae_coef, loss, Dx,
                                 static_cast<__nv_bfloat16*>(dF_bf16), gm,
                                 MgArgs{Fu, labels, num_classes, w, lo, hi, edm_loss});
  return launch_status();
}

int mdt_flow_mg_loss(const float* F, const float* Fu, const float* xt, const float* y, const float* eps,
                     const float* t, const float* labels, int num_classes, const float* mask, const float* gl,
                     float mae_coef, float w, float lo, float hi, float* loss, float* edm_loss, float* x_hat,
                     void* dF_bf16, int B, int C, int R, int p, void* stream) {
  if (!F || !xt || !y || !eps || !t || !loss || B <= 0 || !mg_args_ok(Fu, labels, num_classes, w, lo, hi))
    return MDT_ERR_ARG;
  if (dF_bf16 && !gl) return MDT_ERR_ARG;
  PatchGeom gm;
  if (int rc = make_geom(&gm, C, R, p)) return rc;
  auto kern = gm.pd <= kMaxPD ? flow_mg_loss_kernel<true> : flow_mg_loss_kernel<false>;
  kern<<<B, 256, 0, S(stream)>>>(F, xt, y, eps, t, mask, gl, mae_coef, loss, x_hat,
                                 static_cast<__nv_bfloat16*>(dF_bf16), gm,
                                 MgArgs{Fu, labels, num_classes, w, lo, hi, edm_loss});
  return launch_status();
}

}  // extern "C"

