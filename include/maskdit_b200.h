/* maskdit_b200 — C ABI of the H100 (sm_90a) MaskDiT hot path.
 *
 * The reference (Anima-Lab/MaskDiT) is pure Python/PyTorch and has no FFI layer; its seam for this path is the
 * Python registries `Precond_models`, `DiT_models` (models/maskdit.py:709-715,779-781), `Losses`
 * (train_utils/loss.py:66-68) and `edm_sampler` (sample.py:30-66).  The Python shim in `maskdit_b200/` implements
 * those registries and calls the functions below through ctypes.  Every function:
 *   - takes raw DEVICE pointers + sizes + a `cudaStream_t` (passed as void*), no torch types;
 *   - is asynchronous on that stream, allocates nothing, frees nothing (caller owns all buffers);
 *   - returns MDT_OK (0) or a negative MDT_ERR_* code; the shim raises on non-zero.
 * Each declaration cites the reference code (file:line in /root/reference) whose arithmetic it replaces.
 */
#ifndef MASKDIT_B200_H_
#define MASKDIT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MDT_OK 0
#define MDT_ERR_ARG (-1)    /* bad shape / alignment / null pointer */
#define MDT_ERR_CUDA (-2)   /* launch failed; see cudaGetLastError */
#define MDT_ERR_DRIVER (-3) /* cuTensorMapEncodeTiled entry point unavailable */
#define MDT_ERR_TMAP (-4)   /* tensor-map encode rejected the operand */
#define MDT_ERR_UNSUPPORTED (-5)

/* Precondition kinds of a model handle (mdt_model_set_precond) and of the kernels that depend on it */
#define MDT_PRECOND_EDM 0   /* sigma: EDM noise level; c_in = 1/sqrt(sigma^2 + sigma_data^2), c_noise = ln(sigma)/4 */
#define MDT_PRECOND_FLOW 1  /* sigma holds the flow time t in [0, 1]; c_in = 1, c_noise = t                            */

const char* mdt_status_string(int status);
int mdt_abi_version(void);
/* BLOCK_N * 10 + CTAs-per-tile (always 1) of the last mdt_gemm_bf16 launch (tests). */
int mdt_gemm_last_config(void);
/* Bit set of the GEMM instances launched since the last reset: bit (BLOCK_N/64 - 2) * 2 + (CTAs - 1), i.e. 128/1 = 0,
 * 128/2 = 1, 192/1 = 2, 192/2 = 3, 256/1 = 4, 256/2 = 5.  reset != 0 clears it after reading.                        */
int mdt_gemm_configs_seen(int reset);

/* ------------------------------------------------------------------------------------------------------------
 * bf16 tensor-core GEMM (wgmma / TMA):  out[M,N] (+)= sum_k A[m,k] * B[n,k], fp32 accumulate.
 * Replaces every nn.Linear forward and its autograd dgrad/wgrad: timm Attention.qkv/proj and Mlp.fc1/fc2
 * (ctor sites models/maskdit.py:178,182), adaLN_modulation (:185,206,227), DecoderLayer.linear (:203),
 * FinalLayer.linear (:224), TimestepEmbedder.mlp (:34-38), LabelEmbedder.embedding_table (:75).
 *   a_mn / b_mn = 0: operand stored [rows, K] with K contiguous ("K-major", row stride lda/ldb elements)
 *               = 1: operand stored [K, rows] with rows contiguous ("MN-major")
 * ------------------------------------------------------------------------------------------------------------ */
enum { MDT_EPI_STORE = 0,      /* out = act(acc + bias [+ resid])            out bf16 or fp32            */
       MDT_EPI_GELU = 1,       /* aux = bf16(acc+bias); out = bf16(gelu_tanh(aux))      (Mlp.fc1 + act)   */
       MDT_EPI_GATE_RESID = 2, /* y = acc+bias; aux = bf16(y) (optional); out_f32 = resid + gate[row/rpg]*y
                                  (DiTBlock residual update, models/maskdit.py:190-191)                   */
       MDT_EPI_DGELU = 3,      /* out = bf16(acc * gelu_tanh'(aux))          (backward through GELU)      */
       MDT_EPI_ATOMIC = 4 };   /* out_f32 += acc via red.global.add, stream-K schedule (wgrad, long-K)    */
enum { MDT_ACT_NONE = 0, MDT_ACT_SILU = 1 };

typedef struct mdt_gemm_args {
  const void* A; /* bf16 */
  const void* B; /* bf16 */
  int M, N, K;
  int lda, ldb;  /* row strides in elements (multiple of 8) */
  int a_mn, b_mn;
  int epi, act;
  void* out;
  int ldo;       /* multiple of 8 */
  int out_fp32;  /* 1: float output, 0: bf16 output */
  const float* bias; /* [N] or NULL */
  void* aux;     /* bf16 [M, ld_aux], see epilogue kinds */
  int ld_aux;
  const float* resid; /* fp32 [M, ld_resid] or NULL */
  int ld_resid;
  const float* gate;  /* fp32 [M / rows_per_group, ld_gate] */
  int ld_gate;
  int rows_per_group;
  int block_n;   /* 0 = auto, or 128/192/256 */
  float* colsum; /* MDT_EPI_DGELU only, may be NULL: colsum[n] += sum_m out[m,n] (the bf16-rounded outputs), i.e. the
                    bias gradient of the layer whose pre-activation gradient this GEMM produces (fp32 red.add)      */
} mdt_gemm_args;

int mdt_gemm_bf16(const mdt_gemm_args* args, void* stream);
/* The host-side decisions mdt_gemm_bf16 would take for `args`, without launching anything (needs no device: host
 * tests pin the dispatch with it; pointers in `args` are only checked for alignment, never dereferenced):
 * out10 = {BLOCK_N, CTAs per tile (always 1), k-slices, paired half-tile order (0/1), half-width last
 * column tile (0/1), row tiles, column tiles, k-blocks of 64, work units, grid size in CTAs}.                        */
int mdt_gemm_plan(const mdt_gemm_args* args, long long* out10);
/* Measurement aid (bench.py roofline): while enabled, every mdt_gemm_bf16 launch of this process - also the step
 * driver's - is bracketed by CUDA events on its stream; mdt_gemm_profile_read returns the launch count and fills
 * ms[i] (device time) / flops[i] (2 M N K) for i < cap.  Enabling clears the previous recording.                   */
int mdt_gemm_profile_enable(int on);
int mdt_gemm_profile_read(float* ms, double* flops, int cap);

/* ------------------------------------------------------------------------------------------------------------
 * Mask index path (integer, bit-exact).  get_mask, models/maskdit.py:88-113: ids_shuffle = argsort(noise),
 * ids_restore = argsort(ids_shuffle), ids_keep = ids_shuffle[:, :len_keep], mask = (ids_restore >= len_keep).
 * Ties in `noise` are broken by ascending index (= torch.argsort(stable=True)).
 *   noise [B,L] f32 -> ids_keep [B,len_keep] i64, ids_restore [B,L] i64, mask [B,L] f32 (0 keep / 1 remove)
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_mask_indices(const float* noise, int B, int L, int len_keep, int64_t* ids_keep, int64_t* ids_restore,
                     float* mask, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * PatchEmbed + pos_embed + mask_out_token + EDM c_in scaling, fused.
 * models/maskdit.py:475 (x_embedder(x) + pos_embed), :126 (gather kept tokens), :764-769 (c_in * x).
 *   x [B,C,R,R] f32, sigma [B] f32 or NULL (c_in = 1/sqrt(sigma_data^2+sigma^2), 1 if NULL),
 *   W [D, C*p*p] f32 (Conv2d weight flattened (c,ph,pw)), bias [D], pos [L,D] f32,
 *   ids_keep [B,T] i64 or NULL (NULL: T == L, identity) -> out [B,T,D] f32
 * Backward: gW [D, C*p*p] += sum g (x) patch, gb [D] += sum g    (no input gradient is needed)
 * Supported: cpp = C*p*p <= 384 (every DiT_models patch size at 4 channels: 16, 64, 256), so one block's patch
 * rows stay within 48 KB of shared memory; MDT_ERR_UNSUPPORTED above.  The backward takes 128 tokens per block for
 * cpp <= 96 and 32 above.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_patch_embed(const float* x, const float* sigma, float sigma_data, const float* W, const float* bias,
                    const float* pos, const int64_t* ids_keep, float* out, int B, int C, int R, int p, int D, int T,
                    void* stream);
int mdt_patch_embed_bwd(const float* x, const float* sigma, float sigma_data, const int64_t* ids_keep,
                        const float* g, float* gW, float* gb, int B, int C, int R, int p, int D, int T, void* stream);

/* TimestepEmbedder.timestep_embedding (models/maskdit.py:41-58) on t = c_noise = ln(sigma)/4 (:767):
 *   out[b] = [cos(t f_k) | sin(t f_k)], f_k = exp(-ln(1e4) k / (dim/2)); out bf16 [B, dim]                  */
int mdt_timestep_freq(const float* sigma, int B, int dim, void* out_bf16, void* stream);
/* The same embedding on c_noise = t, the flow time (rectified flow, SiT).                                         */
int mdt_flow_timestep_freq(const float* t, int B, int dim, void* out_bf16, void* stream);

/* Pointwise helpers around the conditioning MLPs (nn.SiLU at models/maskdit.py:36,184,205,226).
 *   silu:      out_bf16 = silu(a [+ b])  (and out_f32 = a + b if non-NULL)
 *   silu_bwd:  dx = dy * silu'(x)                                                                            */
int mdt_silu(const float* a, const float* b, float* sum_f32, void* out_bf16, long long n, void* stream);
int mdt_silu_bwd(const float* dy, const float* x, float* dx_f32, void* dx_bf16, long long n, void* stream);
int mdt_cast_f32_bf16(const float* in, void* out_bf16, long long n, void* stream);
/* column sums: out[N] (+)= sum_m in[m, n]  (bias gradients) */
int mdt_colsum_bf16(const void* in_bf16, int M, int N, int ld, float* out, void* stream);
int mdt_colsum_f32(const float* in, int M, int N, int ld, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * LayerNorm(no affine, eps) + modulate, models/maskdit.py:19-20,177,179,190-191,202,211,223,232:
 *   out_bf16[m,:] = LN(x[m,:]) * (1 + scale[m / rows_per_group,:]) + shift[m / rows_per_group,:]
 * saves mean/rstd [M] for the backward.  shift/scale are fp32 with row stride ld_mod.
 * Backward (dxmod bf16 -> residual-stream gradient, fp32):
 *   g[m,:] (+)= d LN / dx ; dshift[b,:] += sum_t dxmod ; dscale[b,:] += sum_t dxmod * xhat
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_ln_modulate(const float* x, const float* shift, const float* scale, int ld_mod, int rows_per_group,
                    void* out_bf16, float* mean, float* rstd, int M, int D, float eps, void* stream);
int mdt_ln_modulate_bwd(const void* dxmod_bf16, const float* x, const float* mean, const float* rstd,
                        const float* scale, int ld_mod, int rows_per_group, float* g, int accumulate,
                        float* dshift, float* dscale, int ld_dmod, int M, int D, void* stream);

/* Backward of  x_out = x + gate * y  (models/maskdit.py:190-191) w.r.t. y and gate, plus the bias gradient of the
 * Linear that produced y:  dy_bf16 = g * gate ; dgate[b,:] += sum_t g*y ; dbias[:] += sum_m dy                 */
int mdt_gate_bwd(const float* g, const void* y_bf16, const float* gate, int ld_gate, int rows_per_group,
                 void* dy_bf16, float* dgate, int ld_dgate, float* dbias, int M, int D, void* stream);

/* mdt_ln_modulate_bwd immediately followed by mdt_gate_bwd on the finished residual gradient g, in one pass
 * (the block backward alternates exactly these two: models/maskdit.py:190-191 differentiated right to left).
 * y_bf16 == NULL: LN backward only.  Same arguments and arithmetic as the two separate entry points.          */
int mdt_ln_modulate_bwd_gate(const void* dxmod_bf16, const float* x, const float* mean, const float* rstd,
                             const float* scale, int ld_mod, int rows_per_group, float* g, int accumulate,
                             float* dshift, float* dscale, int ld_dmod, const void* y_bf16, const float* gate,
                             int ld_gate, void* dy_bf16, float* dgate, int ld_dgate, float* dbias, int M, int D,
                             void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Multi-head attention core of timm Attention (ctor models/maskdit.py:178):
 *   qkv [B,T,3,H,dh] bf16 -> out [B,T,H*dh] bf16 = softmax(q k^T / sqrt(dh)) v ; lse [B,H,T] f32 (log-sum-exp)
 * Backward: dqkv [B,T,3,H,dh] bf16 from dout.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_attention_fwd(const void* qkv, void* out, float* lse, int B, int T, int H, int dh, void* stream);
int mdt_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, int B, int T,
                      int H, int dh, void* stream);
/* Introspection for the parity tests (host-side, no launch): which kernel family served the last successful
 * mdt_attention_fwd (which = 0) / mdt_attention_bwd (which = 1) call of this process:
 *   0 mma.sync kernels (T not a multiple of 64, other head_dims), 1 wgmma + TMA kernels; -1 = none yet.          */
int mdt_attention_last_impl(int which);
/* Log of every attention call since the last reset, 4 ints per call: (which, T, head_dim, kernel family).  Returns
 * the number of entries copied (<= cap); out4 == NULL resets the log.  The step driver's internal calls are logged too. */
int mdt_attention_impl_log(int* out4, int cap);

/* ------------------------------------------------------------------------------------------------------------
 * unmask_tokens + decoder_pos_embed (models/maskdit.py:157-163,543-545):
 *   out[b,l,:] = (ids_restore[b,l] < T ? u[b, ids_restore[b,l], :] : mask_token) + pos[l,:]
 * ids_restore NULL = eval path (no masking): out = u + pos.  mask_token NULL: zeros; pos NULL: no position term (the
 * decoder-less DiT's zero-filled output scatter, models/maskdit.py:551-553, is mask_token = pos = NULL).
 * Backward: du_bf16[b,i,:] = g[b, ids_keep[b,i], :] ; dmask_token[:] += sum over removed positions of g.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_unmask_tokens(const float* u, const float* mask_token, const float* pos, const int64_t* ids_restore,
                      float* out, int B, int T, int L, int D, void* stream);
int mdt_unmask_tokens_bwd(const float* g, const int64_t* ids_keep, const int64_t* ids_restore, void* du_bf16,
                          float* dmask_token, int B, int T, int L, int D, void* stream);
/* Row gather: out_bf16[b*T + i, :] = in_bf16[b*L + idx[b*T + i], :], idx [B,T] int64 (ids_keep), D % 4 == 0.  The
 * decoder-less DiT's backward through the zero-filled scatter: the gradient of the kept tokens' rows only.       */
int mdt_gather_rows_bf16(const void* in_bf16, const int64_t* idx, void* out_bf16, int B, int T, int L, int D,
                         void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * unpatchify + EDM preconditioning + EDM/MAE loss, forward and the gradient seed in one pass.
 *   F [B,L,p*p*C] f32 (final_layer output) ; xin [B,C,R,R] noisy input y+n ; y [B,C,R,R] clean ; sigma [B]
 *   D = c_skip*xin + c_out*unpatchify(F)                    models/maskdit.py:411-424,764-771
 *   mask != NULL: loss[b] = mean_{kept}(patch-mean(w (D-y)^2)) + mae_coef * mean_{removed}(MSE(patchify(D), norm-patchify(xin)))
 *                                                            train_utils/loss.py:37,44-52,73-101
 *   mask == NULL: loss[b] = mean(w (D-y)^2)                  loss.py:54
 *   dF_bf16 (optional) = d(sum_b gl[b]*loss[b]) / dF ; Dx (optional) [B,C,R,R] f32.
 * Any pd = p*p*C: up to 64 (patch 2 and 4 at 4 channels) a token's D and xin are held in registers; above (patch 8:
 * pd 256) the later passes re-read F and xin.  The output scaling below has no pd bound.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_edm_loss(const float* F, const float* xin, const float* y, const float* sigma, const float* mask,
                 const float* gl, float sigma_data, float mae_coef, float* loss, float* Dx, void* dF_bf16, int B,
                 int C, int R, int p, void* stream);
/* Learned loss weighting (EDM2 uncertainty weighting, Karras et al. CVPR 2024): per sample
 *   c = ln(sigma) / 4,  phi_j(c) = sqrt(2) cos(freqs_j c + phases_j),  u = sum_{j < channels} w_j phi_j(c)
 * (phi in fp64 rounded to fp32, the sum in fp32; 1 <= channels <= 256).  mdt_edm_loss_logvar is mdt_edm_loss's pass
 * with the EDM term E also summed apart from the MAE term M (mae_coef included): loss[b] = E + M bit for bit as
 * mdt_edm_loss writes it, objective[b] = exp(-u) E + u + M, evaluated as loss + expm1(-u) E + u (so at u = 0 it is
 * loss bit for bit), u[b].  With gl: dF_bf16 = d(sum_b gl[b]*objective[b]) / dF, i.e. the
 * EDM term's seed scaled by gl[b] exp(-u) and the MAE term's by gl[b], and du[b] = gl[b] (1 - exp(-u) E) (both
 * optional, both need gl).  No Dx output.
 * mdt_logvar: u[b] alone, the same bits.  mdt_logvar_wgrad: dw[j] += sum_b du[b] phi_j(c_b), summed over b in index
 * order in fp64 and added once (no atomics: the same bits on every run).                                       */
int mdt_edm_loss_logvar(const float* F, const float* xin, const float* y, const float* sigma, const float* mask,
                        const float* gl, float sigma_data, float mae_coef, const float* freqs, const float* phases,
                        const float* w, int channels, float* objective, float* loss, float* u, float* du,
                        void* dF_bf16, int B, int C, int R, int p, void* stream);
int mdt_logvar(const float* sigma, const float* freqs, const float* phases, const float* w, int channels, int B,
               float* u, void* stream);
int mdt_logvar_wgrad(const float* sigma, const float* freqs, const float* phases, const float* du, int channels, int B,
                     float* dw, void* stream);
/* Step front (train.py:206,209 + train_utils/loss.py:35-39 + utils.py:59-65) in one pass, given pre-drawn randoms:
 *   y  = scale_factor * (mean + exp(0.5 * clamp(logvar, -30, 20)) * eps)   moments [B,2C,R,R] = (mean | logvar)
 *   sigma[b] = exp(P_std * rnd_normal[b] + P_mean) ;  yn = y + noise_unit * sigma[b]
 *   labels[b,:] = 0 where !(drop_u[b] >= drop_prob)   (labels / drop_u may be NULL: no label dropout)
 * eps, noise_unit, y, yn: [B,C,R,R] f32 ; rnd_normal, drop_u, sigma: [B] f32 ; labels [B,num_classes] f32 in place. */
int mdt_step_front(const float* moments, const float* eps, const float* rnd_normal, const float* noise_unit,
                   const float* drop_u, float drop_prob, float scale_factor, float P_mean, float P_std, float* y,
                   float* yn, float* sigma, float* labels, int B, int C, int R, int num_classes, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Rectified flow (linear interpolant, velocity prediction; SiT, Ma et al. 2024).  t in [0, 1], t = 0 data, t = 1 noise:
 *   x_t = (1 - t) x + t eps ; network input x_t unscaled (c_in = 1), c_noise = t ; v^ = unpatchify(F) ; target
 *   v = eps - x ; denoised estimate x^ = x_t - t v^.
 * mdt_flow_loss: F [B,L,p*p*C] f32 ; xt [B,C,R,R] ; y = x [B,C,R,R] clean ; eps [B,C,R,R] the noise ; t [B]
 *   mask != NULL: loss[b] = mean_{kept}(patch-mean((v^-v)^2)) + mae_coef * mean_{removed}(MSE(patchify(x^), norm-patchify(xt)))
 *   mask == NULL: loss[b] = mean((v^-v)^2)
 *   dF_bf16 (optional, needs gl) = d(sum_b gl[b]*loss[b]) / dF ; x_hat (optional) [B,C,R,R] f32.
 *   The kept / removed-row rules and the pd handling are mdt_edm_loss's.
 * mdt_flow_cfg_out: out [B,C,R,R] = unpatchify(Fu + s (Fc - Fu)) with use_cfg (F [2B,...], cond rows first), else
 *   unpatchify(F) (F [B,...]).
 * mdt_flow_step_front: mdt_step_front's latent and label dropout, then t[b] = 1 / (1 + exp(-(P_mean + P_std *
 *   rnd_normal[b]))) and xt = (1 - t) y + t noise_unit, each product and sum rounded separately.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_flow_loss(const float* F, const float* xt, const float* y, const float* eps, const float* t, const float* mask,
                  const float* gl, float mae_coef, float* loss, float* x_hat, void* dF_bf16, int B, int C, int R, int p,
                  void* stream);
int mdt_flow_cfg_out(const float* F, int use_cfg, float cfg_scale, float* out, int B, int C, int R, int p,
                     void* stream);
int mdt_flow_step_front(const float* moments, const float* eps, const float* rnd_normal, const float* noise_unit,
                        const float* drop_u, float drop_prob, float scale_factor, float P_mean, float P_std, float* y,
                        float* xt, float* t, float* labels, int B, int C, int R, int num_classes, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Easy Consistency Tuning (ECT; Geng et al., ICLR 2025) of an EDM network f(x, s) = D(x; s) = c_skip(s) x + c_out(s) F.
 * mdt_ect_step_front: mdt_step_front's latent and label dropout, then, each product and sum rounded separately,
 *   t[b] = exp(P_std * rnd_normal[b] + P_mean) ; r[b] = t * max(0, 1 - qs[0] * (1 + k / (1 + exp(b_coef * t))))
 *   xt = y + t noise_unit ; xr = y + r noise_unit ; sr[b] = r > 0 ? r : t  (the target forward's sigma)
 *   qs: ONE fp32 word on the device, q^-(s+1) of the tuning stage s (a graph replay reads the current stage).
 * mdt_ect_loss: Ft, Fr [B,L,p*p*C] f32 the student's (at xt, t) and the target's (at xr, sr) outputs with the same
 *   kept tokens ; xt, xr, y [B,C,R,R] ; t, r [B].  D_t = c_skip(t) xt + c_out(t) F_t ; D_r = r > 0 ? c_skip(r) xr +
 *   c_out(r) F_r : y (a select: F_r of an r = 0 row is never read into the result) ; delta = D_t - D_r.
 *   S = (L / T) sum_{kept} delta^2 (T = L unmasked) ; loss[b] = (sqrt(S + c^2) - c) / (t - r) + mae_coef * M, M the
 *   mdt_edm_loss MAE term on the removed patches with D = D_t (mask == NULL: M = 0).
 *   dF_bf16 (optional, needs gl) = d(sum_b gl[b] loss[b]) / dF_t ; D_t (optional) [B,C,R,R] f32.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_ect_step_front(const float* moments, const float* eps, const float* rnd_normal, const float* noise_unit,
                       const float* drop_u, float drop_prob, float scale_factor, float P_mean, float P_std,
                       const float* qs, float k, float b_coef, float* y, float* xt, float* xr, float* sr, float* t,
                       float* r, float* labels, int B, int C, int R, int num_classes, void* stream);
int mdt_ect_loss(const float* Ft, const float* Fr, const float* xt, const float* xr, const float* y, const float* t,
                 const float* r, const float* mask, const float* gl, float sigma_data, float c, float mae_coef,
                 float* loss, float* D_t, void* dF_bf16, int B, int C, int R, int p, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Model guidance (MG; the definition is DESIGN §5): the conditional network learns the guided denoiser.
 * mdt_mg_loss: F [B,L,p*p*C] the student's output (conditional, gradient-carrying) ; Fu the no-gradient output of the
 *   same weights on the same xin, sigma and kept tokens with the null (all-zero) label row ; labels [B,num_classes] the
 *   student's label rows (a row is kept when any entry is non-zero).  Per row: w_b = w when the label row is kept and
 *   lo < sigma[b] <= hi, else 0 ; target = y + w_b c_out (F - Fu), and where w_b = 0 exactly y (a select: Fu of such a
 *   row is never read into the result).  loss[b] is mdt_edm_loss's loss with y replaced by the target in the
 *   denoising term (the MAE term unchanged) ; dF_bf16 (optional, needs gl) = d(sum_b gl[b] loss[b]) / dF with the
 *   target held constant ; edm_loss (optional) [B] = mdt_edm_loss's loss against y, bit for bit ; Dx as mdt_edm_loss.
 *   With w_b = 0 on every row, loss and dF_bf16 are mdt_edm_loss's bits.  0 <= w < 1 (w = 1 - 1/s for the
 *   CFG-equivalent scale s), lo < hi.  The pd rules are mdt_edm_loss's.
 * mdt_flow_mg_loss: the same on velocities for mdt_flow_loss: target v' = (eps - y) + w_b (F - Fu), the interval on t,
 *   edm_loss = mdt_flow_loss's loss bit for bit, x_hat as there.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_mg_loss(const float* F, const float* Fu, const float* xin, const float* y, const float* sigma,
                const float* labels, int num_classes, const float* mask, const float* gl, float sigma_data,
                float mae_coef, float w, float lo, float hi, float* loss, float* edm_loss, float* Dx, void* dF_bf16,
                int B, int C, int R, int p, void* stream);
int mdt_flow_mg_loss(const float* F, const float* Fu, const float* xt, const float* y, const float* eps,
                     const float* t, const float* labels, int num_classes, const float* mask, const float* gl,
                     float mae_coef, float w, float lo, float hi, float* loss, float* edm_loss, float* x_hat,
                     void* dF_bf16, int B, int C, int R, int p, void* stream);

/* D only (sampler / generic autograd path): Dx = c_skip*xin + c_out*unpatchify(F); and its backward
 * dF_bf16 = c_out * patchify(gD).                                                                            */
int mdt_edm_precond_out(const float* F, const float* xin, const float* sigma, float sigma_data, float* Dx, int B,
                        int C, int R, int p, void* stream);
int mdt_edm_precond_out_bwd(const float* gD, const float* sigma, float sigma_data, void* dF_bf16, int B, int C, int R,
                            int p, void* stream);

/* Classifier-free guidance combine (forward_with_cfg, models/maskdit.py:580-583) fused with the EDM output scaling:
 *   F [2B,L,p*p*C] (cond rows first, uncond rows second) -> Dx [B,C,R,R] = c_skip*x + c_out*(Fu + s (Fc - Fu))  */
int mdt_cfg_precond_out(const float* F, const float* xin, const float* sigma, float sigma_data, float cfg_scale,
                        float* Dx, int B, int C, int R, int p, void* stream);

/* Guidance by a second network (autoguidance, Karras et al. 2024), the same combine fused with the EDM output scaling:
 *   F_main [B, L_main, p_main²·C], F_guide [B, L_guide, p_guide²·C], each as mdt_forward writes it for its own patch
 *   size -> Dx [B,C,R,R] = c_skip*x + c_out*(Fg + w (Fm - Fg)), fp32, one thread per output pixel.
 *   MDT_ERR_ARG for a NULL pointer, B/C/R <= 0, a patch size that does not divide R, or a non-finite w. */
int mdt_guided_precond_out(const float* F_main, int p_main, const float* F_guide, int p_guide, const float* xin,
                           const float* sigma, float sigma_data, float w, float* Dx, int B, int C, int R,
                           void* stream);

/* EDM Heun sampler state update in fp64 (sample.py:56-64):
 *   mode 0 (Euler):  d_cur = (x_hat - den)/t_hat ; x_next = x_hat + (t_next - t_hat) d_cur
 *   mode 1 (Heun):   d_prime = (x_next - den)/t_next ; x_next = x_hat + (t_next - t_hat)(0.5 d_cur + 0.5 d_prime) */
int mdt_heun_update(int mode, const double* x_hat, const float* denoised, double* d_cur, double* x_next,
                    float* x_next_f32, double t_hat, double t_next, long long n, void* stream);

/* Generalised fp64 sampler update for ablation_sampler (sample.py:73-188; Euler / Heun / churn steps of every
 * discretization, schedule and scaling are linear combinations with host-computed fp64 scalars):
 *   out = a*x + b*y + c*z (x, y fp64; z fp32 network output; y / z may be NULL) ; out_f32 = float(out * f32_scale)
 *   (out or out_f32 may be NULL).                                                                                */
int mdt_lincomb_f64(double a, const double* x, double b, const double* y, double c, const float* z, double* out,
                    float* out_f32, double f32_scale, long long n, void* stream);

/* One multistep DPM-Solver++ step in fp64 (dpm_solver_sampler, DESIGN §5), one launch per network evaluation:
 *   D = F (kind MDT_DPM_DATA: F is the data prediction) or D = x - t*F (MDT_DPM_VELOCITY: F is a flow network's
 *   velocity; x is the state at flow time t) ;  d_out = D ;  x = a*x + b0*D + b1*h1 + b2*h2 (in place) ;
 *   x_f32 = float(x).  Each product and sum is rounded separately, in that order.  h2 / h1 may be NULL (term
 *   omitted; h2 only with h1), x_f32 may be NULL.  MDT_ERR_ARG for a NULL F / x / d_out, n <= 0, an unknown kind or a
 *   non-finite scalar.                                                                                            */
#define MDT_DPM_DATA 0
#define MDT_DPM_VELOCITY 1
int mdt_dpm_update(const float* F, int kind, double t, double* x, double* d_out, const double* h1, const double* h2,
                   double a, double b0, double b1, double b2, float* x_f32, long long n, void* stream);

/* Sampler tail (sample.py:287): img [B,C,H,W] f32 in [-1,1] -> uint8 [B,H,W,C] = clamp((img + 1) * 127.5, 0, 255).  */
int mdt_to_uint8_nhwc(const float* img, unsigned char* out, int B, int C, int H, int W, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Fused AdamW (weight_decay handled as adam_w_mode, train.py:141) + EMA (train_utils/helper.py:47-58) + bf16
 * weight-shadow refresh over flat buffers:  one pass instead of apex multi_tensor_adam + a 376-launch EMA loop.
 *   g is multiplied by grad_scale first (1/world_size after a SUM all-reduce).  ema / w_bf16 may be NULL.
 *   max_blocks > 0 caps the grid (a background launch overlapped with the backward GEMMs needs only a few CTAs).
 *   n % 4 == 0; w, m, v, ema and an fp32 g 16-byte aligned, w_bf16 and a bf16 g 8-byte aligned (MDT_ERR_ARG otherwise):
 *   a flat-buffer slice qualifies when it starts at a multiple of 4 elements.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_adamw_ema(float* w, const float* g, float* m, float* v, float* ema, void* w_bf16, long long n, float lr,
                  float beta1, float beta2, float eps, float weight_decay, int step, float ema_decay,
                  float grad_scale, int max_blocks, void* stream);
/* Same with a bf16 gradient operand: the buffer a bf16 gradient all-reduce produced (SURVEY 8e: 1.46 GB instead of
 * 2.92 GB on the wire, fp32 moments / master weights unchanged).                                                  */
int mdt_adamw_ema_g16(float* w, const void* g_bf16, float* m, float* v, float* ema, void* w_bf16, long long n,
                      float lr, float beta1, float beta2, float eps, float weight_decay, int step, float ema_decay,
                      float grad_scale, int max_blocks, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Non-finite gradient guard: accelerate's GradScaler skips an optimizer step whose gradients hold an inf or NaN
 * (train.py:39-48) while update_ema still runs (train.py:230).  The decision lives on the device, so a step needs
 * no host synchronisation:
 *   flag    one fp32 word, 0 = every checked element finite, 1 (or any non-zero) = skip.  The checks only ever store
 *           1.0f, so repeated calls over chunks accumulate, and a SUM all-reduce of the ranks' flags is their OR.
 *   counts  two int64 words {applied steps, skipped steps}, 8-byte aligned.
 * mdt_nonfinite_check: flag = 1 if any of g[0, n) is inf or NaN (g 16-byte aligned; one read of g).
 * mdt_cast_f32_bf16_check: mdt_cast_f32_bf16 (bit-identical output) that also sets the flag if a STORED bf16 value
 *   is inf or NaN, i.e. also for a finite fp32 value beyond bf16's range (|x| >= 3.3961e38 rounds to inf).
 * mdt_adamw_ema_guarded(_g16): with *flag == 0, mdt_adamw_ema(_g16) at step = counts[0] + 1 (the bias corrections are
 *   computed on the device from the counter), bit for bit; with *flag != 0 only ema = d*ema + (1-d)*w, and w, m, v,
 *   w_bf16 are not written.  Same arguments, alignment rules and grid as mdt_adamw_ema(_g16).  Neither reads or
 *   writes the counters' values beyond counts[0], so every chunk of a step sees the same step number.
 * mdt_optim_guard_advance: counts[*flag != 0] += 1 (one thread), enqueued once per step after its last guarded pass.
 *   The flag is not cleared: the caller zeroes it before the next step's checks.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_nonfinite_check(const float* g, long long n, float* flag, void* stream);
int mdt_cast_f32_bf16_check(const float* in, void* out_bf16, long long n, float* flag, void* stream);
int mdt_adamw_ema_guarded(float* w, const float* g, float* m, float* v, float* ema, void* w_bf16, long long n,
                          float lr, float beta1, float beta2, float eps, float weight_decay, float ema_decay,
                          float grad_scale, const float* flag, const long long* counts, int max_blocks, void* stream);
int mdt_adamw_ema_guarded_g16(float* w, const void* g_bf16, float* m, float* v, float* ema, void* w_bf16, long long n,
                              float lr, float beta1, float beta2, float eps, float weight_decay, float ema_decay,
                              float grad_scale, const float* flag, const long long* counts, int max_blocks,
                              void* stream);
int mdt_optim_guard_advance(const float* flag, long long* counts, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Gradient-norm clipping (torch.nn.utils.clip_grad_norm_; the reference does not clip, train.py:141,211-227).  The
 * norm and the coefficient live on the device, so a clipped step needs no host synchronisation:
 * mdt_grad_sumsq_scratch: the number of fp64 scratch slots mdt_grad_sumsq needs for n elements (>= 1; at most 2112
 *   whatever n), or MDT_ERR_ARG for n <= 0.  Host only, no device.
 * mdt_grad_sumsq: *out = sum of g[i]^2 over [0, n), g fp32 (bf16 = 0, 16-byte aligned) or bf16 (bf16 != 0, 8-byte
 *   aligned), accumulated in fp64: per-block partials in `scratch` (8-byte aligned), then one block sums them into
 *   *out (8-byte aligned) in a fixed order, without atomics.  The grid and the order depend on n alone, so the result
 *   is bit-reproducible whatever mdt_set_sm_budget and mdt_set_deterministic say.  A fp32 square stays below fp64's
 *   maximum: *out is finite exactly when every element is.  flag (may be NULL, 4-byte aligned): set to 1 when an
 *   element is inf or NaN, with mdt_nonfinite_check's convention, so one read of g is both the check and the norm.
 *   Two launches; calls on one stream may share `scratch`.
 * mdt_grad_clip_coef (one thread): norm = fp32(grad_scale * sqrt(sum of sumsq[0, k) in index order)), the sum and the
 *   product in fp64; coef = min(1, max_norm / (norm + 1e-6)) in fp32 as clip_grad_norm_ computes it
 *   (reciprocal(norm + 1e-6) * max_norm, a NaN staying NaN).  max_norm = +inf measures only: coef = 1.  With a finite
 *   max_norm and flag != NULL a non-finite norm sets the flag (a sum that overflowed although every rank's values were
 *   finite).  MDT_ERR_ARG for a NULL sumsq / norm / coef, k < 1, grad_scale <= 0 or NaN, max_norm <= 0 or NaN, sumsq
 *   not 8-byte or norm / coef / flag not 4-byte aligned.
 * mdt_adamw_ema_coef(_g16), mdt_adamw_ema_guarded_coef(_g16): mdt_adamw_ema(_g16) / mdt_adamw_ema_guarded(_g16) with
 *   the gradient scale grad_scale * *coef (coef: one fp32 word on the device, 4-byte aligned, read once
 *   before the loop).  With *coef == 1 they compute the plain entries' bits.  Same arguments, alignment rules and grid
 *   otherwise; MDT_ERR_ARG also for a NULL or misaligned coef.
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_grad_sumsq_scratch(long long n);
int mdt_grad_sumsq(const void* g, long long n, int bf16, double* scratch, double* out, float* flag, void* stream);
int mdt_grad_clip_coef(const double* sumsq, int k, double grad_scale, float max_norm, float* norm, float* coef,
                       float* flag, void* stream);
int mdt_adamw_ema_coef(float* w, const float* g, float* m, float* v, float* ema, void* w_bf16, long long n, float lr,
                       float beta1, float beta2, float eps, float weight_decay, int step, float ema_decay,
                       float grad_scale, const float* coef, int max_blocks, void* stream);
int mdt_adamw_ema_coef_g16(float* w, const void* g_bf16, float* m, float* v, float* ema, void* w_bf16, long long n,
                           float lr, float beta1, float beta2, float eps, float weight_decay, int step, float ema_decay,
                           float grad_scale, const float* coef, int max_blocks, void* stream);
int mdt_adamw_ema_guarded_coef(float* w, const float* g, float* m, float* v, float* ema, void* w_bf16, long long n,
                               float lr, float beta1, float beta2, float eps, float weight_decay, float ema_decay,
                               float grad_scale, const float* coef, const float* flag, const long long* counts,
                               int max_blocks, void* stream);
int mdt_adamw_ema_guarded_coef_g16(float* w, const void* g_bf16, float* m, float* v, float* ema, void* w_bf16,
                                   long long n, float lr, float beta1, float beta2, float eps, float weight_decay,
                                   float ema_decay, float grad_scale, const float* coef, const float* flag,
                                   const long long* counts, int max_blocks, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Power-function EMA profiles (post-hoc EMA, Karras et al., CVPR 2024, §3): k <= 4 fp32 profiles advanced from ONE
 * read of w[0, n):
 *   ema[j][i] += one_minus_beta[j] * (w[i] - ema[j][i])        (fp32, one fused multiply-add; c == 1 stores w exactly)
 * `ema` (k device pointers) and `one_minus_beta` (k coefficients in [0, 1], computed in float64 by the caller and
 * rounded) are HOST arrays, read at the call.  Any n > 0 and any 4-byte aligned slices: when every buffer reaches a
 * 16-byte boundary after the same number of elements the body moves float4s, otherwise every element is scalar.
 * Traffic: (4 + 8k) bytes per element.  MDT_ERR_ARG for a NULL pointer, k outside [1, 4], n <= 0, a pointer not 4-byte
 * aligned or a coefficient outside [0, 1] (NaN included).
 * ------------------------------------------------------------------------------------------------------------ */
int mdt_power_ema(const float* w, float* const* ema, const float* one_minus_beta, int k, long long n, void* stream);

/* Cap on the SMs the persistent kernels (the wgmma GEMM) occupy: n > 0 sizes their grids
 * for n SMs instead of the device's count, leaving the rest to a concurrently running collective (the gradient
 * all-reduce overlapped with the backward); 0 = whole device.  Host-side setting, read at launch.                  */
int mdt_set_sm_budget(int n);
int mdt_get_sm_budget(void);

/* Deterministic mode (on != 0; 0 = default): every floating-point reduction of the backward runs in an order that is a
 * function of the shapes alone, so repeated runs give identical bits whatever the SM count or budget.  Host-side
 * setting of the process, read at launch (the Python layer sets it from torch.are_deterministic_algorithms_enabled()).
 * What changes under it:
 *   - MDT_EPI_ATOMIC GEMMs run one k-slice (mdt_gemm_plan reports it); MDT_EPI_DGELU with a colsum pointer writes its
 *     output, then sums its columns in a fixed order;
 *   - mdt_colsum_* sum in a fixed order; mdt_ln_modulate_bwd, mdt_gate_bwd and mdt_ln_modulate_bwd_gate run one block
 *     per sample (rows_per_group rows);
 *   - mdt_workspace_bytes(training) adds the step driver's scratch for per-block partial sums, after every activation.
 * Entry points whose deterministic variant needs scratch they have no argument for return MDT_ERR_UNSUPPORTED under
 * it: mdt_patch_embed_bwd, mdt_gate_bwd with dbias != NULL, mdt_ln_modulate_bwd_gate with y_bf16 and dbias != NULL,
 * mdt_unmask_tokens_bwd with dmask_token != NULL (the step driver runs all four with workspace scratch).
 * mdt_ln_modulate_bwd needs 16-byte aligned dshift / dscale and ld_dmod % 4 == 0 under it (MDT_ERR_UNSUPPORTED otherwise). */
int mdt_set_deterministic(int on);
int mdt_get_deterministic(void);

/* ============================================================================================================
 * Step driver (SURVEY 8b): the whole network forward / backward as ONE call each over a packed parameter blob and ONE
 * caller-provided workspace — the launch sequence the reference obtains from autograd + torch.compile for
 * `loss = loss_fn(net, ...); loss.mean().backward()` (train.py:179,216-220; DiT.forward models/maskdit.py:467-557).
 * No allocation, no host synchronisation, everything enqueued on `stream`.
 *
 * Packed blob (element offsets shared by the fp32 master w32, the bf16 shadow w16 and the fp32 gradient):
 *   [adaLN_modulation.1.weight of blocks 0..depth-1, decoder_layer, decoder_blocks 0.., final_layer]
 *   [the matching adaLN biases] [all other trainable tensors in registration order] [pos_embed, decoder_pos_embed]
 * every tensor on a 64-element boundary; names = the reference's state-dict keys (models/maskdit.py:242-332).  A
 * handle with a learned loss weighting (mdt_model_set_logvar) adds logvar_linear.weight as the last trainable tensor
 * and logvar_fourier.freqs / .phases after the position tables.
 *
 * Decoder-less DiT (use_decoder=False, the reference's default, models/maskdit.py:254): dec_hidden = dec_depth =
 * dec_heads = dec_mlp_hidden = 0 and has_mask_token = 0.  Any other combination with a zero dec_* field is rejected.
 * There is no decoder_layer, no decoder block, no decoder_pos_embed and no mask token; the final layer reads the
 * encoder width ([p*p*C, hidden], adaLN [2*hidden, hidden]) and the modulation vector is blocks 0..depth-1, final:
 * depth*6*hidden + 2*hidden columns.  Training with a mask runs the final layer on the T kept tokens and scatters them
 * into F with zero rows for the removed tokens (:550-553); the removed rows get no gradient.
 * ============================================================================================================ */
typedef struct mdt_model_cfg {
  int img_resolution, img_channels, patch_size, num_classes; /* EDMPrecond / DiT ctor, models/maskdit.py:722-741     */
  int hidden, depth, heads, mlp_hidden;                      /* encoder DiTBlocks (DiT_models, :645-715)              */
  int dec_hidden, dec_depth, dec_heads, dec_mlp_hidden;      /* decoder (:310-312: 512, 8, 16, 2048); all 0: none     */
  int has_mask_token;                                        /* decoder and mae_loss_coef > 0 (:323-324)              */
  float sigma_data;
} mdt_model_cfg;
typedef struct mdt_model mdt_model; /* host-side layout object: no device memory, no CUDA calls */

int mdt_model_create(const mdt_model_cfg* cfg, mdt_model** out);
void mdt_model_destroy(mdt_model* m);
long long mdt_model_param_count(const mdt_model* m, int trainable_only); /* blob length in elements                  */
int mdt_model_num_tensors(const mdt_model* m);
/* i-th tensor in BLOB order: state-dict key, element offset, element count                                            */
int mdt_model_param_info(const mdt_model* m, int i, char* name, int name_cap, long long* offset, long long* numel);
int mdt_model_mod_width(const mdt_model* m); /* columns of the concatenated adaLN modulation vector                   */

/* Activation recomputation (gradient checkpointing) of the training pass: the first r blocks in forward order (encoder
 * blocks 0..depth-1, then decoder blocks) keep only their output residual (4 bytes per row and channel instead of about
 * 42); their other activations share one recompute slot sized for the largest of them, and mdt_backward re-runs each
 * such block's forward into the slot from its stored input (the adaLN modulation stays resident) before reading them.
 * The forward kernels neither split K nor use atomics, so the gradients are those of r = 0 bit for bit under the
 * deterministic mode.  0 <= r <= depth + dec_depth (MDT_ERR_ARG otherwise), default 0 (nothing recomputed, the plan
 * and launches of a handle without this setting).  Host-side setting of the handle, read by mdt_workspace_bytes
 * (training), mdt_forward (save = 1) and mdt_backward; the inference plan ignores it.  mdt_backward refuses
 * (MDT_ERR_ARG) a workspace laid out for another count: at r > 0 anything but the workspace of the handle's last
 * mdt_forward(save = 1) at the same r, at r = 0 the workspace of a last saving forward that recomputed.              */
int mdt_model_set_recompute(mdt_model* m, int r);
int mdt_model_get_recompute(const mdt_model* m); /* -1 for a NULL handle */

/* Learned loss weighting u(sigma) (mdt_edm_loss_logvar) with `channels` Fourier features: lays the handle out again with
 * three more tensors, `logvar_linear.weight` [1, channels] at the end of the trainable region and
 * `logvar_fourier.freqs`, `logvar_fourier.phases` [channels] in the frozen region after the position tables.  0 (the
 * default) is the layout without them.  MDT_ERR_ARG for channels < 0 or > 256, and once the handle has sized or laid
 * out a workspace (mdt_workspace_bytes, mdt_forward).                                                               */
int mdt_model_set_logvar(mdt_model* m, int channels);

/* Precondition kind of the handle: MDT_PRECOND_EDM (the default) or MDT_PRECOND_FLOW, where mdt_forward /
 * mdt_backward read their `sigma` argument as the flow time t: the patch embedding (forward and backward) applies
 * c_in = 1 and the timestep frequencies take c_noise = t.  The layout does not change.  MDT_ERR_ARG for another kind. */
int mdt_model_set_precond(mdt_model* m, int kind);

/* Workspace bytes for batch B with T kept tokens per sample (T <= 0: no token dropping, T = L).
 * training != 0: every activation the backward needs stays resident (+ the backward's scratch; with recomputation only
 * the recomputed blocks' output residuals and the slot); else inference.                                              */
long long mdt_workspace_bytes(const mdt_model* m, int B, int T, int training);

/* F [B*L, p*p*C] f32 = DiT.forward on x_in [B,C,R,R] (UNscaled network input, c_in applied inside), sigma [B],
 * labels [B,num_classes] f32 (NULL iff num_classes == 0), ids_keep [B,T] / ids_restore [B,L] int64 (both NULL: all
 * tokens).  save != 0 keeps the activations in `workspace` (256-byte aligned) for mdt_backward.                        */
int mdt_forward(const mdt_model* m, const float* w32, const void* w16, const float* x_in, const float* sigma,
                const float* labels, const int64_t* ids_keep, const int64_t* ids_restore, int B, int T, int save,
                void* workspace, long long workspace_bytes, float* F_out, void* stream);

/* grad (flat f32, blob offsets, trainable region) += d(loss)/d(params) given dF [B*L, p*p*C] bf16 and the workspace
 * of the matching mdt_forward(save = 1).  `on_ready(user, lo, hi)` (may be NULL) is called on the host as soon as the
 * kernels that finalise the gradient elements [lo, hi) of one block have been enqueued (DDP-bucket-style overlap).     */
typedef void (*mdt_grad_ready_fn)(void* user, long long lo, long long hi);
int mdt_backward(const mdt_model* m, const float* w32, const void* w16, float* grad, const float* x_in,
                 const float* sigma, const int64_t* ids_keep, const int64_t* ids_restore, const void* dF_bf16, int B,
                 int T, void* workspace, long long workspace_bytes, mdt_grad_ready_fn on_ready, void* user,
                 void* stream);

/* Data-parallel gradient exchange (train.py:178 DDP -> SURVEY 8e: ONE sum-all-reduce of the flat gradient buffer over
 * NVLink).  NCCL is resolved at run time from the process's libnccl.so.2 (MDT_ERR_DRIVER when absent).
 *   mdt_nccl_unique_id: rank 0 fills 128 bytes, the host code ships them to every rank (any side channel);
 *   mdt_nccl_comm_create: ncclCommInitRank (max_ctas > 0: ncclCommInitRankConfig with maxCTAs, a communicator that
 *   shares the GPU with the backward, see mdt_set_sm_budget); mdt_allreduce_grads: in-place SUM of fp32 (bf16 = 0) or
 *   bf16 elements.                                                                                                  */
int mdt_nccl_unique_id(void* id128);
int mdt_nccl_comm_create(const void* id128, int rank, int world, int max_ctas, void** comm);
int mdt_nccl_comm_destroy(void* comm);
int mdt_allreduce_grads(void* comm, void* grad, long long n, int bf16, void* stream);

/* Sharded optimizer state (ZeRO stage 1: the all-reduce split into its reduce-scatter and all-gather halves).  Both
 * collectives run in place on `buf`, which holds world * count_per_rank elements; rank r's share is
 * buf + r * count_per_rank.
 *   mdt_reduce_scatter_grads: rank r's share becomes the SUM over the ranks of that share (fp32, or bf16 when
 *   bf16 != 0); the rest of `buf` is left undefined.
 *   mdt_allgather: every rank's share is copied to the same place on every rank.  dtype MDT_DTYPE_F32, _BF16 or _F64.
 * MDT_ERR_ARG for a NULL pointer, count_per_rank <= 0 or another dtype; MDT_ERR_DRIVER when the process's NCCL lacks
 * ncclReduceScatter / ncclAllGather / ncclCommUserRank.                                                             */
#define MDT_DTYPE_F32 0
#define MDT_DTYPE_BF16 1
#define MDT_DTYPE_F64 2
int mdt_reduce_scatter_grads(void* comm, void* buf, long long count_per_rank, int bf16, void* stream);
int mdt_allgather(void* comm, void* buf, long long count_per_rank, int dtype, void* stream);

/* The fp32-read set of the handle's training step: the [lo, hi) element ranges of the trainable region that some
 * launch of mdt_forward / mdt_backward or of the training losses reads from `w32` rather than the bf16 shadow `w16`
 * (the patch embedder, every bias of a GEMM epilogue, the adaLN biases, the mask token, the learned weighting's w).
 * Sorted, disjoint, merged where adjacent, each hi rounded up to the 64-element tensor boundary.  Writes at most `cap`
 * pairs to lohi (may be NULL with cap 0) and returns the number of ranges, or a negative status.  A sharded optimizer
 * all-gathers these ranges of w32 after its update; every other master element may be stale on a rank between steps. */
int mdt_model_fp32_read_ranges(const mdt_model* m, long long* lohi, int cap);

/* dst[seg[3i+1] + j] = src[seg[3i] + j] for j < seg[3i+2], for each of the nseg segments (a device table of int64
 * triples {src offset, dst offset, count}, in fp32 elements).  Segments must not overlap in dst.  The sharded
 * optimizer packs and unpacks the fp32-read set with it.                                                          */
int mdt_copy_segments_f32(const float* src, float* dst, const long long* seg, int nseg, void* stream);

/* ============================================================================================================
 * SD-VAE: decode, the sampler tail (sample.py:275 `vae.decode(z)`; autoencoder.py:306-453), and encode, the latent
 * extraction (extract_latent.py:66; autoencoder.py:212-303,431-442).  Activations are pixel-major
 * fp32 row matrices [B*H*W, C]; every convolution is mdt_gemm_bf16 on an im2col operand built by mdt_vae_im2col with
 * the GroupNorm(32) affine, the swish and the nearest-2x upsample of its source fused in.  The host sequencing is
 * maskdit_b200/vae.py (same state-dict keys as FrozenAutoencoderKL: `decoder.*`, `post_quant_conv.*`, `encoder.*`,
 * `quant_conv.*`).
 * ============================================================================================================ */
/* out [B*P, C] f32 = post_quant_conv(z / scale_factor), z [B,C,h,w] NCHW (autoencoder.py:449-451); C <= 8           */
int mdt_vae_post_quant(const float* z, const float* W, const float* bias, float scale_factor, float* out, int B,
                       int C, int P, void* stream);
/* GroupNorm(32) statistics (Normalize, autoencoder.py:34-35) of x [B,P,C] f32: sums [B,32,2] f64 = (sum, sum of squares),
 * deterministic (fixed-order two-pass reduction); scratch: B * ceil(P/256) * 64 floats                              */
int mdt_vae_gn_stats(const float* x, double* sums, float* scratch, int B, int P, int C, void* stream);
/* A [B*H*W, Kp] bf16, A[(b,y,x),(ky,kx,c)] = f(src[b,(y+ky-pad)/up,(x+kx-pad)/up,c]) (0 outside); ks = 1 | 3; up = 1 | 2;
 * f = identity (sums NULL) | GroupNorm affine | GroupNorm affine + swish (silu != 0): ResnetBlock / Upsample /
 * norm_out inputs (autoencoder.py:49-53,117-137,404-406); columns >= ks*ks*C are zero.                              */
int mdt_vae_im2col(const float* src, const double* sums, const float* gamma, const float* beta, int silu, int ks,
                   int up, void* A_bf16, int B, int H, int W, int C, int Kp, void* stream);
/* The same with a stride and an explicit low-side padding: A[(b,y,x),(ky,kx,c)] = f(src[b, s*y+ky-pad, s*x+kx-pad, c]),
 * 0 outside the s*H x s*W source; stride = 1 | 2 (up must be 1 when stride = 2), 0 <= pad < ks.  Downsample
 * (autoencoder.py:56-75: pad (0,1,0,1) + 3x3 stride-2 conv) is ks = 3, stride = 2, pad = 0.  mdt_vae_im2col is
 * stride = 1, pad = ks / 2.                                                                                       */
int mdt_vae_im2col_strided(const float* src, const double* sums, const float* gamma, const float* beta, int silu,
                           int ks, int up, int stride, int pad, void* A_bf16, int B, int H, int W, int C, int Kp,
                           void* stream);
/* P [rows, cols] bf16 = softmax(scale * S) along columns (AttnBlock, autoencoder.py:185-187)                        */
int mdt_vae_softmax_rows(const float* S, float scale, void* P_bf16, int rows, int cols, void* stream);
/* x [B,P,ldx] f32 (first C columns) -> out [B,C,P] f32: the NCHW image `decode` returns                             */
int mdt_vae_rows_to_nchw(const float* x, float* out, int B, int P, int C, int ldx, void* stream);
/* Encode half (FrozenAutoencoderKL.encode_moments / encode, autoencoder.py:212-303,431-446):
 * img [B,3,H,W] f32 NCHW -> rows [B*H*W, 4] f32 (channel 3 zero; flip != 0: horizontally mirrored, the --xflip pass
 * of extract_latent.py:87), the conv_in operand.                                                                  */
int mdt_vae_image_to_rows(const float* img, float* rows, int B, int H, int W, int flip, void* stream);
/* moments [B,C,P] f32 NCHW = quant_conv(x), x [B*P, ldx] f32 (conv_out rows, first C valid), W [C,C], C <= 8 even;
 * eps [B,C/2,P] or NULL: z [B,C/2,P] = scale_factor * (mean + exp(0.5 * clamp(logvar,-30,20)) * eps) (sample,
 * autoencoder.py:436-442).                                                                                         */
int mdt_vae_quant_moments(const float* x, int ldx, const float* W, const float* bias, const float* eps,
                          float scale_factor, float* moments, float* z, int B, int C, int P, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MASKDIT_B200_H_ */
