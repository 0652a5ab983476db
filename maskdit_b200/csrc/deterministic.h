// Internal declarations of the deterministic mode (mdt_set_deterministic), shared by api.cu, driver.cu and
// elementwise.cu.  With the setting on, every floating-point reduction runs in an order fixed by the shapes alone:
// no float atomic receives more than one contribution per address per launch.  Where that needs per-block partials,
// the caller passes scratch; a NULL scratch under the setting is MDT_ERR_UNSUPPORTED (the library never allocates).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mdt {

extern int g_deterministic;

// out[n] += sum_m in[m, n] in a fixed order (one block per 32-column strip, rows summed lane by lane, lanes in order)
int colsum_ordered(const void* in, int in_bf16, int M, int N, long long ld, float* out, cudaStream_t stream);

// Scratch (floats) the deterministic variants below need: the largest of the three for the given shapes.
long long det_scratch_floats(int B, int T, int L, int D, int Dd, int cpp, int has_mask_token);

// The public entry points with a scratch argument (scratch is ignored when the setting is off).
int ln_modulate_bwd_gate_s(const void* dxmod_bf16, const float* x, const float* mean, const float* rstd,
                           const float* scale, int ld_mod, int rows_per_group, float* g, int accumulate, float* dshift,
                           float* dscale, int ld_dmod, const void* y_bf16, const float* gate, int ld_gate,
                           void* dy_bf16, float* dgate, int ld_dgate, float* dbias, int M, int D, float* scratch,
                           cudaStream_t stream);
int patch_embed_bwd_s(const float* x, const float* sigma, float sigma_data, const int64_t* ids_keep, const float* g,
                      float* gW, float* gb, int B, int C, int R, int p, int D, int T, float* scratch,
                      cudaStream_t stream);
int unmask_tokens_bwd_s(const float* g, const int64_t* ids_restore, void* du_bf16, float* dmask_token, int B, int T,
                        int L, int D, float* scratch, cudaStream_t stream);

}  // namespace mdt
