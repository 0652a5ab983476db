// extern "C" surface that is not tied to one kernel file: status strings, ABI version, GEMM entry.
#include "deterministic.h"
#include "gemm.h"

#include <vector>

namespace mdt {
extern int g_gemm_last_config, g_gemm_configs_seen;
int g_sm_budget = 0;  // mdt_set_sm_budget: SMs the persistent kernels may occupy (0 = all)
}

extern "C" {

const char* mdt_status_string(int status) {
  switch (status) {
    case MDT_OK: return "ok";
    case MDT_ERR_ARG: return "invalid argument (shape / alignment / null pointer)";
    case MDT_ERR_CUDA: return "CUDA launch failure";
    case MDT_ERR_DRIVER: return "cuTensorMapEncodeTiled driver entry point unavailable";
    case MDT_ERR_TMAP: return "tensor map encode failed";
    case MDT_ERR_UNSUPPORTED: return "unsupported configuration";
    default: return "unknown status";
  }
}

int mdt_abi_version(void) { return 2; }  // 2: mdt_gemm_args.colsum, step driver, gradient exchange

int mdt_set_sm_budget(int n) {
  if (n < 0) return MDT_ERR_ARG;
  mdt::g_sm_budget = n;
  return MDT_OK;
}
int mdt_get_sm_budget(void) { return mdt::g_sm_budget; }

int mdt_set_deterministic(int on) {
  mdt::g_deterministic = on != 0;
  return MDT_OK;
}
int mdt_get_deterministic(void) { return mdt::g_deterministic; }

int mdt_gemm_last_config(void) { return mdt::g_gemm_last_config; }
int mdt_gemm_configs_seen(int reset) {
  const int v = mdt::g_gemm_configs_seen;
  if (reset) mdt::g_gemm_configs_seen = 0;
  return v;
}

// Per-launch device timing of the GEMM family inside a real step (bench.py's roofline.achieved): while enabled, every
// mdt_gemm_bf16 launch - also the step driver's internal ones - is bracketed by a pair of CUDA events on the launching
// stream.  Enqueued from C++ the events add no host-side bubbles (the Python-paced variant of this measurement moved
// between 0.73 and 0.81 of peak on identical code).
namespace {
struct GemmProbe {
  cudaEvent_t e0, e1;
  double flops;
};
std::vector<GemmProbe> g_probes;
bool g_probe_on = false;
}  // namespace

int mdt_gemm_profile_enable(int on) {
  if (on && !g_probe_on) {
    for (auto& p : g_probes) cudaEventDestroy(p.e0), cudaEventDestroy(p.e1);
    g_probes.clear();
  }
  g_probe_on = on != 0;
  return MDT_OK;
}

// Returns the number of recorded launches; fills ms[i] / flops[i] for i < cap (synchronises on each launch's end event).
int mdt_gemm_profile_read(float* ms, double* flops, int cap) {
  const int n = static_cast<int>(g_probes.size());
  for (int i = 0; i < n && i < cap; ++i) {
    if (cudaEventSynchronize(g_probes[i].e1) != cudaSuccess) return MDT_ERR_CUDA;
    float t = 0.f;
    if (cudaEventElapsedTime(&t, g_probes[i].e0, g_probes[i].e1) != cudaSuccess) return MDT_ERR_CUDA;
    if (ms) ms[i] = t;
    if (flops) flops[i] = g_probes[i].flops;
  }
  return n;
}

int mdt_gemm_plan(const mdt_gemm_args* args, long long* out10) {
  if (!args || !out10) return MDT_ERR_ARG;
  mdt::GemmPlan pl;
  const int rc = mdt::gemm_plan(*args, &pl);
  if (rc != MDT_OK) return rc;
  const long long v[10] = {pl.block_n, pl.cg, pl.splits, pl.pair_halves, pl.narrow_last,
                           pl.num_m_tiles, pl.num_n_tiles, pl.num_kb, pl.units, pl.grid};
  for (int i = 0; i < 10; ++i) out10[i] = v[i];
  return MDT_OK;
}

// Deterministic mode: the DGELU epilogue's column sum (one reduction per tile and column) is replaced by an ordered
// column sum of the stored bf16 output, the same values the fused sum adds.
static int gemm_run(const mdt_gemm_args& a, cudaStream_t stream) {
  if (!mdt::g_deterministic || a.epi != MDT_EPI_DGELU || !a.colsum) return mdt::gemm_launch(a, stream);
  mdt_gemm_args b = a;
  b.colsum = nullptr;
  const int rc = mdt::gemm_launch(b, stream);
  return rc == MDT_OK ? mdt::colsum_ordered(a.out, 1, a.M, a.N, a.ldo, a.colsum, stream) : rc;
}

int mdt_gemm_bf16(const mdt_gemm_args* args, void* stream) {
  if (!args || !args->A || !args->B || !args->out) return MDT_ERR_ARG;
  if (!g_probe_on) return gemm_run(*args, static_cast<cudaStream_t>(stream));
  GemmProbe p;
  if (cudaEventCreate(&p.e0) != cudaSuccess || cudaEventCreate(&p.e1) != cudaSuccess) return MDT_ERR_CUDA;
  p.flops = 2.0 * args->M * args->N * args->K;
  cudaEventRecord(p.e0, static_cast<cudaStream_t>(stream));
  const int rc = gemm_run(*args, static_cast<cudaStream_t>(stream));
  cudaEventRecord(p.e1, static_cast<cudaStream_t>(stream));
  g_probes.push_back(p);
  return rc;
}

}  // extern "C"
