// Step driver: the whole MaskDiT network forward / backward as ONE C-ABI call each (SURVEY 8b: mdt_forward,
// mdt_backward, mdt_workspace_bytes over a packed parameter blob and ONE caller-provided workspace), plus the data-
// parallel gradient exchange (mdt_nccl_*, mdt_allreduce_grads).
//
// This is the launch sequence of DiT.forward + forward_encoder (models/maskdit.py:467-557) and of its hand-written
// backward, issued from C++ on the caller's stream: ~280 launches forward, ~500 backward, no allocation (every
// activation is a fixed slice of the workspace, planned once per (B, T, mode)), no Python between launches.  The
// reference gets this sequencing from autograd + torch.compile (train.py:179,216-220); the per-kernel entry points
// it is built from stay exported (the parity tests drive them one by one; the tests' reference `maskdit_b200/engine.py::
// Engine` issues the same sequence from Python and must agree bit for bit in the forward).
//
// Packed parameter blob (fp32 master `w32`, bf16 shadow `w16`, fp32 gradient `grad`: same element offsets):
//   [adaLN_modulation.1.weight of blocks 0..depth-1, decoder_layer, decoder_blocks 0..dec_depth-1, final_layer]
//   [the matching adaLN biases] [every other trainable tensor in registration order] [pos_embed, decoder_pos_embed]
// (with mdt_model_set_logvar: logvar_linear.weight the last trainable tensor, logvar_fourier.* after the tables)
// each tensor starting on a 64-element boundary.  The decoder-less DiT (use_decoder=False, models/maskdit.py:254,
// 308-331: all four dec_* fields 0) has no decoder_layer, decoder blocks, decoder_pos_embed or mask token, and its
// final layer reads the encoder width.  `build_layout` is the only place these offsets are decided:
// `mdt_model_param_info` enumerates them and `maskdit_b200/flat.py` lays the nn.Module's parameters out from it.
#include <dlfcn.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "common.cuh"
#include "deterministic.h"
#include "../../include/maskdit_b200.h"

namespace {

typedef long long i64;
constexpr i64 kAlign = 64;  // elements
inline i64 round_up(i64 n, i64 a = kAlign) { return (n + a - 1) / a * a; }

struct Tensor {
  i64 off = -1, numel = 0;
};

struct BlockP {
  Tensor qkv_w, qkv_b, proj_w, proj_b, fc1_w, fc1_b, fc2_w, fc2_b;
  int dim, heads, dh, h4;
  i64 mod_off;
  i64 lo, hi;  // gradient range of the block's non-adaLN tensors (final once the block's backward is enqueued)
};

struct NamedTensor {
  std::string name;
  Tensor* t;
  i64 numel;
  int group;  // 0 adaLN weight, 1 adaLN bias, 2 other trainable, 3 frozen
  int rank;   // order inside groups 0/1
};

}  // namespace

struct mdt_model {
  mdt_model_cfg cfg;
  int D, Dd, L, G, pd, NA, H4e, H4d, Kp;
  bool has_dec;  // false: decoder-less DiT, the final layer runs on the encoder's T kept tokens (width D)
  int Df;        // final-layer input width: Dd, or D without a decoder
  std::vector<BlockP> enc, dec;
  Tensor pos, dpos, mask_token, xw, xb, t0w, t0b, t2w, t2b, ytab, dlw, dlb, flw, flb;
  std::vector<Tensor> ada_w, ada_b;  // per head, in blob order
  i64 ada_w_off, ada_b_off;
  i64 off_declayer, off_final;
  i64 n_train, n_total;
  std::vector<NamedTensor> named;  // registration order
  std::vector<int> order;          // blob order (indices into named)
  int recompute = 0;               // blocks whose activations the backward recomputes (mdt_model_set_recompute)
  int logvar_channels = 0;         // learned loss weighting u(sigma) (mdt_model_set_logvar); 0: none
  Tensor lv_freqs, lv_phases, lv_w;
  int precond = MDT_PRECOND_EDM;   // how mdt_forward / mdt_backward read `sigma` (mdt_model_set_precond)
  mutable bool planned = false;    // a workspace was sized or laid out: the layout is final
  // the workspace of the last mdt_forward(save = 1) and the recompute count it was laid out for: mdt_backward refuses
  // to read a workspace with another count's plan
  mutable const void* fwd_ws = nullptr;
  mutable int fwd_r = 0;
};

namespace {

void build_layout(mdt_model* m) {
  const mdt_model_cfg& c = m->cfg;
  const int D = c.hidden, Dd = c.dec_hidden;
  m->D = D, m->Dd = Dd;
  m->has_dec = c.dec_hidden > 0;
  m->Df = m->has_dec ? Dd : D;
  m->G = c.img_resolution / c.patch_size;
  m->L = m->G * m->G;
  m->pd = c.patch_size * c.patch_size * c.img_channels;
  m->H4e = c.mlp_hidden, m->H4d = c.dec_mlp_hidden;
  m->Kp = static_cast<int>(round_up(c.num_classes, 8));
  m->enc.resize(c.depth);
  m->dec.resize(c.dec_depth);
  m->ada_w.resize(c.depth + c.dec_depth + (m->has_dec ? 2 : 1));
  m->ada_b.resize(c.depth + c.dec_depth + (m->has_dec ? 2 : 1));
  auto& nm = m->named;
  auto add = [&](const std::string& name, Tensor* t, i64 numel, int group, int rank = 0) {
    nm.push_back(NamedTensor{name, t, numel, group, rank});
  };
  // registration order of the reference module (models/maskdit.py:242-332)
  add("model.pos_embed", &m->pos, static_cast<i64>(m->L) * D, 3);
  if (m->has_dec) add("model.decoder_pos_embed", &m->dpos, static_cast<i64>(m->L) * Dd, 3);
  if (c.has_mask_token) add("model.mask_token", &m->mask_token, Dd, 2);
  add("model.x_embedder.proj.weight", &m->xw, static_cast<i64>(D) * m->pd, 2);
  add("model.x_embedder.proj.bias", &m->xb, D, 2);
  add("model.t_embedder.mlp.0.weight", &m->t0w, static_cast<i64>(D) * 256, 2);
  add("model.t_embedder.mlp.0.bias", &m->t0b, D, 2);
  add("model.t_embedder.mlp.2.weight", &m->t2w, static_cast<i64>(D) * D, 2);
  add("model.t_embedder.mlp.2.bias", &m->t2b, D, 2);
  if (c.num_classes > 0) add("model.y_embedder.embedding_table.weight", &m->ytab, static_cast<i64>(D) * c.num_classes, 2);
  int head = 0;
  i64 mod = 0;
  auto add_block = [&](const std::string& p, BlockP& b, int dim, int heads, int h4) {
    b.dim = dim, b.heads = heads, b.dh = dim / heads, b.h4 = h4, b.mod_off = mod;
    mod += 6 * dim;
    add(p + ".attn.qkv.weight", &b.qkv_w, 3ll * dim * dim, 2);
    add(p + ".attn.qkv.bias", &b.qkv_b, 3ll * dim, 2);
    add(p + ".attn.proj.weight", &b.proj_w, static_cast<i64>(dim) * dim, 2);
    add(p + ".attn.proj.bias", &b.proj_b, dim, 2);
    add(p + ".mlp.fc1.weight", &b.fc1_w, static_cast<i64>(h4) * dim, 2);
    add(p + ".mlp.fc1.bias", &b.fc1_b, h4, 2);
    add(p + ".mlp.fc2.weight", &b.fc2_w, static_cast<i64>(dim) * h4, 2);
    add(p + ".mlp.fc2.bias", &b.fc2_b, dim, 2);
    add(p + ".adaLN_modulation.1.weight", &m->ada_w[head], 6ll * dim * D, 0, head);
    add(p + ".adaLN_modulation.1.bias", &m->ada_b[head], 6ll * dim, 1, head);
    ++head;
  };
  for (int i = 0; i < c.depth; ++i) add_block("model.blocks." + std::to_string(i), m->enc[i], D, c.heads, m->H4e);
  m->off_declayer = -1;
  if (m->has_dec) {
    m->off_declayer = mod;
    mod += 2 * D;
    add("model.decoder_layer.linear.weight", &m->dlw, static_cast<i64>(Dd) * D, 2);
    add("model.decoder_layer.linear.bias", &m->dlb, Dd, 2);
    add("model.decoder_layer.adaLN_modulation.1.weight", &m->ada_w[head], 2ll * D * D, 0, head);
    add("model.decoder_layer.adaLN_modulation.1.bias", &m->ada_b[head], 2ll * D, 1, head);
    ++head;
    for (int i = 0; i < c.dec_depth; ++i)
      add_block("model.decoder_blocks." + std::to_string(i), m->dec[i], Dd, c.dec_heads, m->H4d);
  }
  const int Df = m->Df;
  m->off_final = mod;
  mod += 2 * Df;
  add("model.final_layer.linear.weight", &m->flw, static_cast<i64>(m->pd) * Df, 2);
  add("model.final_layer.linear.bias", &m->flb, m->pd, 2);
  add("model.final_layer.adaLN_modulation.1.weight", &m->ada_w[head], 2ll * Df * D, 0, head);
  add("model.final_layer.adaLN_modulation.1.bias", &m->ada_b[head], 2ll * Df, 1, head);
  // learned loss weighting (EDMPrecond registers it after model.*): the weight ends the trainable region, the Fourier
  // features follow the position tables
  if (m->logvar_channels > 0) {
    add("logvar_fourier.freqs", &m->lv_freqs, m->logvar_channels, 3);
    add("logvar_fourier.phases", &m->lv_phases, m->logvar_channels, 3);
    add("logvar_linear.weight", &m->lv_w, m->logvar_channels, 2);
  }
  m->NA = static_cast<int>(mod);
  // blob order: group 0 by rank, group 1 by rank, group 2 in registration order, group 3 last
  i64 off = 0;
  for (int g = 0; g < 4; ++g) {
    if (g == 3) m->n_train = off;
    std::vector<int> idx;
    for (size_t i = 0; i < nm.size(); ++i)
      if (nm[i].group == g) idx.push_back(static_cast<int>(i));
    if (g < 2)
      for (size_t a = 0; a < idx.size(); ++a)  // insertion sort by rank (already nearly ordered)
        for (size_t b = a; b > 0 && nm[idx[b - 1]].rank > nm[idx[b]].rank; --b) std::swap(idx[b - 1], idx[b]);
    for (int i : idx) {
      nm[i].t->off = off, nm[i].t->numel = nm[i].numel;
      off += round_up(nm[i].numel);
      m->order.push_back(i);
    }
  }
  m->n_total = off;
  m->ada_w_off = m->ada_w[0].off;
  m->ada_b_off = m->ada_b[0].off;
  for (auto* blocks : {&m->enc, &m->dec})
    for (BlockP& b : *blocks) b.lo = b.qkv_w.off, b.hi = b.fc2_b.off + round_up(b.fc2_b.numel);
}

// ---- workspace plan ------------------------------------------------------------------------------------------------
struct Arena {
  i64 off = 0;
  i64 take(i64 bytes) {
    const i64 o = off;
    off += (bytes + 255) & ~255ll;
    return o;
  }
};

struct BlockBuf {
  i64 xm1, mean1, rstd1, qkv, O, lse, X1, y1, xm2, mean2, rstd2, a, hpre, X2, y2;
};

struct Plan {
  i64 X0, tf, th_pre, th, c, c2, y16, y16p, wyp, sc, mod;
  std::vector<BlockBuf> enc, dec;
  i64 xmd, mean_d, rstd_d, u, Z, xf, mean_f, rstd_f;
  i64 fk;  // decoder-less + masked: final-layer output of the kept tokens [B*T, pd] f32, in the backward their dF bf16
  // backward scratch
  i64 dmod, dxf, Gz, dyA, dyB, dh, dxm, dO, dqkv, du, dxmd, Ge, dmod16, dsc, dc32, dc16, dth, dpre32, dpre16, ytmp;
  i64 det;  // deterministic mode only: per-block partial sums (after everything else, so no other offset moves)
  i64 total;
};

// Training plan with recomputation (mdt_model_set_recompute, r > 0): the first r blocks in forward order (encoder blocks
// first, then decoder blocks) keep only their output residual X2, the next block's input.  Their other slices all point
// into ONE recompute slot, laid out after the final layer's slices, as large per slice as the largest recomputed block's
// (plus a second mean1 / rstd1, see mdt_backward).  mdt_forward writes a recomputed block's activations into the slot;
// mdt_backward re-runs the block's forward there from its stored input before reading them.
Plan make_plan(const mdt_model* m, int B, int T, bool save, bool with_backward) {
  Plan p;
  Arena a;
  const int D = m->D, Dd = m->Dd, L = m->L, NA = m->NA;
  const int r = save ? m->recompute : 0;
  i64 need_md = 0, need_m = 0, need_mh = 0, need_lse = 0;  // slot: largest M * dim, M, M * mlp hidden, lse bytes
  auto grow = [](i64& n, i64 v) { n = v > n ? v : n; };
  const i64 Me = static_cast<i64>(B) * T, Md = static_cast<i64>(B) * L;
  p.X0 = a.take(Me * D * 4);
  p.tf = a.take(B * 256ll * 2);
  p.th_pre = a.take(static_cast<i64>(B) * D * 4);
  p.th = a.take(static_cast<i64>(B) * D * 2);
  p.c = a.take(static_cast<i64>(B) * D * 4);
  p.c2 = a.take(static_cast<i64>(B) * D * 4);
  p.y16 = a.take(static_cast<i64>(B) * m->Kp * 2 + 16);
  p.y16p = a.take(static_cast<i64>(B) * m->Kp * 2 + 16);
  p.wyp = a.take(static_cast<i64>(D) * m->Kp * 2 + 16);
  p.sc = a.take(static_cast<i64>(B) * D * 2);
  p.mod = a.take(static_cast<i64>(B) * NA * 4);
  auto plan_blocks = [&](const std::vector<BlockP>& bl, std::vector<BlockBuf>& out, i64 M, int tokens, int first) {
    out.resize(bl.size());
    const i64 scratch0 = a.off;
    for (size_t i = 0; i < bl.size(); ++i) {
      if (!save) a.off = scratch0;  // inference: every block reuses one set of temporaries, residual in place
      const int d = bl[i].dim, h4 = bl[i].h4;
      BlockBuf& b = out[i];
      if (first + static_cast<int>(i) < r) {  // recomputed: only the output residual stays, the rest is in the slot
        grow(need_md, M * d), grow(need_m, M), grow(need_mh, M * h4), grow(need_lse, 2ll * B * bl[i].heads * tokens * 4);
        b.X2 = a.take(M * d * 4);
        continue;
      }
      b.xm1 = a.take(M * d * 2);
      b.mean1 = save ? a.take(M * 4) : -1;
      b.rstd1 = save ? a.take(M * 4) : -1;
      b.qkv = a.take(M * 3 * d * 2);
      b.O = a.take(M * d * 2);
      b.lse = save ? a.take(2ll * B * bl[i].heads * tokens * 4) : -1;
      b.X1 = save ? a.take(M * d * 4) : -1;
      b.y1 = save ? a.take(M * d * 2) : -1;
      b.xm2 = a.take(M * d * 2);
      b.mean2 = save ? a.take(M * 4) : -1;
      b.rstd2 = save ? a.take(M * 4) : -1;
      b.a = a.take(M * h4 * 2);
      b.hpre = save ? a.take(M * h4 * 2) : -1;
      b.X2 = save ? a.take(M * d * 4) : -1;
      b.y2 = save ? a.take(M * d * 2) : -1;
    }
  };
  plan_blocks(m->enc, p.enc, Me, T, 0);
  p.xmd = p.mean_d = p.rstd_d = p.u = p.Z = p.fk = p.Gz = p.du = p.dxmd = -1;
  if (m->has_dec) {
    p.xmd = a.take(Me * D * 2);
    p.mean_d = a.take(Me * 4);
    p.rstd_d = a.take(Me * 4);
    p.u = a.take(Me * Dd * 4);
    p.Z = a.take(Md * Dd * 4);
    plan_blocks(m->dec, p.dec, Md, L, static_cast<int>(m->enc.size()));
  }
  const i64 Mf = m->has_dec ? Md : Me;  // final-layer rows
  p.xf = a.take(Mf * m->Df * 2);
  p.mean_f = a.take(Mf * 4);
  p.rstd_f = a.take(Mf * 4);
  if (!m->has_dec) p.fk = a.take(Me * m->pd * 4);
  if (r > 0) {  // the recompute slot, in BlockBuf order (no X2), then the second mean1 / rstd1
    BlockBuf s;
    s.xm1 = a.take(need_md * 2);
    s.mean1 = a.take(need_m * 4);
    s.rstd1 = a.take(need_m * 4);
    s.qkv = a.take(need_md * 3 * 2);
    s.O = a.take(need_md * 2);
    s.lse = a.take(need_lse);
    s.X1 = a.take(need_md * 4);
    s.y1 = a.take(need_md * 2);
    s.xm2 = a.take(need_md * 2);
    s.mean2 = a.take(need_m * 4);
    s.rstd2 = a.take(need_m * 4);
    s.a = a.take(need_mh * 2);
    s.hpre = a.take(need_mh * 2);
    s.y2 = a.take(need_md * 2);
    const i64 mean1b = a.take(need_m * 4), rstd1b = a.take(need_m * 4);
    const int ne = static_cast<int>(p.enc.size());
    for (int g = 0; g < r; ++g) {
      BlockBuf& b = g < ne ? p.enc[g] : p.dec[g - ne];
      s.X2 = b.X2;
      b = s;
      if (g % 2) b.mean1 = mean1b, b.rstd1 = rstd1b;
    }
  }
  if (with_backward) {
    const i64 Mmax_d = Me * D > Md * Dd ? Me * D : Md * Dd;                    // max over (enc, dec) of M * dim
    const i64 Mmax_h = Me * m->H4e > Md * m->H4d ? Me * m->H4e : Md * m->H4d;  // M * mlp hidden
    p.dmod = a.take(static_cast<i64>(B) * NA * 4);
    p.dxf = a.take(Mf * m->Df * 2);
    if (m->has_dec) p.Gz = a.take(Md * Dd * 4);
    p.dyA = a.take(Mmax_d * 2);
    p.dyB = a.take(Mmax_d * 2);
    p.dh = a.take(Mmax_h * 2);
    p.dxm = a.take(Mmax_d * 2);
    p.dO = a.take(Mmax_d * 2);
    p.dqkv = a.take(Mmax_d * 3 * 2);
    if (m->has_dec) p.du = a.take(Me * Dd * 2), p.dxmd = a.take(Me * D * 2);
    p.Ge = a.take(Me * D * 4);
    p.dmod16 = a.take(static_cast<i64>(B) * NA * 2);
    p.dsc = a.take(static_cast<i64>(B) * D * 4);
    p.dc32 = a.take(static_cast<i64>(B) * D * 4);
    p.dc16 = a.take(static_cast<i64>(B) * D * 2);
    p.dth = a.take(static_cast<i64>(B) * D * 4);
    p.dpre32 = a.take(static_cast<i64>(B) * D * 4);
    p.dpre16 = a.take(static_cast<i64>(B) * D * 2);
    p.ytmp = a.take(static_cast<i64>(D) * m->Kp * 4);
  }
  p.det = -1;
  if (with_backward && mdt::g_deterministic)
    p.det = a.take(mdt::det_scratch_floats(B, T, L, D, Dd, m->pd, m->cfg.has_mask_token) * 4);
  p.total = a.off;
  return p;
}

// ---- launch helpers ------------------------------------------------------------------------------------------------
struct Ctx {
  const mdt_model* m;
  const float* w32;
  const __nv_bfloat16* w16;
  float* grad;
  char* ws;
  void* stream;
  int rc = MDT_OK;
  float* scratch = nullptr;  // Plan::det (deterministic mode)
  template <class T>
  T* at(i64 off) const { return off < 0 ? nullptr : reinterpret_cast<T*>(ws + off); }
  const float* W32(const Tensor& t) const { return w32 + t.off; }
  const __nv_bfloat16* W16(const Tensor& t) const { return w16 + t.off; }
  float* Gd(const Tensor& t) const { return grad + t.off; }
  void ck(int r) {
    if (rc == MDT_OK && r != MDT_OK) rc = r;
  }
};

struct Gemm {
  mdt_gemm_args a;
  Gemm(const void* A, const void* B, i64 M, i64 N, i64 K, bool a_mn = false, bool b_mn = false) {
    memset(&a, 0, sizeof(a));
    a.A = A, a.B = B, a.M = static_cast<int>(M), a.N = static_cast<int>(N), a.K = static_cast<int>(K);
    a.a_mn = a_mn, a.b_mn = b_mn;
    a.lda = static_cast<int>(a_mn ? M : K), a.ldb = static_cast<int>(b_mn ? N : K);
    a.ldo = static_cast<int>(N), a.rows_per_group = 1;
  }
  Gemm& out32(float* o, int ldo = 0) { a.out = o, a.out_fp32 = 1; if (ldo) a.ldo = ldo; return *this; }
  Gemm& out16(void* o) { a.out = o, a.out_fp32 = 0; return *this; }
  Gemm& ldb(int v) { a.ldb = v; return *this; }
  Gemm& bias(const float* b) { a.bias = b; return *this; }
  Gemm& epi(int e) { a.epi = e; return *this; }
  Gemm& aux(void* x, int ld) { a.aux = x, a.ld_aux = ld; return *this; }
  Gemm& resid(const float* r, int ld) { a.resid = r, a.ld_resid = ld; return *this; }
  Gemm& colsum(float* cs) { a.colsum = cs; return *this; }
  Gemm& gate(const float* g, int ld, int rpg) { a.gate = g, a.ld_gate = ld, a.rows_per_group = rpg; return *this; }
  void run(Ctx& c) { if (c.rc == MDT_OK) c.ck(mdt_gemm_bf16(&a, c.stream)); }
};

// gout[n_out, k_in] += dY[tokens, n_out]^T @ Xin[tokens, k_in]   (stream-K, fp32 red.add)
void wgrad(Ctx& c, const void* dY, const void* Xin, i64 n_out, i64 k_in, i64 tokens, float* gout) {
  Gemm(dY, Xin, n_out, k_in, tokens, true, true).out32(gout, static_cast<int>(k_in)).epi(MDT_EPI_ATOMIC).run(c);
}

__global__ void add_strided_kernel(float* __restrict__ dst, int ld_dst, const float* __restrict__ src, int ld_src,
                                   int rows, int cols) {
  const i64 i = blockIdx.x * static_cast<i64>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<i64>(rows) * cols) return;
  const int r = static_cast<int>(i / cols), cc = static_cast<int>(i % cols);
  dst[static_cast<i64>(r) * ld_dst + cc] += src[static_cast<i64>(r) * ld_src + cc];
}

struct BlockSaved {  // the tensors one block's backward reads
  const float* X;
  const BlockBuf* b;
};

// DiTBlock.forward (models/maskdit.py:188-192).  X [M, d] f32 -> returns the block output pointer.
float* block_fwd(Ctx& c, const BlockP& s, const BlockBuf& b, float* X, const float* mod, int B, int T, bool save) {
  const int d = s.dim, NA = c.m->NA;
  const i64 M = static_cast<i64>(B) * T, o = s.mod_off;
  void* st = c.stream;
  __nv_bfloat16* xm1 = c.at<__nv_bfloat16>(b.xm1);
  c.ck(mdt_ln_modulate(X, mod + o, mod + o + d, NA, T, xm1, c.at<float>(b.mean1), c.at<float>(b.rstd1),
                       static_cast<int>(M), d, 1e-6f, st));
  __nv_bfloat16* qkv = c.at<__nv_bfloat16>(b.qkv);
  Gemm(xm1, c.W16(s.qkv_w), M, 3 * d, d).out16(qkv).bias(c.W32(s.qkv_b)).run(c);
  __nv_bfloat16* O = c.at<__nv_bfloat16>(b.O);
  c.ck(mdt_attention_fwd(qkv, O, c.at<float>(b.lse), B, T, s.heads, s.dh, st));
  float* X1 = save ? c.at<float>(b.X1) : X;
  Gemm(O, c.W16(s.proj_w), M, d, d).out32(X1).bias(c.W32(s.proj_b)).epi(MDT_EPI_GATE_RESID)
      .aux(c.at<void>(b.y1), d).resid(X, d).gate(mod + o + 2 * d, NA, T).run(c);
  __nv_bfloat16* xm2 = c.at<__nv_bfloat16>(b.xm2);
  c.ck(mdt_ln_modulate(X1, mod + o + 3 * d, mod + o + 4 * d, NA, T, xm2, c.at<float>(b.mean2), c.at<float>(b.rstd2),
                       static_cast<int>(M), d, 1e-6f, st));
  __nv_bfloat16* act = c.at<__nv_bfloat16>(b.a);
  Gemm(xm2, c.W16(s.fc1_w), M, s.h4, d).out16(act).bias(c.W32(s.fc1_b)).epi(MDT_EPI_GELU)
      .aux(c.at<void>(b.hpre), s.h4).run(c);
  float* X2 = save ? c.at<float>(b.X2) : X1;
  Gemm(act, c.W16(s.fc2_w), M, d, s.h4).out32(X2).bias(c.W32(s.fc2_b)).epi(MDT_EPI_GATE_RESID)
      .aux(c.at<void>(b.y2), d).resid(X1, d).gate(mod + o + 5 * d, NA, T).run(c);
  return X2;
}

struct GateNext {  // the MLP-branch gate backward fused into the LN backward that finishes the residual gradient
  const void* y;
  const float* gate;
  float* dgate;
  float* dbias;
  void* dy;
};

void ln_bwd_gate(Ctx& c, const void* dxmod, const float* x, const float* mean, const float* rstd, const float* scale,
                 int rows_per_group, float* g, int accumulate, float* dshift, float* dscale, i64 M, int d,
                 const GateNext* gn) {
  const int NA = c.m->NA;
  c.ck(mdt::ln_modulate_bwd_gate_s(dxmod, x, mean, rstd, scale, NA, rows_per_group, g, accumulate, dshift, dscale, NA,
                                   gn ? gn->y : nullptr, gn ? gn->gate : nullptr, gn ? NA : 0, gn ? gn->dy : nullptr,
                                   gn ? gn->dgate : nullptr, gn ? NA : 0, gn ? gn->dbias : nullptr,
                                   static_cast<int>(M), d, c.scratch, static_cast<cudaStream_t>(c.stream)));
}

GateNext mlp_gate(Ctx& c, const BlockP& s, const BlockBuf& b, const float* mod, float* dmod, void* dy) {
  const i64 o = s.mod_off + 5 * s.dim;
  return GateNext{c.at<void>(b.y2), mod + o, dmod + o, c.Gd(s.fc2_b), dy};
}

struct Refwd {  // a recomputed block: its forward is re-run into the recompute slot from its stored input X
  const BlockP* s;
  const BlockBuf* b;
  float* X;
  int T;
};

void refwd(Ctx& c, const Refwd* r, const float* mod, int B) {
  if (r) block_fwd(c, *r->s, *r->b, r->X, mod, B, r->T, true);
}

// Backward of one DiTBlock.  Gr [M, d] f32 = residual-stream gradient, updated in place; dy2 = gradient of this
// block's MLP-branch output (produced by the caller's LN backward).  `next` = the MLP gate of the block processed
// next (fused into this block's last LN backward, which writes its dy into next->dy).  `pre`: the block processed next
// when it is recomputed; its forward is re-run just before that last LN backward, which reads its y2.
void block_bwd(Ctx& c, const Plan& p, const BlockP& s, const BlockBuf& b, const float* X, float* Gr, const float* mod,
               float* dmod, int B, int T, const void* dy2, const GateNext* next, const Refwd* pre) {
  const int d = s.dim, h4 = s.h4;
  const i64 M = static_cast<i64>(B) * T, o = s.mod_off;
  void* st = c.stream;
  __nv_bfloat16* dh = c.at<__nv_bfloat16>(p.dh);
  // (the fc1 bias gradient = column sums of dh is accumulated by the epilogue that writes dh: no separate pass)
  Gemm(dy2, c.W16(s.fc2_w), M, h4, d, false, true).out16(dh).epi(MDT_EPI_DGELU).aux(c.at<void>(b.hpre), h4)
      .colsum(c.Gd(s.fc1_b)).run(c);
  wgrad(c, dy2, c.at<void>(b.a), d, h4, M, c.Gd(s.fc2_w));
  __nv_bfloat16* dxm = c.at<__nv_bfloat16>(p.dxm);
  Gemm(dh, c.W16(s.fc1_w), M, d, h4, false, true).out16(dxm).run(c);
  wgrad(c, dh, c.at<void>(b.xm2), h4, d, M, c.Gd(s.fc1_w));
  // x1 = x + gate_msa * proj(attn(qkv(xm1))): its gate backward rides on the LN2 backward
  void* dy1 = c.at<void>(p.dyB);
  GateNext g1{c.at<void>(b.y1), mod + o + 2 * d, dmod + o + 2 * d, c.Gd(s.proj_b), dy1};
  ln_bwd_gate(c, dxm, c.at<float>(b.X1), c.at<float>(b.mean2), c.at<float>(b.rstd2), mod + o + 4 * d, T, Gr, 1,
              dmod + o + 3 * d, dmod + o + 4 * d, M, d, &g1);
  __nv_bfloat16* dO = c.at<__nv_bfloat16>(p.dO);
  Gemm(dy1, c.W16(s.proj_w), M, d, d, false, true).out16(dO).run(c);
  wgrad(c, dy1, c.at<void>(b.O), d, d, M, c.Gd(s.proj_w));
  __nv_bfloat16* dqkv = c.at<__nv_bfloat16>(p.dqkv);
  c.ck(mdt_attention_bwd(c.at<void>(b.qkv), c.at<void>(b.O), dO, c.at<float>(b.lse), dqkv, B, T, s.heads, s.dh, st));
  c.ck(mdt_colsum_bf16(dqkv, static_cast<int>(M), 3 * d, 3 * d, c.Gd(s.qkv_b), st));
  Gemm(dqkv, c.W16(s.qkv_w), M, d, 3 * d, false, true).out16(dxm).run(c);
  wgrad(c, dqkv, c.at<void>(b.xm1), 3 * d, d, M, c.Gd(s.qkv_w));
  refwd(c, pre, mod, B);
  ln_bwd_gate(c, dxm, X, c.at<float>(b.mean1), c.at<float>(b.rstd1), mod + o + d, T, Gr, 1, dmod + o, dmod + o + d, M,
              d, next);
}

}  // namespace

extern "C" {

int mdt_model_create(const mdt_model_cfg* cfg, mdt_model** out) {
  if (!cfg || !out) return MDT_ERR_ARG;
  if (cfg->hidden <= 0 || cfg->depth < 0 || cfg->heads <= 0 || cfg->hidden % cfg->heads || cfg->patch_size <= 0 ||
      cfg->img_resolution % cfg->patch_size || cfg->img_channels <= 0 || cfg->num_classes < 0 || cfg->mlp_hidden <= 0)
    return MDT_ERR_ARG;
  // no decoder: every dec_* field 0 and no mask token; otherwise a complete decoder description
  const bool no_dec = cfg->dec_hidden == 0 && cfg->dec_depth == 0 && cfg->dec_heads == 0 && cfg->dec_mlp_hidden == 0;
  if (no_dec ? cfg->has_mask_token != 0
             : (cfg->dec_hidden <= 0 || cfg->dec_depth < 0 || cfg->dec_heads <= 0 || cfg->dec_hidden % cfg->dec_heads ||
                cfg->dec_mlp_hidden <= 0))
    return MDT_ERR_ARG;
  mdt_model* m = new mdt_model();
  m->cfg = *cfg;
  build_layout(m);
  *out = m;
  return MDT_OK;
}

void mdt_model_destroy(mdt_model* m) { delete m; }

long long mdt_model_param_count(const mdt_model* m, int trainable_only) {
  return !m ? -1 : (trainable_only ? m->n_train : m->n_total);
}

int mdt_model_num_tensors(const mdt_model* m) { return m ? static_cast<int>(m->named.size()) : -1; }

int mdt_model_param_info(const mdt_model* m, int i, char* name, int name_cap, long long* offset, long long* numel) {
  if (!m || i < 0 || i >= static_cast<int>(m->order.size())) return MDT_ERR_ARG;
  const NamedTensor& t = m->named[m->order[i]];
  if (name && name_cap > 0) {
    strncpy(name, t.name.c_str(), name_cap - 1);
    name[name_cap - 1] = 0;
  }
  if (offset) *offset = t.t->off;
  if (numel) *numel = t.numel;
  return MDT_OK;
}

int mdt_model_mod_width(const mdt_model* m) { return m ? m->NA : -1; }

int mdt_model_fp32_read_ranges(const mdt_model* m, long long* lohi, int cap) {
  if (!m || cap < 0 || (cap > 0 && !lohi)) return MDT_ERR_ARG;
  // every W32() / w32 + offset read of mdt_forward and mdt_backward, and the loss kernels' logvar w
  std::vector<const Tensor*> ts = {&m->xw, &m->xb, &m->t0b, &m->t2b, &m->flb};
  for (auto* blocks : {&m->enc, &m->dec})
    for (const BlockP& b : *blocks) ts.insert(ts.end(), {&b.qkv_b, &b.proj_b, &b.fc1_b, &b.fc2_b});
  if (m->has_dec) ts.push_back(&m->dlb);
  if (m->cfg.has_mask_token) ts.push_back(&m->mask_token);
  if (m->logvar_channels > 0) ts.push_back(&m->lv_w);
  std::vector<std::pair<i64, i64>> r;
  for (const Tensor* t : ts) r.emplace_back(t->off, t->off + round_up(t->numel));
  r.emplace_back(m->ada_b_off, m->ada_b_off + round_up(m->ada_b.back().off + m->ada_b.back().numel - m->ada_b_off));
  std::sort(r.begin(), r.end());
  std::vector<std::pair<i64, i64>> merged;
  for (const auto& x : r) {
    if (!merged.empty() && x.first <= merged.back().second)
      merged.back().second = std::max(merged.back().second, x.second);
    else
      merged.push_back(x);
  }
  for (size_t i = 0; i < merged.size() && static_cast<int>(i) < cap; ++i)
    lohi[2 * i] = merged[i].first, lohi[2 * i + 1] = merged[i].second;
  return static_cast<int>(merged.size());
}

int mdt_model_set_recompute(mdt_model* m, int r) {
  if (!m || r < 0 || r > static_cast<int>(m->enc.size() + m->dec.size())) return MDT_ERR_ARG;
  m->recompute = r;
  return MDT_OK;
}

int mdt_model_get_recompute(const mdt_model* m) { return m ? m->recompute : -1; }

int mdt_model_set_logvar(mdt_model* m, int channels) {
  if (!m || channels < 0 || channels > 256 || m->planned) return MDT_ERR_ARG;
  m->logvar_channels = channels;
  m->named.clear();
  m->order.clear();
  build_layout(m);
  return MDT_OK;
}

int mdt_model_set_precond(mdt_model* m, int kind) {
  if (!m || (kind != MDT_PRECOND_EDM && kind != MDT_PRECOND_FLOW)) return MDT_ERR_ARG;
  m->precond = kind;
  return MDT_OK;
}

long long mdt_workspace_bytes(const mdt_model* m, int B, int T, int training) {
  if (!m || B <= 0) return -1;
  if (T <= 0) T = m->L;
  m->planned = true;
  return make_plan(m, B, T, training != 0, training != 0).total;
}

int mdt_forward(const mdt_model* m, const float* w32, const void* w16, const float* x_in, const float* sigma,
                const float* labels, const int64_t* ids_keep, const int64_t* ids_restore, int B, int T, int save,
                void* workspace, long long workspace_bytes, float* F_out, void* stream) {
  if (!m || !w32 || !w16 || !x_in || !sigma || !workspace || !F_out || B <= 0) return MDT_ERR_ARG;
  if (T <= 0) T = m->L;
  if ((ids_keep == nullptr) != (ids_restore == nullptr) || (!ids_keep && T != m->L)) return MDT_ERR_ARG;
  if (m->cfg.num_classes > 0 && !labels) return MDT_ERR_ARG;
  m->planned = true;
  const Plan p = make_plan(m, B, T, save != 0, save != 0);
  if (p.total > workspace_bytes || (reinterpret_cast<uintptr_t>(workspace) & 255)) return MDT_ERR_ARG;
  if (save) m->fwd_ws = workspace, m->fwd_r = m->recompute;
  Ctx c{m, w32, static_cast<const __nv_bfloat16*>(w16), nullptr, static_cast<char*>(workspace), stream};
  const mdt_model_cfg& cf = m->cfg;
  const int D = m->D, Dd = m->Dd, L = m->L, NA = m->NA, nc = cf.num_classes;
  const i64 Me = static_cast<i64>(B) * T, Md = static_cast<i64>(B) * L;
  cudaStream_t cs = static_cast<cudaStream_t>(stream);

  float* X = c.at<float>(p.X0);
  // flow: sigma holds t, the input is not scaled (a NULL sigma is c_in = 1) and c_noise = t
  const bool flow = m->precond == MDT_PRECOND_FLOW;
  c.ck(mdt_patch_embed(x_in, flow ? nullptr : sigma, cf.sigma_data, c.W32(m->xw), c.W32(m->xb), c.W32(m->pos),
                       ids_keep, X, B, cf.img_channels, cf.img_resolution, cf.patch_size, D, T, stream));
  // conditioning: c = t_emb(c_noise) + y_emb(labels)   (models/maskdit.py:491-495, :767)
  c.ck(flow ? mdt_flow_timestep_freq(sigma, B, 256, c.at<void>(p.tf), stream)
            : mdt_timestep_freq(sigma, B, 256, c.at<void>(p.tf), stream));
  float* th_pre = c.at<float>(p.th_pre);
  Gemm(c.at<void>(p.tf), c.W16(m->t0w), B, D, 256).out32(th_pre).bias(c.W32(m->t0b)).run(c);
  c.ck(mdt_silu(th_pre, nullptr, nullptr, c.at<void>(p.th), static_cast<i64>(B) * D, stream));
  float* cc = c.at<float>(p.c);
  Gemm(c.at<void>(p.th), c.W16(m->t2w), B, D, D).out32(cc).bias(c.W32(m->t2b)).run(c);
  if (nc > 0) {
    c.ck(mdt_cast_f32_bf16(labels, c.at<void>(p.y16), static_cast<i64>(B) * nc, stream));
    const void* y16 = c.at<void>(p.y16);
    const void* Wy = c.W16(m->ytab);
    int Kp = nc;
    if (nc % 8) {  // toy class counts only (the registry configs use 1000): zero-pad K to a multiple of 8 for TMA strides
      Kp = m->Kp;
      if (cudaMemsetAsync(c.at<void>(p.y16p), 0, static_cast<size_t>(B) * Kp * 2, cs) != cudaSuccess ||
          cudaMemsetAsync(c.at<void>(p.wyp), 0, static_cast<size_t>(D) * Kp * 2, cs) != cudaSuccess ||
          cudaMemcpy2DAsync(c.at<void>(p.y16p), Kp * 2, y16, nc * 2, nc * 2, B, cudaMemcpyDeviceToDevice, cs) !=
              cudaSuccess ||
          cudaMemcpy2DAsync(c.at<void>(p.wyp), Kp * 2, Wy, nc * 2, nc * 2, D, cudaMemcpyDeviceToDevice, cs) !=
              cudaSuccess)
        return MDT_ERR_CUDA;
      y16 = c.at<void>(p.y16p), Wy = c.at<void>(p.wyp);
    }
    float* c2 = c.at<float>(p.c2);
    Gemm(y16, Wy, B, D, Kp).out32(c2).resid(cc, D).run(c);
    cc = c2;
  }
  c.ck(mdt_silu(cc, nullptr, nullptr, c.at<void>(p.sc), static_cast<i64>(B) * D, stream));
  float* mod = c.at<float>(p.mod);
  Gemm(c.at<void>(p.sc), c.w16 + m->ada_w_off, B, NA, D).out32(mod).bias(c.w32 + m->ada_b_off).run(c);

  for (size_t i = 0; i < m->enc.size(); ++i) X = block_fwd(c, m->enc[i], p.enc[i], X, mod, B, T, save != 0);

  i64 o = m->off_final;
  if (!m->has_dec) {
    // FinalLayer on the encoder's tokens (models/maskdit.py:550); training with a mask scatters the kept rows back and
    // fills the removed ones with zeros (:551-553)
    c.ck(mdt_ln_modulate(X, mod + o, mod + o + D, NA, T, c.at<void>(p.xf), save ? c.at<float>(p.mean_f) : nullptr,
                         save ? c.at<float>(p.rstd_f) : nullptr, static_cast<int>(Me), D, 1e-6f, stream));
    float* Fk = ids_restore ? c.at<float>(p.fk) : F_out;
    Gemm(c.at<void>(p.xf), c.W16(m->flw), Me, m->pd, D).out32(Fk).bias(c.W32(m->flb)).run(c);
    if (ids_restore) c.ck(mdt_unmask_tokens(Fk, nullptr, nullptr, ids_restore, F_out, B, T, L, m->pd, stream));
    return c.rc;
  }

  // DecoderLayer (models/maskdit.py:209-213) + unmask_tokens + decoder_pos_embed (:539-545)
  o = m->off_declayer;
  c.ck(mdt_ln_modulate(X, mod + o, mod + o + D, NA, T, c.at<void>(p.xmd), save ? c.at<float>(p.mean_d) : nullptr,
                       save ? c.at<float>(p.rstd_d) : nullptr, static_cast<int>(Me), D, 1e-6f, stream));
  float* u = c.at<float>(p.u);
  Gemm(c.at<void>(p.xmd), c.W16(m->dlw), Me, Dd, D).out32(u).bias(c.W32(m->dlb)).run(c);
  float* Z = c.at<float>(p.Z);
  c.ck(mdt_unmask_tokens(u, cf.has_mask_token ? c.W32(m->mask_token) : nullptr, c.W32(m->dpos), ids_restore, Z, B, T, L,
                         Dd, stream));
  for (size_t i = 0; i < m->dec.size(); ++i) Z = block_fwd(c, m->dec[i], p.dec[i], Z, mod, B, L, save != 0);
  // FinalLayer (models/maskdit.py:230-234)
  o = m->off_final;
  c.ck(mdt_ln_modulate(Z, mod + o, mod + o + Dd, NA, L, c.at<void>(p.xf), save ? c.at<float>(p.mean_f) : nullptr,
                       save ? c.at<float>(p.rstd_f) : nullptr, static_cast<int>(Md), Dd, 1e-6f, stream));
  Gemm(c.at<void>(p.xf), c.W16(m->flw), Md, m->pd, Dd).out32(F_out).bias(c.W32(m->flb)).run(c);
  return c.rc;
}

int mdt_backward(const mdt_model* m, const float* w32, const void* w16, float* grad, const float* x_in,
                 const float* sigma, const int64_t* ids_keep, const int64_t* ids_restore, const void* dF_bf16, int B,
                 int T, void* workspace, long long workspace_bytes, mdt_grad_ready_fn on_ready, void* user,
                 void* stream) {
  if (!m || !w32 || !w16 || !grad || !x_in || !sigma || !dF_bf16 || !workspace || B <= 0) return MDT_ERR_ARG;
  if (T <= 0) T = m->L;
  if ((ids_keep == nullptr) != (ids_restore == nullptr) || (!ids_keep && T != m->L)) return MDT_ERR_ARG;
  const Plan p = make_plan(m, B, T, true, true);
  if (p.total > workspace_bytes || (reinterpret_cast<uintptr_t>(workspace) & 255)) return MDT_ERR_ARG;
  // the workspace must be laid out for this recompute count: at r > 0 it is the last saving forward's, at r = 0 it is
  // not the last saving forward's if that one recomputed
  const int r = m->recompute;
  if (r ? (m->fwd_ws != workspace || m->fwd_r != r) : (m->fwd_ws == workspace && m->fwd_r != 0)) return MDT_ERR_ARG;
  Ctx c{m, w32, static_cast<const __nv_bfloat16*>(w16), grad, static_cast<char*>(workspace), stream};
  c.scratch = c.at<float>(p.det);
  const mdt_model_cfg& cf = m->cfg;
  const int D = m->D, Dd = m->Dd, L = m->L, NA = m->NA, nc = cf.num_classes, pd = m->pd;
  const i64 Me = static_cast<i64>(B) * T, Md = static_cast<i64>(B) * L;
  cudaStream_t cs = static_cast<cudaStream_t>(stream);
  const float* mod = c.at<float>(p.mod);
  float* dmod = c.at<float>(p.dmod);
  if (cudaMemsetAsync(dmod, 0, static_cast<size_t>(B) * NA * 4, cs) != cudaSuccess) return MDT_ERR_CUDA;

  const int ne = static_cast<int>(m->enc.size());
  void* dyA = c.at<void>(p.dyA);
  // Recomputation (r > 0).  The LN backward that ends block i's backward (or the final / decoder layer's) also runs the
  // MLP-gate backward of block i-1 (the block processed next), which reads block i-1's y2.  So a recomputed block's
  // forward is re-run into the slot right before that LN backward; only block i's mean1 / rstd1 are still read after
  // the re-run, and consecutive recomputed blocks keep those in different copies (make_plan).
  Refwd rf;
  auto recomputed = [&](bool dec, int i) -> const Refwd* {
    if ((dec ? ne + i : i) >= r) return nullptr;
    const std::vector<BlockBuf>& bufs = dec ? p.dec : p.enc;
    rf = Refwd{dec ? &m->dec[i] : &m->enc[i], &bufs[i],
               c.at<float>(i > 0 ? bufs[i - 1].X2 : (dec ? p.Z : p.X0)), dec ? L : T};
    return &rf;
  };
  // the LN backward that starts the encoder's residual-stream gradient: of the decoder layer, or of the final layer
  // when there is no decoder (its adaLN offset, input gradient and saved statistics)
  i64 o = m->off_final;
  const void* dx_top = c.at<void>(p.dxf);
  const float *mean_top = c.at<float>(p.mean_f), *rstd_top = c.at<float>(p.rstd_f);
  if (!m->has_dec) {
    // ---- final layer on the kept tokens: the rows of removed tokens are constant zeros in the forward
    // (models/maskdit.py:551-553), so their dF (the MAE term's gradient seed) is dropped
    const void* dFk = dF_bf16;
    if (ids_keep) {
      c.ck(mdt_gather_rows_bf16(dF_bf16, ids_keep, c.at<void>(p.fk), B, T, L, pd, stream));
      dFk = c.at<void>(p.fk);
    }
    wgrad(c, dFk, c.at<void>(p.xf), pd, D, Me, c.Gd(m->flw));
    c.ck(mdt_colsum_bf16(dFk, static_cast<int>(Me), pd, pd, c.Gd(m->flb), stream));
    Gemm(dFk, c.W16(m->flw), Me, D, pd, false, true).out16(c.at<void>(p.dxf)).run(c);
  } else {
    // ---- final layer
    const int nd = static_cast<int>(m->dec.size());
    const float* Z_out = nd ? c.at<float>(p.dec[nd - 1].X2) : c.at<float>(p.Z);
    wgrad(c, dF_bf16, c.at<void>(p.xf), pd, Dd, Md, c.Gd(m->flw));
    c.ck(mdt_colsum_bf16(dF_bf16, static_cast<int>(Md), pd, pd, c.Gd(m->flb), stream));
    Gemm(dF_bf16, c.W16(m->flw), Md, Dd, pd, false, true).out16(c.at<void>(p.dxf)).run(c);
    float* Gz = c.at<float>(p.Gz);
    // every LN backward finishes the residual-stream gradient that the NEXT gate backward consumes: one fused pass
    {
      GateNext gn;
      if (nd) gn = mlp_gate(c, m->dec[nd - 1], p.dec[nd - 1], mod, dmod, dyA), refwd(c, recomputed(true, nd - 1), mod, B);
      ln_bwd_gate(c, c.at<void>(p.dxf), Z_out, c.at<float>(p.mean_f), c.at<float>(p.rstd_f), mod + o + Dd, L, Gz, 0,
                  dmod + o, dmod + o + Dd, Md, Dd, nd ? &gn : nullptr);
    }
    // ---- decoder blocks (last to first)
    for (int i = nd - 1; i >= 0; --i) {
      const float* Xin = i > 0 ? c.at<float>(p.dec[i - 1].X2) : c.at<float>(p.Z);
      GateNext gn;
      if (i > 0) gn = mlp_gate(c, m->dec[i - 1], p.dec[i - 1], mod, dmod, dyA);
      block_bwd(c, p, m->dec[i], p.dec[i], Xin, Gz, mod, dmod, B, L, dyA, i > 0 ? &gn : nullptr,
                i > 0 ? recomputed(true, i - 1) : nullptr);
      if (on_ready && c.rc == MDT_OK) on_ready(user, m->dec[i].lo, m->dec[i].hi);
    }
    // ---- unmask + decoder layer
    float* tok_g = (cf.has_mask_token && ids_restore) ? c.Gd(m->mask_token) : nullptr;
    c.ck(mdt::unmask_tokens_bwd_s(Gz, ids_restore, c.at<void>(p.du), tok_g, B, T, L, Dd, c.scratch, cs));
    o = m->off_declayer;
    wgrad(c, c.at<void>(p.du), c.at<void>(p.xmd), Dd, D, Me, c.Gd(m->dlw));
    c.ck(mdt_colsum_bf16(c.at<void>(p.du), static_cast<int>(Me), Dd, Dd, c.Gd(m->dlb), stream));
    Gemm(c.at<void>(p.du), c.W16(m->dlw), Me, D, Dd, false, true).out16(c.at<void>(p.dxmd)).run(c);
    dx_top = c.at<void>(p.dxmd), mean_top = c.at<float>(p.mean_d), rstd_top = c.at<float>(p.rstd_d);
  }
  float* Ge = c.at<float>(p.Ge);
  const float* X_enc = ne ? c.at<float>(p.enc[ne - 1].X2) : c.at<float>(p.X0);
  {
    GateNext gn;
    if (ne) gn = mlp_gate(c, m->enc[ne - 1], p.enc[ne - 1], mod, dmod, dyA), refwd(c, recomputed(false, ne - 1), mod, B);
    ln_bwd_gate(c, dx_top, X_enc, mean_top, rstd_top, mod + o + D, T, Ge, 0, dmod + o, dmod + o + D, Me, D,
                ne ? &gn : nullptr);
  }
  // ---- encoder blocks
  for (int i = ne - 1; i >= 0; --i) {
    const float* Xin = i > 0 ? c.at<float>(p.enc[i - 1].X2) : c.at<float>(p.X0);
    GateNext gn;
    if (i > 0) gn = mlp_gate(c, m->enc[i - 1], p.enc[i - 1], mod, dmod, dyA);
    block_bwd(c, p, m->enc[i], p.enc[i], Xin, Ge, mod, dmod, B, T, dyA, i > 0 ? &gn : nullptr,
              i > 0 ? recomputed(false, i - 1) : nullptr);
    if (on_ready && c.rc == MDT_OK) on_ready(user, m->enc[i].lo, m->enc[i].hi);
  }
  // ---- patch embedding (no input gradient needed)
  c.ck(mdt::patch_embed_bwd_s(x_in, m->precond == MDT_PRECOND_FLOW ? nullptr : sigma, cf.sigma_data, ids_keep, Ge, c.Gd(m->xw), c.Gd(m->xb), B, cf.img_channels,
                              cf.img_resolution, cf.patch_size, D, T, c.scratch, cs));
  // ---- adaLN projections of all blocks at once, then the conditioning MLPs
  void* dmod16 = c.at<void>(p.dmod16);
  c.ck(mdt_cast_f32_bf16(dmod, dmod16, static_cast<i64>(B) * NA, stream));
  wgrad(c, dmod16, c.at<void>(p.sc), NA, D, B, grad + m->ada_w_off);
  c.ck(mdt_colsum_f32(dmod, B, NA, NA, grad + m->ada_b_off, stream));
  float* dsc = c.at<float>(p.dsc);
  if (cudaMemsetAsync(dsc, 0, static_cast<size_t>(B) * D * 4, cs) != cudaSuccess) return MDT_ERR_CUDA;
  Gemm(dmod16, c.w16 + m->ada_w_off, B, D, NA, false, true).out32(dsc).epi(MDT_EPI_ATOMIC).run(c);  // long K: stream-K
  const float* cc = nc > 0 ? c.at<float>(p.c2) : c.at<float>(p.c);
  c.ck(mdt_silu_bwd(dsc, cc, c.at<float>(p.dc32), c.at<void>(p.dc16), static_cast<i64>(B) * D, stream));
  if (nc > 0) {
    if (nc % 8 == 0) {
      wgrad(c, c.at<void>(p.dc16), c.at<void>(p.y16), D, nc, B, c.Gd(m->ytab));
    } else {
      const int Kp = m->Kp;
      float* tmp = c.at<float>(p.ytmp);
      if (cudaMemsetAsync(tmp, 0, static_cast<size_t>(D) * Kp * 4, cs) != cudaSuccess) return MDT_ERR_CUDA;
      wgrad(c, c.at<void>(p.dc16), c.at<void>(p.y16p), D, Kp, B, tmp);
      const i64 n = static_cast<i64>(D) * nc;
      add_strided_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, cs>>>(c.Gd(m->ytab), nc, tmp, Kp, D, nc);
    }
  }
  wgrad(c, c.at<void>(p.dc16), c.at<void>(p.th), D, D, B, c.Gd(m->t2w));
  c.ck(mdt_colsum_f32(c.at<float>(p.dc32), B, D, D, c.Gd(m->t2b), stream));
  float* dth = c.at<float>(p.dth);
  if (cudaMemsetAsync(dth, 0, static_cast<size_t>(B) * D * 4, cs) != cudaSuccess) return MDT_ERR_CUDA;
  Gemm(c.at<void>(p.dc16), c.W16(m->t2w), B, D, D, false, true).out32(dth).epi(MDT_EPI_ATOMIC).run(c);
  c.ck(mdt_silu_bwd(dth, c.at<float>(p.th_pre), c.at<float>(p.dpre32), c.at<void>(p.dpre16), static_cast<i64>(B) * D,
                    stream));
  wgrad(c, c.at<void>(p.dpre16), c.at<void>(p.tf), D, 256, B, c.Gd(m->t0w));
  c.ck(mdt_colsum_f32(c.at<float>(p.dpre32), B, D, D, c.Gd(m->t0b), stream));
  if (c.rc == MDT_OK && cudaGetLastError() != cudaSuccess) return MDT_ERR_CUDA;
  return c.rc;
}

// ---- data-parallel gradient exchange (train.py:178 DDP; SURVEY 8e: ONE sum-all-reduce of the flat gradient buffer) --
// NCCL is resolved at run time from the libnccl the process already has (PyTorch bundles it): no link-time dependency,
// and the library still loads on a box without NCCL (these entry points then return MDT_ERR_DRIVER).
namespace {
typedef struct { char internal[128]; } NcclUid;
// ncclConfig_t as of NCCL 2.28 (nccl.h: ncclConfig_v22800); older libraries read only the prefix they know (`size`).
struct NcclConfig {
  size_t size;
  unsigned int magic, version;
  int blocking, cgaClusterSize, minCTAs, maxCTAs;
  const char* netName;
  int splitShare, trafficClass;
  const char* commName;
  int collnetEnable, CTAPolicy, shrinkShare, nvlsCTAs, nChannelsPerNetPeer, nvlinkCentricSched;
};
struct NcclApi {
  int (*GetUniqueId)(NcclUid*) = nullptr;
  int (*CommInitRank)(void**, int, NcclUid, int) = nullptr;
  int (*CommInitRankConfig)(void**, int, NcclUid, int, NcclConfig*) = nullptr;
  int (*GetVersion)(int*) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  // the sharded optimizer's halves of the all-reduce (optional: only mdt_reduce_scatter_grads / mdt_allgather need them)
  int (*ReduceScatter)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommUserRank)(void*, int*) = nullptr;
  bool ok = false;
};
NcclApi& nccl() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* h = dlopen("libnccl.so.2", RTLD_LAZY | RTLD_NOLOAD);
    if (!h) h = dlopen("libnccl.so.2", RTLD_LAZY);
    if (!h) h = dlopen("libnccl.so", RTLD_LAZY);
    if (h) {
      api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
      api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
      api.CommInitRankConfig =
          reinterpret_cast<decltype(api.CommInitRankConfig)>(dlsym(h, "ncclCommInitRankConfig"));
      api.GetVersion = reinterpret_cast<decltype(api.GetVersion)>(dlsym(h, "ncclGetVersion"));
      api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
      api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(dlsym(h, "ncclAllReduce"));
      api.ReduceScatter = reinterpret_cast<decltype(api.ReduceScatter)>(dlsym(h, "ncclReduceScatter"));
      api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(h, "ncclAllGather"));
      api.CommUserRank = reinterpret_cast<decltype(api.CommUserRank)>(dlsym(h, "ncclCommUserRank"));
      api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllReduce;
    }
  }
  return api;
}
}  // namespace

int mdt_nccl_unique_id(void* id128) {
  if (!id128) return MDT_ERR_ARG;
  if (!nccl().ok) return MDT_ERR_DRIVER;
  NcclUid u;
  if (nccl().GetUniqueId(&u) != 0) return MDT_ERR_CUDA;
  memcpy(id128, &u, sizeof(u));
  return MDT_OK;
}

int mdt_nccl_comm_create(const void* id128, int rank, int world, int max_ctas, void** comm) {
  if (!id128 || !comm || rank < 0 || world <= 0 || rank >= world || max_ctas < 0) return MDT_ERR_ARG;
  if (!nccl().ok) return MDT_ERR_DRIVER;
  NcclUid u;
  memcpy(&u, id128, sizeof(u));
  if (max_ctas > 0 && nccl().CommInitRankConfig && nccl().GetVersion) {
    // a communicator confined to `max_ctas` CTAs: it runs NEXT TO the backward's persistent GEMMs (mdt_set_sm_budget)
    int ver = 0;
    nccl().GetVersion(&ver);
    NcclConfig cfg;
    const int undef = static_cast<int>(0x80000000);  // NCCL_CONFIG_UNDEF_INT
    cfg.size = sizeof(cfg), cfg.magic = 0xcafebeef, cfg.version = static_cast<unsigned>(ver);
    cfg.blocking = undef, cfg.cgaClusterSize = undef, cfg.minCTAs = undef, cfg.maxCTAs = max_ctas;
    cfg.netName = nullptr, cfg.splitShare = undef, cfg.trafficClass = undef, cfg.commName = nullptr;
    cfg.collnetEnable = undef, cfg.CTAPolicy = undef, cfg.shrinkShare = undef, cfg.nvlsCTAs = undef;
    cfg.nChannelsPerNetPeer = undef, cfg.nvlinkCentricSched = undef;
    return nccl().CommInitRankConfig(comm, world, u, rank, &cfg) == 0 ? MDT_OK : MDT_ERR_CUDA;
  }
  return nccl().CommInitRank(comm, world, u, rank) == 0 ? MDT_OK : MDT_ERR_CUDA;
}

int mdt_nccl_comm_destroy(void* comm) {
  if (!comm) return MDT_ERR_ARG;
  if (!nccl().ok) return MDT_ERR_DRIVER;
  return nccl().CommDestroy(comm) == 0 ? MDT_OK : MDT_ERR_CUDA;
}

int mdt_allreduce_grads(void* comm, void* grad, long long n, int bf16, void* stream) {
  if (!comm || !grad || n <= 0) return MDT_ERR_ARG;
  if (!nccl().ok) return MDT_ERR_DRIVER;
  // ncclDataType_t: ncclFloat32 = 7, ncclBfloat16 = 9 ; ncclRedOp_t: ncclSum = 0
  return nccl().AllReduce(grad, grad, static_cast<size_t>(n), bf16 ? 9 : 7, 0, comm, static_cast<cudaStream_t>(stream)) == 0
             ? MDT_OK
             : MDT_ERR_CUDA;
}

int mdt_reduce_scatter_grads(void* comm, void* buf, long long count_per_rank, int bf16, void* stream) {
  if (!comm || !buf || count_per_rank <= 0) return MDT_ERR_ARG;
  if (!nccl().ok || !nccl().ReduceScatter || !nccl().CommUserRank) return MDT_ERR_DRIVER;
  int rank = 0;
  if (nccl().CommUserRank(comm, &rank) != 0) return MDT_ERR_CUDA;
  const size_t esz = bf16 ? 2 : 4;
  char* recv = static_cast<char*>(buf) + static_cast<size_t>(rank) * static_cast<size_t>(count_per_rank) * esz;
  return nccl().ReduceScatter(buf, recv, static_cast<size_t>(count_per_rank), bf16 ? 9 : 7, 0, comm,
                              static_cast<cudaStream_t>(stream)) == 0
             ? MDT_OK
             : MDT_ERR_CUDA;
}

int mdt_allgather(void* comm, void* buf, long long count_per_rank, int dtype, void* stream) {
  if (!comm || !buf || count_per_rank <= 0) return MDT_ERR_ARG;
  // ncclDataType_t: ncclFloat32 = 7, ncclFloat64 = 8, ncclBfloat16 = 9
  int nd = 0;
  size_t esz = 0;
  switch (dtype) {
    case MDT_DTYPE_F32: nd = 7, esz = 4; break;
    case MDT_DTYPE_BF16: nd = 9, esz = 2; break;
    case MDT_DTYPE_F64: nd = 8, esz = 8; break;
    default: return MDT_ERR_ARG;
  }
  if (!nccl().ok || !nccl().AllGather || !nccl().CommUserRank) return MDT_ERR_DRIVER;
  int rank = 0;
  if (nccl().CommUserRank(comm, &rank) != 0) return MDT_ERR_CUDA;
  const char* send = static_cast<char*>(buf) + static_cast<size_t>(rank) * static_cast<size_t>(count_per_rank) * esz;
  return nccl().AllGather(send, buf, static_cast<size_t>(count_per_rank), nd, comm, static_cast<cudaStream_t>(stream)) == 0
             ? MDT_OK
             : MDT_ERR_CUDA;
}

}  // extern "C"
