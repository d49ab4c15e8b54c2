// Host-side sequencing of the matcher forward + the C ABI (include/mvm_b200.h).
// Mirrors MultiViewMatcher.multi_match in eval mode (multi_view_matcher.py:217-320) on
// point-major activations: kenc -> L x {qkv, attention, merge, mlp} -> final_proj ->
// per pair {score GEMM, Sinkhorn, mutual NN, confidence head}.  Every launch is
// stream-ordered; no host sync, no allocation: the whole call is CUDA-graph capturable.
#include "../../include/mvm_b200.h"
#include "common.cuh"
#include "kernels.cuh"
#include <cuda_fp16.h>

namespace {

struct Workspace {
  float *DT, *H3, *H4, *X, *QKV, *VT, *KLO, *VTLO, *MSG, *MRG, *H, *MD;
  float* sink_ws;
  int* match_ws;
  float *FEAT, *SC, *CF1, *CF2, *CC0, *CC1;
  size_t total;
};

size_t align_up(size_t x) { return (x + 255) & ~size_t(255); }

Workspace carve(char* base, int batch, int n_views, int n_pad, int n_pairs, int has_conf) {
  Workspace w;
  size_t off = 0;
  const size_t rows = (size_t)batch * n_views * n_pad;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align_up(bytes);
    return p;
  };
  w.DT = (float*)take(rows * 256 * 4);
  w.H3 = (float*)take(rows * 128 * 4);
  w.H4 = (float*)take(rows * 256 * 4);
  w.X = (float*)take(rows * 256 * 4);
  w.QKV = (float*)take(rows * 768 * 4);
  w.VT = (float*)take(rows * 256 * 4);
  w.KLO = (float*)take(rows * 256 * 4);
  w.VTLO = (float*)take(rows * 256 * 4);
  w.MSG = (float*)take(rows * 256 * 4);
  w.MRG = (float*)take(rows * 256 * 4);
  w.H = (float*)take(rows * 512 * 4);
  w.MD = (float*)take(rows * 256 * 4);
  const size_t probs = (size_t)n_pairs * batch;
  w.sink_ws = (float*)take(sinkhorn_ws_floats(n_pairs, batch, n_pad) * 4);
  w.match_ws = (int*)take(probs * 3 * (size_t)n_pad * 4);
  const size_t crow = has_conf ? probs * n_pad : 0;
  w.FEAT = (float*)take(crow * 512 * 4);
  w.SC = (float*)take(crow * 4);
  w.CF1 = (float*)take(crow * 512 * 4);
  w.CF2 = (float*)take(crow * 256 * 4);
  w.CC0 = (float*)take(crow * 256 * 4);
  w.CC1 = (float*)take(crow * 256 * 4);
  w.total = off;
  return w;
}

GemmDesc make_gemm(const float* A, int lda, const float* W, int K, const float* bias, float* C,
                   int ldc, int M, int N, int relu) {
  GemmDesc g;
  g.A = A; g.lda = lda; g.A2 = nullptr; g.lda2 = 0; g.K1 = K;
  g.W = W; g.ldw = K; g.Whi = nullptr; g.Wlo = nullptr; g.Whi16 = nullptr; g.Wlo16 = nullptr; g.wscale = 0.f;
  g.bias = bias; g.R = nullptr; g.ldr = 0;
  g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K; g.alpha = 1.f; g.relu = relu;
  g.batch = 1; g.sA = g.sA2 = g.sW = g.sR = g.sC = 0;
  return g;
}

// PROCESS DEFAULTS of the per-call options (mvm_matcher_options).  They are read once, at the top of
// mvm_matcher_forward, to fill the options of that call; nothing below this point reads or writes a global,
// so two models / two streams / two threads may run forwards concurrently (each with its own workspace).
// math mode: 3 = 3xTF32 on the tensor cores (fp32-faithful, DEFAULT), 1 = single-pass TF32, 0 = fp32 CUDA cores
int g_math_mode = 3;
int g_score_tc = 1;                     // score GEMM on the tensor cores in mode 3 (mvm_debug_set_score_kernel)
int g_gemm_split = 1;                   // operand planes of the mode-3 GEMMs: 1 = fp16 hi/lo (default, needs the packed half planes), 0 = tf32
int g_attn_split = 1;                   // operand planes of the mode-3 attention: 1 = fp16 hi/lo (default), 0 = tf32 hi/lo

// everything a forward needs to know beyond its arguments, by value
struct Ctx {
  int math_mode, score_tc, gemm_tile, gemm_persist, sinkhorn_variant, attn_split;
  long long hi_off, lo_off;             // tf32 planes of the weights (mvm_matcher_weights)
  const float* flat_base;               // start of the flat fp32 weight buffer the half planes mirror element for element
  const __half* w16_hi; const __half* w16_lo; float w16_scale;   // fp16 planes of w16_scale * W (null: tf32x3 GEMMs)
};

// the W planes of a GEMM: tf32 (always, the one-tile kernels use them) and, when packed, the half-precision ones
void set_planes(const Ctx& cx, GemmDesc& g) {
  if (cx.math_mode == 3 && cx.lo_off != 0) {
    g.Whi = g.W + cx.hi_off; g.Wlo = g.W + cx.lo_off;
    if (cx.w16_hi) {
      const long long e = g.W - cx.flat_base;
      g.Whi16 = cx.w16_hi + e; g.Wlo16 = cx.w16_lo + e; g.wscale = cx.w16_scale;
    }
  }
}

int run_gemm(const Ctx& cx, const GemmDesc& g_in, cudaStream_t s) {
  GemmDesc g = g_in;
  set_planes(cx, g);
  if (cx.math_mode != 0 && g.batch == 1 && g.N % 128 == 0 && g.K % 32 == 0 && g.K1 % 32 == 0 && g.ldc % 4 == 0)
    return launch_gemm_tc(g, cx.math_mode, nullptr, 0, 0, s, nullptr, nullptr, cx.gemm_tile, cx.gemm_persist);
  return launch_gemm_simt(g, s);
}

// The QKV projection of a GNN layer, x [rows, 256] -> [rows, 768], with its W planes already in the descriptor (qkv_desc
// + the caller's planes).  K and V leave as the operand planes of the attention that follows: fp16 hi / lo planes (hp,
// the fp16x3 attention), or V^T [rows / n_pad, 256, n_pad] (VT) and, in 3xTF32, the tf32 remainders of K and V^T.
GemmDesc qkv_desc(const float* X, const float* W, const float* bias, float* qkv, int rows) {
  return make_gemm(X, 256, W, 256, bias, qkv, 768, rows, 768, 0);
}
int run_qkv(const GemmDesc& gq, int n_pass, int n_pad, const HalfPlanes* hp, float* VT, float* KLO, float* VTLO,
            int gemm_tile, int gemm_persist, cudaStream_t s) {
  if (hp) {
    MvmProfScope prof__(MVM_TAG_GEMM, s);      // (launch_gemm_tc opens the scope on the other path)
    return launch_gemm_tc_persist(gq, nullptr, 512, n_pad, nullptr, nullptr, s, hp);
  }
  return launch_gemm_tc(gq, n_pass, VT, 512, n_pad, s, KLO, VTLO, gemm_tile, gemm_persist);
}

#define MVM_TRY(x)            \
  do {                        \
    int rc__ = (x);           \
    if (rc__ != MVM_OK) return rc__; \
  } while (0)

int fill_pair_table(PairTable& tab, const mvm_pair_io* pairs, int n_pairs, int n_views,
                    const int* counts, int batch) {
  MVM_REQUIRE(n_pairs >= 1 && n_pairs <= MVM_MAX_PAIRS);
  tab.n_pairs = n_pairs;
  tab.n_views = n_views;
  long long off = 0;
  for (int p = 0; p < n_pairs; ++p) {
    const int a = pairs[p].view_a, b = pairs[p].view_b;
    MVM_REQUIRE(a >= 0 && b >= 0 && a < n_views && b < n_views && a != b);
    tab.a[p] = a; tab.b[p] = b;
    tab.m[p] = counts[a]; tab.n[p] = counts[b];
    tab.scores[p] = pairs[p].scores;
    tab.matches_a[p] = pairs[p].matches_a; tab.matches_b[p] = pairs[p].matches_b;
    tab.ms_a[p] = pairs[p].mscores_a; tab.ms_b[p] = pairs[p].mscores_b;
    tab.conf[p] = pairs[p].conf;
    tab.ws_off[p] = off;
    off += (long long)batch * (counts[a] + counts[b] + 2);
  }
  return MVM_OK;
}

}  // namespace

extern "C" {

void mvm_debug_set_score_kernel(int tc) { g_score_tc = tc ? 1 : 0; }
void mvm_debug_set_attention_split(int fp16) { g_attn_split = fp16 ? 1 : 0; }
void mvm_debug_set_gemm_split(int fp16) { g_gemm_split = fp16 ? 1 : 0; }

const char* mvm_version(void) { return "mvm_b200 0.1 sm_90a"; }

size_t mvm_matcher_workspace_bytes(int batch, int n_views, int n_pad, int n_pairs, int has_conf) {
  return carve(nullptr, batch, n_views, n_pad, n_pairs, has_conf).total;
}

void mvm_matcher_options_default(mvm_matcher_options* o) {
  if (!o) return;
  o->math_mode = g_math_mode;
  o->score_kernel = g_score_tc;
  o->gemm_tile = mvm_default_gemm_tile();
  o->gemm_kernel = mvm_default_gemm_persistent();
  o->sinkhorn_variant = 0;
  o->attention_split = g_attn_split;
  o->gemm_split = g_gemm_split;
}

int mvm_matcher_forward(const mvm_matcher_weights* w, int batch, int n_views, int n_pad,
                        const int* counts, const float* kpts, const float* kscores,
                        const float* desc, float img_w, float img_h, int sinkhorn_iters,
                        float match_threshold, const mvm_pair_io* pairs, int n_pairs,
                        void* workspace, size_t workspace_bytes, void* stream_) {
  return mvm_matcher_forward_ex(w, batch, n_views, n_pad, counts, kpts, kscores, desc, img_w, img_h, sinkhorn_iters,
                                match_threshold, pairs, n_pairs, workspace, workspace_bytes, nullptr, stream_);
}

int mvm_matcher_forward_ex(const mvm_matcher_weights* w, int batch, int n_views, int n_pad,
                           const int* counts, const float* kpts, const float* kscores,
                           const float* desc, float img_w, float img_h, int sinkhorn_iters,
                           float match_threshold, const mvm_pair_io* pairs, int n_pairs,
                           void* workspace, size_t workspace_bytes, const mvm_matcher_options* opt, void* stream_) {
  float view_wh[MVM_MAX_VIEWS][2];
  for (int t = 0; t < MVM_MAX_VIEWS; ++t) { view_wh[t][0] = img_w; view_wh[t][1] = img_h; }
  return mvm_matcher_forward_views(w, batch, n_views, n_pad, counts, kpts, kscores, desc, &view_wh[0][0], sinkhorn_iters,
                                   match_threshold, pairs, n_pairs, workspace, workspace_bytes, opt, stream_);
}

int mvm_matcher_forward_views(const mvm_matcher_weights* w, int batch, int n_views, int n_pad,
                              const int* counts, const float* kpts, const float* kscores,
                              const float* desc, const float* view_wh, int sinkhorn_iters,
                              float match_threshold, const mvm_pair_io* pairs, int n_pairs,
                              void* workspace, size_t workspace_bytes, const mvm_matcher_options* opt, void* stream_) {
  return mvm_matcher_forward_ragged(w, batch, n_views, n_pad, counts, nullptr, kpts, kscores, desc, view_wh, sinkhorn_iters,
                                    match_threshold, pairs, n_pairs, workspace, workspace_bytes, opt, stream_);
}

int mvm_matcher_forward_ragged(const mvm_matcher_weights* w, int batch, int n_views, int n_pad,
                               const int* counts, const int* slot_counts, const float* kpts, const float* kscores,
                               const float* desc, const float* view_wh, int sinkhorn_iters,
                               float match_threshold, const mvm_pair_io* pairs, int n_pairs,
                               void* workspace, size_t workspace_bytes, const mvm_matcher_options* opt, void* stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  mvm_matcher_options o;
  if (opt) o = *opt; else mvm_matcher_options_default(&o);
  MVM_REQUIRE(o.math_mode == 0 || o.math_mode == 1 || o.math_mode == 3);
  MVM_REQUIRE(o.sinkhorn_variant >= 0 && o.sinkhorn_variant <= 4);
  // device counts reach the tensor-core kernels of math mode 3 only (the SIMT attention and score kernels keep host counts)
  MVM_REQUIRE(!slot_counts || (o.math_mode == 3 && o.score_kernel));
  MVM_REQUIRE(w && counts && kpts && kscores && desc && view_wh && pairs && workspace && sinkhorn_iters >= 1);
  MVM_REQUIRE(batch >= 1 && n_views >= 2 && n_views <= MVM_MAX_VIEWS);
  MVM_REQUIRE(n_pad >= 64 && n_pad % 64 == 0);
  MVM_REQUIRE(w->n_layers >= 0 && w->n_layers <= MVM_MAX_LAYERS);
  for (int t = 0; t < n_views; ++t) MVM_REQUIRE(counts[t] >= 1 && counts[t] <= n_pad);
  Workspace ws = carve((char*)workspace, batch, n_views, n_pad, n_pairs, w->has_conf);
  if (ws.total > workspace_bytes) return MVM_ERR_WORKSPACE;

  Ctx cx;
  cx.math_mode = o.math_mode; cx.score_tc = o.score_kernel ? 1 : 0; cx.gemm_tile = o.gemm_tile == 128 ? 128 : 256;
  cx.gemm_persist = o.gemm_kernel ? 1 : 0; cx.sinkhorn_variant = o.sinkhorn_variant;
  cx.hi_off = w->hi_offset; cx.lo_off = w->lo_offset;
  // the fp16x3 attention needs the persistent GEMM (its epilogue writes the half-precision planes) and pre-split weights
  cx.attn_split = (o.attention_split == 1 && cx.math_mode == 3 && cx.lo_off != 0) ? 1 : 0;
  const bool g16 = o.gemm_split == 1 && cx.math_mode == 3 && cx.gemm_persist && w->w16_hi && w->w16_lo && w->flat_base && w->w16_scale > 0.f;
  cx.flat_base = w->flat_base;
  cx.w16_hi = g16 ? (const __half*)w->w16_hi : nullptr;
  cx.w16_lo = g16 ? (const __half*)w->w16_lo : nullptr;
  cx.w16_scale = w->w16_scale;
  const int V = batch * n_views;
  const int rows = V * n_pad;
  AttnSegs segs;
  segs.n_views = n_views;
  for (int t = 0; t < 8; ++t) segs.counts[t] = t < n_views ? counts[t] : 0;
  segs.slot = slot_counts;

  // keypoint encoder + descriptor add (multi_view_matcher.py:265-269)
  MVM_TRY(launch_transpose_cn(desc, ws.DT, V, 256, n_pad, s));
  MVM_TRY(launch_kenc_front(kpts, kscores, w->kenc_w, w->kenc_b, ws.H3, rows, view_wh, n_views, n_pad, s));
  MVM_TRY(run_gemm(cx, make_gemm(ws.H3, 128, w->kenc_w[3], 128, w->kenc_b[3], ws.H4, 256, rows, 256, 1), s));
  {
    GemmDesc g = make_gemm(ws.H4, 256, w->kenc_w[4], 256, w->kenc_b[4], ws.X, 256, rows, 256, 0);
    g.R = ws.DT; g.ldr = 256;
    MVM_TRY(run_gemm(cx, g, s));
  }

  // attentional GNN (multi_view_matcher.py:87-100 / superglue.py:131-140)
  for (int l = 0; l < w->n_layers; ++l) {
    const mvm_layer_weights& L = w->layers[l];
    if (cx.attn_split == 1) {
      // fp16x3: K and V^T leave the QKV GEMM as half-precision hi / lo planes (carved out of the tf32 lo-plane
      // buffers: two fp16 planes fill one fp32 plane exactly)
      __half* kh = reinterpret_cast<__half*>(ws.KLO);
      __half* vh = reinterpret_cast<__half*>(ws.VTLO);
      HalfPlanes hp = {kh, kh + (size_t)rows * 256, vh, vh + (size_t)rows * 256};
      GemmDesc gq = qkv_desc(ws.X, L.w_qkv, L.b_qkv, ws.QKV, rows);
      set_planes(cx, gq);
      MVM_TRY(run_qkv(gq, cx.math_mode, n_pad, &hp, nullptr, nullptr, nullptr, cx.gemm_tile, cx.gemm_persist, s));
      MVM_TRY(launch_attention_h3(ws.QKV, (const __half*)hp.kh, (const __half*)hp.kl, (const __half*)hp.vh,
                                  (const __half*)hp.vl, ws.MSG, batch, n_pad, segs, L.is_cross, s));
    } else if (cx.math_mode != 0) {
      // tensor-core path: the QKV GEMM epilogue also writes V^T [view, 256, n_pad] for the P.V product
      float* klo = cx.math_mode == 3 ? ws.KLO : nullptr;
      float* vtlo = cx.math_mode == 3 ? ws.VTLO : nullptr;
      GemmDesc gq = qkv_desc(ws.X, L.w_qkv, L.b_qkv, ws.QKV, rows);
      if (cx.math_mode == 3 && cx.lo_off != 0) { gq.Whi = gq.W + cx.hi_off; gq.Wlo = gq.W + cx.lo_off; }
      MVM_TRY(run_qkv(gq, cx.math_mode, n_pad, nullptr, ws.VT, klo, vtlo, cx.gemm_tile, cx.gemm_persist, s));
      MVM_TRY(launch_attention_tc(ws.QKV, ws.VT, ws.MSG, batch, n_pad, segs, L.is_cross, cx.math_mode, s, klo, vtlo));
    } else {
      MVM_TRY(run_gemm(cx, make_gemm(ws.X, 256, L.w_qkv, 256, L.b_qkv, ws.QKV, 768, rows, 768, 0), s));
      MVM_TRY(launch_attention_simt(ws.QKV, ws.MSG, batch, n_pad, segs, L.is_cross, s));
    }
    // attn.merge (superglue.py:109) is linear and feeds mlp.0 directly (:121): packing.py folds it into the
    // message half of mlp.0 (w_merge == NULL); an unfolded weight set still runs the separate GEMM
    const float* msg = ws.MSG;
    if (L.w_merge) {
      MVM_TRY(run_gemm(cx, make_gemm(ws.MSG, 256, L.w_merge, 256, L.b_merge, ws.MRG, 256, rows, 256, 0), s));
      msg = ws.MRG;
    }
    {
      GemmDesc g = make_gemm(ws.X, 256, L.w_mlp0, 512, L.b_mlp0, ws.H, 512, rows, 512, 1);
      g.A2 = msg; g.lda2 = 256; g.K1 = 256;      // cat([x, message]) by K-split
      MVM_TRY(run_gemm(cx, g, s));
    }
    {
      GemmDesc g = make_gemm(ws.H, 512, L.w_mlp1, 512, L.b_mlp1, ws.X, 256, rows, 256, 0);
      g.R = ws.X; g.ldr = 256;                   // desc = desc + delta
      MVM_TRY(run_gemm(cx, g, s));
    }
  }

  // final projection once per view (the reference redoes it per pair, :276)
  MVM_TRY(run_gemm(cx, make_gemm(ws.X, 256, w->w_final, 256, w->b_final, ws.MD, 256, rows, 256, 0), s));

  PairTable tab;
  MVM_TRY(fill_pair_table(tab, pairs, n_pairs, n_views, counts, batch));
  tab.slot = slot_counts;
  // score matrices: tensor cores in the 3xTF32 mode (the K_lo / V^T_lo planes of the GNN are free again and
  // hold the tf32 planes of the descriptors), fp32 CUDA cores otherwise
  if (cx.math_mode == 3 && cx.score_tc) MVM_TRY(launch_score_gemm_tc(ws.MD, ws.KLO, ws.VTLO, n_pad, tab, batch, 1.0f / 16.0f, s));
  else MVM_TRY(launch_score_gemm_simt(ws.MD, n_pad, tab, batch, 1.0f / 16.0f, s));
  MVM_TRY(launch_sinkhorn(tab, batch, w->bin_score, sinkhorn_iters, ws.sink_ws, s, cx.sinkhorn_variant));
  MVM_TRY(launch_extract_matches(tab, batch, n_pad, match_threshold, ws.match_ws, s));

  if (w->has_conf) {
    const long long crow = (long long)n_pairs * batch * n_pad;
    MVM_TRY(launch_conf_gather(ws.MD, tab, batch, n_pad, ws.FEAT, ws.SC, s));
    MVM_TRY(run_gemm(cx, make_gemm(ws.FEAT, 512, w->conf_wf0, 512, w->conf_bf0, ws.CF1, 512, (int)crow, 512, 1), s));
    MVM_TRY(run_gemm(cx, make_gemm(ws.CF1, 512, w->conf_wf1, 512, w->conf_bf1, ws.CF2, 256, (int)crow, 256, 1), s));
    MVM_TRY(launch_conf_c0(ws.SC, w->conf_wc0, w->conf_bc0, ws.CC0, crow, s));
    {
      GemmDesc g = make_gemm(ws.CC0, 256, w->conf_wc1, 256, w->conf_bc1, ws.CC1, 256, (int)crow, 256, 1);
      g.R = ws.CF2; g.ldr = 256;                 // out_f + out_c
      MVM_TRY(run_gemm(cx, g, s));
    }
    MVM_TRY(launch_conf_final(ws.CC1, w->conf_wl, w->conf_bl, tab, batch, n_pad, s));
  }
  return MVM_OK;
}

int mvm_linear(const float* A, int lda, const float* A2, int lda2, int K1, const float* W,
               int ldw, const float* bias, const float* R, int ldr, float* C, int ldc, int M,
               int N, int K, float alpha, int relu, void* stream) {
  MVM_REQUIRE(A && W && C);
  GemmDesc g = make_gemm(A, lda, W, K, bias, C, ldc, M, N, relu);
  g.ldw = ldw; g.alpha = alpha;
  if (A2) { g.A2 = A2; g.lda2 = lda2; g.K1 = K1; }
  if (R) { g.R = R; g.ldr = ldr; }
  return launch_gemm_simt(g, (cudaStream_t)stream);
}

int mvm_set_math_mode(int mode) {
  MVM_REQUIRE(mode == 0 || mode == 1 || mode == 3);
  g_math_mode = mode;
  return MVM_OK;
}
int mvm_get_math_mode(void) { return g_math_mode; }

int mvm_linear_tc(const float* A, int lda, const float* A2, int lda2, int K1, const float* W, int ldw,
                  const float* bias, const float* R, int ldr, float* C, int ldc, int M, int N, int K,
                  float alpha, int relu, int n_pass, void* stream) {
  MVM_REQUIRE(A && W && C && (n_pass == 1 || n_pass == 3));
  GemmDesc g = make_gemm(A, lda, W, K, bias, C, ldc, M, N, relu);
  g.ldw = ldw; g.alpha = alpha;
  if (A2) { g.A2 = A2; g.lda2 = lda2; g.K1 = K1; }
  if (R) { g.R = R; g.ldr = ldr; }
  return launch_gemm_tc(g, n_pass, nullptr, 0, 0, (cudaStream_t)stream);
}

int mvm_linear_tc_presplit(const float* A, int lda, const float* A2, int lda2, int K1, const float* W_hi,
                           const float* W_lo, int ldw, const float* bias, const float* R, int ldr, float* C, int ldc,
                           int M, int N, int K, float alpha, int relu, void* stream) {
  MVM_REQUIRE(A && W_hi && W_lo && C);
  GemmDesc g = make_gemm(A, lda, W_hi, K, bias, C, ldc, M, N, relu);
  g.ldw = ldw; g.alpha = alpha; g.Whi = W_hi; g.Wlo = W_lo;
  if (A2) { g.A2 = A2; g.lda2 = lda2; g.K1 = K1; }
  if (R) { g.R = R; g.ldr = ldr; }
  return launch_gemm_tc(g, 3, nullptr, 0, 0, (cudaStream_t)stream);
}

int mvm_pair_scores(const float* mdesc, float* hi, float* lo, int batch, int n_views, int n_pad, int n_pairs, const int* pa,
                    const int* pb, const int* m, const int* n, float* const* scores, float alpha, void* stream) {
  MVM_REQUIRE(mdesc && hi && lo && pa && pb && m && n && scores && batch >= 1 && n_views >= 2 && n_views <= MVM_MAX_VIEWS);
  MVM_REQUIRE(n_pairs >= 1 && n_pairs <= MVM_MAX_PAIRS && n_pad >= 64 && n_pad % 64 == 0);
  PairTable tab;
  memset(&tab, 0, sizeof(tab));
  tab.n_pairs = n_pairs; tab.n_views = n_views;
  for (int p = 0; p < n_pairs; ++p) {
    MVM_REQUIRE(pa[p] >= 0 && pa[p] < n_views && pb[p] >= 0 && pb[p] < n_views && scores[p]);
    MVM_REQUIRE(m[p] >= 1 && m[p] <= n_pad && n[p] >= 1 && n[p] <= n_pad);
    tab.a[p] = pa[p]; tab.b[p] = pb[p]; tab.m[p] = m[p]; tab.n[p] = n[p]; tab.scores[p] = scores[p];
  }
  return launch_score_gemm_tc(mdesc, hi, lo, n_pad, tab, batch, alpha, (cudaStream_t)stream);
}

int mvm_linear_tc_presplit_splitk(const float* A, int lda, const float* W_hi, const float* W_lo, int ldw, float* C, int ldc,
                                  int M, int N, int K, float alpha, int ksplit, float* ws, void* stream) {
  MVM_REQUIRE(A && W_hi && W_lo && C && ws && ksplit >= 2 && M % 128 == 0 && N % 128 == 0 && K % (32 * ksplit) == 0);
  MVM_REQUIRE(lda % 4 == 0 && ldw % 4 == 0 && ldc % 4 == 0);
  GemmDesc g = make_gemm(A, lda, W_hi, K, nullptr, C, ldc, M, N, 0);
  g.ldw = ldw; g.alpha = alpha; g.Whi = W_hi; g.Wlo = W_lo;
  MvmProfScope prof__(MVM_TAG_GEMM, (cudaStream_t)stream);
  int rc = launch_gemm_tc_persist(g, nullptr, 0, 0, nullptr, nullptr, (cudaStream_t)stream, nullptr, ksplit, ws);
  if (rc != MVM_OK) return rc;
  return launch_splitk_reduce(ws, C, M, N, ldc, ksplit, (cudaStream_t)stream);
}

int mvm_linear_tc_h16(const float* A, int lda, const float* A2, int lda2, int K1, const void* W16_hi, const void* W16_lo,
                      float wscale, int ldw, const float* bias, const float* R, int ldr, float* C, int ldc, int M, int N, int K,
                      float alpha, int relu, void* stream) {
  MVM_REQUIRE(A && W16_hi && W16_lo && C && wscale > 0.f && K % 64 == 0 && N % 128 == 0);
  GemmDesc g = make_gemm(A, lda, reinterpret_cast<const float*>(W16_hi), K, bias, C, ldc, M, N, relu);
  g.ldw = ldw; g.alpha = alpha; g.Whi = g.W; g.Wlo = g.W;       // (the tf32 planes are not read in the fp16 mode)
  g.Whi16 = W16_hi; g.Wlo16 = W16_lo; g.wscale = wscale;
  if (A2) { g.A2 = A2; g.lda2 = lda2; g.K1 = K1; MVM_REQUIRE(K1 % 64 == 0); }
  if (R) { g.R = R; g.ldr = ldr; }
  return launch_gemm_tc_persist(g, nullptr, 0, 0, nullptr, nullptr, (cudaStream_t)stream);
}

int mvm_qkv_projection(const float* X, const float* W_hi, const float* W_lo, const void* W16_hi, const void* W16_lo,
                       float wscale, const float* bias, float* qkv, int rows, int n_pad, int planes16, void* k_hi,
                       void* k_lo, void* v_hi, void* v_lo, void* stream) {
  MVM_REQUIRE(X && W_hi && W_lo && qkv && k_lo && v_hi && v_lo && n_pad >= 64 && n_pad % 64 == 0 && rows % n_pad == 0);
  MVM_REQUIRE(!planes16 || k_hi);
  MVM_REQUIRE(!W16_hi == !W16_lo && (!W16_hi || wscale > 0.f));
  // the GNN layer's launch (run_qkv), with the process defaults of the options
  GemmDesc gq = qkv_desc(X, W_hi, bias, qkv, rows);
  gq.Whi = W_hi; gq.Wlo = W_lo;
  if (!planes16) return run_qkv(gq, 3, n_pad, nullptr, (float*)v_hi, (float*)k_lo, (float*)v_lo, -1, -1, (cudaStream_t)stream);
  if (W16_hi) { gq.Whi16 = W16_hi; gq.Wlo16 = W16_lo; gq.wscale = wscale; }
  HalfPlanes hp = {k_hi, k_lo, v_hi, v_lo};
  return run_qkv(gq, 3, n_pad, &hp, nullptr, nullptr, nullptr, -1, -1, (cudaStream_t)stream);
}

int mvm_attention(const float* qkv, float* out, int batch, int n_views, int n_pad,
                  const int* counts, int is_cross, void* stream) {
  MVM_REQUIRE(qkv && out && counts && n_views >= 1 && n_views <= 8);
  AttnSegs segs;
  segs.n_views = n_views;
  for (int t = 0; t < 8; ++t) segs.counts[t] = t < n_views ? counts[t] : 0;
  return launch_attention_simt(qkv, out, batch, n_pad, segs, is_cross, (cudaStream_t)stream);
}

size_t mvm_sinkhorn_workspace_floats(int n_pairs, int batch, int n_max) {
  return sinkhorn_ws_floats(n_pairs, batch, (n_max + 63) / 64 * 64);
}

int mvm_log_optimal_transport(float* scores, int batch, int m, int n, float bin_score, int iters,
                              float* ws, void* stream) {
  MVM_REQUIRE(scores && ws && batch >= 1 && m >= 1 && n >= 1);
  PairTable tab;
  tab.n_pairs = 1; tab.n_views = 2; tab.a[0] = 0; tab.b[0] = 1; tab.m[0] = m; tab.n[0] = n;
  tab.scores[0] = scores; tab.ws_off[0] = 0;
  return launch_sinkhorn(tab, batch, bin_score, iters, ws, (cudaStream_t)stream);
}

int mvm_log_optimal_transport_ex(float* scores, int batch, int m, int n, float bin_score, int iters, float* ws,
                                 int variant, void* stream) {
  MVM_REQUIRE(scores && ws && batch >= 1 && m >= 1 && n >= 1 && variant >= 0 && variant <= 4);
  PairTable tab;
  tab.n_pairs = 1; tab.n_views = 2; tab.a[0] = 0; tab.b[0] = 1; tab.m[0] = m; tab.n[0] = n;
  tab.scores[0] = scores; tab.ws_off[0] = 0;
  return launch_sinkhorn(tab, batch, bin_score, iters, ws, (cudaStream_t)stream, variant);
}

int mvm_sinkhorn_max_active_clusters(int m, int n) {
  const int C = sinkhorn_cluster_size(m, n);
  return C > 0 ? sinkhorn_cluster_max_active(C, n) : 0;
}

int mvm_attention_tc(const float* qkv, const float* vt, float* out, int batch, int n_views, int n_pad,
                     const int* counts, int is_cross, int n_pass, const float* klo, const float* vtlo, void* stream) {
  MVM_REQUIRE(qkv && vt && out && counts && n_views >= 1 && n_views <= 8 && (n_pass == 1 || n_pass == 3));
  AttnSegs segs;
  segs.n_views = n_views;
  for (int t = 0; t < 8; ++t) segs.counts[t] = t < n_views ? counts[t] : 0;
  MVM_REQUIRE(n_pass == 1 || (klo && vtlo));
  return launch_attention_tc(qkv, vt, out, batch, n_pad, segs, is_cross, n_pass, (cudaStream_t)stream, klo, vtlo);
}

int mvm_attention_h3(const float* qkv, const void* kh, const void* kl, const void* vh, const void* vl, float* out,
                     int batch, int n_views, int n_pad, const int* counts, int is_cross, void* stream) {
  MVM_REQUIRE(qkv && kh && kl && vh && vl && out && counts && n_views >= 1 && n_views <= 8);
  AttnSegs segs;
  segs.n_views = n_views;
  for (int t = 0; t < 8; ++t) segs.counts[t] = t < n_views ? counts[t] : 0;
  return launch_attention_h3(qkv, (const __half*)kh, (const __half*)kl, (const __half*)vh, (const __half*)vl, out, batch,
                             n_pad, segs, is_cross, (cudaStream_t)stream);
}

int mvm_log_optimal_transport_logdomain(float* scores, int batch, int m, int n, float bin_score, int iters,
                                        float* ws, void* stream) {
  MVM_REQUIRE(scores && ws && batch >= 1 && m >= 1 && n >= 1);
  PairTable tab;
  tab.n_pairs = 1; tab.n_views = 2; tab.a[0] = 0; tab.b[0] = 1; tab.m[0] = m; tab.n[0] = n;
  tab.scores[0] = scores; tab.ws_off[0] = 0;
  return launch_sinkhorn_log(tab, batch, bin_score, iters, ws, (cudaStream_t)stream);
}

int mvm_log_optimal_transport_ref(float* scores, int batch, int m, int n, float bin_score,
                                  int iters, float* ws, void* stream) {
  MVM_REQUIRE(scores && ws && batch >= 1 && m >= 1 && n >= 1);
  PairTable tab;
  tab.n_pairs = 1; tab.n_views = 2; tab.a[0] = 0; tab.b[0] = 1; tab.m[0] = m; tab.n[0] = n;
  tab.scores[0] = scores; tab.ws_off[0] = 0;
  return launch_sinkhorn_ref(tab, batch, bin_score, iters, ws, (cudaStream_t)stream);
}

int mvm_extract_matches(const float* scores, int batch, int m, int n, float match_threshold,
                        int64_t* matches0, int64_t* matches1, float* mscores0, float* mscores1,
                        void* ws, void* stream) {
  MVM_REQUIRE(scores && matches0 && matches1 && mscores0 && mscores1 && ws);
  PairTable tab;
  tab.n_pairs = 1; tab.n_views = 2; tab.a[0] = 0; tab.b[0] = 1; tab.m[0] = m; tab.n[0] = n;
  tab.scores[0] = const_cast<float*>(scores);
  tab.matches_a[0] = matches0; tab.matches_b[0] = matches1;
  tab.ms_a[0] = mscores0; tab.ms_b[0] = mscores1;
  const int n_pad = ((m > n ? m : n) + 63) / 64 * 64;
  return launch_extract_matches(tab, batch, n_pad, match_threshold, (int*)ws, (cudaStream_t)stream);
}

}  // extern "C"
