// Internal launch prototypes (host side) of the matcher kernels.
#pragma once
#include "common.cuh"

constexpr int MVM_MAX_PAIRS = 28;  // C(8,2)

// Per-pair table passed BY VALUE to the pair-stage kernels (score GEMM, Sinkhorn, match
// extraction, confidence head): one launch covers every (pair, batch) problem and the
// whole forward stays CUDA-graph capturable (no host->device table copies).
struct PairTable {
  int n_pairs;
  int n_views;                 // views per tuple (slot of view t in tuple b = b*n_views + t)
  int a[MVM_MAX_PAIRS], b[MVM_MAX_PAIRS];   // view ids, a < b
  int m[MVM_MAX_PAIRS], n[MVM_MAX_PAIRS];   // true keypoint counts of a and b
  float* scores[MVM_MAX_PAIRS];             // [batch, m+1, n+1]
  int64_t* matches_a[MVM_MAX_PAIRS];        // [batch, m]
  int64_t* matches_b[MVM_MAX_PAIRS];        // [batch, n]
  float* ms_a[MVM_MAX_PAIRS];
  float* ms_b[MVM_MAX_PAIRS];
  float* conf[MVM_MAX_PAIRS];               // [batch, m] (or nullptr)
  long long ws_off[MVM_MAX_PAIRS];          // float offset of this pair's (u,v) scratch
  // ragged batches (mvm_matcher_forward_ragged): device [batch * n_views] true count of every view slot; m / n above are
  // then the capacities, which set every stride.  nullptr: every slot holds exactly m / n keypoints.
  const int* slot = nullptr;
};
typedef PairTable SinkhornTable;

// view_wh: host float[n_views][2], (width, height) of each view slot; row r belongs to slot (r / n_pad) % n_views
int launch_kenc_front(const float* kpts, const float* kscores, const float* const* w,
                      const float* const* b, float* h3, int n_points, const float* view_wh, int n_views,
                      int n_pad, cudaStream_t stream);
int launch_transpose_cn(const float* in, float* out, int n_views_total, int C, int n_pad,
                        cudaStream_t stream);

// What every GEMM launch needs of its descriptor, checked on the host before any CUDA call (a bad call returns
// MVM_ERR_INVALID instead of failing a tensor-map encode or faulting in the kernel).  `ops` names the kernel family:
//   GEMM_SIMT     fp32 CUDA cores: float4 loads of A, A2 and W (16-byte aligned, lda / lda2 / ldw multiples of 4),
//                 K and K1 multiples of 16
//   GEMM_TC_TF32  tensor cores with tf32 operands: TMA boxes of A, A2 and the W planes (16-byte aligned base, row
//                 pitch a multiple of 16 bytes), K and K1 multiples of 32, N of 128, float2 epilogue stores and residual
//                 loads (C and R 8-byte aligned, ldc / ldr multiples of 4)
//   GEMM_TC_F16   as GEMM_TC_TF32 with W given as fp16 planes (ldw a multiple of 8), K and K1 multiples of 64
// Always: M >= 1, K >= one k-block, and K1 == K without A2 (0 < K1 < K with it).
enum { GEMM_SIMT = 0, GEMM_TC_TF32 = 1, GEMM_TC_F16 = 2 };
inline bool mvm_aligned(const void* p, unsigned bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }
inline bool gemm_desc_valid(const GemmDesc& d, int ops) {
  const bool tc = ops != GEMM_SIMT;
  const int bk = ops == GEMM_SIMT ? 16 : ops == GEMM_TC_TF32 ? 32 : 64;
  if (!d.A || !d.C || d.M < 1 || d.N < 1 || d.K < bk || d.K % bk != 0 || d.K1 % bk != 0) return false;
  if (d.A2 ? (d.K1 <= 0 || d.K1 >= d.K) : d.K1 != d.K) return false;
  if (!mvm_aligned(d.A, 16) || d.lda % 4 != 0) return false;
  if (d.A2 && (!mvm_aligned(d.A2, 16) || d.lda2 % 4 != 0)) return false;
  // W operand: raw fp32 (SIMT, the raw-W tensor-core kernels) or its pre-split tf32 / fp16 planes
  if (ops == GEMM_SIMT && !d.W) return false;
  if (ops == GEMM_TC_TF32 && !d.W && !(d.Whi && d.Wlo)) return false;
  if (ops == GEMM_TC_F16 && !(d.Whi16 && d.Wlo16 && d.wscale > 0.f)) return false;
  const void* w[5] = {d.W, d.Whi, d.Wlo, d.Whi16, d.Wlo16};
  for (const void* p : w)
    if (p && !mvm_aligned(p, 16)) return false;
  if (d.ldw % (ops == GEMM_TC_F16 ? 8 : 4) != 0) return false;
  if (!tc) return d.batch >= 1;
  return d.batch == 1 && d.N % 128 == 0 && mvm_aligned(d.C, 8) && d.ldc % 4 == 0 &&
         (!d.R || (mvm_aligned(d.R, 8) && d.ldr % 4 == 0));
}

// tensor-core GEMM (gemm_tc.cu): n_pass 3 = fp32-faithful 3xTF32, 1 = single-pass TF32
// gemm_tile (128 / 256) and gemm_persist (0 / 1) select the kernel; -1 = the process defaults
int launch_gemm_tc(const GemmDesc& d, int n_pass, float* VT, int vt_col0, int n_pad, cudaStream_t stream,
                   float* KLO = nullptr, float* VTLO = nullptr, int gemm_tile = -1, int gemm_persist = -1);
int mvm_default_gemm_tile();
int mvm_default_gemm_persistent();
// persistent schedule of the same kernel with pre-split W planes (tf32, or fp16 when d.Whi16 / d.Wlo16 are given)
// hp != nullptr (QKV projection, vt_col0 = 512): the K third and V^T leave as half-precision hi / lo planes for
// launch_attention_h3 instead of the fp32 / tf32 buffers (kh, kl, vh, vl: all [rows, 256], as __half; V stays key-major)
struct HalfPlanes { void* kh; void* kl; void* vh; void* vl; };
int launch_gemm_tc_persist(const GemmDesc& d, float* VT, int vt_col0, int n_pad, float* KLO, float* VTLO,
                           cudaStream_t stream, const HalfPlanes* hp = nullptr, int ksplit = 1, float* slabs = nullptr);
int launch_splitk_reduce(const float* slabs, float* C, int M, int N, int ldc, int ksplit, cudaStream_t stream);
// every (pair, tuple) score matrix in one launch of the GEMM kernel (3xTF32); hi / lo: scratch [rows, 256]
struct PairTable;
int launch_score_gemm_tc(const float* mdesc, float* hi, float* lo, int n_pad, const PairTable& tab, int batch,
                         float alpha, cudaStream_t stream);

struct AttnSegs {
  int n_views;
  int counts[8];
  const int* slot = nullptr;   // as PairTable::slot: counts[] are then the capacities
};

// Keypoints of view t of tuple b: the capacity `cap` without device counts, else slot[b * n_views + t] clamped to
// [0, cap], so that no count a caller passes can move an access outside the capacity-sized buffers.
__device__ __forceinline__ int slot_count(const int* slot, int b, int n_views, int t, int cap) {
  return slot ? min(max(__ldg(slot + b * n_views + t), 0), cap) : cap;
}
// What every attention launch needs of its segments, checked on the host before any CUDA call: 1..8 views, cross
// attention over at least two, every count in [0, n_pad] (a larger count walks the key loop into the next view's rows),
// and a source key for every query view that has a query row (without one the softmax denominator is 0: NaN output)
inline bool attn_segs_valid(const AttnSegs& segs, int n_pad, int is_cross) {
  if (segs.n_views < 1 || segs.n_views > 8 || (is_cross && segs.n_views < 2)) return false;
  for (int t = 0; t < segs.n_views; ++t)
    if (segs.counts[t] < 0 || segs.counts[t] > n_pad) return false;
  for (int t = 0; t < segs.n_views; ++t) {
    int keys = 0;
    for (int s = 0; s < segs.n_views; ++s)
      if (is_cross ? s != t : s == t) keys += segs.counts[s];
    if (segs.counts[t] > 0 && keys == 0) return false;
  }
  return true;
}
// klo / vtlo: tf32 remainder planes of K [rows,256] and V^T (n_pass == 3; K and V^T then hold the rn_tf32 parts)
int launch_attention_tc(const float* qkv, const float* vt, float* out, int batch, int n_pad, AttnSegs segs,
                        int is_cross, int n_pass, cudaStream_t stream, const float* klo = nullptr,
                        const float* vtlo = nullptr);
int launch_attention_simt(const float* qkv, float* out, int batch, int n_pad, AttnSegs segs,
                          int is_cross, cudaStream_t stream);
// fp32-faithful attention with half-precision operand planes (fp16x3, attention_h3.cu); planes as in HalfPlanes
struct __half;
int launch_attention_h3(const float* qkv, const __half* kh, const __half* kl, const __half* vh, const __half* vl,
                        float* out, int batch, int n_pad, AttnSegs segs, int is_cross, cudaStream_t stream);

// scores[p][bi] inner block = mdesc[a] . mdesc[b]^T * alpha   (mdesc: [views, n_pad, 256])
int launch_score_gemm_simt(const float* mdesc, int n_pad, const PairTable& tab, int batch,
                           float alpha, cudaStream_t stream);

int launch_sinkhorn_ref(const SinkhornTable& tab, int batch, float bin_score, int iters,
                        float* ws, cudaStream_t stream);
// production dispatch (sinkhorn_exp.cu): cluster kernel up to 1024 x 1024, multi-CTA kernel beyond;
// variant 0 = automatic, 1 = multi-CTA kernel, 2 = cluster kernel
int launch_sinkhorn(const SinkhornTable& tab, int batch, float bin_score, int iters, float* ws,
                    cudaStream_t stream, int variant = 0);
int launch_sinkhorn_multicta(const SinkhornTable& tab, int batch, float bin_score, int iters, float* ws,
                             cudaStream_t stream);
// one thread-block cluster per problem (sinkhorn_cl.cu)
int sinkhorn_cluster_size(int max_m, int max_n);
int sinkhorn_cluster_max_active(int C, int n);
int launch_sinkhorn_cluster(const SinkhornTable& tab, int batch, float bin_score, int iters, int C,
                            cudaStream_t stream, int rr = 0);
int launch_sinkhorn_log(const SinkhornTable& tab, int batch, float bin_score, int iters, float* ws,
                        cudaStream_t stream);
size_t sinkhorn_ws_floats(int n_pairs, int batch, int n_pad);

// idx_ws: ints [n_pairs*batch*2*n_pad] + floats; see match.cu
int launch_extract_matches(const PairTable& tab, int batch, int n_pad, float thresh, int* idx_ws,
                           cudaStream_t stream);

// feat [n_pairs*batch*n_pad, 512] = cat(mdesc_a[i], mdesc_b[match(i)]); sc [rows] = Z[i, match(i)]
int launch_conf_gather(const float* mdesc, const PairTable& tab, int batch, int n_pad, float* feat,
                       float* sc, cudaStream_t stream);
int launch_conf_c0(const float* sc, const float* w, const float* b, float* out, long long rows,
                   cudaStream_t stream);
int launch_conf_final(const float* h, const float* wl, float bl, const PairTable& tab, int batch,
                      int n_pad, cudaStream_t stream);
