/* mvm_b200.h -- C ABI of libmvm_b200.so, the H100 (sm_90a) drop-in for the hot path of
 * barbararoessle/e2e_multi_view_matching.
 *
 * The reference has no FFI layer: the path sits behind Python callables.  Each entry point
 * below is what a binding for that callable would call (INTEGRATION.md shows the ctypes
 * stubs).  Conventions: plain device pointers + sizes, an explicit CUDA stream (passed as
 * void* == cudaStream_t), int status return (0 ok, 1 invalid argument, 2 launch failure,
 * 3 workspace too small).  Nothing throws across the ABI, every call is stream-ordered and
 * re-entrant per stream; the only state on the call path is the caller-provided workspace (process-wide
 * defaults exist for the options struct, see mvm_matcher_options; per-device function attributes and
 * tensor-map descriptors are cached under a mutex).
 *
 * Activation layout inside the library is point-major [view, keypoint, channel]; the
 * reference's channel-first [B, C, N] tensors are accepted at the boundary.
 */
#ifndef MVM_B200_H
#define MVM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MVM_DESC_DIM 256
#define MVM_HEADS 4
#define MVM_MAX_VIEWS 8
#define MVM_MAX_LAYERS 64

/* One AttentionalPropagation layer (superglue.py:112-121), repacked:
 * BatchNorm folded into the preceding 1x1 conv; q/k/v rows and merge columns permuted from
 * the reference's channel = d*4 + h interleave (superglue.py:106,109) to head-contiguous
 * h*64 + d; q,k,v stacked into one [768,256] matrix.  All matrices row-major [out, in]. */
typedef struct mvm_layer_weights {
  const float* w_qkv;   /* [768,256] */
  const float* b_qkv;   /* [768]     */
  const float* w_merge; /* [256,256]; NULL = folded into w_mlp0 (what packing.py does by default):      */
  const float* b_merge; /* [256]      w_mlp0[:,256:] <- w_mlp0[:,256:] @ w_merge, b_mlp0 += w_mlp0[:,256:] @ b_merge */
  const float* w_mlp0;  /* [512,512]  mlp.0 with mlp.1 (BN) folded */
  const float* b_mlp0;  /* [512]     */
  const float* w_mlp1;  /* [256,512]  mlp.3 */
  const float* b_mlp1;  /* [256]     */
  int is_cross;         /* 0 = 'self', 1 = 'cross' */
} mvm_layer_weights;

/* Whole matcher (multi_view_matcher.py:103-148).  Device pointers; BN folded everywhere. */
typedef struct mvm_matcher_weights {
  int n_layers;
  /* tf32 hi / lo copies of the whole flat weight buffer for the 3xTF32 mode, as float offsets from any
   * weight pointer below (0 = not provided: the GEMM splits the weight tiles on chip) */
  long long hi_offset, lo_offset;
  /* KeypointEncoder 3->32->64->128->256->256 (multi_view_matcher.py:24-37) */
  const float* kenc_w[5];
  const float* kenc_b[5];
  mvm_layer_weights layers[MVM_MAX_LAYERS];
  const float* w_final; /* [256,256] final_proj */
  const float* b_final;
  float bin_score;
  /* ConfidenceMLP (multi_view_matcher.py:39-53); has_conf = 0 skips it */
  int has_conf;
  const float* conf_wf0; const float* conf_bf0; /* [512,512] layers_f.0 (+BN) */
  const float* conf_wf1; const float* conf_bf1; /* [256,512] layers_f.3 (+BN) */
  const float* conf_wc0; const float* conf_bc0; /* [256] each: layers_c.0 (1->256, +BN) */
  const float* conf_wc1; const float* conf_bc1; /* [256,256] layers_c.3 (+BN) */
  const float* conf_wl;  float conf_bl;         /* [256], scalar: layers.0 */
  /* fp16x3 GEMMs (optional; NULL = tf32x3): half-precision hi / lo planes of w16_scale * (the whole flat weight buffer
   * starting at flat_base), element for element; w16_scale is a power of two that lifts the lo plane out of the fp16
   * subnormals (packing.py uses 64) */
  const float* flat_base;
  const void* w16_hi; const void* w16_lo;
  float w16_scale;
} mvm_matcher_weights;

/* Outputs of one view pair (a < b), batch-major, exactly the tensors the reference returns
 * (multi_view_matcher.py:308-315): matches{a}_{a}_{b} [B,n_a] int64 (-1 = none),
 * matches{b}_{a}_{b} [B,n_b], matching_scores (fp32), scores_{a}_{b} [B,n_a+1,n_b+1],
 * conf_scores_{a}_{b} [B,n_a,1].  conf may be NULL when has_conf == 0. */
typedef struct mvm_pair_io {
  int view_a, view_b;
  int64_t* matches_a; int64_t* matches_b;
  float* mscores_a;   float* mscores_b;
  float* scores;
  float* conf;
} mvm_pair_io;

/* Gathers the per-view inputs of a matcher call -- the reference's `data` dict, keypoints{i} [B,n_i,2], scores{i}
 * [B,n_i], descriptors{i} [B,256,n_i] (models/models/multi_view_matcher.py:229-262) -- into the zero-padded
 * view-slot-major buffers mvm_matcher_forward reads (kpts [B,T,n_pad,2], scores [B,T,n_pad], desc [B,T,256,n_pad]).
 * kpts / scores / desc: HOST arrays of n_views device pointers; counts[t] = n_t <= n_pad.  One launch. */
int mvm_pack_views(const float* const* kpts, const float* const* scores, const float* const* desc,
                   const int* counts, int batch, int n_views, int n_pad, float* out_kpts, float* out_scores,
                   float* out_desc, void* stream);

/* Bytes of scratch mvm_matcher_forward needs for this shape. */
size_t mvm_matcher_workspace_bytes(int batch, int n_views, int n_pad, int n_pairs, int has_conf);

/* MultiViewMatcher.forward in eval mode (multi_view_matcher.py:322-332; multi_match
 * :217-320; with n_views == 2 it is also SuperGlue/`match`, :150-215, superglue.py:230-285).
 *   batch     tuples; n_views views per tuple; view v of tuple b is slot b*n_views + v
 *   n_pad     row stride of the per-view buffers (multiple of 64, >= max count)
 *   counts    host int[n_views]: true keypoints per view (shared by the batch)
 *   kpts      [batch*n_views, n_pad, 2]  pixel x,y        (device)
 *   kscores   [batch*n_views, n_pad]                       (device)
 *   desc      [batch*n_views, 256, n_pad] channel-first    (device)
 *   img_w/h   image size used by normalize_keypoints (superglue.py:65-72), the same for every view
 *             (mvm_matcher_forward_views takes one size per view)
 *   pairs     host array of n_pairs descriptors with device output pointers
 *   match_threshold  0 for MultiViewMatcher (:297), 0.2 for SuperGlue (superglue.py:275) */
int mvm_matcher_forward(const mvm_matcher_weights* w, int batch, int n_views, int n_pad,
                        const int* counts, const float* kpts, const float* kscores,
                        const float* desc, float img_w, float img_h, int sinkhorn_iters,
                        float match_threshold, const mvm_pair_io* pairs, int n_pairs,
                        void* workspace, size_t workspace_bytes, void* stream);

/* Per-call options: the forward reads its configuration from this struct only (no process-global state on the
 * call path), so concurrent forwards on different streams / threads with different options are safe as long as
 * each has its own workspace.  mvm_matcher_options_default fills in the process defaults (math mode 3, tensor-core
 * score kernel, 256-wide persistent GEMM, automatic Sinkhorn kernel), which mvm_set_math_mode / the mvm_debug_*
 * hooks below change for callers of the plain mvm_matcher_forward. */
typedef struct mvm_matcher_options {
  int math_mode;        /* 3 = 3xTF32 on the tensor cores (fp32-faithful), 1 = single-pass TF32, 0 = fp32 CUDA cores */
  int score_kernel;     /* 1 = score matrices on the tensor cores (math mode 3), 0 = fp32 CUDA cores */
  int gemm_tile;        /* 128 | 256: tile width of the one-tile-per-CTA GEMM (when gemm_kernel == 0) */
  int gemm_kernel;      /* 1 = persistent 3xTF32 GEMM, 0 = one tile per CTA */
  int sinkhorn_variant; /* 0 = automatic (see mvm_log_optimal_transport_ex) */
  int attention_split;  /* math mode 3: operand planes of attention, 0 = tf32 hi/lo (3 x tf32 wgmma), 1 = fp16 hi/lo
                         * (3 x f16 wgmma: same 22-bit operands, half the tensor-pipe time) */
  int gemm_split;       /* the same choice for the 1x1-conv GEMMs (1 needs mvm_matcher_weights.w16_*) */
} mvm_matcher_options;
void mvm_matcher_options_default(mvm_matcher_options* opt);
int mvm_matcher_forward_ex(const mvm_matcher_weights* w, int batch, int n_views, int n_pad,
                           const int* counts, const float* kpts, const float* kscores,
                           const float* desc, float img_w, float img_h, int sinkhorn_iters,
                           float match_threshold, const mvm_pair_io* pairs, int n_pairs,
                           void* workspace, size_t workspace_bytes, const mvm_matcher_options* opt /* NULL = defaults */,
                           void* stream);

/* mvm_matcher_forward_ex with one image size per view slot, for pairs whose images differ in size (the pairwise
 * matcher normalises each view by its own image, multi_view_matcher.py:165-166, superglue.py:245-246):
 *   view_wh   HOST float[n_views][2]: (width, height) of view slot t, shared by the batch; keypoint k of slot t is
 *             normalised as (k - wh/2) / (0.7 * max(w, h)) in fp32.
 * mvm_matcher_forward and _ex call this with every entry equal to (img_w, img_h); the results are bitwise the same. */
int mvm_matcher_forward_views(const mvm_matcher_weights* w, int batch, int n_views, int n_pad,
                              const int* counts, const float* kpts, const float* kscores,
                              const float* desc, const float* view_wh, int sinkhorn_iters,
                              float match_threshold, const mvm_pair_io* pairs, int n_pairs,
                              void* workspace, size_t workspace_bytes, const mvm_matcher_options* opt /* NULL = defaults */,
                              void* stream);

/* ---- individual stages (exported for stage-parity tests and for callers that only need
 * one stage; same semantics as the fused forward) -------------------------------------- */

/* C[M,N] = act(alpha*[A|A2] W^T + bias) + R, fp32 CUDA cores (superglue.py:51-62). */
int mvm_linear(const float* A, int lda, const float* A2, int lda2, int K1, const float* W,
               int ldw, const float* bias, const float* R, int ldr, float* C, int ldc, int M,
               int N, int K, float alpha, int relu, void* stream);

/* Same contract on the tensor cores (tf32 wgmma, TMA-fed, accumulators in registers).
 * n_pass = 3: fp32-faithful 3xTF32 (operands split hi/lo on chip); n_pass = 1: single-pass TF32.
 *
 * Operand rules of every GEMM entry below and of mvm_linear, checked on the host before any CUDA call; a call that
 * breaks one returns 1 (invalid argument):
 *   M >= 1, N >= 1; K and K1 multiples of the k-block and K >= one k-block: 32 here and in the _presplit / _splitk
 *   entries, 64 in mvm_linear_tc_h16, 16 in mvm_linear; K1 == K without A2, 0 < K1 < K with it;
 *   A, A2 and W (or its planes) 16-byte aligned, lda, lda2 and ldw multiples of 4 (ldw of 8 for the fp16 planes): the
 *   tensor-core kernels load them by TMA, mvm_linear by float4;
 *   tensor cores only: N % 128 == 0, C and R 8-byte aligned with ldc, ldr multiples of 4 (float2 epilogue);
 *   the _splitk entry: C and ws 16-byte aligned, M and N multiples of 128, K of 32 * ksplit, ksplit >= 2.
 * Leading dimensions may exceed the logical widths (column slices of wider buffers).  R may be C itself (an in-place
 * residual, as every GNN layer's mlp.1 does): each output element reads its residual before it is stored. */
int mvm_linear_tc(const float* A, int lda, const float* A2, int lda2, int K1, const float* W,
                  int ldw, const float* bias, const float* R, int ldr, float* C, int ldc, int M,
                  int N, int K, float alpha, int relu, int n_pass, void* stream);

/* The production 3xTF32 path: W given as its two tf32 planes W_hi = rn_tf32(W), W_lo = rn_tf32(W - W_hi)
 * (what packing.py stores next to the raw weights).  Persistent schedule, A split on chip in
 * registers.  Same shape requirements as mvm_linear_tc. */
int mvm_linear_tc_presplit(const float* A, int lda, const float* A2, int lda2, int K1, const float* W_hi,
                           const float* W_lo, int ldw, const float* bias, const float* R, int ldr, float* C,
                           int ldc, int M, int N, int K, float alpha, int relu, void* stream);

/* mvm_linear_tc_presplit for GEMMs with few output tiles and a very long contraction (the weight gradients of training:
 * M, N <= 768, K = all points of the batch): K is cut into ksplit slices computed by different CTAs of the persistent
 * kernel into ws [ksplit, M, N] and summed in fixed order.  M, N multiples of 128, K of 32 * ksplit; no bias / residual. */
int mvm_linear_tc_presplit_splitk(const float* A, int lda, const float* W_hi, const float* W_lo, int ldw, float* C, int ldc,
                                  int M, int N, int K, float alpha, int ksplit, float* ws, void* stream);

/* fp16x3 on the persistent schedule: W16_hi / W16_lo = fp16 planes of wscale * W (hi = fp16(wscale W), lo = fp16(wscale W - hi));
 * K and K1 multiples of 64, N of 128.
 * Range of A, which is split on chip the same way (hi = fp16(a), lo = fp16(a - hi)): hi + lo keeps the 22 bits of the
 * 3xTF32 split only while lo is an fp16 normal, i.e. |a| >= 2^-3; below that lo is exact to 2^-24 absolute, so every
 * element costs up to 2^-25 |w| of error however small it is, and rows made of small elements lose relative accuracy.
 * |a| >= 65520 makes hi infinite: the output is inf or NaN where fp32 is finite.  Use the tf32 entries for operands
 * outside the range given in DESIGN.md section 3. */
int mvm_linear_tc_h16(const float* A, int lda, const float* A2, int lda2, int K1, const void* W16_hi, const void* W16_lo,
                      float wscale, int ldw, const float* bias, const float* R, int ldr, float* C, int ldc, int M, int N, int K,
                      float alpha, int relu, void* stream);

/* The QKV projection of one GNN layer as mvm_matcher_forward_views launches it in math mode 3, with the process
 * defaults of the options: x = X[rows, 256] . W[768, 256]^T + bias, W given as its tf32 planes W_hi / W_lo and,
 * optionally, as the fp16 planes of wscale * W (W16_hi / W16_lo, both or neither; they select fp16x3).  Columns
 * [0, 256) of qkv [rows, 768] receive Q = x.  rows a multiple of n_pad (a multiple of 64).
 *   planes16 = 1 (the fp16x3 attention): K and V leave as half-precision planes of [rows, 256], key-major:
 *     k_hi = fp16_rn(x_K), k_lo = fp16_rn(x_K - k_hi), v_hi / v_lo the same of x_V; the persistent kernel, whose
 *     sum order is that of mvm_linear_tc_h16 (fp16 planes) or mvm_linear_tc_presplit (tf32), so x is their output.
 *   planes16 = 0 (the tf32 attention): qkv[:, 256:512] = rn_tf32(x_K) and k_lo [rows, 256] = rn_tf32(x_K - that);
 *     v_hi [rows / n_pad, 256, n_pad] = rn_tf32 of V^T by view slot, v_lo its remainder; k_hi is not used.  The
 *     kernel mvm_linear_tc_presplit would pick.
 * The K and V thirds of qkv that go to planes are not written. */
int mvm_qkv_projection(const float* X, const float* W_hi, const float* W_lo, const void* W16_hi, const void* W16_lo,
                       float wscale, const float* bias, float* qkv, int rows, int n_pad, int planes16, void* k_hi,
                       void* k_lo, void* v_hi, void* v_lo, void* stream);

/* Math mode of the matcher's GEMMs/attention inside mvm_matcher_forward: 0 = fp32 CUDA cores,
 * 3 = 3xTF32 on the tensor cores (fp32-faithful), 1 = single-pass TF32 (torch 1.10's Ampere default). */
int mvm_set_math_mode(int mode);
int mvm_get_math_mode(void);

/* Multi-head attention over key/value segments (superglue.py:87-109 with the multi-view
 * cross source of multi_view_matcher.py:92-95).  qkv [n_views_total, n_pad, 768]
 * (q|k|v, head-contiguous); view v attends to its own keys (is_cross = 0) or to all other
 * views of its tuple in ascending order (is_cross = 1).  out [n_views_total, n_pad, 256].
 * The three attention entry points below share these conditions, and return 1 (invalid argument) before any CUDA call
 * when the first three fail: 1 <= n_views <= 8 (cross attention: at least 2); every counts[t] in [0, n_pad]; every
 * view with counts[t] >= 1 has at least one source key (in cross attention, some other view has a nonzero count).
 * Rows at and beyond counts[t] of qkv (and of the K / V planes) must be FINITE: masked keys get P = 0, and their V
 * rows are still multiplied by it (0 x inf = NaN); their values do not otherwise reach rows below the counts.  Output
 * rows at and beyond counts[t] are unspecified. */
int mvm_attention(const float* qkv, float* out, int batch, int n_views, int n_pad,
                  const int* counts, int is_cross, void* stream);

/* The same attention on the tensor cores (wgmma/TMA flash kernel).  vt [n_views_total, 256,
 * n_pad] holds V^T per head (written by the QKV GEMM epilogue); the v third of qkv is not read.
 * n_pass == 3 (3xTF32): the k third of qkv and vt must hold rn_tf32 values and klo [rows,256] / vtlo
 * their tf32-rounded remainders (the QKV GEMM epilogue writes all four); NULL for n_pass == 1. */
int mvm_attention_tc(const float* qkv, const float* vt, float* out, int batch, int n_views, int n_pad,
                     const int* counts, int is_cross, int n_pass, const float* klo, const float* vtlo,
                     void* stream);

/* fp32-faithful attention with HALF-PRECISION operand planes (fp16x3: hi = fp16(x), lo = fp16(x - hi); three
 * f16 MMAs per product, half the tensor-pipe time of the tf32 variant at the same 22-bit operand precision).
 * kh, kl, vh, vl [n_views_total * n_pad, 256] are fp16 buffers, point-major like K and V themselves (the QKV GEMM
 * epilogue writes them inside mvm_matcher_forward; V is read as an MN-major tensor-core operand, no transposed copy);
 * the q third of qkv is read as fp32. */
int mvm_attention_h3(const float* qkv, const void* kh, const void* kl, const void* vh, const void* vl, float* out,
                     int batch, int n_views, int n_pad, const int* counts, int is_cross, void* stream);

/* log_optimal_transport (superglue.py:143-172).  scores: [batch, m+1, n+1] buffers whose
 * inner [m,n] block holds the raw scores on entry; on exit the full coupling matrix
 * Z + u + v - norm.  ws: mvm_sinkhorn_workspace_floats(1, batch, max(m,n)) floats.
 * mvm_log_optimal_transport is the production kernel (shared-memory-resident, stabilised scaling
 * domain, FMA inner loops); _logdomain is the same multi-CTA layout iterating in the log domain
 * exactly like the reference; _ref is the one-CTA-per-problem kernel that walks the matrix in
 * L2/HBM (both kept as on-device cross-checks).
 * iters: Sinkhorn iterations, >= 1 (the reference runs 100).  Every entry point, and mvm_matcher_forward with
 * sinkhorn_iters, returns 1 (invalid argument) for iters < 1 without launching anything. */
size_t mvm_sinkhorn_workspace_floats(int n_pairs, int batch, int n_max);
int mvm_log_optimal_transport(float* scores, int batch, int m, int n, float bin_score,
                              int iters, float* ws, void* stream);
/* variant 0 = what mvm_log_optimal_transport picks (one thread-block cluster per problem when m, n <= 1024 and
 * the device can co-schedule the cluster, else the multi-CTA kernel, launched cooperatively); 1 = multi-CTA
 * kernel; 2 / 3 = cluster kernel, one 16-row group per warp (1024 threads) with 8 / 6 of every 16 rows in registers;
 * 4 = cluster kernel, two row groups per warp (512 threads x 128 registers; the default of variant 0).  2-4 fail when
 * the problem does not fit a cluster. */
int mvm_log_optimal_transport_ex(float* scores, int batch, int m, int n, float bin_score, int iters,
                                 float* ws, int variant, void* stream);
/* co-resident clusters the device offers for an m x n problem (0: the cluster kernel is not used) */
int mvm_sinkhorn_max_active_clusters(int m, int n);
int mvm_log_optimal_transport_ref(float* scores, int batch, int m, int n, float bin_score,
                                  int iters, float* ws, void* stream);
int mvm_log_optimal_transport_logdomain(float* scores, int batch, int m, int n, float bin_score,
                                        int iters, float* ws, void* stream);

/* Mutual-nearest-neighbour extraction (multi_view_matcher.py:288-300).
 * ws: 3 * batch * round_up(max(m,n), 64) 4-byte words. */
int mvm_extract_matches(const float* scores, int batch, int m, int n, float match_threshold,
                        int64_t* matches0, int64_t* matches1, float* mscores0,
                        float* mscores1, void* ws, void* stream);

/* ---- two-view pose (pose_optimization/two_view/) ------------------------------------- */

/* estimate_relative_pose_w8pt (estimate_relative_pose.py:84-128): weighted eight-point on
 * matched keypoints, one CTA per batch element, fp64 on chip.
 *   kpts0/1 [B,N,2] pixels (kpts1 already gathered by the matches), intr0/1 [B,4] = fx,fy,cx,cy,
 *   conf [B,N] (un-normalised), T_gt [B,16] target pose for choose_closest (else NULL).
 * Outputs: T021 [B,16] row-major 4x4; kpts{0,1}_norm [B,N,2]; conf_norm [B,N] = conf/(sum+1e-6);
 * pos_depth_mask / inliers [B,N] bytes (inliers only when determine_inliers); F_out [B,9] the
 * normalised essential matrix (may be NULL).  n_valid [B] (device, may be NULL): effective
 * keypoints per item when the arrays are padded to n; success [B] (may be NULL) is 0 for items
 * with fewer than 8 keypoints (the reference returns (None, None), :85-86). */
int mvm_w8pt(const float* kpts0, const float* kpts1, const float* intr0, const float* intr1,
             const float* conf, int batch, int n, const float* T_gt, int choose_closest,
             int determine_inliers, float* T021, float* kpts0_norm, float* kpts1_norm,
             float* conf_norm, unsigned char* pos_depth_mask, unsigned char* inliers,
             float* F_out, const int* n_valid, unsigned char* success, void* stream);

/* Backward of mvm_w8pt with respect to conf: one CTA per batch element, fp64 on chip.  The inputs are
 * mvm_w8pt's (no n_valid: all n keypoints count), its output T021 [B,16], grad_T021 [B,16] and
 * grad_conf_norm [B,N] (the gradient reaching conf_norm; may be NULL).  The kernel re-runs the
 * forward's solve and candidate choice and differentiates the reference's steps in closed form: the
 * smallest right-singular vector of the weighted design matrix, the rank-2 projection,
 * normalize_transformation and decompose_essential_matrix of the chosen candidate.  Output
 * grad_conf [B,N].  Items with fewer than 8 non-zero weights (the vector is not unique), or whose
 * recomputed pose differs from T021 in any bit, get NaN; items with n < 8 get 0. */
int mvm_w8pt_backward(const float* kpts0, const float* kpts1, const float* intr0, const float* intr1,
                      const float* conf, int batch, int n, const float* T_gt, int choose_closest,
                      const float* T021, const float* grad_T021, const float* grad_conf_norm,
                      float* grad_conf, void* stream);

/* estimate_pose (models/models/utils.py:288-312): OpenCV's findEssentialMat(method=RANSAC) + recoverPose, restated
 * (tests/ransac_oracle.py), one CTA per batch element, fp64 on chip, the whole batch in one launch.
 *   kpts0/1 [B,N,2] pixels (kpts1 already gathered by the matches), intr0/1 [B,4] = fx,fy,cx,cy, n_valid [B] (device,
 *   may be NULL = N): effective matches per item.  Points normalised in fp64 as (k - c) / f; inlier threshold
 *   thresh_px / mean(fx0, fy1, fx0, fy1) on OpenCV's error (x2'Ex1)^2 / (Ex1_0^2 + Ex1_1^2 + E'x2_0^2 + E'x2_1^2),
 *   rounded to float; prob / max_iters: OpenCV's confidence and iteration cap (the reference: 0.99999, 1000).
 *   Samples come from splitmix64(seed, hypothesis, draw, attempt), independent of the batch position.
 * Outputs: T021 [B,16] row-major 4x4 (R | unit t of recoverPose; identity when success = 0); kpts{0,1}_norm [B,N,2];
 * inliers [B,N] bytes = the mask recoverPose leaves (RANSAC inliers at depth 0..50 in both cameras: estimate_pose's
 * positional 1e9 is the R output of the recoverPose overload it resolves to, so OpenCV's fixed threshold of 50
 * applies); n_inliers [B] its
 * count; E_out [B,10,9] doubles = findEssentialMat's E (unit Frobenius norm, largest entry positive): the chosen
 * model (n_models = 1) for n_valid > 5, every solution of the five-point problem (n_models <= 10) for n_valid == 5;
 * iterations [B] = hypotheses the sequential RANSAC loop consumed (0 for n_valid <= 5); success [B] = 0 for fewer
 * than 5 matches, when no model reaches 5 inliers, or when no match passes recoverPose (the reference's None).
 * With n_valid == 5 the pose is that of the first solution with a nonzero count (each recoverPose call keeps only the
 * matches the previous one left, so no later count can be larger), and the solutions come in ascending order of the
 * solver's hidden variable, not in OpenCV's order: the 5-match pose is not the reference's.
 * Returns 1 (invalid argument) before launching when a pointer other than n_valid is NULL, batch < 1, n < 1,
 * n > 2048 (the matches of a pair are held in shared memory), thresh_px <= 0, prob outside [0, 1] or max_iters < 1. */
int mvm_ransac_essential(const float* kpts0, const float* kpts1, const float* intr0, const float* intr1,
                         int batch, int n, const int* n_valid, float thresh_px, double prob, int max_iters,
                         unsigned long long seed, float* T021, float* kpts0_norm, float* kpts1_norm,
                         unsigned char* inliers, int* n_inliers, double* E_out, int* n_models,
                         int* iterations, unsigned char* success, void* stream);

/* run_bundle_adjust_2_view -> BundleAdjustGaussNewton2View.run
 * (estimate_relative_pose.py:138-143, bundle_adjust_gauss_newton_2_view.py:127-201):
 * LM with the reference's schedule, Schur-complement step, one CTA per batch element.
 *   conf [B,N]: entries <= 0 are invalid matches; items with <= 6 valid matches get
 *   valid_batch = 0 and T_out = T_init.  pts_ws: B*N*3 doubles.  trace: [B,n_iterations+1]
 *   residual norms per evaluation, or NULL.  n_valid [B] (may be NULL): effective keypoints per
 *   item; mask [B,N] (may be NULL): matches with mask == 0 are dropped (the callers'
 *   `confidence[~pos_depth_mask] = 0`, eval_pairs.py:251-252). */
int mvm_ba2view(const float* kpts0_norm, const float* kpts1_norm, const float* conf,
                const float* T_init, int batch, int n, int n_iterations, float* T_out,
                unsigned char* valid_batch, double* pts_ws, float* trace, const int* n_valid,
                const unsigned char* mask, void* stream);

/* ---- multi-view stage (pose_optimization/multi_view/) -------------------------------- */

/* Order-preserving compaction of the valid matches of every (tuple, pair):
 * valid = matches >= 0 and conf > conf_thresh (bundle_adjust_io.py:66-98, eval_pairs.py:215-222).
 * kpts [B*T, n_pad, 2]; pairs[p].matches_a / .conf are the matcher outputs of that pair.
 * Outputs [B, P, n_pad, ...] zero padded; n_valid [B, P] (device). */
int mvm_gather_matches(const float* kpts, int n_views, int n_pad, const int* counts,
                       const mvm_pair_io* pairs, int n_pairs, int batch, float conf_thresh,
                       float* mkpts_a, float* mkpts_b, float* mconf, int* n_valid, void* stream);

/* Maximum-spanning-tree initial extrinsics (bundle_adjust_io.py:135-172).  T_rel [B,P,16] relative
 * poses a->b, weight [B,P] edge weights (number of matches), success [B,P]; extr [B,T,16] doubles,
 * world->cam, view 0 = identity; on_tree [B,P] (may be NULL). */
int mvm_spanning_tree_init(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch,
                           const float* T_rel, const int* weight, const unsigned char* success,
                           double* extr, unsigned char* on_tree, void* stream);

/* Replacement of the `ba_initializer` binary (ba_init.cpp:77-91: Theia RobustRotationEstimator, initialised
 * from the spanning-tree rotations, then LeastUnsquaredDeviationPositionEstimator; restated in
 * oracle/ba_init.py).  Edges = successful pairs with >= min_inliers inliers or on the spanning tree
 * (bundle_adjust_io.py:181-190; the reference uses min_inliers = 20).  extr_tree / extr_out [B,T,16]
 * doubles (world->cam), inliers [B,P,n_pad] bytes (NULL: edges = success && on_tree, for callers that
 * already hold the edge list, e.g. `ba_init_in.csv`), n_edges_out [B] (may be NULL). */
int mvm_ba_initialize(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch, int n_pad,
                      const double* extr_tree, const float* T_rel, const unsigned char* success,
                      const unsigned char* on_tree, const unsigned char* inliers, int min_inliers,
                      double* extr_out, int* n_edges_out, void* stream);

/* Global bundle adjustment replacing the `bundle_adjuster` binary (ba_problem.cpp:115-157,
 * ba_problem.h:60-151, problem construction bundle_adjust_io.py:193-259): camera 0 fixed, one 3-D
 * point per pairwise match triangulated from extr_init, weights c / (0.5 (sum c + 1e-3)),
 * Ceres-style trust-region LM with a Schur complement, fp64.  xn_a/xn_b [B,P,n_pad,2] normalised
 * observations, conf [B,P,n_pad], n_valid [B,P], extr_init [B,T,16] doubles, extr_out [B,T,16]. */
size_t mvm_mvba_workspace_bytes(int n_views, int n_pairs, int batch, int n_pad);
int mvm_multi_view_ba(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch,
                      int n_pad, const float* xn_a, const float* xn_b, const float* conf,
                      const int* n_valid, const double* extr_init, float* extr_out,
                      int max_iterations, int* iterations_out, double* cost_out, void* workspace,
                      size_t workspace_bytes, void* stream);

/* Same solver for a problem stated the way `ba_in.csv` states it (ba_problem.cpp:8-95, written by
 * write_bundle_adjust_problem, bundle_adjust_io.py:193-259): points_init [B,P,n_pad,3] doubles are the given
 * 3-D points (NULL = triangulate as above); weights_prenormalized != 0: conf already holds the per-observation
 * weights of the file (no re-normalisation); extr_out_f64 [B,T,16] (may be NULL) receives the result in fp64
 * (`ba_out.csv` is written with 12 significant digits, ba_problem.cpp:97-113). */
int mvm_multi_view_ba_ex(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch,
                         int n_pad, const float* xn_a, const float* xn_b, const float* conf,
                         const int* n_valid, const double* extr_init, const double* points_init,
                         int weights_prenormalized, float* extr_out, double* extr_out_f64, int max_iterations,
                         int* iterations_out, double* cost_out, void* workspace, size_t workspace_bytes,
                         void* stream);

/* The general form of the reference's BaProblem for pairwise tracks (ba_problem.h:60-151): one weight per
 * OBSERVATION.  conf [B,P,n_pad] weighs the view-a observation of a point, conf_b the view-b observation
 * (NULL = the same weight, i.e. mvm_multi_view_ba_ex).  With weights_prenormalized != 0 and points_init given this
 * is exactly the problem `ba_in.csv` states -- the reference's own gtest scenes (test_ba_problem.cpp:40-67, weight =
 * depth in each camera) run through it (tests/test_mv_gpu.py). */
int mvm_multi_view_ba_obs(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch,
                          int n_pad, const float* xn_a, const float* xn_b, const float* conf, const float* conf_b,
                          const int* n_valid, const double* extr_init, const double* points_init,
                          int weights_prenormalized, float* extr_out, double* extr_out_f64, int max_iterations,
                          int* iterations_out, double* cost_out, void* workspace, size_t workspace_bytes,
                          void* stream);

/* Two-view DLT of every match of every (tuple, pair) with the given world->cam extrinsics
 * (cv2.triangulatePoints in write_bundle_adjust_problem, bundle_adjust_io.py:219-225).
 * points_out [B,P,n_pad,3] doubles (zero beyond n_valid). */
int mvm_triangulate_pairs(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch, int n_pad,
                          const float* xn_a, const float* xn_b, const int* n_valid, const double* extr,
                          double* points_out, void* stream);

/* ---- SuperPoint front-end (models/models/superpoint.py:147-229; SURVEY.md §8 f-3) --------------------------- */

/* Device pointers.  3x3 convolutions conv1a, conv1b, conv2a, conv2b, conv3a, conv3b, conv4a, conv4b, convPa, convDa in
 * that order, each repacked to [tap = 3*ky + kx][Cin][Cout]; the 1x1 heads convPb [65,256] and convDb [256,256] row-major
 * [out, in] as in the state dict. */
typedef struct mvm_superpoint_weights {
  const float* w[10];
  const float* b[10];
  const float* w_pb; const float* b_pb;
  const float* w_db; const float* b_db;
} mvm_superpoint_weights;

size_t mvm_superpoint_workspace_bytes(int batch, int height, int width);

/* Dense part of SuperPoint.forward (:150-170, :213-216): image [batch, height, width] fp32 (grayscale in [0,1]; any
 * height, width >= 16) -> scores_nms [batch, 8*floor(height/8), 8*floor(width/8)] (softmax keypoint scores after
 * simple_nms, 0 where suppressed) and dense_desc [batch, floor(height/8), floor(width/8), 256] (L2-normalised, channels
 * last).  The three 2x2 pools floor odd sizes like nn.MaxPool2d, so the last height % 8 rows and width % 8 columns of the
 * image have no score, as in the reference (:169-172). */
int mvm_superpoint_dense(const mvm_superpoint_weights* w, const float* image, int batch, int height, int width,
                         int nms_radius, float* scores_nms, float* dense_desc, void* workspace, size_t workspace_bytes,
                         void* stream);

/* sample_descriptors (:86-100) for one image: keypoints [n,2] (x, y) pixels, dense_desc [h, w, 256] of that image ->
 * descriptors [256, n] (bilinear, align_corners=True, L2-normalised). */
int mvm_superpoint_sample(const float* dense_desc, const float* keypoints, int n, int h, int w, float* descriptors,
                          void* stream);

/* Largest max_keypoints mvm_superpoint_select takes: the chosen keypoints are sorted in shared memory. */
#define MVM_SUPERPOINT_MAX_SELECT 16384

/* Keypoint selection of SuperPoint.forward (:181-189) for a whole batch in one launch, without host synchronisation:
 * scores_nms [batch, height, width] as mvm_superpoint_dense writes it (height, width multiples of 8) -> counts [batch]
 * int32 = the number of candidates (score > keypoint_threshold, at least remove_borders pixels inside every edge), and
 * keypoints [batch, max_keypoints, 2] (x, y as float) with scores [batch, max_keypoints]:
 *   - counts[b] <= max_keypoints: every candidate in raster order (what nonzero + top_k_keypoints gives), zeros after;
 *   - counts[b] >  max_keypoints: the max_keypoints largest scores in descending order (top_k_keypoints).  Tie rule:
 *     among equal scores the lower raster index y * width + x comes first, also when the tie straddles the cut.
 * 1 <= max_keypoints <= min(height * width, MVM_SUPERPOINT_MAX_SELECT); scores_nms 16-byte aligned. */
int mvm_superpoint_select(const float* scores_nms, int batch, int height, int width, float keypoint_threshold,
                          int remove_borders, int max_keypoints, float* keypoints, float* scores, int* counts,
                          void* stream);

/* mvm_superpoint_sample for a batch in one launch: dense_desc [batch, h, w, 256], keypoints [batch, max_keypoints, 2],
 * counts [batch] -> descriptors [batch, 256, max_keypoints], the matcher's layout.  The same device code as
 * mvm_superpoint_sample, so the descriptors are bitwise those of the per-image call; columns at or past counts[b] are
 * zero. */
int mvm_superpoint_sample_batch(const float* dense_desc, const float* keypoints, const int* counts, int batch,
                                int max_keypoints, int h, int w, float* descriptors, void* stream);

/* ---- training path (SURVEY.md §8 a20 / f-2): losses, ground-truth matches, train-mode BatchNorm, backward kernels ---- */

/* compute_match_loss (helpers.py:228-241): weighted NLL of the ground-truth assignment on the log-couplings.
 * log_p [bs, ft, ft] (ft = keypoints + 1), gt_indices [bs, 2, ft] int64 (-1 = dustbin = last index), gt_weights
 * [bs, 2, ft]; partial_ws: bs doubles; loss: one float.  Backward: grad_log_p [bs, ft, ft] = d loss / d log_p * grad_loss. */
int mvm_match_loss_forward(const float* log_p, const int64_t* gt_indices, const float* gt_weights, int bs, int ft,
                           double* partial_ws, float* loss, void* stream);
int mvm_match_loss_backward(const int64_t* gt_indices, const float* gt_weights, const float* grad_loss, int bs, int ft,
                            float* grad_log_p, void* stream);

/* BatchNorm1d in TRAINING mode on point-major activations x -> y [rows, C] (row stride ld; y may be x), optionally followed
 * by ReLU -- the MLPs of the train branch (multi_view_matcher.py:8-22 with self.training).  Statistics over the rows whose
 * index inside their n_pad-row view slot is < n_valid, restricted to the slots s with s % slot_mod == slot_rem (1, 0 =
 * every slot; the pairwise train path normalises each view separately); biased variance for the normalisation,
 * running_mean / running_var (may both be NULL) updated with `momentum` and the unbiased variance like
 * torch.nn.BatchNorm1d.  save_stats (may be NULL): [2 C] = mean | 1 / sqrt(var + eps) for the backward.  ws: 3 C doubles. */
int mvm_batchnorm_train(const float* x, float* y, int rows, int C, int ld, int n_pad, int n_valid, int slot_mod,
                        int slot_rem, const float* gamma, const float* beta, float eps, int relu, float* running_mean,
                        float* running_var, float momentum, float* save_stats, double* ws, void* stream);
/* its backward (what autograd computes for BatchNorm1d(+ReLU) in training mode): dy holds the gradient w.r.t. y on entry
 * and the gradient w.r.t. x on return (rows outside the statistics are left untouched); x = the forward's input, y = its
 * output (ReLU mask; may be NULL when relu == 0); dgamma / dbeta [C] are overwritten or, with accumulate != 0, added to.
 * ws: 2 C doubles. */
int mvm_batchnorm_train_backward(const float* x, const float* y, float* dy, int rows, int C, int ld, int n_pad, int n_valid,
                                 int slot_mod, int slot_rem, const float* gamma, const float* save_stats, int relu,
                                 float* dgamma, float* dbeta, int accumulate, double* ws, void* stream);
/* out[c] (+)= sum_r x[r, c]: the bias gradient of a Conv1d(k=1) from the gradient of its output.  ws: C doubles. */
int mvm_colsum(const float* x, int rows, int C, int ld, float* out, int accumulate, double* ws, void* stream);
/* Backward of the ConfidenceMLP of the train branch (stage 2 of training; multi_view_matcher.py:39-53, 302-306), the two
 * steps the GEMM / BatchNorm / colsum kernels do not cover.  Rows are pair-major, r = (p * batch + b) * n + i.  Both are
 * deterministic (fixed summation order, fp64 accumulators, no floating-point atomics).  ws: mvm_conf_backward_ws_doubles(rows).
 * Tail: conf [rows] = the sigmoid outputs, g_conf [rows] = the gradient w.r.t. them, h [rows, 256] = out_f + out_c,
 * w_last [256] -> g_h [rows, 256] = g_conf c (1 - c) w_last, dw_last [256] and db_last [1] (overwritten). */
#define MVM_CONF_MAX_PAIRS 28
size_t mvm_conf_backward_ws_doubles(int rows);
int mvm_conf_tail_backward(const float* conf, const float* g_conf, const float* h, const float* w_last, int rows,
                           float* g_h, float* dw_last, float* db_last, double* ws, size_t ws_doubles, void* stream);
/* Gather transpose: g_x [rows, 512] = the gradient w.r.t. cat[m0, m1g]; g_pre_c0 [rows, 256] = the gradient w.r.t. the
 * pre-BatchNorm output of the score-input layer (K = 1), add [rows] its input, w_c0 [256] its weight; i0 [rows] int64 in
 * [-1, n).  slot_a / slot_b: host arrays (n_pairs <= MVM_CONF_MAX_PAIRS) of the pairs' view slots.  Adds
 * g_x[r, :256] to g_md[b, slot_a[p], i] and g_x[r, 256:] to g_md[b, slot_b[p], i0 (-1 -> n - 1)] (g_md [batch, n_views,
 * n_pad, 256]; rows without a contribution are not written), sum_k g_pre_c0[r, k] w_c0[k] to
 * g_scores[p * batch + b, i, i0 (-1 -> n)] (g_scores [n_pairs * batch, n + 1, n + 1]), and writes dw_c0[k] =
 * sum_r g_pre_c0[r, k] add[r].  The range of i0 is read back (one stream synchronisation) and checked before the
 * gathers launch. */
int mvm_conf_gather_backward(const float* g_x, const float* g_pre_c0, const float* add, const float* w_c0,
                             const int64_t* i0, int n_pairs, int batch, int n, int n_views, int n_pad, const int* slot_a,
                             const int* slot_b, float* g_md, float* g_scores, float* dw_c0, double* ws, size_t ws_doubles,
                             void* stream);
/* A / B hook (process-wide): 0 skips the read-back of the i0 range in mvm_conf_gather_backward (the caller then
 * guarantees i0 in [-1, n)); default 1. */
void mvm_debug_set_conf_i0_check(int on);
/* x [R, C] (row stride ld) -> transposed copies [C, R] (row stride ldo): raw (may be NULL) and / or the tf32 planes
 * hi = rn_tf32(x), lo = rn_tf32(x - hi) (both or neither) that mvm_linear_tc_presplit takes as its W operand: the operand
 * staging of the backward GEMMs (dX = dY W: W^T planes; dW = dY^T X: dY^T raw and X^T planes). */
int mvm_transpose_split(const float* x, int R, int C, int ld, float* raw, float* hi, float* lo, long long ldo, void* stream);

/* Backward of the multi-head attention with multi-view key segments (autograd of superglue.py:87-109 with the sources of
 * multi_view_matcher.py:65-86): qkv [batch*n_views, n_pad, 768] (q | k | v, head-contiguous, as mvm_attention takes it),
 * out = the forward's output and dout the gradient w.r.t. it, both [batch*n_views, n_pad, 256] -> dqkv like qkv.  Rows
 * beyond counts[t] are masked (zero gradient).  ws: 2 * batch*n_views * 4 * n_pad floats.  Deterministic. */
int mvm_attention_backward(const float* qkv, const float* out, const float* dout, float* dqkv, float* ws, int batch,
                           int n_views, int n_pad, const int* counts, int is_cross, void* stream);
/* process default of its kernels: 1 = tile products on the tensor cores (mma.sync TF32 x 3 split passes, default),
 * 0 = fp32 CUDA cores (cross-check) */
int mvm_debug_set_attention_backward_variant(int variant);

/* Every (pair, tuple) score matrix of a call in one launch of the tensor-core GEMM (3xTF32):
 * scores[p][bi] inner [m_p, n_p] block = mdesc[view a_p of tuple bi] . mdesc[view b_p of tuple bi]^T * alpha, written
 * into buffers laid out [batch, m_p + 1, n_p + 1] (multi_view_matcher.py:278-280; the dustbin row / column are not
 * touched).  mdesc: [batch * n_views * n_pad, 256] point-major; hi / lo: scratch of the same size; pa / pb / m / n and
 * scores: host arrays of n_pairs entries (scores: device pointers). */
int mvm_pair_scores(const float* mdesc, float* hi, float* lo, int batch, int n_views, int n_pad, int n_pairs, const int* pa,
                    const int* pb, const int* m, const int* n, float* const* scores, float alpha, void* stream);

/* log_optimal_transport for training (superglue.py:143-172): problem b reads its m x n scores at
 * scores + b * scores_stride with row stride scores_ld (packed [batch, m, n]: ld = n, stride = m n; the inner block of
 * the [batch, m+1, n+1] buffers mvm_pair_scores fills: ld = n + 1, stride = (m+1)(n+1)); alpha = device scalar
 * (bin_score) -> couplings out [batch, m+1, n+1], keeping the potentials of every iteration in pot
 * (mvm_sinkhorn_train_pot_floats floats); the backward turns dZ (gradient w.r.t. the couplings on entry) into the exact
 * gradient of the unrolled iterations w.r.t. the augmented score matrix (inner block = d scores) and adds the dustbin
 * entries to *d_alpha (device double, zeroed by the caller).  m, n <= 1055. */
size_t mvm_sinkhorn_train_pot_floats(int batch, int m, int n, int iters);
int mvm_sinkhorn_train_forward(const float* scores, long long scores_ld, long long scores_stride, const float* alpha, int batch,
                               int m, int n, int iters, float* out, float* pot, void* stream);
int mvm_sinkhorn_train_backward(const float* scores, long long scores_ld, long long scores_stride, const float* alpha,
                                const float* pot, int batch, int m, int n, int iters, float* dZ, double* d_alpha, void* stream);

/* compute_gt_matches_of_image_pair (helpers.py:121-203, with transform_kpts :115-119 and set_weight :205-213):
 * ground-truth assignment of an image pair from depth maps and poses, without the [bs, N, N] error matrix.
 * kpts0/1 [bs, n, 2] pixel x,y (truncated like .long()); K0/K1, T0to1 [bs, 4, 4]; depth0/1 [bs, H, W];
 * indices [bs, 2, n+1] int64 (-1 = unmatched; last entry = dustbin), weights [bs, 2, n+1] (class-balanced, 0 = dropped).
 * A keypoint outside the image is clamped to the border (the reference raises an IndexError there). */
size_t mvm_gt_matches_workspace_bytes(int bs, int n);
int mvm_gt_matches_pair(const float* kpts0, const float* kpts1, const float* K0, const float* K1, const float* T0to1,
                        const float* depth0, const float* depth1, int bs, int n, int H, int W,
                        float max_matched_reproj_err, float min_unmatched_reproj_err, long long* indices,
                        float* weights, void* workspace, size_t workspace_bytes, void* stream);

/* ---- instrumentation ----------------------------------------------------------------- */
/* Kernels launched by the library since load (bench.py's gpu_launches). */
unsigned long long mvm_launch_count(void);
/* Optional CUDA-event profiler: when enabled every kernel-class scope is bracketed by events on
 * its launching stream; collect() returns summed milliseconds / scope counts per class
 * (0 gemm, 1 attention, 2 sinkhorn, 3 score gemm, 4 match extraction, 5 confidence head,
 * 6 keypoint encoder, 7 w8pt, 8 two-view BA, 9 multi-view BA, 10 misc). */
void mvm_profile_enable(int on);
int mvm_profile_collect(double* ms_per_tag, int* n_per_tag, int n_tags);

/* ---- debug / A-B hooks (process-wide defaults; not used on the mvm_matcher_forward_ex call path) ------------ */
void mvm_debug_set_score_kernel(int tensor_cores);      /* default of mvm_matcher_options.score_kernel */
void mvm_debug_set_gemm_tile(int bn);                   /* default of .gemm_tile (128 | 256) */
void mvm_debug_set_gemm_kernel(int persistent);         /* default of .gemm_kernel */
void mvm_debug_set_attention_split(int fp16);           /* default of .attention_split */
void mvm_debug_set_attention_h3_variant(int v);         /* fp16-plane attention kernel: 1 = one softmax group, two CTAs per SM
                                                          (default), 0 = two softmax groups, one CTA per SM (A/B comparison) */
void mvm_debug_set_gemm_split(int fp16);                /* default of .gemm_split */
/* clock64 phase traces of CTA 0 (device buffers of 8 / 6 / 8 long long; NULL switches the trace off) */
void mvm_debug_set_attention_timing(long long* buf);
void mvm_debug_set_sinkhorn_timing(long long* buf);
void mvm_debug_set_mvba_timing(long long* buf);

/* Library/build info: returns "mvm_b200 <version> sm_90a". */
const char* mvm_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MVM_B200_H */
