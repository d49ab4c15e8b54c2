// Weighted eight-point relative pose, one CTA per pair problem, fp64 register/shared-memory
// resident (no cuSOLVER).  Reference: estimate_relative_pose_w8pt and find_fundamental,
// pose_optimization/two_view/estimate_relative_pose.py:34-128, with the kornia 0.7.0 helpers
// restated in SURVEY.md appendix A.5 (normalize_points, normalize_transformation,
// motion_from_essential[_choose_solution], triangulate_points, depth_from_point,
// symmetrical_epipolar_distance).
//
// Differences by design (same mathematics):
//  * the N x 9 weighted design matrix is never materialised (nor the [B,N,N] diag_embed of
//    :68-69): its 9x9 normal matrix is accumulated in fp64 and the smallest eigenvector taken
//    with a warp-cooperative Jacobi sweep == last right-singular vector of X (:72-73)
//  * 3x3 SVDs via Jacobi on E^T E; the (U, V) sign/det canonicalisation of kornia's
//    decompose_essential_matrix is applied analytically (u2 = u0 x u1, v2 = v0 x v1)
//  * the four candidate triangulations of the cheirality vote are reused for pos_depth_mask.
//
// mvm_w8pt_backward differentiates the reference's computation (the torch.svd steps of find_fundamental and
// decompose_essential_matrix) with respect to the confidences, in closed form: it re-runs the forward's solve and
// candidate choice with the same device code, then chains the 3x3 steps on one thread and the per-match
// eigenvector gradient across the block.
#include "../../include/mvm_b200.h"
#include "common.cuh"
#include "linalg_small.cuh"

namespace {

constexpr int NT = 256;

__device__ __forceinline__ double block_sum(double v, double* red) {
  // red: >= 8 doubles of shared scratch
  v = warp_sum_d(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < NT / 32; ++w) s += red[w];
  return s;
}

struct W8ptArgs {
  const float* kpts0; const float* kpts1;   // [B,N,2] pixels
  const float* intr0; const float* intr1;   // [B,4]: fx, fy, cx, cy
  const float* conf;                        // [B,N]
  const float* T_gt;                        // [B,16] or null (choose_closest)
  const int* n_valid;                       // [B] effective keypoints per item (<= N) or null
  unsigned char* success;                   // [B] or null: 0 when an item has < 8 keypoints
  int N;
  int choose_closest, determine_inliers;
  float* T021;                              // [B,16]
  float* k0n; float* k1n;                   // [B,N,2]
  float* conf_n;                            // [B,N]
  unsigned char* pos_depth;                 // [B,N]
  unsigned char* inliers;                   // [B,N] or null
  float* F_out;                             // [B,9] or null
};

// SVD pieces of a 3x3 via eigen-decomposition of M^T M: V (columns sorted by descending
// singular value) and the singular values.
__device__ void svd3_V(const double M[9], double V[9], double sig[3]) {
  double a[3][3], v[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += M[k * 3 + i] * M[k * 3 + j];
      a[i][j] = s;
    }
  jacobi_eig_reg<3, 10>(a, v);
  int o[3] = {0, 1, 2};
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2 - i; ++j)
      if (a[o[j]][o[j]] < a[o[j + 1]][o[j + 1]]) { const int t = o[j]; o[j] = o[j + 1]; o[j + 1] = t; }
  for (int c = 0; c < 3; ++c) {
    sig[c] = sqrt(fmax(a[o[c]][o[c]], 0.0));
    for (int r = 0; r < 3; ++r) V[r * 3 + c] = v[r][o[c]];
  }
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

__device__ void mat3mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += A[i * 3 + k] * B[k * 3 + j];
      C[i * 3 + j] = s;
    }
}

__device__ double rot_err(const double* R, const float* Tg) {
  // compute_pose_error.py:3-12: acos(clamp((tr(R0^T R1) - 1) / 2))
  double tr = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) tr += R[k * 3 + i] * (double)Tg[k * 4 + i];
  double c = (tr - 1.0) * 0.5;
  c = fmin(1.0, fmax(-1.0, c));
  return fabs(acos(c));
}
__device__ double transl_err(const double* t, const float* Tg) {
  // compute_pose_error.py:14-21
  const double g[3] = {(double)Tg[3], (double)Tg[7], (double)Tg[11]};
  const double n = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]) * sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
  if (!(n > 1e-6)) return 0.0;
  double c = (t[0] * g[0] + t[1] * g[1] + t[2] * g[2]) / n;
  c = fmin(1.0, fmax(-1.0, c));
  return fabs(acos(c));
}

// Block state of one item, shared by the forward and the backward kernel.  The backward re-runs the
// forward's solve and candidate choice with the same code, so it differentiates exactly the pose the
// forward returned.
struct W8ptSmem {
  double red[NT / 32];
  double M[81], V[81];            // normal matrix (eigenvalues on the diagonal after Jacobi), eigenvectors
  double part[NT / 32][45];
  double E[9], R[2][9], t[3];     // normalised essential matrix, candidate rotations, translation
  int cnt[4];
  int choice;
  int mi;                         // column of V taken as F
  double Fv[9], Fsig[3];          // 3x3 SVD of F: right singular vectors (columns), singular values
  double Epre[9];                 // T2^T Fp T1 before normalize_transformation
  double U[9], Vc[9], se[3];      // canonical U, V of E (columns, det +1) and its singular values
};

// Normalised camera coordinates and weight of match i.  The forward reads back what it wrote; the
// backward recomputes them with the forward's fp32 expressions, which gives the same bits.
struct W8ptPtsStored {
  const float* k0n; const float* k1n; const float* cn;
  __device__ __forceinline__ void xy(int i, float& x0, float& y0, float& x1, float& y1) const {
    x0 = k0n[2 * i]; y0 = k0n[2 * i + 1]; x1 = k1n[2 * i]; y1 = k1n[2 * i + 1];
  }
  __device__ __forceinline__ float w(int i) const { return cn[i]; }
};
struct W8ptPtsRecomputed {
  const float* k0; const float* k1; const float* cf;
  float fx0, fy0, cx0, cy0, fx1, fy1, cx1, cy1, sum_conf;
  __device__ __forceinline__ void xy(int i, float& x0, float& y0, float& x1, float& y1) const {
    x0 = (k0[2 * i] - cx0) / fx0; y0 = (k0[2 * i + 1] - cy0) / fy0;
    x1 = (k1[2 * i] - cx1) / fx1; y1 = (k1[2 * i + 1] - cy1) / fy1;
  }
  __device__ __forceinline__ float w(int i) const { return cf[i] / sum_conf; }
};

// Hartley scales, the weighted normal matrix and its eigenvectors, F, its rank-2 projection, E and
// the candidate decomposition (:53-82, kornia decompose_essential_matrix).  Needs the point means.
template <class Pts>
__device__ __forceinline__ void w8pt_solve(const Pts& pts, int N, double mx0, double my0, double mx1,
                                           double my1, double& sc0, double& sc1, W8ptSmem& s) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // Hartley normalisation (kornia normalize_points): scale = sqrt(2) / (mean dist + 1e-8)
  double d0 = 0, d1 = 0;
  for (int i = tid; i < N; i += NT) {
    float px0, py0, px1, py1;
    pts.xy(i, px0, py0, px1, py1);
    const double ax = px0 - mx0, ay = py0 - my0;
    const double bx = px1 - mx1, by = py1 - my1;
    d0 += sqrt(ax * ax + ay * ay);
    d1 += sqrt(bx * bx + by * by);
  }
  d0 = block_sum(d0, s.red) / N; d1 = block_sum(d1, s.red) / N;
  sc0 = sqrt(2.0) / (d0 + 1e-8); sc1 = sqrt(2.0) / (d1 + 1e-8);

  // 9x9 normal matrix of the weighted design rows (:65-69), fp64, upper triangle (45 entries)
  double acc[45];
#pragma unroll
  for (int e = 0; e < 45; ++e) acc[e] = 0.0;
  for (int i = tid; i < N; i += NT) {
    float px0, py0, px1, py1;
    pts.xy(i, px0, py0, px1, py1);
    const double x1 = sc0 * (px0 - mx0), y1 = sc0 * (py0 - my0);
    const double x2 = sc1 * (px1 - mx1), y2 = sc1 * (py1 - my1);
    const double w = (double)pts.w(i);
    const double r[9] = {w * x2 * x1, w * x2 * y1, w * x2, w * y2 * x1, w * y2 * y1, w * y2, w * x1, w * y1, w};
    int e = 0;
#pragma unroll
    for (int p = 0; p < 9; ++p)
#pragma unroll
      for (int q = p; q < 9; ++q) acc[e++] += r[p] * r[q];
  }
#pragma unroll
  for (int e = 0; e < 45; ++e) acc[e] = warp_sum_d(acc[e]);
  if (lane == 0)
#pragma unroll
    for (int e = 0; e < 45; ++e) s.part[warp][e] = acc[e];
  __syncthreads();
  if (tid < 45) {
    double sum = 0.0;
    for (int w = 0; w < NT / 32; ++w) sum += s.part[w][tid];
    // unpack upper-triangle index tid -> (p,q)
    int p = 0, e = tid;
    while (e >= 9 - p) { e -= 9 - p; ++p; }
    const int q = p + e;
    s.M[p * 9 + q] = sum;
    s.M[q * 9 + p] = sum;
  }
  __syncthreads();
  if (warp == 0) jacobi_eig9_warp(s.M, s.V, lane);
  __syncthreads();

  if (tid == 0) {
    int mi = 0;
    for (int i = 1; i < 9; ++i)
      if (s.M[i * 9 + i] < s.M[mi * 9 + mi]) mi = i;
    if (N == 8) {
      // The reference takes V[..., -1] of the REDUCED svd(X) (:72-73).  With exactly 8 matches X is 8 x 9, the
      // reduced V has only 8 columns and its last one belongs to the smallest of the 8 NON-ZERO singular values --
      // not to the null vector.  Reproduce that: second-smallest eigenvalue of the 9 x 9 normal matrix.
      int m2 = mi == 0 ? 1 : 0;
      for (int i = 0; i < 9; ++i)
        if (i != mi && s.M[i * 9 + i] < s.M[m2 * 9 + m2]) m2 = i;
      mi = m2;
    }
    s.mi = mi;
    double F[9];
    for (int i = 0; i < 9; ++i) F[i] = s.V[i * 9 + mi];
    // rank-2 projection (:76-79): F - (F v3) v3^T with v3 the smallest right-singular vector
    double V[9], sig[3];
    svd3_V(F, V, sig);
    for (int i = 0; i < 9; ++i) s.Fv[i] = V[i];
    for (int i = 0; i < 3; ++i) s.Fsig[i] = sig[i];
    double Fv[3];
    for (int i = 0; i < 3; ++i) Fv[i] = F[i * 3 + 0] * V[2] + F[i * 3 + 1] * V[5] + F[i * 3 + 2] * V[8];
    double Fp[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Fp[i * 3 + j] = F[i * 3 + j] - Fv[i] * V[j * 3 + 2];
    // de-normalise (:80): T2^T Fp T1 with T = [[s,0,-s mx],[0,s,-s my],[0,0,1]]
    const double T1[9] = {sc0, 0, -sc0 * mx0, 0, sc0, -sc0 * my0, 0, 0, 1};
    const double T2t[9] = {sc1, 0, 0, 0, sc1, 0, -sc1 * mx1, -sc1 * my1, 1};
    double tmp[9], E[9];
    mat3mul(Fp, T1, tmp);
    mat3mul(T2t, tmp, E);
    for (int i = 0; i < 9; ++i) s.Epre[i] = E[i];
    // normalize_transformation (:82)
    if (fabs(E[8]) > 1e-8) {
      const double inv = 1.0 / (E[8] + 1e-8);
      for (int i = 0; i < 9; ++i) E[i] *= inv;
    }
    for (int i = 0; i < 9; ++i) s.E[i] = E[i];
    // motion_from_essential: E = U S V^T; canonical U = [u0,u1,u0xu1], V = [v0,v1,v0xv1]
    double Ve[9], se[3];
    svd3_V(E, Ve, se);
    double u0[3], u1[3], u2[3], v0[3] = {Ve[0], Ve[3], Ve[6]}, v1[3] = {Ve[1], Ve[4], Ve[7]}, v2[3];
    for (int i = 0; i < 3; ++i) {
      u0[i] = (E[i * 3] * v0[0] + E[i * 3 + 1] * v0[1] + E[i * 3 + 2] * v0[2]) / se[0];
      u1[i] = (E[i * 3] * v1[0] + E[i * 3 + 1] * v1[1] + E[i * 3 + 2] * v1[2]) / se[1];
    }
    // re-orthonormalise u1 against u0 (guards tiny fp64 drift)
    double dot = u0[0] * u1[0] + u0[1] * u1[1] + u0[2] * u1[2];
    for (int i = 0; i < 3; ++i) u1[i] -= dot * u0[i];
    double nu = sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
    for (int i = 0; i < 3; ++i) u1[i] /= nu;
    cross3(u0, u1, u2);
    cross3(v0, v1, v2);
    // R1 = U W V^T, R2 = U W^T V^T, W = [[0,-1,0],[1,0,0],[0,0,1]]
    // U W = [u1, -u0, u2];  U W^T = [-u1, u0, u2]
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        s.R[0][i * 3 + j] = u1[i] * v0[j] - u0[i] * v1[j] + u2[i] * v2[j];
        s.R[1][i * 3 + j] = -u1[i] * v0[j] + u0[i] * v1[j] + u2[i] * v2[j];
      }
    for (int i = 0; i < 3; ++i) {
      s.t[i] = u2[i];
      s.U[i * 3 + 0] = u0[i]; s.U[i * 3 + 1] = u1[i]; s.U[i * 3 + 2] = u2[i];
      s.Vc[i * 3 + 0] = v0[i]; s.Vc[i * 3 + 1] = v1[i]; s.Vc[i * 3 + 2] = v2[i];
      s.se[i] = se[i];
    }
    for (int c = 0; c < 4; ++c) s.cnt[c] = 0;
  }
  __syncthreads();
}

// Candidate choice -> s.choice: closest to the target pose (:95-107) or the cheirality vote (:109).
template <class Pts>
__device__ __forceinline__ void w8pt_choose(const Pts& pts, int N, int choose_closest, const float* Tg,
                                            W8ptSmem& s) {
  const int tid = threadIdx.x, lane = tid & 31;
  if (choose_closest) {
    // training branch (:95-107): candidate closest to the target pose
    if (tid == 0) {
      double best = 1e6;
      int bc = -1;
      for (int c = 0; c < 4; ++c) {
        const double* R = s.R[c >> 1];
        const double sg = (c & 1) ? -1.0 : 1.0;
        const double t[3] = {sg * s.t[0], sg * s.t[1], sg * s.t[2]};
        const double err = rot_err(R, Tg) + transl_err(t, Tg);
        if (err < best) { best = err; bc = c; }
      }
      s.choice = bc;
    }
    __syncthreads();
  } else {
    // cheirality vote (:109): triangulate every point for the 4 candidates
    int cnt[4] = {0, 0, 0, 0};
    for (int i = tid; i < N; i += NT) {
      float px0, py0, px1, py1;
      pts.xy(i, px0, py0, px1, py1);
      const double x1 = px0, y1 = py0, x2 = px1, y2 = py1;
#pragma unroll 1
      for (int c = 0; c < 4; ++c) {
        const double* R = s.R[c >> 1];
        const double sg = (c & 1) ? -1.0 : 1.0;
        const double t[3] = {sg * s.t[0], sg * s.t[1], sg * s.t[2]};
        double X[3];
        triangulate_dlt(R, t, x1, y1, x2, y2, X);
        const double dpt1 = X[2];
        const double dpt2 = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2];
        if (dpt1 > 0.0 && dpt2 > 0.0) cnt[c]++;
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      int v = cnt[c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) atomicAdd(&s.cnt[c], v);
    }
    __syncthreads();
    if (tid == 0) {
      int bc = 0;
      for (int c = 1; c < 4; ++c)
        if (s.cnt[c] > s.cnt[bc]) bc = c;   // first maximum wins (torch.max)
      s.choice = bc;
    }
    __syncthreads();
  }
}

// The fp32 T021 of the chosen candidate, as the forward writes it.
__device__ __forceinline__ void w8pt_pose(const W8ptSmem& s, float* T) {
  const int c = s.choice;
  if (c < 0) {  // no candidate beat 1e6: identity (:98)
    for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.f : 0.f;
    return;
  }
  const double* R = s.R[c >> 1];
  const double sg = (c & 1) ? -1.0 : 1.0;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T[i * 4 + j] = (float)R[i * 3 + j];
    T[i * 4 + 3] = (float)(sg * s.t[i]);
  }
  T[12] = 0.f; T[13] = 0.f; T[14] = 0.f; T[15] = 1.f;
}

// Two CTAs per SM (128 registers): a batch larger than the SM count, e.g. the 140 pairs of a cfg3 step, runs in one
// wave; at one CTA per SM the launch takes 1.55x as long on an H100.
__global__ void __launch_bounds__(NT, 2) w8pt_kernel(W8ptArgs a) {
  __shared__ W8ptSmem s;

  const int b = blockIdx.x, NS = a.N, tid = threadIdx.x;
  const int N = a.n_valid ? min(max(a.n_valid[b], 0), NS) : NS;   // effective count; NS = row stride
  const float* k0 = a.kpts0 + (long long)b * NS * 2;
  const float* k1 = a.kpts1 + (long long)b * NS * 2;
  const float* cf = a.conf + (long long)b * NS;
  const float fx0 = a.intr0[b * 4 + 0], fy0 = a.intr0[b * 4 + 1], cx0 = a.intr0[b * 4 + 2], cy0 = a.intr0[b * 4 + 3];
  const float fx1 = a.intr1[b * 4 + 0], fy1 = a.intr1[b * 4 + 1], cx1 = a.intr1[b * 4 + 2], cy1 = a.intr1[b * 4 + 3];
  float* k0n = a.k0n + (long long)b * NS * 2;
  float* k1n = a.k1n + (long long)b * NS * 2;
  float* cn = a.conf_n + (long long)b * NS;
  // padding rows beyond the effective count: neutral outputs
  for (int i = N + tid; i < NS; i += NT) {
    k0n[2 * i] = 0.f; k0n[2 * i + 1] = 0.f; k1n[2 * i] = 0.f; k1n[2 * i + 1] = 0.f; cn[i] = 0.f;
    a.pos_depth[(long long)b * NS + i] = 0;
    if (a.inliers) a.inliers[(long long)b * NS + i] = 0;
  }
  if (N < 8) {   // fewer than 8 keypoints: no estimate (estimate_relative_pose.py:85-86)
    if (tid < 16) a.T021[b * 16 + tid] = (tid % 5 == 0) ? 1.f : 0.f;
    // the keypoints are still normalised: the multi-view BA takes every pair's matches, estimated or not
    // (write_bundle_adjust_problem, bundle_adjust_io.py:193-225), from these buffers
    for (int i = tid; i < N; i += NT) {
      k0n[2 * i] = (k0[2 * i] - cx0) / fx0; k0n[2 * i + 1] = (k0[2 * i + 1] - cy0) / fy0;
      k1n[2 * i] = (k1[2 * i] - cx1) / fx1; k1n[2 * i + 1] = (k1[2 * i + 1] - cy1) / fy1;
      cn[i] = 0.f;
      a.pos_depth[(long long)b * NS + i] = 0;
      if (a.inliers) a.inliers[(long long)b * NS + i] = 0;
    }
    if (tid == 0 && a.success) a.success[b] = 0;
    if (tid < 9 && a.F_out) a.F_out[b * 9 + tid] = 0.f;
    return;
  }
  if (tid == 0 && a.success) a.success[b] = 1;

  // confidence normalisation (:87-88) and camera normalisation (:9-14, :89-90), fp32 like the ref
  double csum = 0.0;
  for (int i = tid; i < N; i += NT) csum += (double)cf[i];
  csum = block_sum(csum, s.red);
  const float sum_conf = (float)csum + 1e-6f;
  double mx0 = 0, my0 = 0, mx1 = 0, my1 = 0;
  for (int i = tid; i < N; i += NT) {
    const float x0 = (k0[2 * i] - cx0) / fx0, y0 = (k0[2 * i + 1] - cy0) / fy0;
    const float x1 = (k1[2 * i] - cx1) / fx1, y1 = (k1[2 * i + 1] - cy1) / fy1;
    k0n[2 * i] = x0; k0n[2 * i + 1] = y0; k1n[2 * i] = x1; k1n[2 * i + 1] = y1;
    cn[i] = cf[i] / sum_conf;
    mx0 += x0; my0 += y0; mx1 += x1; my1 += y1;
  }
  mx0 = block_sum(mx0, s.red) / N; my0 = block_sum(my0, s.red) / N;
  mx1 = block_sum(mx1, s.red) / N; my1 = block_sum(my1, s.red) / N;

  const W8ptPtsStored pts{k0n, k1n, cn};
  double sc0, sc1;
  w8pt_solve(pts, N, mx0, my0, mx1, my1, sc0, sc1, s);
  if (tid < 9 && a.F_out) a.F_out[b * 9 + tid] = (float)s.E[tid];
  w8pt_choose(pts, N, a.choose_closest, a.choose_closest ? a.T_gt + b * 16 : nullptr, s);

  if (tid == 0) w8pt_pose(s, a.T021 + b * 16);
  __syncthreads();

  // positive-depth mask with the chosen pose (:113-118) and inliers (:121-125)
  {
    // the reference triangulates with the fp32 pose it just wrote
    double R[9], t[3];
    const float* T = a.T021 + b * 16;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) R[i * 3 + j] = (double)T[i * 4 + j];
      t[i] = (double)T[i * 4 + 3];
    }
    const double thresh = 3.0 / (((double)fx0 + fy0 + fx1 + fy1) / 4.0);
    for (int i = tid; i < N; i += NT) {
      const double x1 = k0n[2 * i], y1 = k0n[2 * i + 1], x2 = k1n[2 * i], y2 = k1n[2 * i + 1];
      double X[3];
      triangulate_dlt(R, t, x1, y1, x2, y2, X);
      const double dpt2 = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2];
      const bool pos = X[2] > 0.0 && dpt2 > 0.0;
      a.pos_depth[(long long)b * NS + i] = pos ? 1 : 0;
      if (a.inliers) {
        const double* E = s.E;
        const double l1[3] = {E[0] * x1 + E[1] * y1 + E[2], E[3] * x1 + E[4] * y1 + E[5], E[6] * x1 + E[7] * y1 + E[8]};
        const double l2[3] = {E[0] * x2 + E[3] * y2 + E[6], E[1] * x2 + E[4] * y2 + E[7], E[2] * x2 + E[5] * y2 + E[8]};
        const double num = x2 * l1[0] + y2 * l1[1] + l1[2];
        const double d = num * num * (1.0 / (l1[0] * l1[0] + l1[1] * l1[1]) + 1.0 / (l2[0] * l2[0] + l2[1] * l2[1]));
        a.inliers[(long long)b * NS + i] = (pos && sqrt(d) <= thresh) ? 1 : 0;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Backward: d(T021, conf_norm) -> d conf.  Differentiates what the reference computes (its torch.svd
// steps), not the forward's Jacobi iterations; every step below is a closed form of fp64 scalars.
// ------------------------------------------------------------------------------------------------
struct W8ptBwdArgs {
  const float* kpts0; const float* kpts1; const float* intr0; const float* intr1; const float* conf;
  const float* T_gt;                        // [B,16] or null
  const float* T021;                        // [B,16] the forward's pose
  const float* gT;                          // [B,16]
  const float* g_cn;                        // [B,N] or null
  float* g_conf;                            // [B,N]
  int N, choose_closest;
};

// Gradient of a loss through the eigenvector v_j of a symmetric n x n matrix A = sum_i x_i x_i^T
// (or F^T F): the coefficients c_k = (v_k . g_v) / (lam_k - lam_j), k != j, so that
// g_A = -sum_k c_k sym(v_k v_j^T).
template <int n>
__device__ __forceinline__ void eigvec_coeffs(const double* V, int ldv, const double* lam, int j,
                                              const double* gv, double* c) {
  for (int k = 0; k < n; ++k) {
    if (k == j) { c[k] = 0.0; continue; }
    double d = 0.0;
    for (int i = 0; i < n; ++i) d += V[i * ldv + k] * gv[i];
    c[k] = d / (lam[k] - lam[j]);
  }
}

// 3x3 steps of the backward (tid 0): d T021 -> d E (decompose_essential_matrix) -> d Epre
// (normalize_transformation) -> d Fp (T2^T Fp T1) -> d F (rank-2 projection).  Returns g_f [9].
__device__ void w8pt_backward_3x3(const W8ptSmem& s, const float* gT, double sc0, double sc1, double mx0,
                                  double my0, double mx1, double my1, double gf[9]) {
  const int c = s.choice;
  for (int i = 0; i < 9; ++i) gf[i] = 0.0;
  if (c < 0) return;   // identity pose: no dependence on the confidences
  const double sg = (c & 1) ? -1.0 : 1.0;
  // decompose_essential_matrix.  With U^T dU = Omega_U, V^T dV = Omega_V (skew) and
  // P = U^T dE V:  U^T dR V = Omega_U W - W Omega_V and U^T du2 = Omega_U e2, where
  // Omega_U[p][q] = (P_pq s_q + P_qp s_p) / (s_q^2 - s_p^2), Omega_V[p][q] = (P_pq s_p + P_qp s_q) / (s_q^2 - s_p^2).
  // E has rank 2 (s_2 = 0); the (0,1) pair enters R only through (P01 - P10) / (s0 + s1), which stays finite
  // when s0 = s1 (an exact essential matrix).
  const double* U = s.U;
  const double* V = s.Vc;
  double Gb[9], h[3];
  for (int p = 0; p < 3; ++p) {
    for (int q = 0; q < 3; ++q) {
      double acc = 0.0;
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) acc += U[i * 3 + p] * (double)gT[i * 4 + j] * V[j * 3 + q];
      Gb[p * 3 + q] = acc;
    }
    double acc = 0.0;
    for (int i = 0; i < 3; ++i) acc += U[i * 3 + p] * sg * (double)gT[i * 4 + 3];
    h[p] = acc;
  }
  // W for R1 = U W V^T, W^T for R2
  const double W0[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1};
  double W[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) W[i * 3 + j] = (c >> 1) ? W0[j * 3 + i] : W0[i * 3 + j];
  // <Gb, Omega_U W - W Omega_V> = <Gb W^T, Omega_U> - <W^T Gb, Omega_V>
  double A[9], Bm[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double sa = 0.0, sb = 0.0;
      for (int k = 0; k < 3; ++k) { sa += Gb[i * 3 + k] * W[j * 3 + k]; sb += W[k * 3 + i] * Gb[k * 3 + j]; }
      A[i * 3 + j] = sa; Bm[i * 3 + j] = sb;
    }
  const double al01 = A[1] - A[3];
  const double al02 = A[2] - A[6] + h[0], al12 = A[5] - A[7] + h[1];
  const double be02 = -(Bm[2] - Bm[6]), be12 = -(Bm[5] - Bm[7]);
  const double s0 = s.se[0], s1 = s.se[1];
  double Q[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  Q[1] = al01 / (s0 + s1);
  Q[3] = -al01 / (s0 + s1);
  Q[2] = -be02 / s0; Q[6] = -al02 / s0;
  Q[5] = -be12 / s1; Q[7] = -al12 / s1;
  double gE[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double acc = 0.0;
      for (int p = 0; p < 3; ++p)
        for (int q = 0; q < 3; ++q) acc += U[i * 3 + p] * Q[p * 3 + q] * V[j * 3 + q];
      gE[i * 3 + j] = acc;
    }
  // normalize_transformation: E = Epre / (Epre[8] + 1e-8) when |Epre[8]| > 1e-8
  if (fabs(s.Epre[8]) > 1e-8) {
    const double d = s.Epre[8] + 1e-8;
    double dot = 0.0;
    for (int i = 0; i < 9; ++i) dot += gE[i] * s.Epre[i];
    for (int i = 0; i < 9; ++i) gE[i] /= d;
    gE[8] -= dot / (d * d);
  }
  // Epre = T2^T Fp T1  ->  g_Fp = T2 g_E T1^T
  const double T1[9] = {sc0, 0, -sc0 * mx0, 0, sc0, -sc0 * my0, 0, 0, 1};
  const double T2[9] = {sc1, 0, -sc1 * mx1, 0, sc1, -sc1 * my1, 0, 0, 1};
  double T1t[9], tmp[9], G[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) T1t[i * 3 + j] = T1[j * 3 + i];
  mat3mul(gE, T1t, tmp);
  mat3mul(T2, tmp, G);
  // Fp = F (I - v3 v3^T), v3 the smallest right-singular vector of F, i.e. the eigenvector of F^T F with the
  // smallest eigenvalue: g_F = G (I - v3 v3^T) + F (g_A + g_A^T), g_v3 = -(F^T G + G^T F) v3.
  double F[9];
  for (int i = 0; i < 9; ++i) F[i] = s.V[i * 9 + s.mi];
  const double* Fv = s.Fv;
  const double v3[3] = {Fv[2], Fv[5], Fv[8]};
  double Fv3[3], Gv3[3];
  for (int i = 0; i < 3; ++i) {
    Fv3[i] = F[i * 3] * v3[0] + F[i * 3 + 1] * v3[1] + F[i * 3 + 2] * v3[2];
    Gv3[i] = G[i * 3] * v3[0] + G[i * 3 + 1] * v3[1] + G[i * 3 + 2] * v3[2];
  }
  double gv3[3];
  for (int j = 0; j < 3; ++j) {
    double acc = 0.0;
    for (int i = 0; i < 3; ++i) acc += F[i * 3 + j] * Gv3[i] + G[i * 3 + j] * Fv3[i];
    gv3[j] = -acc;
  }
  const double lam[3] = {s.Fsig[0] * s.Fsig[0], s.Fsig[1] * s.Fsig[1], s.Fsig[2] * s.Fsig[2]};
  double ck[3];
  eigvec_coeffs<3>(Fv, 3, lam, 2, gv3, ck);
  // g_A + g_A^T = -sum_k c_k (v_k v3^T + v3 v_k^T)
  double gA2[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double acc = 0.0;
      for (int k = 0; k < 2; ++k) acc -= ck[k] * (Fv[i * 3 + k] * v3[j] + v3[i] * Fv[j * 3 + k]);
      gA2[i * 3 + j] = acc;
    }
  mat3mul(F, gA2, tmp);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) gf[i * 3 + j] = G[i * 3 + j] - Gv3[i] * v3[j] + tmp[i * 3 + j];
}

__global__ void __launch_bounds__(NT) w8pt_backward_kernel(W8ptBwdArgs a) {
  __shared__ W8ptSmem s;
  __shared__ double s_ck[9];
  __shared__ int s_bad;

  const int b = blockIdx.x, N = a.N, tid = threadIdx.x;
  const float* k0 = a.kpts0 + (long long)b * N * 2;
  const float* k1 = a.kpts1 + (long long)b * N * 2;
  const float* cf = a.conf + (long long)b * N;
  const float* gcn = a.g_cn ? a.g_cn + (long long)b * N : nullptr;
  float* gc = a.g_conf + (long long)b * N;
  const float fx0 = a.intr0[b * 4 + 0], fy0 = a.intr0[b * 4 + 1], cx0 = a.intr0[b * 4 + 2], cy0 = a.intr0[b * 4 + 3];
  const float fx1 = a.intr1[b * 4 + 0], fy1 = a.intr1[b * 4 + 1], cx1 = a.intr1[b * 4 + 2], cy1 = a.intr1[b * 4 + 3];
  if (N < 8) {   // no estimate, nothing depends on the confidences
    for (int i = tid; i < N; i += NT) gc[i] = 0.f;
    return;
  }

  // the forward's prologue, without its stores
  double csum = 0.0;
  for (int i = tid; i < N; i += NT) csum += (double)cf[i];
  csum = block_sum(csum, s.red);
  const float sum_conf = (float)csum + 1e-6f;
  const W8ptPtsRecomputed pts{k0, k1, cf, fx0, fy0, cx0, cy0, fx1, fy1, cx1, cy1, sum_conf};
  double mx0 = 0, my0 = 0, mx1 = 0, my1 = 0;
  for (int i = tid; i < N; i += NT) {
    float x0, y0, x1, y1;
    pts.xy(i, x0, y0, x1, y1);
    mx0 += x0; my0 += y0; mx1 += x1; my1 += y1;
  }
  mx0 = block_sum(mx0, s.red) / N; my0 = block_sum(my0, s.red) / N;
  mx1 = block_sum(mx1, s.red) / N; my1 = block_sum(my1, s.red) / N;
  double sc0, sc1;
  w8pt_solve(pts, N, mx0, my0, mx1, my1, sc0, sc1, s);
  w8pt_choose(pts, N, a.choose_closest, a.choose_closest ? a.T_gt + b * 16 : nullptr, s);

  if (tid == 0) {
    // the recomputed pose must be the forward's, bit for bit
    float T[16];
    w8pt_pose(s, T);
    int bad = 0;
    for (int i = 0; i < 16; ++i) bad |= __float_as_uint(T[i]) != __float_as_uint(a.T021[b * 16 + i]);
    s_bad = bad;
    double gf[9];
    w8pt_backward_3x3(s, a.gT + b * 16, sc0, sc1, mx0, my0, mx1, my1, gf);
    double lam[9];
    for (int k = 0; k < 9; ++k) lam[k] = s.M[k * 9 + k];
    eigvec_coeffs<9>(s.V, 9, lam, s.mi, gf, s_ck);
  }
  __syncthreads();

  // per match: g_w_i = 2 w_i x_i^T g_M x_i = -2 w_i (x_i . f) sum_k c_k (x_i . v_k), plus the gradient reaching
  // conf_norm; then through the normalisation w = c / (sum c + 1e-6)
  const int mi = s.mi;
  auto grad_w = [&](int i, double& w) {
    float px0, py0, px1, py1;
    pts.xy(i, px0, py0, px1, py1);
    const double x1 = sc0 * (px0 - mx0), y1 = sc0 * (py0 - my0);
    const double x2 = sc1 * (px1 - mx1), y2 = sc1 * (py1 - my1);
    w = (double)pts.w(i);
    const double r[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
    double xf = 0.0, acc = 0.0;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      double xv = 0.0;
#pragma unroll
      for (int j = 0; j < 9; ++j) xv += r[j] * s.V[j * 9 + k];
      if (k == mi) xf = xv;
      acc += s_ck[k] * xv;
    }
    double g = -2.0 * w * xf * acc;
    if (gcn) g += (double)gcn[i];
    return g;
  };
  double gwc = 0.0, nz = 0.0;
  for (int i = tid; i < N; i += NT) {
    double w;
    gwc += grad_w(i, w) * (double)cf[i];
    nz += (w != 0.0) ? 1.0 : 0.0;
  }
  gwc = block_sum(gwc, s.red);
  nz = block_sum(nz, s.red);
  // fewer than 8 non-zero weights: the eigenvector is not unique and has no gradient
  const bool nan_item = s_bad || nz < 8.0;
  const double S = csum + 1e-6;
  for (int i = tid; i < N; i += NT) {
    double w;
    const double g = grad_w(i, w);
    gc[i] = nan_item ? __int_as_float(0x7fc00000) : (float)(g / S - gwc / (S * S));
  }
}
}  // namespace

extern "C" int mvm_w8pt(const float* kpts0, const float* kpts1, const float* intr0,
                        const float* intr1, const float* conf, int batch, int n,
                        const float* T_gt, int choose_closest, int determine_inliers, float* T021,
                        float* kpts0_norm, float* kpts1_norm, float* conf_norm,
                        unsigned char* pos_depth_mask, unsigned char* inliers, float* F_out,
                        const int* n_valid, unsigned char* success, void* stream) {
  MvmProfScope prof__(MVM_TAG_W8PT, (cudaStream_t)stream);
  MVM_REQUIRE(kpts0 && kpts1 && intr0 && intr1 && conf && T021 && kpts0_norm && kpts1_norm &&
              conf_norm && pos_depth_mask);
  MVM_REQUIRE(batch >= 1 && n >= 1);
  MVM_REQUIRE(!choose_closest || T_gt != nullptr);
  MVM_REQUIRE(!determine_inliers || inliers != nullptr);
  W8ptArgs a;
  a.kpts0 = kpts0; a.kpts1 = kpts1; a.intr0 = intr0; a.intr1 = intr1; a.conf = conf; a.T_gt = T_gt;
  a.n_valid = n_valid; a.success = success;
  a.N = n; a.choose_closest = choose_closest; a.determine_inliers = determine_inliers;
  a.T021 = T021; a.k0n = kpts0_norm; a.k1n = kpts1_norm; a.conf_n = conf_norm;
  a.pos_depth = pos_depth_mask; a.inliers = determine_inliers ? inliers : nullptr; a.F_out = F_out;
  w8pt_kernel<<<batch, NT, 0, (cudaStream_t)stream>>>(a);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

extern "C" int mvm_w8pt_backward(const float* kpts0, const float* kpts1, const float* intr0,
                                 const float* intr1, const float* conf, int batch, int n,
                                 const float* T_gt, int choose_closest, const float* T021,
                                 const float* grad_T021, const float* grad_conf_norm, float* grad_conf,
                                 void* stream) {
  MvmProfScope prof__(MVM_TAG_W8PT, (cudaStream_t)stream);
  MVM_REQUIRE(kpts0 && kpts1 && intr0 && intr1 && conf && T021 && grad_T021 && grad_conf);
  MVM_REQUIRE(batch >= 1 && n >= 1);
  MVM_REQUIRE(!choose_closest || T_gt != nullptr);
  W8ptBwdArgs a;
  a.kpts0 = kpts0; a.kpts1 = kpts1; a.intr0 = intr0; a.intr1 = intr1; a.conf = conf;
  a.T_gt = choose_closest ? T_gt : nullptr; a.T021 = T021; a.gT = grad_T021; a.g_cn = grad_conf_norm;
  a.g_conf = grad_conf; a.N = n; a.choose_closest = choose_closest;
  w8pt_backward_kernel<<<batch, NT, 0, (cudaStream_t)stream>>>(a);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
